"""The random draws of one `render()` call, in the reference's order.

`Map3DGenerator.render` consumes the global torch RNG four times (SURVEY.md §7 hard part 5):
  1. `torch.rand(z_vals.shape)`  [B,R,S,1]   ray jitter            volume_rendering.py:126
  2. `torch.randn((B,1))` theta               unused camera sample  volume_rendering.py:194 ('gaussian')
  3. `torch.randn((B,1))` phi                 unused camera sample  volume_rendering.py:195
  4. `torch.randn(sigmas.shape)` [B,R,S,1]   sigma noise (drawn even when noise_std == 0)  :24
Issuing the same calls on the same device keeps a seeded run bit-compatible with the reference
and lets tests hand identical tensors to the oracle and to the kernels.
"""
import torch


def draw_render_noise(batch, rays, steps, device, sample_dist="gaussian"):
    u = torch.rand((batch, rays, steps, 1), device=device)
    if sample_dist == "uniform":
        torch.rand((batch, 1), device=device)
        torch.rand((batch, 1), device=device)
    elif sample_dist in ("normal", "gaussian"):
        torch.randn((batch, 1), device=device)
        torch.randn((batch, 1), device=device)
    elif sample_dist is None or sample_dist == "none":
        pass
    else:
        raise RuntimeError(f"sample_dist={sample_dist!r} is not used by any shipped curriculum")
    noise = torch.randn((batch, rays, steps, 1), device=device)
    return u, noise


class HierarchicalNoise:
    """The sigma-noise draws of a hierarchical_sample=True render: `coarse` [B,R,S,1] of the coarse integration
    (map3d_generator.py:453), `u_pdf` [B*R,S] of sample_pdf (volume_rendering.py:288) and `final` [B,R,2S,1] of the
    integration over the merged samples, in depth order (map3d_generator.py:513)."""

    def __init__(self, coarse, u_pdf, final):
        self.coarse, self.u_pdf, self.final = coarse, u_pdf, final


def draw_hierarchical_noise(batch, rays, steps, device, sample_dist="gaussian"):
    """Draws of one hierarchical render in the reference's order: jitter, the two camera draws, coarse noise, u_pdf,
    final noise.  Returns (u, HierarchicalNoise)."""
    u, coarse = draw_render_noise(batch, rays, steps, device, sample_dist)
    u_pdf = torch.rand(batch * rays, steps, device=device)
    final = torch.randn((batch, rays, 2 * steps, 1), device=device)
    return u, HierarchicalNoise(coarse, u_pdf, final)


def draw(batch, rays, steps, device, cfg):
    """The draws of one render under `cfg`: (u, noise), noise a HierarchicalNoise when hierarchical_sample is set."""
    if cfg.get("hierarchical_sample", False):
        return draw_hierarchical_noise(batch, rays, steps, device, cfg.get("sample_dist", None))
    return draw_render_noise(batch, rays, steps, device, cfg.get("sample_dist", None))
