"""Latent inversion (3dhumangan_b200/inversion.py): the image loss kernel against fp64 torch, and the optimisation loop end
to end -- a target rendered from a hidden latent, recovered from another seed with the generator in eval mode and frozen."""
import copy
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu

SPREAD = 2e-4       # run-to-run bound of a seeded inversion: 10x the measured 1.6e-5 / 1.9e-5 (loss curve), 3e-6 / 5e-6 (image)


@pytest.mark.parametrize("kind", ["l2", "charbonnier"])
@pytest.mark.parametrize("masked", [False, True])
def test_image_loss_matches_fp64(kind, masked):
    ops = importlib.import_module("3dhumangan_b200.ops.trainer_ops")
    B, H, W = 3, 132, 70                      # ragged: 9240 pixels, not a multiple of the block size
    g = torch.Generator().manual_seed(7)
    pred = torch.randn(B, 3, H, W, generator=g)
    target = torch.randn(B, 3, H, W, generator=g)
    mask = (torch.rand(B, 1, H, W, generator=g) > 0.4).float() * (0.5 + torch.rand(B, 1, H, W, generator=g)) if masked else None
    pd = pred.double().requires_grad_(True)
    d = pd - target.double()
    rho = d * d if kind == "l2" else torch.sqrt(d * d + 1e-3 ** 2)
    ref = (rho * (mask.double() if masked else 1.0)).mean()
    ref.backward()
    pc = pred.cuda().requires_grad_(True)
    loss = ops.image_loss(pc, target.cuda(), None if mask is None else mask.cuda(), kind=kind)
    (loss * 3.0).backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - float(ref)) < 1e-6 * abs(float(ref))
    assert (pc.grad.cpu().double() / 3.0 - pd.grad).abs().max() < 1e-6 * pd.grad.abs().max()
    again = ops.image_loss(pred.cuda(), target.cuda(), None if mask is None else mask.cuda(), kind=kind)
    assert torch.equal(again, loss.detach())
    with pytest.raises(RuntimeError, match="not built"):
        ops.image_loss(pc, target.cuda(), kind="lpips")


def _released_like(pkg, which):
    """-> eval-mode generator with trained-looking statistics (three train-mode forwards), cfg, conditions (B = 1)."""
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    if which == "420":            # the released checkpoint's curriculum as apps/sample_from_generator.py runs it
        cfg = pkg.configs.extract_metadata(copy.deepcopy(pkg.configs.MAP3DBN512L), 0)
        cfg.update(dataset_length=16, gen_height=512, gen_width=256, render_height=96, render_width=48, num_steps=32)
    else:
        cfg = pkg.configs.baseline_config("tiny")
        cfg.update(gen_height=32, gen_width=32, render_height=8, render_width=8, num_steps=16)
    cfg.update(last_back=True, nerf_noise=0.0)
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).cuda()
    G.set_device(torch.device("cuda:0"))
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(1, seed=1).items()}
    G.train()
    with torch.no_grad():
        for _ in range(3):
            G(torch.randn(1, cfg["latent_dim"], device="cuda"), cond, **dict(cfg, last_back=False))
    G.eval()
    return G, cfg, cond


@pytest.mark.parametrize("which", ["tiny", "420"])
def test_inversion_recovers_a_hidden_latent(pkg, which):
    inv = importlib.import_module("3dhumangan_b200.inversion")
    G, cfg, cond = _released_like(pkg, which)
    state = {k: v.clone() for k, v in G.state_dict().items()}
    flags = [p.requires_grad for p in G.parameters()]
    torch.manual_seed(11)
    with torch.no_grad():
        target = G(torch.randn(1, cfg["latent_dim"], device="cuda"), cond, **cfg)["rgbs"]
    runs = [inv.invert(G, target, cond, space="film", steps=60, lr=0.02, seed=5, **cfg) for _ in range(2)]
    torch.cuda.synchronize()
    losses = runs[0]["losses"]
    print(f"{which}: loss {losses[0]:.4e} -> {losses[-1]:.4e} ({losses[0] / losses[-1]:.1f}x) in {len(losses)} steps")
    assert len(losses) == 60 and all(l == l for l in losses)
    assert losses[-1] * 10 <= losses[0]
    # same seed, same curve -- up to the order of the shared-memory float atomics of the data-gradient kernels' S1 / S2
    # sums, which differs between runs
    spread = max(abs(a - b) / b for a, b in zip(runs[1]["losses"], losses))
    image_spread = float((runs[1]["image"] - runs[0]["image"]).norm() / runs[0]["image"].norm())
    print(f"{which}: second run differs by {spread:.2e} (loss curve), {image_spread:.2e} (final image)")
    assert spread < SPREAD and image_spread < SPREAD
    assert runs[0]["image"].shape == target.shape
    # the checkpoint is as it was: parameters, buffers, mode, requires_grad flags
    assert all(torch.equal(v, state[k]) for k, v in G.state_dict().items())
    assert not G.training and [p.requires_grad for p in G.parameters()] == flags
    assert all(p.grad is None for p in G.parameters())


def test_inversion_in_z_space_and_with_a_mask(pkg):
    inv = importlib.import_module("3dhumangan_b200.inversion")
    G, cfg, cond = _released_like(pkg, "tiny")
    torch.manual_seed(11)
    with torch.no_grad():
        target = G(torch.randn(1, cfg["latent_dim"], device="cuda"), cond, **cfg)["rgbs"]
    mask = torch.zeros(1, 1, 32, 32, device="cuda")
    mask[..., 8:24, 8:24] = 1.0
    G.train()
    res = inv.invert(G, target, cond, space="z", steps=20, lr=0.05, seed=5, mask=mask, loss="charbonnier", **cfg)
    assert G.training                             # restored
    assert set(res["variables"]) == {"z"} and res["losses"][-1] < res["losses"][0]
    with pytest.raises(RuntimeError, match="not built"):
        inv.invert(G, target, cond, space="w+", steps=1, **cfg)
