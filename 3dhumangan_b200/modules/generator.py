"""`lib.generators` surface: Map3DGenerator (reference: lib/generators/map3d_generator.py:101-523).

Same constructor (`Map3DGenerator(neural_field_cls, **config)`), attributes (`step`, `epoch`,
`latent_pool`, `set_device`, `generate_avg_latent`), call signatures (every call receives the whole
merged config as **kwargs and swallows what it does not need) and `state_dict()` names / shapes /
order as the reference, so released checkpoints load with `strict=True` and the reference's
trainer / sample app can drive it.  The forward pass is three fused device programs instead of the
reference's ~150 ATen launches:

    hg_geo_features   rays + jitter + camera transform + exact nearest-vertex search + 31-d feature
    hg_render_mlp     FiLM-SIREN MLP + volume integration, one kernel, only [rays, 260] leaves the SM
    hg_spade_conv x18 SPADE half-blocks with BatchNorm / modulation / ToRGB fused around wgmma GEMMs

There is no CPU or eager-PyTorch fallback: without a CUDA device and lib3dhg_sm90a.so the
forward raises RuntimeError.  With autograd enabled on parameters or inputs that require grad, `forward` runs the
training kernels (modules/render_train.py, modules/synthesis_train.py) and its outputs are differentiable: in
train() mode with batch statistics, in eval() mode with the running statistics and no buffer written (latent
inversion through `synthesize`, fine-tuning with frozen statistics).
"""
from __future__ import annotations

import math
import os
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import abi, rng
from . import render_ops, synthesis_ops


def _precision_passes(kwargs=None):
    """'fp32x3' (default): bf16x3 split GEMMs, meets the 1e-3-of-fp32 contract; 'bf16': single pass."""
    mode = (kwargs or {}).get("hg_precision", os.environ.get("HG3D_PRECISION", "fp32x3"))
    if mode not in ("fp32x3", "bf16"):
        raise RuntimeError(f"hg3d: unknown precision mode {mode!r}")
    return 3 if mode == "fp32x3" else 1


# ------------------------------------------------------------------------------------------------
# parameter holders with the reference's names
# ------------------------------------------------------------------------------------------------
class LatentPool(nn.Module):
    """lib/components/util.py:18-29.  On CUDA the lookup and its dense gradient run on hg_latent_pool_gather /
    hg_latent_pool_grad (`ops.trainer_ops.latent_pool_gather`); a CPU pool is indexed by torch."""

    def __init__(self, pool_size, latent_dim):
        super().__init__()
        self.latents = nn.Parameter(torch.zeros([pool_size, latent_dim]), requires_grad=True)

    def init(self, latents):
        with torch.no_grad():
            self.latents.copy_(latents)

    def forward(self, indices):
        if self.latents.is_cuda:
            from ..ops.trainer_ops import latent_pool_gather
            return latent_pool_gather(self.latents, torch.as_tensor(indices))
        return self.latents[indices]


def _kaiming_leaky_(w, a=0.2):
    with torch.no_grad():
        nn.init.kaiming_normal_(w, a=a, mode="fan_in", nonlinearity="leaky_relu")


class MappingNetwork(nn.Module):
    """z -> (freq, phase) for the SIREN (lib/components/mapping_networks.py:13-41).  The four dense layers run on the
    wgmma GEMM (`ops.dense`, fp32 via the bf16x3 split), LeakyReLU on `ops.bias_act`; the `nn.Linear` /
    `nn.LeakyReLU` children only hold the parameters under the reference's state_dict names."""

    def __init__(self, latent_dim, map_hidden_dim, map_output_dim):
        super().__init__()
        self.network = nn.Sequential(nn.Linear(latent_dim, map_hidden_dim), nn.LeakyReLU(0.2, inplace=True),
                                     nn.Linear(map_hidden_dim, map_hidden_dim), nn.LeakyReLU(0.2, inplace=True),
                                     nn.Linear(map_hidden_dim, map_hidden_dim), nn.LeakyReLU(0.2, inplace=True),
                                     nn.Linear(map_hidden_dim, map_output_dim))
        for m in self.network:
            if isinstance(m, nn.Linear):
                _kaiming_leaky_(m.weight)
        with torch.no_grad():
            self.network[-1].weight *= 0.25

    def forward(self, z):
        from ..ops import bias_act
        from ..ops.dense import dense
        x = z.to(torch.float32)
        x = x * (x.square().mean(dim=1, keepdim=True) + 1e-8).rsqrt()
        for m in self.network:
            if isinstance(m, nn.Linear):
                x = dense(x, m.weight, m.bias)
            else:
                x = bias_act.bias_act(x, None, act="lrelu", alpha=m.negative_slope, gain=1.0)
        half = x.shape[-1] // 2
        return x[..., :half], x[..., half:]


class FullyConnectedLayer(nn.Module):
    """StyleGAN-style equalised-lr dense layer (mapping_networks.py:92-121): the product on the wgmma GEMM with the
    weight gain folded into the operand packing (`ops.dense`), bias + activation through the `bias_act` kernel."""

    def __init__(self, in_features, out_features, bias=True, activation="linear", lr_multiplier=1, bias_init=0):
        super().__init__()
        self.activation = activation
        self.weight = nn.Parameter(torch.randn([out_features, in_features]) / lr_multiplier)
        self.bias = nn.Parameter(torch.full([out_features], np.float32(bias_init))) if bias else None
        self.weight_gain = lr_multiplier / np.sqrt(in_features)
        self.bias_gain = lr_multiplier

    def forward(self, x):
        from ..ops import bias_act
        from ..ops.dense import dense
        b = self.bias
        if b is not None and self.bias_gain != 1:
            b = b * self.bias_gain
        if self.activation == "linear":
            return dense(x, self.weight, b, gain=self.weight_gain)
        return bias_act.bias_act(dense(x, self.weight, None, gain=self.weight_gain), b, act=self.activation)


class TwoPartMappingNetwork(nn.Module):
    """z -> (implicit, superres) styles (mapping_networks.py:124-216); only `superres` is consumed."""

    def __init__(self, z_dim, c_dim, implicit_dim, w_dim, num_ws, trunk_layers=6, branch_layers=2, embed_features=None,
                 layer_features=None, activation="lrelu", lr_multiplier=0.01):
        super().__init__()
        if c_dim != 0:
            raise RuntimeError("hg3d: conditional mapping (c_dim > 0) is not used by any shipped curriculum")
        self.z_dim, self.c_dim, self.implicit_dim, self.w_dim, self.num_ws = z_dim, c_dim, implicit_dim, w_dim, num_ws
        self.trunk_layers, self.branch_layers = trunk_layers, branch_layers
        layer_features = w_dim if layer_features is None else layer_features
        trunk = [z_dim] + [layer_features] * trunk_layers
        implicit = [layer_features] * branch_layers + [implicit_dim]
        superres = [layer_features] * branch_layers + [w_dim]
        for i in range(trunk_layers):
            setattr(self, f"trunk{i}", FullyConnectedLayer(trunk[i], trunk[i + 1], activation=activation, lr_multiplier=lr_multiplier))
        for i in range(branch_layers):
            setattr(self, f"implicit{i}", FullyConnectedLayer(implicit[i], implicit[i + 1],
                                                              activation="linear" if i == branch_layers - 1 else activation,
                                                              lr_multiplier=lr_multiplier))
        getattr(self, f"implicit{branch_layers - 1}").weight_gain *= 0.2
        for i in range(branch_layers):
            setattr(self, f"superres{i}", FullyConnectedLayer(superres[i], superres[i + 1], activation=activation,
                                                              lr_multiplier=lr_multiplier))

    def forward(self, z, c=None, **_):
        x = z.to(torch.float32)
        x = x * (x.square().mean(dim=1, keepdim=True) + 1e-8).rsqrt()
        for i in range(self.trunk_layers):
            x = getattr(self, f"trunk{i}")(x)
        xi, xs = x, x
        for i in range(self.branch_layers):
            xi = getattr(self, f"implicit{i}")(xi)
        for i in range(self.branch_layers):
            xs = getattr(self, f"superres{i}")(xs)
        if self.num_ws is not None:
            xs = xs.unsqueeze(1).repeat([1, self.num_ws, 1])
        return xi, xs


class _SinAct(nn.Module):
    def forward(self, x):
        return torch.sin(x)


class SynthesisInput(nn.Module):
    """Parameter holder of lib/components/map3d_layers.py:241-275 (evaluated by hg_synth_input)."""

    def __init__(self, input_dim, output_dim, num_layers=1):
        super().__init__()
        if num_layers != 1 or input_dim != 2:
            raise RuntimeError("hg3d: SynthesisInput is built for the shipped configuration (2 coords, 1 layer)")
        conv = nn.Conv2d(input_dim, output_dim, kernel_size=1)
        nn.init.uniform_(conv.weight, -math.sqrt(9 / input_dim), math.sqrt(9 / input_dim))
        self.network = nn.Sequential(conv, _SinAct())


class SynthesisStyleInput(nn.Module):
    """Parameter holder of map3d_layers.py:278-327.  Only reached with `disable_render=True`, which
    no shipped curriculum sets; its tensors exist so that checkpoints load strictly."""

    def __init__(self, input_dim, latent_dim, output_dim, num_layers=1):
        super().__init__()
        self.latent_dim = latent_dim
        self.from_coords = nn.Sequential(nn.Conv2d(input_dim, latent_dim, kernel_size=1), _SinAct())
        nn.init.uniform_(self.from_coords[0].weight, -math.sqrt(9 / input_dim), math.sqrt(9 / input_dim))
        net = [nn.Conv2d(latent_dim * 2, output_dim, kernel_size=1), nn.LeakyReLU(0.2, inplace=True)]
        _kaiming_leaky_(net[0].weight)
        for _ in range(1, num_layers - 1):
            layer = nn.Conv2d(output_dim, output_dim, kernel_size=1)
            _kaiming_leaky_(layer.weight)
            net += [layer, nn.LeakyReLU(0.2, inplace=True)]
        self.network = nn.Sequential(*net)


class SPADE2d(nn.Module):
    """Parameter holder of map3d_layers.py:153-190 (SyncBatchNorm affine + running stats, shared/gamma/beta convs)."""

    def __init__(self, input_dim, feature_dim, normalization="instance_norm"):
        super().__init__()
        if normalization != "batch_norm":
            raise RuntimeError("hg3d: only spatial_normalization='batch_norm' (all shipped curricula) is built")
        self.normalization = normalization
        self.first_norm = nn.SyncBatchNorm(input_dim)
        self.mlp_shared = nn.Sequential(nn.Conv2d(feature_dim, 128, kernel_size=1), nn.ReLU())
        self.mlp_gamma = nn.Conv2d(128, input_dim, kernel_size=1)
        self.mlp_beta = nn.Conv2d(128, input_dim, kernel_size=1)


class SPADEBlock(nn.Module):
    """Parameter holder of map3d_layers.py:193-238: two spectral-normed 1x1 convs + two SPADE2d."""

    def __init__(self, in_dim, out_dim, style_dim, normalization="instance_norm"):
        super().__init__()
        self.in_dim, self.out_dim, self.style_dim = in_dim, out_dim, style_dim
        self.conv_0 = nn.utils.spectral_norm(nn.Conv2d(in_dim, out_dim, kernel_size=1))
        self.conv_1 = nn.utils.spectral_norm(nn.Conv2d(out_dim, out_dim, kernel_size=1))
        self.spade_0 = SPADE2d(in_dim, style_dim, normalization)
        self.spade_1 = SPADE2d(out_dim, style_dim, normalization)


class ToRGB(nn.Module):
    """map3d_layers.py:330-352."""

    def __init__(self, in_dim, dim_rgb=3, use_conv=True):
        super().__init__()
        self.linear = nn.Conv2d(in_dim, dim_rgb, 1)
        with torch.no_grad():
            self.linear.weight *= 0.25


class SynthesisNetwork(nn.Module):
    """Parameter holder of map3d_generator.py:14-97 (`network.m3d_k`, `to_rgbs.m3d_k`)."""

    def __init__(self, input_dim, style_dim, hidden_dim=256, num_blocks=8, mod_blocks=tuple(range(8)), name_prefix="m3d",
                 spatial_normalization="instance_norm", map3d_mode="isolated", **kwargs):
        super().__init__()
        self.style_dim, self.num_blocks, self.mod_blocks, self.map3d_mode = style_dim, num_blocks, list(mod_blocks), map3d_mode
        self.normalization = spatial_normalization
        network, to_rgbs = OrderedDict(), OrderedDict()
        out_dim = input_dim
        for i in range(num_blocks):
            in_dim, out_dim = out_dim, hidden_dim
            network[f"{name_prefix}_{i}"] = SPADEBlock(in_dim, out_dim, style_dim, spatial_normalization)
            to_rgbs[f"{name_prefix}_{i}"] = ToRGB(out_dim, 3, use_conv=True)
        self.network = nn.ModuleDict(network)
        self.to_rgbs = nn.ModuleDict(to_rgbs)


# ------------------------------------------------------------------------------------------------
# the generator
# ------------------------------------------------------------------------------------------------
class Map3DGenerator(nn.Module):
    def __init__(self, neural_field_cls, **kwargs):
        super().__init__()
        self.latent_dim = kwargs["latent_dim"]
        self.hidden_dim = kwargs["hidden_dim"]
        self.feature_dim = kwargs["feature_dim"]
        self.geo_feature_dim = kwargs["geo_feature_dim"]
        self.label_dim = kwargs["label_dim"]
        self.gen_height = kwargs["gen_height"]
        self.gen_width = kwargs["gen_width"]
        self.disable_modulation = kwargs.get("disable_modulation", False)
        self.legacy_mode = kwargs.get("legacy_mode", False)
        if isinstance(neural_field_cls, str):
            from . import implicit
            neural_field_cls = getattr(implicit, neural_field_cls)
        self.neural_field = neural_field_cls(
            output_dim=kwargs["feature_dim"] + 4, latent_dim=kwargs["latent_dim"], input_dim=kwargs["input_dim"],
            hidden_dim=kwargs["hidden_dim"], geo_feature_dim=kwargs["geo_feature_dim"], feature_dim=kwargs["feature_dim"],
            num_blocks=kwargs["neural_field_blocks"], device=None)
        self.synthesis_input = SynthesisInput(
            input_dim=2 + (kwargs["semantic_dim"] if kwargs.get("2d_semantic_input", False) else 0) +
            (1 if kwargs.get("2d_label_input", False) else 0), output_dim=kwargs["feature_dim"])
        self.synthesis_style_input = SynthesisStyleInput(
            input_dim=1 if "segments" in kwargs["condition_modal_gen"] else 3, latent_dim=kwargs["latent_dim"],
            output_dim=kwargs["feature_dim"], num_layers=3)
        self.synthesis_network = SynthesisNetwork(
            input_dim=kwargs["feature_dim"] + (kwargs["latent_dim"] if kwargs.get("2d_latent_input", False) else 0),
            style_dim=kwargs["feature_dim"], hidden_dim=kwargs["hidden_dim"], num_blocks=kwargs["synthesis_blocks"],
            mod_blocks=kwargs["mod_blocks"], map3d_mode=kwargs.get("map3d_mode", "isolated"),
            spatial_normalization=kwargs.get("spatial_normalization", "instance_norm"))
        self.neural_field_mapping_network = MappingNetwork(
            latent_dim=kwargs["latent_dim"], map_hidden_dim=kwargs["hidden_dim"],
            map_output_dim=2 * kwargs["neural_field_blocks"] * kwargs["hidden_dim"])
        self.synthesis_mapping_network = TwoPartMappingNetwork(
            z_dim=kwargs["latent_dim"], c_dim=0, implicit_dim=1, w_dim=kwargs["feature_dim"], num_ws=1, trunk_layers=7,
            branch_layers=1, lr_multiplier=0.01)
        self.epoch = 0
        self.step = 0
        self.side_length = kwargs["side_length"]
        self.latent_pool = LatentPool(kwargs["dataset_length"], kwargs["latent_dim"])
        self._cfg = {k: v for k, v in kwargs.items() if isinstance(k, str)}

    # -------------------------------------------------------------------------------- reference API
    def set_device(self, device):
        self.device = device
        self.neural_field.device = device

    def generate_avg_latent(self):
        """Average freq / phase / style over 10 000 fresh latents (map3d_generator.py:182-194)."""
        z = torch.randn((10000, self.latent_dim), device=self.neural_field.device)
        freq, phase = self.neural_field_mapping_network(z)
        _, styles = self.synthesis_mapping_network(z)
        self.avg_latent = (z.mean(dim=0, keepdim=True), freq.mean(dim=0, keepdim=True),
                           phase.mean(dim=0, keepdim=True), styles.mean(dim=0, keepdim=True))
        return self.avg_latent

    # -------------------------------------------------------------------------------- internals
    def _params(self):
        return OrderedDict(list(self.named_parameters()) + list(self.named_buffers()))

    def _wants_grad(self, *inputs):
        """Autograd is on and a parameter or one of `inputs` (a frozen generator asked for d / d latent) requires grad."""
        return torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters())
                                            or any(t is not None and t.requires_grad for t in inputs))

    def _guard(self, kwargs):
        for key, bad in (("disable_render", True), ("disable_synthesis", True), ("2d_label_input", True),
                         ("2d_latent_input", True)):
            if kwargs.get(key, False) == bad:
                raise RuntimeError(f"hg3d: {key}={bad} is not used by any shipped curriculum and is not built")
        if kwargs.get("feature_map_interpolation", "bilinear") != "bilinear":
            raise RuntimeError("hg3d: only bilinear feature-map interpolation is built")

    def _cfg_for(self, kwargs, render_height, render_width):
        cfg = dict(self._cfg)
        cfg.update({k: v for k, v in kwargs.items() if isinstance(k, str)})
        cfg.update(render_height=render_height, render_width=render_width, gen_height=self.gen_height,
                   gen_width=self.gen_width, hidden_dim=self.hidden_dim, feature_dim=self.feature_dim,
                   legacy_mode=self.legacy_mode)
        cfg.setdefault("num_steps", 24)
        return cfg

    def _run(self, freq, phase, styles, conditions, cfg, passes, want_records=False):
        """-> (rgbs, rgbs_render, depth); with `want_records` (differentiable path only) also the render's (rec, z_vals)."""
        B = freq.shape[0]
        dev = freq.device
        Rh, Rw, S = cfg["render_height"], cfg["render_width"], cfg["num_steps"]
        P = self._params()
        cond = {k: conditions[k] for k in ("skeletons_xyz", "vertices", "tpose_vertices", "fk_matrices", "lbs_weights",
                                           "cam2world_matrices", "intrinsics", "scales")}
        u, noise = rng.draw(B, Rh * Rw, S, dev, cfg)
        wants_grad = self._wants_grad(freq, phase, styles)
        if (want_records or cfg.get("hg_records") is not None) and not wants_grad:
            raise RuntimeError("hg3d: hg_records re-uses the point records of a differentiable render; the inference kernels "
                               "rebuild them in the fused pass")
        if self.hidden_dim != 256 and not wants_grad:
            # hidden_dim 384 (MAP3DBN) / 420 (MAP3DBN512L, the released checkpoint): the zero-padded 2 x 256 path on the
            # general blocked-GEMM engine (modules/wide_ops.py); under autograd it runs inside GeneratorCore below
            from . import wide_ops
            feats, rgb01, depth = wide_ops.render_forward_wide(P, freq, phase, cond, cfg, u, noise, passes=passes)
            rgb = wide_ops.synthesis_forward_wide(P, feats, styles.reshape(B, -1), cfg, training=self.training, passes=passes)
            rgb_render = (rgb01 * 2 - 1).reshape(B, Rh, Rw, 3).permute(0, 3, 1, 2)
            return rgb, rgb_render, depth
        if wants_grad:
            # training step of the generator, or gradients through it in eval mode: layer-by-layer renderer + taped
            # synthesis network (render_train.py, synthesis_train.py); the fused inference kernels below keep nothing
            # for a backward pass
            from . import render_train
            names, tensors = render_train.core_parameters(self)
            rgb, rgb_render, depth, rec, z_vals = render_train.GeneratorCore.apply(self, cond, cfg, u, noise, passes, names, freq,
                                                                                   phase, styles.reshape(B, -1), *tensors)
            return (rgb, rgb_render, depth, (rec, z_vals)) if want_records else (rgb, rgb_render, depth)
        r = render_ops.render_forward(P, freq, phase, cond, cfg, u, noise, passes=passes)
        ray = r["ray_out"]                                                   # [B,R,260]
        rgb = synthesis_ops.synthesis_forward(P, ray, styles.reshape(B, -1), cfg, training=self.training, passes=passes)
        rgb_render = (ray[..., 256:259] * 2 - 1).reshape(B, Rh, Rw, 3).permute(0, 3, 1, 2)
        depth = ray[..., 259:260]
        return rgb, rgb_render, depth

    # -------------------------------------------------------------------------------- forward paths
    def _forward_eager(self, latent, conditions, cfg, passes):
        zz = latent if cfg.get("neural_field_latent_input", True) else torch.zeros_like(latent)
        freq, phase = self.neural_field_mapping_network(zz)
        _, styles = self.synthesis_mapping_network(latent)
        return self._run(freq, phase, styles, conditions, cfg, passes)

    def _forward_graphed(self, latent, conditions, cfg, passes):
        """Replay the whole forward (~400 kernel launches + ~300 small torch ops) as ONE CUDA graph.
        Captured once per (shapes, mode) key; inputs are copied into static buffers, parameters and
        buffers are read / updated in place by the replay (running stats, spectral-norm u/v, RNG offsets)."""
        keys = ("skeletons_xyz", "vertices", "tpose_vertices", "fk_matrices", "lbs_weights", "cam2world_matrices",
                "intrinsics", "scales")
        # every plain config value is part of the key: scalars such as clamp_mode, ray_start/ray_end, side_length,
        # sample_dist, legacy_mode are baked into the captured launches, and a curriculum step may change them
        plain = tuple(sorted((k, repr(v)) for k, v in cfg.items()
                             if isinstance(v, (bool, int, float, str, type(None), list, tuple)) and not k.startswith("hg_")))
        sig = (tuple(latent.shape), tuple(tuple(conditions[k].shape) for k in keys), self.training, passes,
               str(latent.device), plain)
        if not hasattr(self, "_graphs"):
            self._graphs = {}
        entry = self._graphs.get(sig)
        if entry is None:
            static_z = latent.clone()
            static_c = {k: conditions[k].detach().float().contiguous().clone() for k in keys}
            # Warm-up outside the capture (lazy inits, allocator).  It must not count as a forward: module
            # buffers (running statistics, spectral-norm u/v, num_batches_tracked) and the RNG stream are restored.
            saved = {k: b.detach().clone() for k, b in self.named_buffers()}
            rng_state = torch.cuda.get_rng_state(latent.device)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._forward_eager(static_z, static_c, cfg, passes)
            torch.cuda.current_stream().wait_stream(side)
            for k, b in self.named_buffers():
                b.copy_(saved[k])
            torch.cuda.set_rng_state(rng_state, latent.device)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                outs = self._forward_eager(static_z, static_c, cfg, passes)
            entry = self._graphs[sig] = (graph, static_z, static_c, outs)
        graph, static_z, static_c, outs = entry
        static_z.copy_(latent, non_blocking=True)
        for k in keys:
            static_c[k].copy_(conditions[k], non_blocking=True)
        graph.replay()
        return tuple(o.clone() for o in outs)

    def forward(self, latent, conditions, render_height, render_width, latent_indices=None, **kwargs):
        """-> {"rgbs": [B,3,Hg,Wg], "rgbs_render": [B,3,Rh,Rw]}  (map3d_generator.py:208-280).
        `hg_cuda_graph=True` (or HG3D_CUDA_GRAPH=1) replays the forward as a CUDA graph.
        With autograd enabled and parameters that require grad (the generator step of the trainer) the training
        kernels run instead (render_train.GeneratorCore): outputs carry a grad_fn, `loss.backward()` fills `.grad`."""
        self._guard(kwargs)
        if self._wants_grad(latent):
            cfg = self._cfg_for(kwargs, render_height, render_width)
            if latent_indices is not None:
                latent = self.latent_pool(latent_indices)
            rgb, rgb_render, _ = self._forward_eager(latent, conditions, cfg, _precision_passes(kwargs))
            return {"rgbs": rgb, "rgbs_render": rgb_render}
        with torch.no_grad():
            cfg = self._cfg_for(kwargs, render_height, render_width)
            if latent_indices is not None:
                latent = self.latent_pool(latent_indices)
            passes = _precision_passes(kwargs)
            use_graph = kwargs.get("hg_cuda_graph", os.environ.get("HG3D_CUDA_GRAPH", "0") == "1")
            multi = torch.distributed.is_available() and torch.distributed.is_initialized() \
                and torch.distributed.get_world_size() > 1 and self.training
            if use_graph and multi and not kwargs.get("hg_cuda_graph_nccl", os.environ.get("HG3D_CUDA_GRAPH_NCCL", "0") == "1"):
                use_graph = False      # SyncBatchNorm all-reduces (NCCL) are captured only on explicit request
            if use_graph and getattr(self, "_graph_broken", False):
                use_graph = False
            if use_graph:
                try:
                    rgb, rgb_render, _ = self._forward_graphed(latent, conditions, cfg, passes)
                except RuntimeError as err:          # capture refused (e.g. a collective that cannot be captured here)
                    if "hg3d:" in str(err):
                        raise
                    self._graph_broken = True
                    import warnings
                    warnings.warn(f"hg3d: CUDA-graph capture failed ({str(err)[:200]}); launching eagerly from now on")
                    rgb, rgb_render, _ = self._forward_eager(latent, conditions, cfg, passes)
            else:
                rgb, rgb_render, _ = self._forward_eager(latent, conditions, cfg, passes)
        return {"rgbs": rgb, "rgbs_render": rgb_render}

    def synthesize(self, freq, phase, styles, conditions, render_height, render_width, **kwargs):
        """`forward` from the mapped space: freq / phase [B, 4*hidden_dim] of `neural_field_mapping_network`, styles
        [B,1,feature_dim] of `synthesis_mapping_network` -> the dict of `forward`, differentiable in the three tensors
        (truncation and mapped-space optimisation are the caller's).  Under autograd the dict also holds `hg_records`, the
        point records (rec, z_vals) of this render: passed back as `hg_records=` they replace ray sampling, nearest-vertex
        search and geometry features of a later call with the same pose, camera and jitter (they carry no gradient)."""
        self._guard(kwargs)
        cfg = self._cfg_for(kwargs, render_height, render_width)
        if self._wants_grad(freq, phase, styles):
            rgb, rgb_render, _, records = self._run(freq, phase, styles, conditions, cfg, _precision_passes(kwargs),
                                                    want_records=True)
            return {"rgbs": rgb, "rgbs_render": rgb_render, "hg_records": records}
        with torch.no_grad():
            rgb, rgb_render, _ = self._run(freq, phase, styles, conditions, cfg, _precision_passes(kwargs))
        return {"rgbs": rgb, "rgbs_render": rgb_render}

    def truncated_codes(self, latent, truncation_psi, cfg, averages=None):
        """latent -> (freq, phase, styles) as `staged_forward` maps them (map3d_generator.py:282-379): the SIREN's codes from
        the latent or, with neural_field_latent_input False, from a zero latent; truncation_psi < 1 pulls all three towards
        the averages of `generate_avg_latent` (fresh draws on every call), or towards `averages` = (freq, phase, styles)
        when they are given."""
        zz = latent if cfg.get("neural_field_latent_input", True) else torch.zeros_like(latent)
        freq, phase = self.neural_field_mapping_network(zz)
        _, styles = self.synthesis_mapping_network(latent)
        if truncation_psi < 1.0:
            if averages is None:
                self.generate_avg_latent()
                _, afreq, aphase, astyles = self.avg_latent
            else:
                afreq, aphase, astyles = averages
            freq = afreq + truncation_psi * (freq - afreq)
            phase = aphase + truncation_psi * (phase - aphase)
            styles = astyles + truncation_psi * (styles - astyles)
        return freq, phase, styles

    def staged_forward(self, latent, conditions, render_height, render_width, truncation_psi, **kwargs):
        """Inference entry of apps/sample_from_generator.py (map3d_generator.py:282-379): truncation
        towards the average latent, depth map in [-1,1] on the CPU, skeleton passthrough.  The
        reference chunks points to bound memory (max_points); the fused kernel needs no chunking."""
        self._guard(kwargs)
        with torch.no_grad():
            cfg = self._cfg_for(kwargs, render_height, render_width)
            B = latent.shape[0]
            freq, phase, styles = self.truncated_codes(latent, truncation_psi, cfg)
            rgb, rgb_render, depths = self._run(freq, phase, styles, conditions, cfg, _precision_passes(kwargs))
            focals = conditions["intrinsics"][:, 0, 0]
            scales = conditions["scales"].float()
            depth = depths - (focals / scales).view(B, 1, 1)
            depth = torch.clamp(depth / (cfg["depth_length"] / 2.0), -1.0, 1.0)
            depth_map = depth.reshape(B, render_height, render_width).unsqueeze(1).contiguous().cpu()
        return {"rgbs": rgb, "rgbs_render": rgb_render, "depths": depth_map, "skeletons": conditions["skeletons_xyz"]}
