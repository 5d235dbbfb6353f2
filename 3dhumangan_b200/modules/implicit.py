"""`lib.implicit_funcitions` surface: COORDCONCATSIREN (reference: lib/implicit_funcitions/modulated.py:6-75).

The module owns the parameters under the reference's names (`first_layer_coord.layer.*`,
`first_layer_mod.layer.*`, `network.{i}.layer.*`, `sigma_layer.*`, `color_layer_sine.layer.*`,
`color_layer_linear.*`, `feature_layer_linear.*`) and evaluates the MLP with the fused sm_90a
kernel.  Inside `Map3DGenerator` the MLP never runs on its own (it is fused with the ray
integration in `hg_render_mlp`); `forward()` is provided for callers that want raw
per-point outputs and uses the same kernel with one sample per "ray".
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn


class _LinearHolder(nn.Module):
    """`SineLayer` / `FiLMLayer` parameter holder: a single `layer = nn.Linear` (pigan_layers.py:63-87)."""

    def __init__(self, in_dim, out_dim):
        super().__init__()
        self.layer = nn.Linear(in_dim, out_dim)


def _uniform_(w, bound):
    with torch.no_grad():
        w.uniform_(-bound, bound)


class COORDCONCATSIREN(nn.Module):
    def __init__(self, input_dim=2, latent_dim=100, hidden_dim=256, geo_feature_dim=88, output_dim=1, feature_dim=32,
                 num_blocks=9, device=None):
        super().__init__()
        self.device = device
        self.input_dim, self.latent_dim, self.hidden_dim = input_dim, latent_dim, hidden_dim
        self.geo_feature_dim, self.output_dim, self.feature_dim = geo_feature_dim, output_dim, feature_dim
        self.first_layer_coord = _LinearHolder(input_dim, hidden_dim)
        self.first_layer_mod = _LinearHolder(geo_feature_dim, hidden_dim)
        self.network = nn.ModuleList([_LinearHolder(2 * hidden_dim, hidden_dim)] +
                                     [_LinearHolder(hidden_dim, hidden_dim) for _ in range(num_blocks - 1)])
        self.sigma_layer = nn.Linear(hidden_dim, 1)
        self.color_layer_sine = _LinearHolder(hidden_dim + 3, hidden_dim)
        self.color_layer_linear = nn.Linear(hidden_dim, 3)
        self.feature_layer_linear = nn.Linear(hidden_dim, feature_dim)
        # SIREN initialisation: frequency_init(25) everywhere, 1/fan_in on the two first layers
        # (modulated.py:32-38, pigan_layers.py:27-52)
        for lin in [h.layer for h in self.network] + [self.sigma_layer, self.color_layer_sine.layer,
                                                      self.color_layer_linear, self.feature_layer_linear]:
            _uniform_(lin.weight, math.sqrt(6 / lin.weight.shape[1]) / 25)
        for lin in (self.first_layer_coord.layer, self.first_layer_mod.layer):
            _uniform_(lin.weight, 1 / lin.weight.shape[1])

    def forward(self, input, frequencies, phase_shifts, geo_feature, ray_directions, input_scaler=1.0,
                geo_feature_scaler=1.0, **kwargs):
        """[B,N,3], [B,4H], [B,4H], [B,N,G], [B,N,3] -> [B,N,3+F+1] (rgb, features, sigma) (modulated.py:41-75)."""
        from . import render_ops
        return render_ops.siren_points(self, input, frequencies, phase_shifts, geo_feature, ray_directions,
                                       input_scaler, geo_feature_scaler)
