"""The conditioning pieces of the reference's downstream tasks (downstream_tasks/test_flow_latent_inpainting.py and
test_flow_latent_semantic_syn.py): ``WrapperCondFlow``, ``SpatialRescaler`` (models/encoder.py) and their
``sample_from_model(model, x_0, args)``.

A concat-conditioned ``UNetModel`` (``in_channels`` = 4 + condition channels) wrapped in ``WrapperCondFlow(model, cond)``
runs every native solver: the solver entry finds ``cond`` on the wrapper and stores it in the native context
(lfm_set_condition), and each network evaluation reads the state and the stored condition.  ``SpatialRescaler`` runs once
per batch on the conditioning input, not on the solver path, so it stays in torch.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import solvers


class WrapperCondFlow(nn.Module):
    """downstream_tasks/test_flow_latent_*.py: ``forward(t, x) = model(t, cat([x, cond], 1))``."""

    def __init__(self, model, cond):
        super().__init__()
        self.model = model
        self.cond = cond

    def forward(self, t, x):
        return self.model(t, torch.cat([x, self.cond], 1))


class SpatialRescaler(nn.Module):
    """models/encoder.py SpatialRescaler: ``n_stages`` interpolations by ``multiplier``, then an optional bias-free 1x1 conv
    (key ``channel_mapper.weight``)."""

    def __init__(self, n_stages=1, method="bilinear", multiplier=0.5, in_channels=3, out_channels=None, bias=False):
        super().__init__()
        if n_stages < 0:
            raise ValueError("n_stages must be >= 0")
        if method not in ("nearest", "linear", "bilinear", "trilinear", "bicubic", "area"):
            raise ValueError(f"unknown interpolation method {method!r}")
        self.n_stages, self.method, self.multiplier = n_stages, method, multiplier
        self.remap_output = out_channels is not None
        if self.remap_output:
            self.channel_mapper = nn.Conv2d(in_channels, out_channels, 1, bias=bias)

    def forward(self, x):
        for _ in range(self.n_stages):
            x = F.interpolate(x, scale_factor=self.multiplier, mode=self.method)
        if self.remap_output:
            x = self.channel_mapper(x)
        return x

    def encode(self, x):
        return self(x)


def sample_from_model(model, x_0, args):
    """downstream_tasks/test_flow_latent_*.py sample_from_model: ``odeint(model, x_0, t=[1, 0], method=args.method, ...)``
    with no model_kwargs.  Returns the [2, B, 4, H, W] trajectory (x_0, x_final).  The reference sets
    ``model.count_nfe`` when it does not compute the FID; that attribute changes nothing here."""
    if not getattr(args, "compute_fid", False):
        model.count_nfe = True
    sargs = SimpleNamespace(method=args.method, step_size=getattr(args, "step_size", 0.01), perturb=getattr(args, "perturb", False),
                            atol=args.atol, rtol=args.rtol, cfg_scale=1.0, compute_nfe=False)
    return solvers.sample_from_model(model, x_0, {}, sargs)
