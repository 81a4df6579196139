"""The conditioning pieces of the reference's downstream tasks (downstream_tasks/test_flow_latent_inpainting.py and
test_flow_latent_semantic_syn.py): ``WrapperCondFlow``, ``SpatialRescaler`` (models/encoder.py) and their
``sample_from_model(model, x_0, args)``.

A concat-conditioned ``UNetModel`` (``in_channels`` = 4 + condition channels) wrapped in ``WrapperCondFlow(model, cond)``
runs every native solver: the solver entry finds ``cond`` on the wrapper and stores it in the native context
(lfm_set_condition), and each network evaluation reads the state and the stored condition.  ``SpatialRescaler`` runs once
per batch on the conditioning input, not on the solver path.  Its float ``forward`` stays in torch; semantic synthesis calls
``forward_labels``, which computes the condition of a label map in one native kernel (lfm_label_condition) without building
the one-hot.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, solvers


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

    @torch.no_grad()
    def forward_labels(self, labels):
        """``self(F.one_hot(labels.long(), in_channels).permute(0, 3, 1, 2).float())`` for a ``[B, H, W]`` uint8 or int64 label
        map on a CUDA device, in one native kernel (lfm_label_condition): on one-hot input the bilinear halvings are the
        2^n_stages-pixel block class counts over the block area, exactly, so the one-hot is never built.  Labels are checked to
        lie in ``[0, in_channels)`` as ``F.one_hot`` checks them (one reduction on the device); -> ``[B, out_channels, H / f,
        W / f]`` fp32 with f = 2^n_stages."""
        if self.method != "bilinear" or self.multiplier != 0.5:
            raise NotImplementedError(f"forward_labels computes bilinear halvings only (method {self.method!r}, multiplier "
                                      f"{self.multiplier})")
        if not self.remap_output:
            raise NotImplementedError("forward_labels needs the 1x1 channel_mapper (out_channels)")
        if self.channel_mapper.bias is not None:
            raise NotImplementedError("forward_labels computes a bias-free channel_mapper only (bias=True)")
        if not torch.is_tensor(labels) or labels.dim() != 3 or labels.dtype not in (torch.uint8, torch.int64):
            raise ValueError(f"labels must be a [B, H, W] uint8 or int64 tensor, got "
                             f"{tuple(labels.shape) if torch.is_tensor(labels) else type(labels).__name__}"
                             f"{' ' + str(labels.dtype) if torch.is_tensor(labels) else ''}")
        B, H, W = labels.shape
        f = 2 ** self.n_stages
        if H % f != 0 or W % f != 0 or B < 1 or H < 1 or W < 1:
            raise ValueError(f"label map sides must be positive multiples of 2^n_stages = {f}, got {tuple(labels.shape)}")
        if not labels.is_cuda:
            raise ValueError("labels must be on a CUDA device (no CPU path)")
        K, O = self.channel_mapper.in_channels, self.channel_mapper.out_channels
        lo, hi = labels.aminmax()
        lo, hi = int(lo), int(hi)
        if lo < 0 or hi >= K:
            raise ValueError(f"labels must lie in [0, {K}) (the one-hot's classes), got values in [{lo}, {hi}]")
        labels = labels.to(torch.uint8).contiguous()
        w = self.channel_mapper.weight.to(device=labels.device, dtype=torch.float32).reshape(O, K).contiguous()
        out = torch.empty(B, O, H // f, W // f, device=labels.device, dtype=torch.float32)
        with torch.cuda.device(labels.device):
            stream = torch.cuda.current_stream(labels.device).cuda_stream
            _lib.check(_lib.load().lfm_label_condition(labels.data_ptr(), B, H, W, K, self.n_stages, w.data_ptr(), O,
                                                       out.data_ptr(), stream))
        return out


def sample_from_model(model, x_0, args):
    """downstream_tasks/test_flow_latent_*.py sample_from_model: ``odeint(model, x_0, t=[1, 0], method=args.method, ...)``
    with no model_kwargs.  Returns the [2, B, 4, H, W] trajectory (x_0, x_final).  The reference sets
    ``model.count_nfe`` when it does not compute the FID; that attribute changes nothing here."""
    if not getattr(args, "compute_fid", False):
        model.count_nfe = True
    sargs = SimpleNamespace(method=args.method, step_size=getattr(args, "step_size", 0.01), perturb=getattr(args, "perturb", False),
                            atol=args.atol, rtol=args.rtol, cfg_scale=1.0, compute_nfe=False)
    return solvers.sample_from_model(model, x_0, {}, sargs)
