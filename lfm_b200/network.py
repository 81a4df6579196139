"""Host-side mirror of the reference's network interface for the sampling path.

``create_network(config)`` / ``DiT_models[...]`` (reference models/__init__.py:6-17, models/DiT.py:355-415)
return a :class:`DiT` whose *parameters* are ordinary ``nn.Module`` state (same ``state_dict`` keys and
shapes as the reference - SURVEY.md 8(b) - so ``load_state_dict(ckpt, strict=True)``, ``.parameters()``,
``.eval()``, ``.to(device)`` behave identically), and whose *compute* is liblfm_b200.so: ``model(t, x, y)`` and
``model.forward_with_cfg(t, x, y, cfg_scale)`` call the C ABI (include/lfm_b200.h) on the current CUDA stream.
There is no PyTorch implementation of the forward pass in this package and no fallback: without an H100 and the
built library the call raises.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch
import torch.nn as nn

from . import _lib


def _pos_embed_2d(dim: int, grid: int) -> torch.Tensor:
    """Fixed 2-D sin-cos table, column-first (reference models/DiT.py:299-346)."""
    def one(d, pos):
        omega = 1.0 / 10000 ** (np.arange(d // 2, dtype=np.float64) / (d / 2.0))
        out = np.einsum("m,d->md", pos.reshape(-1), omega)
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)

    gh = np.arange(grid, dtype=np.float32)
    gw = np.arange(grid, dtype=np.float32)
    mesh = np.stack(np.meshgrid(gw, gh), axis=0).reshape(2, 1, grid, grid)
    emb = np.concatenate([one(dim // 2, mesh[0]), one(dim // 2, mesh[1])], axis=1)
    return torch.from_numpy(emb).float().unsqueeze(0)


class _Holder(nn.Module):
    """Parameter container: exists only so that state_dict keys match the reference's module tree."""


class _NativeNet(nn.Module):
    """Shared plumbing: lazily create the native context, upload the state_dict (strict), call lfm_forward."""

    max_batch_hint = None
    table_rows = 0

    def _init_native(self):
        self._ctx = None
        self._ctx_rows = 0
        self._ctx_device = None
        self._uploaded_version = None
        self._dirty = True          # parameters may differ from the uploaded copy: do the full version walk
        self._probe = None          # O(1) fingerprint (first / last parameter) checked on every call
        self.last_stats = None

    def _version(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _quick_probe(self):
        ps = self._probe_params
        return tuple((p.data_ptr(), p._version) for p in ps)

    # everything that can change parameters through the nn.Module interface marks the native copy stale; direct in-place
    # edits of a parameter tensor are caught by the O(1) probe when they touch the first / last parameter, otherwise
    # call mark_dirty().  (Round 1 walked all 252-428 tensors on every model(t, x) call: ~100 us per NFE for callers that
    # drive the solver from Python, e.g. the reference's own odeint or --measure_time.)
    def mark_dirty(self):
        self._dirty = True

    def _apply(self, fn, *a, **k):
        self._dirty = True
        object.__setattr__(self, "_probe_cache", None)   # .to() / .to_empty() may replace the Parameter objects
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._dirty = True
        object.__setattr__(self, "_probe_cache", None)
        return super().load_state_dict(*a, **k)

    def _release(self):
        if getattr(self, "_ctx", None) is not None:
            _lib.load().lfm_destroy(self._ctx)
            self._ctx = None
            self._ctx_rows = 0

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _create_ctx(self, lib, dev_index):  # -> ctypes handle
        raise NotImplementedError

    def _native_state_dict(self):
        """The entries uploaded to the native context (lfm_set_param, strict on both sides)."""
        return self.state_dict()

    def _finalize_rows(self, rows: int) -> int:
        """Rows the native workspace is sized for when a context is (re)created for `rows`."""
        return max(rows, self.max_batch_hint or 0)

    def native(self, rows: int, device: torch.device):
        """Return the lfm_ctx handle, (re)creating it and uploading the weights when needed."""
        lib = _lib.load()
        if device.type != "cuda":
            raise RuntimeError("lfm_b200 runs on a CUDA device (H100, sm_90a) only; got tensors on " + str(device))
        dev_index = device.index if device.index is not None else torch.cuda.current_device()
        if (self._ctx is not None and not self._dirty and rows <= self._ctx_rows and self._ctx_device == dev_index
                and self._quick_probe() == self._probe):
            return self._ctx                     # fast path: nothing changed since the upload
        ver = self._version()
        if (self._ctx is not None and rows <= self._ctx_rows and self._ctx_device == dev_index
                and ver == self._uploaded_version):
            self._dirty = False
            self._probe = self._quick_probe()
            return self._ctx
        self._release()
        ctx = self._create_ctx(lib, dev_index)
        try:
            for key, p in self._native_state_dict().items():
                t = p.detach().to(torch.float32).contiguous()
                shape = (C.c_int64 * t.dim())(*t.shape)
                _lib.check(lib.lfm_set_param(ctx, key.encode(), C.c_void_p(t.data_ptr()), 0, shape, t.dim()), ctx)
            max_rows = self._finalize_rows(rows)
            _lib.check(lib.lfm_finalize(ctx, max_rows), ctx)
        except Exception:
            lib.lfm_destroy(ctx)
            raise
        self._ctx, self._ctx_rows, self._ctx_device, self._uploaded_version = ctx, max_rows, dev_index, ver
        self._dirty = False
        self._probe = self._quick_probe()
        return ctx

    @property
    def _probe_params(self):
        ps = getattr(self, "_probe_cache", None)
        if ps is None:
            allp = list(self.parameters())
            ps = (allp[0], allp[-1]) if allp else ()
            object.__setattr__(self, "_probe_cache", ps)
        return ps

    @staticmethod
    def _stream(device):
        return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)

    def _prep(self, t, x, y):
        if not x.is_cuda:
            raise RuntimeError("lfm_b200: x must be a CUDA tensor (no CPU path)")
        x = x.to(torch.float32).contiguous()
        B = x.shape[0]
        t = torch.as_tensor(t, dtype=torch.float32, device=x.device).reshape(-1).contiguous()
        if t.numel() not in (1, B):
            raise ValueError(f"t has {t.numel()} elements, expected 1 or {B}")
        if y is not None:
            y = torch.as_tensor(y, device=x.device).to(torch.int64).contiguous()
            if y.numel() != B:
                raise ValueError(f"y has {y.numel()} labels, expected {B}")
            self._check_table_index(y)
        return t, x, y, B

    def uses_labels(self):
        return True

    def _check_table_index(self, y):
        """The failure the reference's ``nn.Embedding`` raises on an out-of-range index (the device kernels clamp)."""
        if y.numel() and (int(y.min()) < 0 or int(y.max()) >= self.table_rows):
            raise IndexError(f"label out of range for the embedding table ({self.table_rows} rows)")

    def check_label_range(self, y):
        """Validation of user-facing labels (solver entry points)."""
        self._check_table_index(y)

    def _forward_native(self, t, x, y, cfg_scale=1.0):
        B = x.shape[0]
        ctx = self.native(B, x.device)
        v = x.new_empty((B, self.out_channels) + tuple(x.shape[2:]))
        _lib.check(_lib.load().lfm_forward(ctx, t.data_ptr(), t.numel(), x.data_ptr(), y.data_ptr() if y is not None else None,
                                           B, float(cfg_scale), v.data_ptr(), self._stream(x.device)), ctx)
        return v

    def launch_count(self) -> int:
        return int(_lib.load().lfm_launch_count(self._ctx)) if self._ctx is not None else 0


class DiT(_NativeNet):
    """H100-native DiT velocity network with the reference's constructor (models/DiT.py:157-169).

    ``fp8=True`` (not a reference option; off by default) runs each block's attn.qkv and mlp.fc1 GEMMs on e4m3 operands:
    per-token activation scales from the LayerNorm-modulate pass, per-output-channel weight scales taken at upload from the
    fp32 parameters (include/lfm_b200.h, lfm_set_fp8).  The results then differ from the bf16 path's by that rounding."""

    def __init__(self, img_resolution=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4.0, label_dropout=0.1, num_classes=1000, learn_sigma=False, max_batch=None, fp8=False):
        super().__init__()
        if learn_sigma:
            raise NotImplementedError("learn_sigma=True is not used by the LFM sampling path")
        D, Hd = hidden_size, int(hidden_size * mlp_ratio)
        self.in_channels = self.out_channels = in_channels
        self.patch_size, self.num_heads, self.num_classes = patch_size, num_heads, num_classes
        self.hidden_size, self.depth, self.mlp_hidden, self.img_resolution = D, depth, Hd, img_resolution
        self.label_dropout = label_dropout
        self.table_rows = num_classes + (1 if label_dropout > 0 else 0)  # models/DiT.py:79-81
        self.max_batch_hint = max_batch
        self.fp8 = bool(fp8)

        self.x_embedder = _Holder()
        self.x_embedder.proj = nn.Conv2d(in_channels, D, kernel_size=patch_size, stride=patch_size, bias=True)
        self.t_embedder = _Holder()
        self.t_embedder.mlp = nn.Sequential(nn.Linear(256, D), nn.SiLU(), nn.Linear(D, D))
        self.y_embedder = _Holder()
        self.y_embedder.embedding_table = nn.Embedding(self.table_rows, D)
        grid = img_resolution // patch_size
        self.pos_embed = nn.Parameter(torch.zeros(1, grid * grid, D), requires_grad=False)
        blocks = []
        for _ in range(depth):
            b = _Holder()
            b.attn = _Holder()
            b.attn.qkv = nn.Linear(D, 3 * D)
            b.attn.proj = nn.Linear(D, D)
            b.mlp = _Holder()
            b.mlp.fc1 = nn.Linear(D, Hd)
            b.mlp.fc2 = nn.Linear(Hd, D)
            b.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(D, 6 * D))
            blocks.append(b)
        self.blocks = nn.ModuleList(blocks)
        self.final_layer = _Holder()
        self.final_layer.linear = nn.Linear(D, patch_size * patch_size * in_channels)
        self.final_layer.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(D, 2 * D))
        self.initialize_weights()
        self.requires_grad_(False)
        self._init_native()

    # -- reference models/DiT.py:193-228 (same distributions; adaLN and output layers start at zero) ----------
    def initialize_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                nn.init.zeros_(m.bias)
        self.pos_embed.data.copy_(_pos_embed_2d(self.hidden_size, self.img_resolution // self.patch_size))
        w = self.x_embedder.proj.weight.data
        nn.init.xavier_uniform_(w.view(w.shape[0], -1))
        nn.init.zeros_(self.x_embedder.proj.bias)
        nn.init.normal_(self.y_embedder.embedding_table.weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        for b in self.blocks:
            nn.init.zeros_(b.adaLN_modulation[-1].weight)
            nn.init.zeros_(b.adaLN_modulation[-1].bias)
        nn.init.zeros_(self.final_layer.adaLN_modulation[-1].weight)
        nn.init.zeros_(self.final_layer.adaLN_modulation[-1].bias)
        nn.init.zeros_(self.final_layer.linear.weight)
        nn.init.zeros_(self.final_layer.linear.bias)

    def _create_ctx(self, lib, dev_index):
        desc = _lib.ModelDesc(0, self.img_resolution, self.patch_size, self.in_channels, self.hidden_size, self.depth,
                              self.num_heads, self.mlp_hidden, self.table_rows)
        ctx = C.c_void_p()
        _lib.check(lib.lfm_create(C.byref(desc), dev_index, C.byref(ctx)))
        if self.fp8:
            rc = lib.lfm_set_fp8(ctx, 1)
            if rc != 0:
                msg = _lib.last_error(ctx)
                lib.lfm_destroy(ctx)
                raise RuntimeError("liblfm_b200: " + msg)
        return ctx

    # -- model(t, x, y)  (reference models/DiT.py:252-272) -----------------------------------------------------
    def forward(self, t, x, y=None, **kwargs):
        t, x, y, B = self._prep(t, x, y)
        return self._forward_native(t, x, y)

    # -- model.forward_with_cfg(t, x, y, cfg_scale)  (reference models/DiT.py:274-290) ------------------------
    def forward_with_cfg(self, t, x, y=None, cfg_scale=1.0, **kwargs):
        t, x, y, B = self._prep(t, x, y)
        if B % 2:
            raise ValueError("forward_with_cfg expects the doubled batch [x, x]")
        if y is None:
            y = torch.full((B,), self.table_rows - 1, dtype=torch.int64, device=x.device)
        if cfg_scale > 1.0:
            return self._forward_native(t, x, y, cfg_scale)
        # cfg_scale <= 1: g = u + s (c - u) still holds; evaluate the plain doubled batch and combine here
        half = x[: B // 2]
        out = self.forward(t, torch.cat([half, half], 0), y)
        c, u = out[: B // 2], out[B // 2:]
        g = u + cfg_scale * (c - u)
        return torch.cat([g, g], 0)

def _dit(depth, hidden_size, patch_size, num_heads):
    def make(**kwargs):
        return DiT(depth=depth, hidden_size=hidden_size, patch_size=patch_size, num_heads=num_heads, **kwargs)
    return make


# reference models/DiT.py:355-415
DiT_models = {
    "DiT-XL/2": _dit(28, 1152, 2, 16), "DiT-XL/4": _dit(28, 1152, 4, 16), "DiT-XL/8": _dit(28, 1152, 8, 16),
    "DiT-L/2": _dit(24, 1024, 2, 16), "DiT-L/4": _dit(24, 1024, 4, 16), "DiT-L/8": _dit(24, 1024, 8, 16),
    "DiT-B/2": _dit(12, 768, 2, 12), "DiT-B/4": _dit(12, 768, 4, 12), "DiT-B/8": _dit(12, 768, 8, 12),
    "DiT-S/2": _dit(12, 384, 2, 6), "DiT-S/4": _dit(12, 384, 4, 6), "DiT-S/8": _dit(12, 384, 8, 6),
}


def create_network(config):
    """reference models/__init__.py:6-17: UNetModel (--use_origin_adm), the EDM family (model_type without "DiT":
    only "adm" = DhariwalUNet is native) or a DiT.  ``config.fp8`` (absent = False) selects the DiT's FP8 mode, which
    the UNets do not have."""
    fp8 = bool(getattr(config, "fp8", False))
    if fp8 and (getattr(config, "use_origin_adm", False) or "DiT" not in config.model_type):
        raise ValueError("fp8 is implemented for the DiT models only, not for the ADM / EDM UNets "
                         f"(model_type {config.model_type!r}, use_origin_adm {getattr(config, 'use_origin_adm', False)})")
    if getattr(config, "use_origin_adm", False):
        return get_flow_model(config)
    if "DiT" not in config.model_type:
        from .edm import get_edm_network
        return get_edm_network(config)
    return DiT_models[config.model_type](
        img_resolution=config.image_size // config.f,
        in_channels=config.num_in_channels,
        label_dropout=config.label_dropout,
        num_classes=config.num_classes,
        fp8=fp8,
    )


def get_flow_model(config):
    """reference models/__init__.py:20-70: the OpenAI-ADM UNetModel selected by --use_origin_adm."""
    from .unet import UNetModel
    if getattr(config, "layout", False):
        raise NotImplementedError("UNetModelAttn (--layout, cross-attention conditioning) is outside the hot path")
    return UNetModel(
        image_size=config.image_size // 8,
        in_channels=config.num_in_channels,
        model_channels=config.nf,
        out_channels=config.num_out_channels,
        num_res_blocks=config.num_res_blocks,
        attention_resolutions=config.attn_resolutions,
        dropout=config.dropout,
        channel_mult=config.ch_mult,
        conv_resample=config.resamp_with_conv,
        dims=2,
        num_classes=config.num_classes,
        use_checkpoint=False,
        use_fp16=False,
        num_heads=config.num_heads,
        num_head_channels=config.num_head_channels,
        num_heads_upsample=config.num_head_upsample,
        use_scale_shift_norm=config.use_scale_shift_norm,
        resblock_updown=config.resblock_updown,
        use_new_attention_order=config.use_new_attention_order,
    )
