"""Host-side mirror of the reference's EDM-style ADM network ``DhariwalUNet`` (models/EDM.py:716-861), the class
``create_network`` returns for ``--model_type adm`` without ``--use_origin_adm`` (ffhq_adm / bed_adm / imnet_adm
presets, models/__init__.py:10-11 -> ``get_edm_network`` models/EDM.py:864-937).

Parameters and buffers live in an ``nn.Module`` tree with the reference's ``state_dict`` keys and order
(``map_layer{0,1}``, ``map_label``, ``enc.{r}x{r}_{conv,down,block{i}}``, ``dec.{r}x{r}_{in0,in1,up,block{i}}`` with
``norm0 conv0 affine norm1 conv1 skip norm2 qkv proj``, the constant ``resample_filter`` buffers of the up / down
blocks, ``out_norm``, ``out_conv``); the compute is liblfm_b200.so (``lfm_create_edm``).  No PyTorch forward, no fallback.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn

from . import _lib
from .network import _Holder, _NativeNet


class _W(nn.Module):
    """A leaf with the reference's parameter names.  Initialisation follows ``weight_init`` (EDM.py:27-36) with
    DhariwalUNet's ``init`` / ``init_zero`` dictionaries (EDM.py:741-742)."""

    def __init__(self, shape, fan_in, bias=True, scale=math.sqrt(1 / 3), mode="kaiming_uniform", resample=False):
        super().__init__()
        if mode == "kaiming_uniform":
            w = math.sqrt(3 / fan_in) * (torch.rand(*shape) * 2 - 1)
            b = math.sqrt(3 / fan_in) * (torch.rand(shape[0]) * 2 - 1)
        else:  # kaiming_normal
            w = math.sqrt(1 / fan_in) * torch.randn(*shape)
            b = math.sqrt(1 / fan_in) * torch.randn(shape[0])
        self.weight = nn.Parameter(w * scale)
        if bias:
            self.bias = nn.Parameter(b * scale)
        if resample:
            self.register_buffer("resample_filter", torch.full((1, 1, 2, 2), 0.25))


class _Resample(nn.Module):
    """``Conv2d(kernel=0, up / down)``: the weight-free skip of a resampling block - only the constant buffer."""

    def __init__(self):
        super().__init__()
        self.register_buffer("resample_filter", torch.full((1, 1, 2, 2), 0.25))


class _Norm(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))


def _unet_block(cin, cout, emb, attention=False, up=False, down=False):
    """UNetBlock.__init__ (EDM.py:188-252): registration order = state_dict order."""
    b = _Holder()
    resample = up or down
    b.norm0 = _Norm(cin)
    b.conv0 = _W((cout, cin, 3, 3), cin * 9, resample=resample)
    b.affine = _W((2 * cout, emb), emb)
    b.norm1 = _Norm(cout)
    b.conv1 = _W((cout, cout, 3, 3), cout * 9, scale=0.0)
    if cout != cin:
        b.skip = _W((cout, cin, 1, 1), cin, resample=resample)
    elif resample:
        b.skip = _Resample()
    if attention:
        b.norm2 = _Norm(cout)
        b.qkv = _W((3 * cout, cout, 1, 1), cout)
        b.proj = _W((cout, cout, 1, 1), cout, scale=0.0)
    return b


class DhariwalUNet(_NativeNet):
    """H100-native DhariwalUNet with the reference's constructor (models/EDM.py:717-733)."""

    def __init__(self, img_resolution, in_channels, out_channels, label_dim=0, augment_dim=0, model_channels=192,
                 channel_mult=(1, 2, 3, 4), channel_mult_emb=4, num_blocks=3, attn_resolutions=(32, 16, 8), dropout=0.10,
                 label_dropout=0, use_context=False, max_batch=None):
        super().__init__()
        if use_context:
            raise NotImplementedError("use_context=True (UNetBlockWithContext, model_type adm_context) is outside the hot path")
        if augment_dim:
            raise NotImplementedError("augment_dim != 0 is not used by get_edm_network (EDM.py:911)")
        if channel_mult_emb != 4:
            raise NotImplementedError("channel_mult_emb must be 4 (EDM.py:913)")
        self.img_resolution, self.in_channels, self.out_channels = img_resolution, in_channels, out_channels
        self.label_dim, self.label_dropout = int(label_dim), label_dropout
        self.model_channels, self.num_blocks = model_channels, num_blocks
        self.channel_mult = tuple(int(m) for m in channel_mult)
        self.attn_resolutions = tuple(int(a) for a in attn_resolutions)
        self.table_rows = self.label_dim + 1     # the extra index = a dropped label (all-zero one-hot)
        self.max_batch_hint = max_batch
        self.use_context = False
        E = model_channels * channel_mult_emb
        self.map_layer0 = _W((E, model_channels), model_channels)
        self.map_layer1 = _W((E, E), E)
        if self.label_dim:
            self.map_label = _W((E, self.label_dim), self.label_dim, bias=False, scale=math.sqrt(self.label_dim),
                                mode="kaiming_normal")
        # encoder (EDM.py:764-782)
        self.enc = nn.ModuleDict()
        cout = in_channels
        for level, mult in enumerate(self.channel_mult):
            res = img_resolution >> level
            if level == 0:
                cin, cout = cout, model_channels * mult
                self.enc[f"{res}x{res}_conv"] = _W((cout, cin, 3, 3), cin * 9)
            else:
                self.enc[f"{res}x{res}_down"] = _unet_block(cout, cout, E, down=True)
            for idx in range(num_blocks):
                cin, cout = cout, model_channels * mult
                self.enc[f"{res}x{res}_block{idx}"] = _unet_block(cin, cout, E, attention=res in self.attn_resolutions)
        skips = [model_channels * self.channel_mult[0]]
        for level, mult in enumerate(self.channel_mult):
            if level:
                skips.append(model_channels * self.channel_mult[level - 1])
            skips += [model_channels * mult] * num_blocks
        # decoder (EDM.py:785-805)
        self.dec = nn.ModuleDict()
        for level, mult in reversed(list(enumerate(self.channel_mult))):
            res = img_resolution >> level
            if level == len(self.channel_mult) - 1:
                self.dec[f"{res}x{res}_in0"] = _unet_block(cout, cout, E, attention=True)
                self.dec[f"{res}x{res}_in1"] = _unet_block(cout, cout, E)
            else:
                self.dec[f"{res}x{res}_up"] = _unet_block(cout, cout, E, up=True)
            for idx in range(num_blocks + 1):
                cin = cout + skips.pop()
                cout = model_channels * mult
                self.dec[f"{res}x{res}_block{idx}"] = _unet_block(cin, cout, E, attention=res in self.attn_resolutions)
        self.out_norm = _Norm(cout)
        self.out_conv = _W((out_channels, cout, 3, 3), cout * 9, scale=0.0)
        self.requires_grad_(False)
        self._init_native()

    def _create_ctx(self, lib, dev_index):
        cm, ar = self.channel_mult, self.attn_resolutions
        d = _lib.EdmDesc(self.img_resolution, self.in_channels, self.out_channels, self.label_dim, self.model_channels,
                         len(cm), (C.c_int32 * 8)(*cm), self.num_blocks, len(ar), (C.c_int32 * 8)(*ar))
        ctx = C.c_void_p()
        _lib.check(lib.lfm_create_edm(C.byref(d), dev_index, C.byref(ctx)))
        return ctx

    def uses_labels(self):
        return bool(self.label_dim)          # without map_label a y argument is ignored (EDM.py:823)

    def check_label_range(self, y):
        if y.numel() and (int(y.min()) < 0 or int(y.max()) >= self.label_dim):
            raise RuntimeError("Class values must be smaller than num_classes.")   # what F.one_hot raises

    def _labels(self, y, B, drop_half_label):
        """one_hot(y, label_dim) semantics (EDM.py:824): labels must be class ids; a dropped label is encoded as
        index label_dim (the all-zero row of the native table)."""
        if not self.label_dim or y is None:
            return None                      # map_label is None, or the label term is skipped (EDM.py:823)
        y = torch.as_tensor(y).to(torch.int64)
        if y.numel() != B:
            raise ValueError(f"y has {y.numel()} labels, expected {B}")
        self.check_label_range(y)
        if drop_half_label:
            y = y.clone()
            y[B // 2:] = self.label_dim
        return y

    # model(t, x, y)   (EDM.py:812-845)
    def forward(self, noise_labels, x, y=None, augment_labels=None, drop_half_label=False, **kwargs):
        y = self._labels(y, x.shape[0], drop_half_label)
        t, x, y, B = self._prep(noise_labels, x, y)
        return self._forward_native(t, x, y)

    # model.forward_with_cfg(t, x, y, cfg_scale)   (EDM.py:847-861)
    def forward_with_cfg(self, noise_labels, x, y=None, augment_labels=None, cfg_scale=1.0, **kwargs):
        B = x.shape[0]
        if B % 2:
            raise ValueError("forward_with_cfg expects the doubled batch [x, x]")
        if cfg_scale > 1.0:
            y = self._labels(y, B, True)
            t, x, y, B = self._prep(noise_labels, x, y)
            return self._forward_native(t, x, y, cfg_scale)
        half = x[: B // 2]
        out = self.forward(noise_labels, torch.cat([half, half], 0), y, drop_half_label=True)
        c, u = out[: B // 2], out[B // 2:]
        g = u + cfg_scale * (c - u)
        return torch.cat([g, g], 0)


def get_edm_network(config):
    """reference models/EDM.py:864-937.  Only ``model_type == "adm"`` (the LFM ADM presets) is native."""
    if config.model_type != "adm":
        raise NotImplementedError(f"model_type '{config.model_type}' (SongUNet / context ADM) is outside the native hot path; "
                                  "'adm' (DhariwalUNet) and the DiT family are native")
    return DhariwalUNet(
        img_resolution=config.image_size // config.f,
        in_channels=config.num_in_channels,
        out_channels=config.num_out_channels,
        label_dim=config.label_dim,
        augment_dim=0,
        model_channels=config.nf,
        channel_mult=config.ch_mult,
        channel_mult_emb=4,
        num_blocks=config.num_res_blocks,
        attn_resolutions=config.attn_resolutions,
        dropout=config.dropout,
        label_dropout=config.label_dropout,
    )
