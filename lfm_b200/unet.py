"""Host-side mirror of the reference's OpenAI-ADM ``UNetModel`` (models/guided_diffusion/unet.py:376-655).

Parameters live in an ``nn.Module`` tree with the reference's ``state_dict`` keys (``time_embed.{0,2}``,
``input_blocks.N.M.{in_layers,emb_layers,out_layers,skip_connection,norm,qkv,proj_out,op}``, ``middle_block``,
``output_blocks``, ``out.{0,2}``); the compute is liblfm_b200.so (wgmma implicit-GEMM convolutions, fused
GroupNorm/SiLU/FiLM, attention).  Only the configuration the LFM presets use is native:
``use_scale_shift_norm=True``, ``resblock_updown=False``, ``conv_resample=True``, legacy attention order, dims=2.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from .network import _Holder, _NativeNet


def _zero(m):
    for p in m.parameters():
        nn.init.zeros_(p)
    return m


def _res_block(cin, cout, emb):
    b = _Holder()
    b.in_layers = nn.Sequential(nn.GroupNorm(32, cin), nn.SiLU(), nn.Conv2d(cin, cout, 3, padding=1))
    b.emb_layers = nn.Sequential(nn.SiLU(), nn.Linear(emb, 2 * cout))
    b.out_layers = nn.Sequential(nn.GroupNorm(32, cout), nn.SiLU(), nn.Dropout(p=0.0),
                                 _zero(nn.Conv2d(cout, cout, 3, padding=1)))       # zero_module, unet.py:198
    b.skip_connection = nn.Identity() if cin == cout else nn.Conv2d(cin, cout, 1)
    return b


def _attn_block(ch):
    b = _Holder()
    b.norm = nn.GroupNorm(32, ch)
    b.qkv = nn.Conv1d(ch, 3 * ch, 1)
    b.proj_out = _zero(nn.Conv1d(ch, ch, 1))                                       # zero_module, unet.py:276
    return b


class _Seq(nn.Module):
    """TimestepEmbedSequential stand-in: children registered as "0", "1", ... (parameter names only)."""

    def __init__(self, *mods):
        super().__init__()
        for i, m in enumerate(mods):
            self.add_module(str(i), m)


class UNetModel(_NativeNet):
    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, num_classes=None, use_checkpoint=False,
                 use_fp16=False, num_heads=1, num_head_channels=-1, num_heads_upsample=-1, use_scale_shift_norm=False,
                 resblock_updown=False, use_new_attention_order=False, max_batch=None):
        super().__init__()
        if not use_scale_shift_norm or resblock_updown or not conv_resample or use_new_attention_order or dims != 2 or use_fp16:
            raise NotImplementedError("native UNetModel implements the LFM preset configuration only: "
                                      "use_scale_shift_norm=True, resblock_updown=False, conv_resample=True, "
                                      "legacy attention order, dims=2, fp32 parameters")
        if num_heads_upsample not in (-1, num_heads):
            raise NotImplementedError("num_heads_upsample != num_heads (a different head count in the output-block "
                                      "attention, unet.py:452-453) is not implemented natively")
        self.dropout = dropout   # a training-time option: the sampling path runs in eval mode, where Dropout is the identity
        self.image_size, self.in_channels, self.model_channels, self.out_channels = image_size, in_channels, model_channels, out_channels
        self.num_res_blocks = num_res_blocks
        self.attention_resolutions = tuple(int(a) for a in attention_resolutions)
        self.channel_mult = tuple(int(m) for m in channel_mult)
        self.num_classes, self.num_heads, self.num_head_channels = num_classes, num_heads, num_head_channels
        self.table_rows = num_classes or 0
        self.max_batch_hint = max_batch
        E = model_channels * 4
        self.time_embed = nn.Sequential(nn.Linear(model_channels, E), nn.SiLU(), nn.Linear(E, E))
        if num_classes is not None:
            self.label_emb = nn.Embedding(num_classes, E)
        ch = int(self.channel_mult[0] * model_channels)
        blocks = [_Seq(nn.Conv2d(in_channels, ch, 3, padding=1))]
        chans, ds = [ch], 1
        for level, mult in enumerate(self.channel_mult):
            for _ in range(num_res_blocks):
                layers = [_res_block(ch, int(mult * model_channels), E)]
                ch = int(mult * model_channels)
                if ds in self.attention_resolutions:
                    layers.append(_attn_block(ch))
                blocks.append(_Seq(*layers))
                chans.append(ch)
            if level != len(self.channel_mult) - 1:
                down = _Holder()
                down.op = nn.Conv2d(ch, ch, 3, stride=2, padding=1)
                blocks.append(_Seq(down))
                chans.append(ch)
                ds *= 2
        self.input_blocks = nn.ModuleList(blocks)
        self.middle_block = _Seq(_res_block(ch, ch, E), _attn_block(ch), _res_block(ch, ch, E))
        outs = []
        for level, mult in list(enumerate(self.channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                ich = chans.pop()
                layers = [_res_block(ch + ich, int(model_channels * mult), E)]
                ch = int(model_channels * mult)
                if ds in self.attention_resolutions:
                    layers.append(_attn_block(ch))
                if level and i == num_res_blocks:
                    up = _Holder()
                    up.conv = nn.Conv2d(ch, ch, 3, padding=1)
                    layers.append(up)
                    ds //= 2
                outs.append(_Seq(*layers))
        self.output_blocks = nn.ModuleList(outs)
        self.out = nn.Sequential(nn.GroupNorm(32, ch), nn.SiLU(), _zero(nn.Conv2d(ch, out_channels, 3, padding=1)))
        self.requires_grad_(False)
        self._init_native()

    def _create_ctx(self, lib, dev_index):
        ar, cm = self.attention_resolutions, self.channel_mult
        d = _lib.UnetDesc(self.image_size, self.in_channels, self.model_channels, self.out_channels, self.num_res_blocks,
                          len(ar), (C.c_int32 * 8)(*ar), len(cm), (C.c_int32 * 8)(*cm), self.num_heads,
                          self.num_head_channels, self.num_classes or 0)
        ctx = C.c_void_p()
        _lib.check(lib.lfm_create_unet(C.byref(d), dev_index, C.byref(ctx)))
        return ctx

    # model(t, x, y)   (unet.py:613-655; a 0-d t is expanded to the batch, :629-630)
    def forward(self, timesteps, x, y=None, **kwargs):
        assert (y is not None) == (self.num_classes is not None), \
            "must specify y if and only if the model is class-conditional"
        t, x, y, B = self._prep(timesteps, x, y)
        if x.dim() != 4 or x.shape[1] != self.in_channels:
            raise ValueError(f"x must be [B, {self.in_channels}, H, W] (got {tuple(x.shape)})")
        return self._forward_native(t, x, y)
