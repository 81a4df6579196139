"""Oracle: the encoder half of the Stable-Diffusion ``AutoencoderKL`` (TEST INFRASTRUCTURE; PARITY UNPINNED).

The inpainting loop (downstream_tasks/test_flow_latent_inpainting.py:147) calls
``first_stage_model.encode(masked_image).latent_dist.sample()``.  ``diffusers`` is absent here, so, like oracle/vae.py for the
decoder, this file RESTATES the published architecture (diffusers ``models/autoencoders/vae.py`` ``Encoder``;
``models/downsampling.py`` ``Downsample2D``; ``models/autoencoders/vae.py`` ``DiagonalGaussianDistribution``; as of
diffusers 0.2x) with the sd-vae-ft-mse config, and parity of the native encoder is anchored on this restatement only:

    encode(x):  h = conv_in(x)                                       3x3, 3 -> 128, pad 1
                for i, ch in enumerate((128, 256, 512, 512)):
                    2 x ResnetBlock2D(-> ch)  (first one changes the width: 1x1 conv_shortcut)
                    if i < 3: Downsample2D(padding=0): F.pad(h, (0, 1, 0, 1)) then conv3x3 stride 2, pad 0
                h = mid.resnets[0](h); h = mid.attentions[0](h); h = mid.resnets[1](h)     (as the decoder's)
                h = conv_out(silu(conv_norm_out(h)))                 GroupNorm(32, 512) -> SiLU -> 3x3, 512 -> 8
                moments = quant_conv(h)                              1x1, 8 -> 8
                mean, logvar = moments.chunk(2, dim=1); logvar = clamp(logvar, -30, 20)

The ResnetBlock2D and attention restatements, the synthetic-weight recipe and the operand-rounding emulation
(``emulate_bf16``) are oracle/vae.py's; the 3-channel conv_in and quant_conv run in fp32 on the native side too.
"""
from __future__ import annotations

import math
import zlib

import torch
import torch.nn.functional as F

from oracle import vae as ovae


def encoder_plan(cfg: ovae.VAEConfig = ovae.VAEConfig()):
    """[(prefix, kind, cin, cout)] in execution order after conv_in; kind in {res, down, attn}."""
    ch = cfg.block_out_channels[0]
    plan = []
    for i, out in enumerate(cfg.block_out_channels):
        for j in range(cfg.layers_per_block):
            plan.append((f"encoder.down_blocks.{i}.resnets.{j}", "res", ch, out))
            ch = out
        if i != len(cfg.block_out_channels) - 1:
            plan.append((f"encoder.down_blocks.{i}.downsamplers.0", "down", ch, ch))
    plan += [("encoder.mid_block.resnets.0", "res", ch, ch), ("encoder.mid_block.attentions.0", "attn", ch, ch),
             ("encoder.mid_block.resnets.1", "res", ch, ch)]
    return plan, ch


def encoder_param_shapes(cfg: ovae.VAEConfig = ovae.VAEConfig(), image_channels: int = 3):
    """Ordered {key: shape} of the ``encoder.*`` and ``quant_conv.*`` entries of the diffusers state dict."""
    plan, c_last = encoder_plan(cfg)
    c0, L2 = cfg.block_out_channels[0], 2 * cfg.latent_channels
    sh = {"encoder.conv_in.weight": (c0, image_channels, 3, 3), "encoder.conv_in.bias": (c0,)}
    for p, kind, cin, cout in plan:
        if kind == "res":
            sh[p + ".norm1.weight"] = (cin,)
            sh[p + ".norm1.bias"] = (cin,)
            sh[p + ".conv1.weight"] = (cout, cin, 3, 3)
            sh[p + ".conv1.bias"] = (cout,)
            sh[p + ".norm2.weight"] = (cout,)
            sh[p + ".norm2.bias"] = (cout,)
            sh[p + ".conv2.weight"] = (cout, cout, 3, 3)
            sh[p + ".conv2.bias"] = (cout,)
            if cin != cout:
                sh[p + ".conv_shortcut.weight"] = (cout, cin, 1, 1)
                sh[p + ".conv_shortcut.bias"] = (cout,)
        elif kind == "attn":
            sh[p + ".group_norm.weight"] = (cin,)
            sh[p + ".group_norm.bias"] = (cin,)
            for n in ("to_q", "to_k", "to_v", "to_out.0"):
                sh[f"{p}.{n}.weight"] = (cin, cin)
                sh[f"{p}.{n}.bias"] = (cin,)
        else:
            sh[p + ".conv.weight"] = (cout, cin, 3, 3)
            sh[p + ".conv.bias"] = (cout,)
    sh["encoder.conv_norm_out.weight"] = (c_last,)
    sh["encoder.conv_norm_out.bias"] = (c_last,)
    sh["encoder.conv_out.weight"] = (L2, c_last, 3, 3)
    sh["encoder.conv_out.bias"] = (L2,)
    sh["quant_conv.weight"] = (L2, L2, 1, 1)
    sh["quant_conv.bias"] = (L2,)
    return sh


def full_param_shapes(cfg: ovae.VAEConfig = ovae.VAEConfig()):
    """{key: shape} of the whole AutoencoderKL checkpoint: the encoder's 108 entries and the decoder's 140."""
    return {**encoder_param_shapes(cfg), **ovae.param_shapes(cfg)}


def synthetic_state_dict(cfg: ovae.VAEConfig = ovae.VAEConfig(), seed: int = 1):
    """oracle.vae.synthetic_state_dict's per-key (seed, crc32(key)) recipe over the full checkpoint: the decoder tensors
    are exactly the decoder-only ones."""
    sd = {}
    for k, shp in encoder_param_shapes(cfg).items():
        g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(k.encode()))
        leaf = k.rsplit(".", 2)[-2]
        if "norm" in leaf:
            sd[k] = (1.0 + 0.1 * torch.randn(shp, generator=g)) if k.endswith("weight") else 0.1 * torch.randn(shp, generator=g)
        elif k.endswith(".bias"):
            sd[k] = 0.02 * torch.randn(shp, generator=g)
        else:
            fan_in = int(math.prod(shp[1:]))
            sd[k] = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(fan_in)
    sd.update(ovae.synthetic_state_dict(cfg, seed))
    return sd


def downsample(x, w, b):
    """Downsample2D(padding=0): F.pad(x, (0, 1, 0, 1)) then conv3x3 stride 2 (operands rounded under emulate_bf16)."""
    return ovae._conv(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)


@torch.no_grad()
def vae_encode(sd, x, cfg: ovae.VAEConfig = ovae.VAEConfig(), emulate_bf16: bool = False):
    """``AutoencoderKL.encode(x).latent_dist`` moments: x [B, 3, S, S] fp32 -> (mean, logvar) [B, 4, S/8, S/8] fp32."""
    was = ovae._EMULATE_BF16
    ovae._EMULATE_BF16 = emulate_bf16
    try:
        plan, _ = encoder_plan(cfg)
        h = F.conv2d(x, sd["encoder.conv_in.weight"], sd["encoder.conv_in.bias"], padding=1)
        for p, kind, cin, cout in plan:
            if kind == "res":
                h = ovae.resnet_block(sd, p, h, cfg)
            elif kind == "attn":
                h = ovae.attention_block(sd, p, h, cfg)
            else:
                h = downsample(h, sd[p + ".conv.weight"], sd[p + ".conv.bias"])
        h = F.silu(ovae._gn(h, sd, "encoder.conv_norm_out", cfg))
        h = ovae._conv(h, sd["encoder.conv_out.weight"], sd["encoder.conv_out.bias"], padding=1)
        moments = F.conv2d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])
    finally:
        ovae._EMULATE_BF16 = was
    mean, logvar = moments.chunk(2, dim=1)
    return mean, torch.clamp(logvar, -30.0, 20.0)


def encode_flops_per_image(cfg: ovae.VAEConfig = ovae.VAEConfig(), image_side: int = 256) -> float:
    """Algorithmic FLOPs (2 x MAC) of one encode: the convolutions, quant_conv, the four attention projections and the two
    attention GEMMs."""
    plan, c_last = encoder_plan(cfg)
    side = image_side
    fl = 2.0 * side * side * 9 * 3 * cfg.block_out_channels[0]
    for p, kind, cin, cout in plan:
        px = side * side
        if kind == "res":
            fl += 2.0 * px * 9 * (cin * cout + cout * cout) + (2.0 * px * cin * cout if cin != cout else 0.0)
        elif kind == "attn":
            fl += 2.0 * px * 4 * cin * cin + 4.0 * px * px * cin
        else:
            side //= 2
            fl += 2.0 * side * side * 9 * cin * cout
    L2 = 2 * cfg.latent_channels
    fl += 2.0 * side * side * (9 * c_last * L2 + L2 * L2)
    return fl
