"""The DiT forward of the FP8 mode (lfm_set_fp8), restated on top of the oracle's layers (oracle/dit.py).

It is the oracle's bf16 emulation (emulate_bf16=True: bf16 operands of every GEMM, bf16 stored activations) with the qkv and fc1
GEMMs replaced by the FP8 mode's arithmetic:
  * the LayerNorm-modulate output v [M, D] is quantised per row:  s = amax|v| / 448 (1 for an all-zero row), codes = e4m3(v / s);
  * the weight [N, K] is quantised per output channel the same way, from its fp32 values;
  * out = (codes_v codes_w^T) s_v s_w + bias, the product summed exactly (fp64 here, fp32 on the device).
Zero-padding the weight rows of DiT-XL's 72-channel heads to 80 only adds rows whose outputs the attention never reads, so the
timm-order weight is quantised here as it is.
"""
import torch
import torch.nn.functional as F

from oracle import dit as odit

E4M3_MAX = 448.0


def quantize_rows(v):
    """Per-row e4m3 quantisation of v [..., K] (fp32): (codes as torch.float8_e4m3fn, scales fp32 [...])."""
    v = v.float()
    amax = v.abs().amax(dim=-1, keepdim=True)
    # a tensor divisor: torch divides by a python scalar as a product with its rounded reciprocal on the GPU
    s = torch.where(amax > 0, amax / torch.full_like(amax, E4M3_MAX), torch.ones_like(amax))
    return (v / s).to(torch.float8_e4m3fn), s.squeeze(-1)


def fp8_linear(x, w, b):
    """x [..., K] @ w[N, K]^T + b on per-row e4m3 operands, fp32 result."""
    qx, sx = quantize_rows(x)
    qw, sw = quantize_rows(w)
    acc = (qx.double() @ qw.double().t()).float()
    return acc * sx.unsqueeze(-1) * sw + b


def _attention(sd, pre, cfg, x):
    B, N, D = x.shape
    H = cfg.num_heads
    dh = D // H
    qkv = odit._r(fp8_linear(x, sd[pre + "qkv.weight"], sd[pre + "qkv.bias"]), True)
    qkv = qkv.reshape(B, N, 3, H, dh).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    s = (q * dh ** -0.5) @ k.transpose(-2, -1)
    e = torch.exp(s - s.amax(dim=-1, keepdim=True))
    o = (odit._r(e, True) @ v) / e.sum(dim=-1, keepdim=True)
    o = odit._r(o.transpose(1, 2).reshape(B, N, D), True)
    return odit._linear(o, sd[pre + "proj.weight"], sd[pre + "proj.bias"], True)


def _mlp(sd, pre, x):
    h = F.gelu(fp8_linear(x, sd[pre + "fc1.weight"], sd[pre + "fc1.bias"]), approximate="tanh")
    return odit._linear(odit._r(h, True), sd[pre + "fc2.weight"], sd[pre + "fc2.bias"], True)


def _block(sd, i, cfg, x, c):
    pre = f"blocks.{i}."
    mod = F.linear(F.silu(c), sd[pre + "adaLN_modulation.1.weight"], sd[pre + "adaLN_modulation.1.bias"])
    sh1, sc1, g1, sh2, sc2, g2 = mod.chunk(6, dim=1)
    x = x + g1.unsqueeze(1) * _attention(sd, pre + "attn.", cfg, odit._ln_mod(x, sh1, sc1))
    x = x + g2.unsqueeze(1) * _mlp(sd, pre + "mlp.", odit._ln_mod(x, sh2, sc2))
    return x


@torch.no_grad()
def dit_forward_fp8(sd, cfg, t, x, y=None):
    """odit.dit_forward(..., emulate_bf16=True) with the FP8 mode's qkv and fc1."""
    t = torch.as_tensor(t, dtype=torch.float32, device=x.device)
    B = x.shape[0]
    h = odit.patch_embed(sd, cfg, x.float(), True)
    c = odit.conditioning(sd, cfg, t, y, B, True)
    if c.shape[0] == 1 and B != 1:
        c = c.expand(B, -1)
    for i in range(cfg.depth):
        h = _block(sd, i, cfg, h, c)
    return odit.unpatchify(cfg, odit.final_layer(sd, cfg, h, c))


@torch.no_grad()
def dit_forward_with_cfg_fp8(sd, cfg, t, x, y, cfg_scale):
    half = x[: len(x) // 2]
    out = dit_forward_fp8(sd, cfg, t, torch.cat([half, half], dim=0), y)
    cond, uncond = torch.split(out, len(out) // 2, dim=0)
    g = uncond + cfg_scale * (cond - uncond)
    return torch.cat([g, g], dim=0)
