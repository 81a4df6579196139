"""The library baseline of bench.py's `gpu_eager_baseline` leg: the reference DiT in plain eager PyTorch on the GPU,
the way a user of the reference would run it on a GPU - `F.scaled_dot_product_attention` (what timm's Attention
dispatches to), optional bf16 autocast, TF32 on (test_flow_latent_ddp.py:23).  Self-contained torch.nn.functional
code over the reference's state_dict keys (models/DiT.py:112-131,252-272; timm PatchEmbed / Attention / Mlp).

BASELINE / TEST TOOLING ONLY: nothing under lfm_b200/ imports this file, and it never calls liblfm_b200.so.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def _modulate(x, shift, scale):
    return x * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1)          # models/DiT.py:20-21


def timestep_embedding(t, dim=256, max_period=10000):
    half = dim // 2                                                   # models/DiT.py:43-63 (cos first, raw t)
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


@torch.no_grad()
def dit_forward(sd, t, x, y=None, *, depth, hidden, heads, patch=2):
    """model(t, x, y) of models/DiT.py:252-272 with the parameters of `sd` (reference key names, CUDA tensors)."""
    B, C, H, W = x.shape
    D, dh = hidden, hidden // heads
    h = F.conv2d(x, sd["x_embedder.proj.weight"], sd["x_embedder.proj.bias"], stride=patch)
    h = h.flatten(2).transpose(1, 2) + sd["pos_embed"]
    t = torch.as_tensor(t, dtype=torch.float32, device=x.device).reshape(-1)
    te = timestep_embedding(t)
    te = F.linear(F.silu(F.linear(te, sd["t_embedder.mlp.0.weight"], sd["t_embedder.mlp.0.bias"])),
                  sd["t_embedder.mlp.2.weight"], sd["t_embedder.mlp.2.bias"])
    table = sd["y_embedder.embedding_table.weight"]
    if y is None:
        y = torch.full((B,), table.shape[0] - 1, dtype=torch.long, device=x.device)   # models/DiT.py:259-260
    c = F.silu(te + table[y])
    T = h.shape[1]
    for i in range(depth):
        p = f"blocks.{i}."
        m = F.linear(c, sd[p + "adaLN_modulation.1.weight"], sd[p + "adaLN_modulation.1.bias"]).chunk(6, dim=1)
        a = _modulate(F.layer_norm(h, (D,), eps=1e-6), m[0], m[1])
        qkv = F.linear(a, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(B, T, 3, heads, dh).permute(2, 0, 3, 1, 4)
        o = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2])   # timm Attention (fused kernel)
        o = F.linear(o.transpose(1, 2).reshape(B, T, D), sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
        h = h + m[2].unsqueeze(1) * o
        a = _modulate(F.layer_norm(h, (D,), eps=1e-6), m[3], m[4])
        a = F.linear(F.gelu(F.linear(a, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]), approximate="tanh"),
                     sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])
        h = h + m[5].unsqueeze(1) * a
    m = F.linear(c, sd["final_layer.adaLN_modulation.1.weight"], sd["final_layer.adaLN_modulation.1.bias"]).chunk(2, dim=1)
    h = _modulate(F.layer_norm(h, (D,), eps=1e-6), m[0], m[1])
    h = F.linear(h, sd["final_layer.linear.weight"], sd["final_layer.linear.bias"])
    g = H // patch
    h = h.reshape(B, g, g, patch, patch, C)
    return torch.einsum("nhwpqc->nchpwq", h).reshape(B, C, H, W).float()


@torch.no_grad()
def euler(sd, x, nodes, *, autocast_bf16, **arch):
    """torchdiffeq fixed-grid Euler over the model-time nodes (the loop bench.py's own arm runs natively)."""
    for k in range(len(nodes) - 1):
        t = nodes[k]
        if autocast_bf16:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                v = dit_forward(sd, t, x, **arch)
        else:
            v = dit_forward(sd, t, x, **arch)
        x = x + (nodes[k + 1] - nodes[k]) * v
    return x
