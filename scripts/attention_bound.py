"""The 256-token attention of DiT-L/2 at batch 64 (B*H = 1024 heads of 256 x 64) on cuda:0: kernel time (CUDA events) against the
least time its bytes and FLOPs allow, and its share of one network evaluation.

    python scripts/attention_bound.py

Bytes: the qkv rows are read once and the output written once (100 MB + 33.5 MB); FLOPs 4 T^2 d per head.  The memory bound uses the
device-to-device copy rate measured in the same process (and the data-sheet HBM rate); the tensor bound the data-sheet dense bf16 rate.
Prints one JSON line."""
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lfm_b200 import _lib  # noqa: E402

B, H, T, DH, L = 64, 16, 256, 64, 24
dev = torch.device("cuda:0")


def event_ms(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


lib = _lib.load()
D = H * DH
qkv = torch.randn(B * T, 3 * D, device=dev).bfloat16()
out = torch.empty(B * T, D, device=dev, dtype=torch.bfloat16)
s = C.c_void_p(torch.cuda.current_stream().cuda_stream)


def attn():
    assert lib.lfm_dbg_attention(C.c_void_p(qkv.data_ptr()), C.c_void_p(out.data_ptr()), B, H, 0, None, s) == 0, _lib.last_error()


src = torch.empty(512 << 20, dtype=torch.uint8, device=dev)   # 512 MB each way: far beyond the 50 MB L2
dst = torch.empty_like(src)
copy_ms = event_ms(lambda: dst.copy_(src), 20)
copy_gbs = 2 * src.numel() / (copy_ms * 1e-3) / 1e9            # bytes read + written per second
attn_ms = min(event_ms(attn, 50) for _ in range(3))
nbytes = qkv.numel() * 2 + out.numel() * 2
flops = 4 * B * H * T * T * DH
net = bench.build_model(dev, max_batch=B)
x = torch.randn(B, 4, 32, 32, device=dev)
t = torch.tensor(0.5, device=dev)
fwd_ms = event_ms(lambda: net(t, x), 10)
gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print(json.dumps({
    "gpu": gpu, "attention_us": round(attn_ms * 1e3, 1), "bytes": nbytes, "flops": flops,
    "copy_rate_gbs": round(copy_gbs, 1), "bound_us_at_copy_rate": round(nbytes / copy_gbs / 1e3, 1),
    "bound_us_at_datasheet_hbm": round(nbytes / 3.35e12 * 1e6, 1), "bound_us_at_datasheet_bf16": round(flops / 989e12 * 1e6, 1),
    "achieved_gbs": round(nbytes / (attn_ms * 1e-3) / 1e9, 1), "achieved_tflops": round(flops / (attn_ms * 1e-3) / 1e12, 1),
    "forward_ms": round(fwd_ms, 3), "attention_share_of_forward": round(L * attn_ms / fwd_ms, 4)}))
