"""The four DiT-L/2 GEMM shapes at batch 64 through (a) torch.matmul (cuBLAS) and (b) lfm_dbg_gemm (the wgmma
kernel with its fused epilogue), a few launches each - run under ncu to compare kernel names / tile shapes / counters:
  ncu --set full --clock-control none -k regex:'nvjet|cutlass|gemm' -c 24 -o gpurun_out/r2_gemm python scripts/gemm_profile.py"""
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lfm_b200 import _lib  # noqa: E402

lib = _lib.load()
dev = torch.device("cuda:0")
M = 16384
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
for name, N, K, epi in (("qkv", 3072, 1024, 0), ("proj", 1024, 1024, 2), ("fc1", 4096, 1024, 1), ("fc2", 1024, 4096, 2)):
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) * 0.03).bfloat16()
    bias = torch.randn(N, device=dev)
    gate = torch.randn(M // 256, N, device=dev)
    o = torch.zeros(M, N, device=dev, dtype=torch.float32 if epi >= 2 else torch.bfloat16)
    torch.cuda.synchronize()
    for _ in range(reps):
        c = a @ w.t()
    torch.cuda.synchronize()
    for _ in range(reps):
        rc = lib.lfm_dbg_gemm(a.data_ptr(), w.data_ptr(), bias.data_ptr(), o.data_ptr(), gate.data_ptr(), N, 256, M, N, K, epi, 0, None)
        assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    print(name, "done", flush=True)
