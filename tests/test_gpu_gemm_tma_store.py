"""The GEMM epilogue's two store paths give the same bits: the register stores, and the sub-tiles staged in shared memory and
written by TMA stores (the residual stream TMA-loaded into the staging buffer first), which the network now takes for its
16-byte aligned outputs.  Each is forced through lfm_dbg_gemm_path at both tile widths, compared bit for bit, and held
elementwise to the fp64 product (the bounds of tests/test_gpu_dit_kernels.py).

The shapes cover the four DiT-L/2 layers at batch 64 (M = 16384), an odd number of 128-row blocks (M = 1100: the last block's
second 64-row half keeps the register stores), M = 1000 and M = 1, an N tail, both sweep directions, and the gated residual with
per-sample gates, one shared gate row (stride 0) and no gate."""
import ctypes as C

import pytest
import torch

from lfm_b200 import _lib
from tests import test_gpu_kernels as tk
from tests.test_gpu_dit_kernels import gemm_expect, gemm_ref

pytestmark = pytest.mark.gpu



def run_path(a, w, bias, x0, gate, gate_stride, rps, M, N, K, epi, bn, reverse, tma):
    out = x0.clone()
    rc = _lib.load().lfm_dbg_gemm_path(C.c_void_p(a.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(bias.data_ptr()),
                                       C.c_void_p(out.data_ptr()), C.c_void_p(gate.data_ptr()) if gate is not None else None,
                                       gate_stride, rps, M, N, K, epi, bn, reverse, tma, None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    return out


def check_paths(M, N, K, epi, reverse=0, gate_mode="sample", rps=256, bn=256, seed=0):
    g = torch.Generator().manual_seed(seed + M + N + K + epi)
    a = torch.randn(M, K, generator=g).cuda().bfloat16()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).cuda().bfloat16()
    bias = torch.randn(N, generator=g).cuda()
    dt = torch.float32 if epi >= 2 else torch.bfloat16
    x0 = torch.randn(M, N, generator=g).cuda().to(dt)
    gate, gate_stride, gate_rows = None, 0, None
    if epi == 2 and gate_mode == "sample":
        gate = torch.randn((M + rps - 1) // rps, N, generator=g).cuda()
        gate_stride = N
        gate_rows = gate[torch.arange(M, device="cuda") // rps]
    elif epi == 2 and gate_mode == "shared":
        gate = torch.randn(1, N, generator=g).cuda()
        gate_rows = gate.expand(M, N)
    base = run_path(a, w, bias, x0, gate, gate_stride, rps, M, N, K, epi, bn, reverse, 0)
    out = run_path(a, w, bias, x0, gate, gate_stride, rps, M, N, K, epi, bn, reverse, 1)
    assert torch.equal(out, base), "the TMA-store epilogue differs from the register stores"
    acc, absacc = gemm_ref(a, w, bias)
    ref, bound = gemm_expect(epi, acc, absacc, K, x0, gate_rows)
    tk.assert_within(out, ref, bound, f"gemm {M}x{N}x{K} epi {epi} block_n {bn} reverse {reverse}")


@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("name,N,K,epi", [("qkv", 3072, 1024, 0), ("proj", 1024, 1024, 2), ("fc1", 4096, 1024, 1),
                                          ("fc2", 1024, 4096, 2)])
def test_dit_l_layers(name, N, K, epi, reverse):
    check_paths(16384, N, K, epi, reverse)


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("epi", [0, 1, 2, 3])
@pytest.mark.parametrize("M,N,K", [(1100, 1024, 256), (1000, 1000, 128), (1, 512, 128)])
def test_ragged_shapes(M, N, K, epi, reverse, bn):
    check_paths(M, N, K, epi, reverse, rps=100, bn=bn)


@pytest.mark.parametrize("gate_mode", ["sample", "shared", "none"])
def test_residual_gates(gate_mode):
    check_paths(1100, 1000, 256, 2, 1, gate_mode=gate_mode, rps=100)


def test_misaligned_output_refuses_tma_store():
    a = torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(256, 64, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(128 * 256 + 8, device="cuda")
    rc = _lib.load().lfm_dbg_gemm_path(C.c_void_p(a.data_ptr()), C.c_void_p(w.data_ptr()), None,
                                       C.c_void_p(out.data_ptr() + 4), None, 0, 1, 128, 256, 64, 3, 256, 0, 1, None)
    assert rc != 0 and "alignment" in _lib.last_error()
