"""The GEMM epilogue stores whole 32-column groups with 16-byte accesses after a transpose within each quad of lanes, and
falls back to the per-8-column stores for the N tail and for an output that is not 16-byte aligned.  Both paths must write
the same bytes: the same product written to an aligned and to a misaligned (4 bytes off) output is compared bit for bit, and both
are held elementwise to the fp64 product (the bounds of tests/test_gpu_dit_kernels.py), so that a mistake both paths share is seen."""
import ctypes as C

import pytest
import torch

from lfm_b200 import _lib
from tests import test_gpu_kernels as tk
from tests.test_gpu_dit_kernels import gemm_expect, gemm_ref

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("epi", [0, 1, 2, 3])
@pytest.mark.parametrize("M,N,K", [(1000, 1000, 256), (384, 2048, 128), (5, 264, 64)])   # N tails of 8 / none / 8 columns
def test_vector_and_scalar_stores_agree(M, N, K, epi, bn):
    g = torch.Generator().manual_seed(M + N + epi)
    a = torch.randn(M, K, generator=g).cuda().bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.05).cuda().bfloat16()
    bias = torch.randn(N, generator=g).cuda()
    gate = torch.randn((M + 255) // 256, N, generator=g).cuda()
    dt = torch.float32 if epi >= 2 else torch.bfloat16
    x0 = torch.randn(M * N, generator=g).cuda().to(dt)
    outs = []
    for off in (0, 2):   # elements: 0 = 16-byte aligned, 2 = 4 (bf16) / 8 (fp32) bytes off, the per-8-column path
        buf = torch.zeros(M * N + 8, device="cuda", dtype=dt)
        buf[off:off + M * N] = x0
        p = C.c_void_p(buf.data_ptr() + off * buf.element_size())
        rc = _lib.load().lfm_dbg_gemm(C.c_void_p(a.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(bias.data_ptr()), p,
                                      C.c_void_p(gate.data_ptr()) if epi == 2 else None, N, 256, M, N, K, epi, bn, None)
        torch.cuda.synchronize()
        assert rc == 0, _lib.last_error()
        outs.append(buf[off:off + M * N].clone())
    assert torch.equal(outs[0], outs[1])
    acc, absacc = gemm_ref(a, w, bias)
    ref, bound = gemm_expect(epi, acc, absacc, K, x0.view(M, N), gate[torch.arange(M, device="cuda") // 256])
    err = (outs[0].double().view(M, N) - ref).norm() / ref.norm()
    assert err < (4e-3 if epi < 2 else 1e-5)
    tk.assert_within(outs[0].view(M, N), ref, bound, f"gemm {M}x{N}x{K} epi {epi} bn {bn}")
