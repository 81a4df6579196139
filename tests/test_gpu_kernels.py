"""Kernel-level parity of the UNet, EDM and VAE programs (H100 only, `-m gpu`): each op runs through the network's own host
code (the lfm_dbg_* entries build and launch it with the helpers run_unet_program uses) and is compared element by element
with a plain fp64 reference of the same operation on the same bf16-rounded operands, computed on the GPU.

Bounds, from the compute types (u = 2^-24 is the fp32 unit roundoff):
  * fp32 results of a K-term bf16 dot product (convolution, batched GEMM).  The products of bf16 operands are exact in fp32;
    the K-term fp32 sum is off by at most K u |a| |w| (the recursive-summation bound).  The tensor cores may truncate
    rather than round inside a k-step, so the bound is taken with 2 u:
        |y - ref| <= c (|A| * |W| + |bias| + |out_0|),   c = (K + 16) 2^-23
    (|A| * |W| is the convolution / product of the absolute values, out_0 the accumulated-into output of the residual
    epilogue; the 16 covers the split-K slab sum, the bias and the residual add).  One wrong tap or a seam column read as zero
    padding moves an element by about sqrt(3 Cin) |a||w|, 100x (Cin 1024) to 300x (Cin 128) more than c |A| * |W|, which
    rel-L2 over a 256 x 256 image would dilute.  Measured: at most 0.003 of this bound (fp32 outputs).
    Also rel-L2 <= 1e-5 up to K = 9216, and 1e-5 K / 9216 beyond.  Within one K slice the tensor cores' fp32 accumulation
    truncates, so its error does not average out but grows linearly in K: rel-L2 = K 2^-30 (within 15 %) at every K measured, 1.1e-6
    at K = 1152, 4.9e-6 at 4608, 9.2e-6 at 9216 and 1.6e-5 at 18432 (the 4 x 4 output blocks' 2048-channel concat input, which
    the network runs as one slice for 64 < batch <= 136); split-K slices add in fp32 with rounding, e.g. 1.1e-6 at K = 9216 in
    8 slices.
  * bf16 results: one bf16 ulp of the reference, plus the fp32 error of what is rounded (the bound above for the conv; for
    GroupNorm 2^-12 |gamma (1 + scale)|, which covers the fp32 statistics: a lane adds at most 16 values per chunk in the
    mean >= 50 std cases, so the variance is off by <= 16 u (1 + (mean / std)^2) ~ 2.4e-3 relative and the output by
    <= 1.2e-3 |y|, inside the half ulp the final rounding leaves; the mean is off by <= 16 u 50 std = 5e-5 std).
    Measured: the conv, batched-GEMM and GroupNorm bf16 outputs reach 0.46 / 0.50 / 0.50 of their bounds (the half ulp of the
    final rounding).
  * attention (bf16 out): the short-grid and flash kernels round P to bf16 before P V, which moves an output by at most
    2^-9 sum_j p_j |v_j|; the bound is one bf16 ulp + 2^-8 (P |V|), twice that.  A wrong softmax scale moves outputs by
    ~0.1 std(v).  Measured: at most 0.52 of the bound.
  * the GroupNorm statistics of the conv epilogue (integer atomics of the sum in units of 2^-28 and of the sum of squares in
    units of 2^-20, one add per warp, 16 rows and one group): each add rounds to half a unit, and the warp's fp32 partial
    of at most 16 cpg values is off by 16 cpg u of its magnitude; plus the conv's own bound above, carried into the sums.
  * split-K results and statistics bins are bit-identical across two calls (fixed-order reduction, integer atomics).
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from lfm_b200 import _lib

pytestmark = pytest.mark.gpu

GN_SCALE, GN_SCALE_SQ = 2.0 ** 28, 2.0 ** 20   # fixed-point units of the statistics bins (gemm.cuh kGnFixScale / kGnFixScaleSq)
REPLICAS = 16                                  # kGnBinReplicas


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def P(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def bf16_ulp(x):
    """The spacing of bf16 numbers at |x| (8 significant bits)."""
    e = torch.floor(torch.log2(x.abs().double().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def dot_c(K):
    return (K + 16) * 2.0 ** -23


def assert_within(out, ref, bound, what):
    err = (out.double() - ref).abs()
    worst = float((err / bound).max())
    assert worst <= 1.0, f"{what}: |out - ref| reaches {worst:.3g} x the bound (max error {float(err.max()):.3g})"


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def picked_block_n(M, N):
    """pick_block_n in lfm_api.cu: the tile width the network uses for an M x N output."""
    tiles256 = -(-M // 128) * -(-N // 256)
    return 128 if (N <= 128 or 2 * tiles256 <= num_sms()) else 256


# ------------------------------------------------------------------------------------------------ 3x3 convolution


def conv_operands(B, side, Cin, Cout, seed, w_std=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, side, side, Cin, generator=g).cuda().bfloat16()
    w = (torch.randn(Cout, 9 * Cin, generator=g) * (w_std if w_std is not None else (9 * Cin) ** -0.5)).cuda().bfloat16()
    bias = (torch.randn(Cout, generator=g) * 0.1).cuda()
    return x, w, bias


def conv_ref(x, w, bias, stride):
    """fp64 conv2d (pad 1) on the bf16 operands, NHWC: the value and the conv of the absolute values."""
    Cout, Cin = w.shape[0], x.shape[-1]
    xd = x.double().permute(0, 3, 1, 2)
    wd = w.double().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2)     # K index (r * 3 + s) * Cin + c
    y = F.conv2d(xd, wd, stride=stride, padding=1).permute(0, 2, 3, 1) + bias.double()
    ya = F.conv2d(xd.abs(), wd.abs(), stride=stride, padding=1).permute(0, 2, 3, 1) + bias.double().abs()
    return y, ya


def run_conv(x, w, bias, out, stride, block_n, epi, ksplit, bins=None):
    B, side, _, Cin = x.shape
    rc = _lib.load().lfm_dbg_conv(P(x), P(w), P(bias), P(out), P(bins), B, side, Cin, w.shape[0], stride, block_n, epi, ksplit, None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()


def check_conv(out, ref, absref, K, what, out0=None):
    scale = absref if out0 is None else absref + out0.double().abs()
    bound = dot_c(K) * scale
    if out.dtype == torch.bfloat16:
        bound = bound + bf16_ulp(ref)
    else:
        rel_tol = 1e-5 * max(1.0, K / 9216)
        assert rel_l2(out, ref) <= rel_tol, f"{what}: rel-L2 {rel_l2(out, ref):.3g}"
    assert_within(out, ref, bound, what)


# (output side, Cin, Cout, B) as the presets pair them: celeb512 UNet (64 x 64 latents, nf 256, mult 1 2 2 2 4), imnet EDM
# (32 x 32, nf 256, mult 1 2 3 4), the VAE decoder (128 / 256 / 512 / 512 channels up to 256 x 256), and the N = 4 output convs
CONV_S1 = [
    (4, 512, 1024, 5), (4, 1024, 1024, 3), (4, 2048, 1024, 1), (4, 1792, 1024, 3),
    (8, 512, 512, 5), (8, 1024, 512, 3), (8, 768, 768, 1),
    (16, 512, 512, 3), (32, 256, 512, 3), (32, 512, 512, 1),
    (64, 256, 256, 3), (64, 512, 256, 1), (64, 512, 512, 1), (64, 256, 4, 3),
    (128, 512, 256, 1), (128, 256, 256, 3), (128, 512, 512, 1),
    (256, 256, 128, 1), (256, 128, 128, 3), (256, 256, 256, 1), (256, 128, 4, 3),
]


@pytest.mark.parametrize("forced", [False, True])   # the tile width the network picks, and the other one (no split-K then)
@pytest.mark.parametrize("side,Cin,Cout,B", CONV_S1)
def test_conv3x3(dev, side, Cin, Cout, B, forced):
    x, w, bias = conv_operands(B, side, Cin, Cout, side * 7 + Cin + Cout + B)
    ref, absref = conv_ref(x, w, bias, 1)
    picked = picked_block_n(B * side * side, Cout)
    block_n, ksplit = (384 - picked, 1) if forced else (0, -1)
    out = torch.full((B, side, side, Cout), float("nan"), device=dev)
    run_conv(x, w, bias, out, 1, block_n, 3, ksplit)
    check_conv(out, ref, absref, 9 * Cin, f"conv {side} {Cin}->{Cout} B{B} bn{block_n}")
    if not forced:   # the bf16 store conv1 uses when its statistics are fused (no split-K for bf16)
        outb = torch.zeros(B, side, side, Cout, device=dev, dtype=torch.bfloat16)
        run_conv(x, w, bias, outb, 1, 0, 0, -1)
        check_conv(outb, ref, absref, 9 * Cin, f"bf16 conv {side} {Cin}->{Cout}")


@pytest.mark.parametrize("side,C,B", [(64, 256, 3), (16, 512, 3), (8, 512, 5)])   # Downsample convs: 64->32, 16->8, 8->4
def test_conv3x3_stride2(dev, side, C, B):
    x, w, bias = conv_operands(B, side, C, C, side + C + B)
    ref, absref = conv_ref(x, w, bias, 2)
    for block_n in (0, 128, 256):
        out = torch.full((B, side // 2, side // 2, C), float("nan"), device=dev)
        run_conv(x, w, bias, out, 2, block_n, 3, -1 if block_n == 0 else 1)
        check_conv(out, ref, absref, 9 * C, f"stride-2 conv {side} {C} bn{block_n}")


@pytest.mark.parametrize("epi", [3, 2])
@pytest.mark.parametrize("ksplit", [-1, 2, 5, 8])   # 5: 144 / 72 K blocks do not divide evenly
@pytest.mark.parametrize("B", [8, 32])
@pytest.mark.parametrize("side,C", [(4, 1024), (8, 512)])   # the tile-starved celeb512 layers the network splits
def test_conv3x3_split_k(dev, side, C, B, ksplit, epi):
    x, w, bias = conv_operands(B, side, C, C, side * 100 + B + ksplit)
    ref, absref = conv_ref(x, w, bias, 1)
    out0 = torch.randn(B, side, side, C, generator=torch.Generator().manual_seed(B)).cuda()
    outs = []
    for _ in range(2):
        out = out0.clone() if epi == 2 else torch.full_like(out0, float("nan"))
        run_conv(x, w, bias, out, 1, 0, epi, ksplit)
        outs.append(out)
    assert torch.equal(outs[0], outs[1]), "split-K result differs between two identical calls"
    if epi == 2:
        check_conv(outs[0], out0.double() + ref, absref, 9 * C, f"split-K {ksplit} accumulate", out0=out0)
    else:
        check_conv(outs[0], ref, absref, 9 * C, f"split-K {ksplit}")


def bins_to_stats(bins, B):
    """[B][replica][group][sum, sumsq] fixed point -> fp64 (S, Q) per (image, group)."""
    t = bins.view(B, REPLICAS, 32, 2).sum(1)   # int64: the totals are exact
    return t[..., 0].double() / GN_SCALE, t[..., 1].double() / GN_SCALE_SQ


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("side,Cin,Cout,B,rms", [
    (64, 256, 128, 3, 1.0),     # cpg 4
    (32, 256, 256, 3, 1.0),     # cpg 8
    (16, 512, 512, 2, 1.0),     # cpg 16
    (8, 1024, 1024, 5, 1.0),    # cpg 32; 2 images per tile, so the last tile's second image is out of bounds
    (256, 128, 128, 1, 1e-2),   # the VAE's last stage (2^18 values per group): small activations
    (256, 128, 128, 1, 500.0),  # ... and large ones: the sum of squares (6.6e10) is past the 2^35 an 2^-28 unit could hold
])
def test_conv_groupnorm_statistics(dev, side, Cin, Cout, B, rms, block_n):
    x, w, bias = conv_operands(B, side, Cin, Cout, side + Cin + Cout, w_std=rms * (9 * Cin) ** -0.5)
    bias = bias * rms
    ref, absref = conv_ref(x, w, bias, 1)
    bins = [torch.zeros(B * REPLICAS * 64, dtype=torch.int64, device=dev) for _ in range(2)]
    out = torch.full((B, side, side, Cout), float("nan"), device=dev)
    for bb in bins:
        run_conv(x, w, bias, out, 1, block_n, 3, 1, bb)
    assert torch.equal(bins[0], bins[1]), "statistics bins differ between two identical calls"
    check_conv(out, ref, absref, 9 * Cin, "conv with statistics")
    S, Q = bins_to_stats(bins[0], B)
    cpg, HW = Cout // 32, side * side
    rg = ref.reshape(B, HW, 32, cpg)
    S_ref, Q_ref = rg.sum((1, 3)), (rg * rg).sum((1, 3))
    adds = HW // 16                               # one add per (warp of 16 rows, group)
    err_y = (dot_c(9 * Cin) * absref).reshape(B, HW, 32, cpg)
    S_bound = adds * 0.5 / GN_SCALE + err_y.sum((1, 3)) + 16 * cpg * 2.0 ** -24 * rg.abs().sum((1, 3))
    Q_bound = adds * 0.5 / GN_SCALE_SQ + (2 * rg.abs() * err_y + err_y ** 2).sum((1, 3)) + 16 * cpg * 2.0 ** -24 * Q_ref
    assert_within(S, S_ref, S_bound, "group sum")
    assert_within(Q, Q_ref, Q_bound, "group sum of squares")


# ------------------------------------------------------------------------------------------------ GroupNorm


def make_bins(x, B, HW, C):
    """The statistics a producing conv would accumulate, spread over all replicas: replica r holds the sums of pixel chunk r."""
    cpg = C // 32
    xd = x.double().reshape(B, HW, 32, cpg)
    bins = torch.zeros(B, REPLICAS, 32, 2, dtype=torch.int64, device=x.device)
    edges = [HW * r // REPLICAS for r in range(REPLICAS + 1)]
    for r in range(REPLICAS):
        part = xd[:, edges[r]:edges[r + 1]]
        bins[:, r, :, 0] = torch.round(part.sum((1, 3)) * GN_SCALE).long()
        bins[:, r, :, 1] = torch.round((part * part).sum((1, 3)) * GN_SCALE_SQ).long()
    return bins.reshape(-1)


# (Ca, Cb, HW, B, eps, film, act, source, max_chunks, copy_out, raw_out, mean / std)
#   source: "f32" = statistics pass over the fp32 source; "bins" = fp32 source with bins; "bf16" = bf16 source with bins
GN_CASES = [
    (128, 0, 65536, 1, 1e-6, None, 1, "f32", 256, False, False, 0),      # VAE last stage, J = 1
    (256, 0, 16384, 2, 1e-6, None, 1, "f32", 256, False, True, 0),       # VAE 128 x 128, + raw_out
    (512, 0, 4096, 3, 1e-6, None, 0, "f32", 256, False, False, 0),       # VAE mid block, no SiLU
    (256, 512, 1024, 2, 1e-5, "sample", 1, "f32", 32, False, True, 0),   # concat 256 + 512: cpg 24, group 10 straddles
    (1024, 1024, 16, 3, 1e-5, "sample", 1, "f32", 32, False, False, 0),  # concat 1024 + 1024 at 4 x 4, J = 16
    (256, 0, 4096, 3, 1e-5, "shared", 1, "f32", 32, True, False, 0),     # identity skip copy, FiLM stride 0
    (384, 0, 256, 2, 1e-5, "sample", 1, "f32", 32, True, True, 0),       # J = 3, both side outputs
    (640, 0, 64, 2, 1e-5, "sample", 1, "f32", 32, False, False, 0),      # J = 5
    (1536, 0, 64, 3, 1e-5, "sample", 0, "f32", 32, False, False, 0),     # J = 12
    (256, 0, 1024, 2, 1e-5, "sample", 1, "f32", 32, False, False, 50),   # mean 50 x std
    (1024, 0, 256, 2, 1e-5, None, 1, "f32", 32, False, False, 50),       # mean 50 x std, J = 8
    (128, 0, 65536, 1, 1e-6, None, 1, "bf16", 32, False, False, 0),      # conv1 output as bf16: the fast path, J = 1
    (256, 0, 4096, 3, 1e-5, "sample", 1, "bf16", 32, False, False, 0),   # J = 2
    (384, 0, 1024, 2, 1e-5, "sample", 1, "bf16", 32, False, False, 0),   # J = 3 (4-pixel groups)
    (512, 0, 1024, 2, 1e-5, "shared", 1, "bf16", 32, False, False, 0),   # J = 4
    (1024, 0, 64, 3, 1e-5, "sample", 1, "bf16", 32, False, False, 0),    # generic pass on a bf16 source, J = 8
    (2048, 0, 16, 2, 1e-5, "sample", 1, "bf16", 32, False, False, 0),    # J = 16, cpg 64
    (256, 0, 4096, 2, 1e-5, "sample", 1, "bins", 32, False, False, 0),   # bins instead of the partials, fp32 source
]


@pytest.mark.parametrize("Ca,Cb,HW,B,eps,film,act,source,max_chunks,copy,raw,mean", GN_CASES)
def test_groupnorm(dev, Ca, Cb, HW, B, eps, film, act, source, max_chunks, copy, raw, mean):
    C_ = Ca + Cb
    g = torch.Generator().manual_seed(C_ + HW + B)
    a = ((torch.randn(B, HW, Ca, generator=g) + mean) * 1.7 + torch.randn(1, 1, Ca, generator=g) * 0.3).cuda()
    b = (torch.randn(B, HW, Cb, generator=g) * 0.6 - 0.4).cuda() if Cb else None
    gamma = (1 + 0.3 * torch.randn(C_, generator=g)).cuda()
    beta = (0.3 * torch.randn(C_, generator=g)).cuda()
    src_bf16 = None
    x = a if b is None else torch.cat([a, b], -1)
    if source == "bf16":
        src_bf16 = x.bfloat16()
        x = src_bf16.float()
    bins = make_bins(x, B, HW, C_) if source in ("bins", "bf16") else None
    if film is None:
        film_t, stride = None, 0
    else:
        rows = B if film == "sample" else 1
        film_t = torch.cat([0.5 * torch.randn(rows, C_, generator=g), torch.randn(rows, C_, generator=g)], 1).cuda()
        stride = 2 * C_ if film == "sample" else 0
    out = torch.full((B, HW, C_), float("nan"), device=dev).bfloat16()
    copy_out = torch.full((B, HW, C_), float("nan"), device=dev) if copy else None
    raw_out = torch.full((B, HW, C_), float("nan"), device=dev).bfloat16() if raw else None
    rc = _lib.load().lfm_dbg_groupnorm(P(a), Ca, P(b), Cb, P(src_bf16), P(bins), max_chunks, P(gamma), P(beta), P(film_t), stride, act,
                                       eps, P(out), P(copy_out), P(raw_out), B, HW, None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    xd = x.double().reshape(B, HW, 32, C_ // 32)
    mu, var = xd.mean((1, 3), keepdim=True), xd.var((1, 3), unbiased=False, keepdim=True)
    y = ((xd - mu) / torch.sqrt(var + eps)).reshape(B, HW, C_) * gamma.double() + beta.double()
    amp = gamma.double().abs().expand(B, 1, C_)
    if film_t is not None:
        f = film_t.double().reshape(-1, 1, 2 * C_)
        y = y * (1 + f[..., :C_]) + f[..., C_:]
        amp = amp * (1 + f[..., :C_]).abs()
    if act:
        y = y * torch.sigmoid(y)
    assert_within(out, y, bf16_ulp(y) + 2.0 ** -12 * amp, "GroupNorm output")
    if copy:
        assert torch.equal(copy_out, x)
    if raw:
        assert torch.equal(raw_out, x.bfloat16())


# ------------------------------------------------------------------------------------------------ batched GEMM (VAE attention)


def run_batched(a, a_rows, a_ld, w, w_rows, w_ld, K, N, out, bias, B, out_hw, epi, batch_m, a_mod, b_rows):
    rc = _lib.load().lfm_dbg_gemm_batched(C.c_void_p(a), a_rows, a_ld, C.c_void_p(w), w_rows, w_ld, K, N, P(out), P(bias), B, out_hw,
                                          epi, batch_m, a_mod, b_rows, None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [256, 1024])
def test_vae_attention_batched_gemms(dev, T, B):
    c = 512
    g = torch.Generator().manual_seed(T + B)
    X = torch.randn(B * T, c, generator=g).cuda().bfloat16()
    Wv = (torch.randn(c, c, generator=g) * c ** -0.5).cuda().bfloat16()
    QK = torch.randn(B * T, 2 * c, generator=g).cuda().bfloat16()
    Pm = torch.softmax(torch.randn(B * T, T, generator=g) * 2, -1).cuda().bfloat16()
    bv = torch.randn(c, generator=g).cuda()
    # V^T_b = Wv X_b^T: A = Wv shared by every image (a_mod = c), group b multiplies W rows [b T, b T + T)
    VT = torch.zeros(B * c, T, device=dev, dtype=torch.bfloat16)
    run_batched(Wv.data_ptr(), c, c, X.data_ptr(), B * T, c, c, T, VT, None, B, c, 0, c, c, T)
    Xd = X.double().reshape(B, T, c)
    ref = (Wv.double() @ Xd.transpose(1, 2)).reshape(B * c, T)
    absref = (Wv.double().abs() @ Xd.abs().transpose(1, 2)).reshape(B * c, T)
    assert_within(VT, ref, bf16_ulp(ref) + dot_c(c) * absref, "V^T")
    # S_b = Q_b K_b^T: column windows [0, c) and [c, 2c) of [Q | K] (row pitch 2c), fp32 out
    S = torch.full((B * T, T), float("nan"), device=dev)
    run_batched(QK.data_ptr(), B * T, 2 * c, QK.data_ptr() + 2 * c, B * T, 2 * c, c, T, S, None, B, T, 3, T, 0, T)
    Q, K = QK.double()[:, :c].reshape(B, T, c), QK.double()[:, c:].reshape(B, T, c)
    ref = (Q @ K.transpose(1, 2)).reshape(B * T, T)
    absref = (Q.abs() @ K.abs().transpose(1, 2)).reshape(B * T, T)
    assert rel_l2(S, ref) <= 1e-5
    assert_within(S, ref, dot_c(c) * absref, "S = Q K^T")
    # O_b = P_b V_b + bv with V_b = (V^T_b)^T (the V^T computed above), bf16 out
    O = torch.zeros(B * T, c, device=dev, dtype=torch.bfloat16)
    run_batched(Pm.data_ptr(), B * T, T, VT.data_ptr(), B * c, T, T, c, O, bv, B, T, 0, T, 0, c)
    Pd, Vd = Pm.double().reshape(B, T, T), VT.double().reshape(B, c, T)
    ref = (Pd @ Vd.transpose(1, 2)).reshape(B * T, c) + bv.double()
    absref = (Pd.abs() @ Vd.abs().transpose(1, 2)).reshape(B * T, c) + bv.double().abs()
    assert_within(O, ref, bf16_ulp(ref) + dot_c(T) * absref, "O = P V + b")


# ------------------------------------------------------------------------------------------------ attention


def attention_ref(q, k, v, head_dim):
    """softmax(q k^T / sqrt(head_dim)) v in fp64 on q, k, v [B, T, heads, ch]; also P |V| (the scale of the bf16-P rounding); both
    [B T, heads ch]."""
    B, T, H, ch = q.shape
    q, k, v = (x.double().transpose(1, 2) for x in (q, k, v))   # [B, heads, T, ch]
    p = torch.softmax((q @ k.transpose(-1, -2)) * head_dim ** -0.5, -1)
    return [o.transpose(1, 2).reshape(B * T, H * ch) for o in (p @ v, p @ v.abs())]


TIMM, HEAD_MAJOR = _lib.QKV_TIMM, _lib.QKV_HEAD_MAJOR
ATTN_BH = [(1, 1), (2, 4), (3, 12), (64, 16), (5, 16), (7, 6), (33, 12), (128, 16)]
# (layout, T, ch, head_dim, heads, B): every route of the table, at the shapes the networks run
ATTN_CASES = (
    [(TIMM, 256, 64, 64, H, B) for B, H in ATTN_BH]             # TMA + wgmma: the DiT /2 presets, EDM 16 x 16
    + [(HEAD_MAJOR, 256, 64, 64, H, B) for B, H in ATTN_BH]     # the same data on flash: ADM 16 x 16
    # DiT geometries outside 256 tokens / head_dim 64: heads zero-padded from 72 to 80 channels, 1024 tokens
    + [(HEAD_MAJOR, 1024, 64, 64, 4, 2), (HEAD_MAJOR, 256, 80, 72, 16, 3), (HEAD_MAJOR, 256, 64, 64, 3, 2), (HEAD_MAJOR, 64, 80, 72, 16, 5),
       (HEAD_MAJOR, 16, 80, 72, 16, 7), (HEAD_MAJOR, 128, 80, 72, 2, 1)]
    # UNet shapes: attention_mma_kernel, flash, SIMT with K / V in shared memory, plain SIMT ((256, 64, 4 heads, B 2) is above)
    + [(HEAD_MAJOR, T, ch, ch, heads, B) for T, ch, heads, B in [
        (16, 64, 4, 5), (16, 128, 2, 3), (16, 256, 4, 8), (64, 64, 2, 3), (64, 128, 4, 4), (64, 256, 2, 2), (1024, 64, 2, 2),
        (16, 32, 4, 3), (16, 96, 2, 3), (64, 32, 4, 2), (64, 96, 2, 3), (256, 32, 2, 2), (256, 96, 2, 2), (256, 128, 2, 2),
        (256, 256, 1, 2)]]
    # head_dim = ch on attention_mma_kernel: the kernel's own ch^-1/2, as the UNets run it
    + [(HEAD_MAJOR, T, ch, ch, 2, 3) for T, ch in [(16, 128), (16, 256), (64, 128), (64, 256), (256, 64)]]
    # 80-channel UNet heads: attention_mma_kernel and flash
    + [(HEAD_MAJOR, 64, 80, 80, 4, 3), (HEAD_MAJOR, 256, 80, 80, 4, 2)]
)


@pytest.mark.parametrize("layout,T,ch,head_dim,heads,B", ATTN_CASES)
def test_attention(dev, layout, T, ch, head_dim, heads, B):
    """lfm_dbg_attention (the op and launch the networks run for the shape) against an fp64 reference on the same bf16 q, k, v.
    Cases that differ only in layout hold the same q, k, v."""
    g = torch.Generator().manual_seed(B * 1000 + heads * 100 + T + ch)
    qkv = torch.randn(B, T, 3, heads, ch, generator=g)
    qkv[..., head_dim:] = 0                                       # the padding channels are zero (zero weight rows)
    qkv = qkv.to(dev).bfloat16()
    ref, pv = attention_ref(*qkv.unbind(2), head_dim)
    rows = qkv if layout == TIMM else qkv.transpose(2, 3)         # {q,k,v} * heads ch + head * ch + c, or head * 3 ch + {q,k,v} * ch + c
    rows = rows.reshape(B * T, 3 * heads * ch).contiguous()
    out = torch.full((B * T, heads * ch), float("nan"), device=dev).bfloat16()
    rc = _lib.load().lfm_dbg_attention(P(rows), P(out), B, T, heads, ch, head_dim, layout, None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    what = f"attention layout {layout} T {T} ch {ch} head_dim {head_dim} heads {heads} B {B}"
    assert rel_l2(out, ref) < 5e-3, what                          # P and O are rounded to bf16
    assert_within(out, ref, bf16_ulp(ref) + 2.0 ** -8 * pv, what)
    if head_dim < ch:
        assert float(out.float().reshape(B * T, heads, ch)[..., head_dim:].abs().max()) == 0.0   # padded output channels are exactly zero


# ------------------------------------------------------------------------------------------------ refusals


def test_unet_attention_shape_without_a_kernel_is_refused(dev):
    """UNetModel(image_size=32, model_channels=128, channel_mult=(1, 2), attention_resolutions=(1,), num_heads=1) would run
    1024 tokens with 128-channel heads, which no attention kernel covers: the constructor refuses it, launching nothing."""
    import lfm_b200
    net = lfm_b200.UNetModel(image_size=32, in_channels=4, model_channels=128, out_channels=4, num_res_blocks=1,
                             attention_resolutions=(1,), channel_mult=(1, 2), num_heads=1, use_scale_shift_norm=True)
    with pytest.raises(RuntimeError, match="1024 tokens"):
        net.native(1, dev)
