"""Kernel-level parity of the DiT forward (H100 only, `-m gpu`): every kernel launch_network makes, run through the same host helper
the network calls (the lfm_dbg_* entries), at the shapes the DiT presets launch, compared element by element with a plain fp64
reference of the same operation on the same bf16- or fp32-rounded operands, computed on the GPU.

Bounds, from the compute types (u = 2^-24 is the fp32 unit roundoff; NV = D / 128, the float4 a lane holds per row):
  * LayerNorm + modulate (ln_modulate_kernel, bf16 out).  The fp32 row sum runs over D / 32 values per lane and a 5-step butterfly, so
    the mean is off by e_mu <= (NV + 9) u mean|x| (the division included).  That error, relative to the row's std, is what matters:
    it moves every normalised value z by e_mu rstd and the variance by (e_mu rstd)^2 relative; the sum of squares, the rsqrt
    (2 ulp) and the products add at most (NV + 32) u |z|:
        |y - ref| <= ulp_bf16(ref) + |1 + scale| ((NV + 32) u |z| + (e_mu rstd)^2 |z| + 2 e_mu rstd) + 2^-23 |ref|
    Rows whose mean is 50x and 1000x their std need the e_mu term (at 1000x it is ~1e-3 of the output); constant rows (variance 0,
    rstd = 1e3) turn the mean's rounding into the whole output error.  Measured: at most 0.50 of this bound (the final rounding's
    half ulp).
  * FinalLayer (fp32): the same LayerNorm without the bf16 rounding, then a D-term fp32 dot product (D / 32 fmas per lane and a
    5-step butterfly, 16 outputs at p = 2, 32 per chunk otherwise): (D / 32 + 8) u (|W| |y| + |b|) + |W| e_y.  A swapped p / q or c
    index moves a pixel by a whole independent output.  Measured: at most 0.013 of this bound.
  * conditioning: the timestep features t f_k with f_k = exp(-ln(1e4) k / half) evaluated in fp32 (the exponent's two roundings,
    expf's 2 ulp and the product: 24 u |t f_k|; cosf / sinf 1 ulp): (32 |t f_k| + 4) u.  Each MLP layer is checked from the
    kernel's own fp32 input: K / 32 fmas per lane, a 5-step butterfly, the bias and the label row, (K / 32 + 8) u (|W| |in| + |b|
    + |table|), through SiLU (slope <= 1.1); SiLU's __expf is ex2.approx of a rounded product (2^-21 + u |v| relative) and its
    division is IEEE: |silu(v)| (2^-21 + 2^-23 (|v| + 2)).  c is rounded to bf16: one ulp more.  Measured: tf 0.12, h1 0.057, c 0.50.
  * patch embed (fp32): a C p^2-term fma chain from the bias, then + pos: (C p^2 + 16) 2^-23 (|W| |patch| + |b| + |pos|).  The CFG
    half (network rows x_rows..2 x_rows read the same latents) must be bit-identical to the first.  Measured: at most 0.071.
  * GEMM (gemm_bf16_wgmma at the qkv / proj / fc1 / fc2 / adaLN shapes of S, B, L and XL): the bound of tests/test_gpu_kernels.py,
    (K + 16) 2^-23 (|A| |W| + |b|), times |gate| plus |x_0| for the gated residual; one bf16 ulp more for bf16 outputs.  GELU
    (fc1) evaluates tanh with tanh.approx.f32, whose maximum relative error the PTX ISA documents as 2^-10.987: 0.5 |x| |tanh| 2^-10.987
    on top, up to |x| 2^-12 in the negative tail where 1 + tanh cancels (at x = -3, ~50 bf16 ulps of the output), plus the fp32
    roundings of the inner polynomial, 2^-21 |x| |inner|, and the accumulation error through GELU's slope (<= 1.13).  Measured: fp32
    outputs 0.005, bf16 0.49, GELU 0.47 of these bounds.
All fractions were measured on an NVIDIA H100 80GB HBM3 at its 700 W power limit.
"""
import ctypes as C
import math

import pytest
import torch

from lfm_b200 import _lib
from tests import test_gpu_kernels as tk

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TANH_REL = 2.0 ** -10.987   # PTX ISA: maximum relative error of tanh.approx.f32
NULL_CLASS = 1000           # ImageNet labels 0..999, then the null row CFG reads


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(*shape, g):
    return torch.randn(*shape, device="cuda", generator=g)


def ptr(t, offset=0):
    """Device address of element `offset` of t."""
    return C.c_void_p(t.data_ptr() + offset * t.element_size())


def done(rc):
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()


def nan_like(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


def modulation_table(rows, D, L, g):
    """A (6 L + 2) D-wide adaLN table of `rows` samples (the layout of the network's mod buffer)."""
    return randn(rows, (6 * L + 2) * D, g=g) * 0.5


def layernorm_ref(x, shift, scale, rows_per_sample):
    """fp64 LayerNorm (eps 1e-6) + modulate of fp32 rows with per-sample [rows, D] shift / scale (one row: shared), and the fp32
    error bound of the kernels' statistics (see the header)."""
    M, D = x.shape
    xd = x.double()
    mu = xd.mean(1, keepdim=True)
    var = ((xd - mu) ** 2).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-6)
    z = (xd - mu) * rstd
    b = torch.arange(M, device=x.device) // rows_per_sample
    sh, sc = shift.double(), scale.double()
    if sh.shape[0] > 1:
        sh, sc = sh[b], sc[b]
    y = z * (1 + sc) + sh
    nv = D // 128
    em = (nv + 9) * U * xd.abs().mean(1, keepdim=True) * rstd
    err = (1 + sc).abs() * (z.abs() * ((nv + 32) * U + em ** 2) + 2 * em) + 2 * U * y.abs()
    return y, err


# ------------------------------------------------------------------------------------------------ LayerNorm + modulate


def ln_rows(kind, M, D, g):
    x = randn(M, D, g=g) * torch.exp(randn(M, 1, g=g) * 0.5)    # rows of different std
    if kind in ("mean50", "mean1000"):
        k = 50.0 if kind == "mean50" else 1000.0
        sign = torch.where(randn(M, 1, g=g) > 0, 1.0, -1.0)
        x = (randn(M, D, g=g) + k * sign) * torch.exp(randn(M, 1, g=g))
    elif kind == "constant":
        x = randn(M, 1, g=g).expand(M, D).contiguous()
        x[::3] = torch.round(x[::3] * 8) / 8                       # some rows sum exactly, the rest do not
    elif kind == "small":
        x = x * 1e-3
    elif kind == "large":
        x = x * 1e3
    return x.contiguous()


# (T, B, modulation, rows): B "sms" gives exactly one 16-row tile per block; 3 and 64 x 256 (DiT-L at batch 64, M = 16384) give
# fewer tiles than SMs and several wraps of the ring
LN_SCENARIOS = [
    (16, "sms", "sample", "normal"), (64, 3, "shared", "normal"), (256, 64, "sample", "normal"), (1024, 5, "sample", "normal"),
    (256, 4, "sample", "mean50"), (64, 6, "shared", "mean1000"), (16, 9, "sample", "mean1000"), (16, 9, "sample", "constant"),
    (1024, 2, "sample", "small"), (256, 3, "sample", "large"),
]


@pytest.mark.parametrize("down", [0, 1])
@pytest.mark.parametrize("T,B,mod,kind", LN_SCENARIOS)
@pytest.mark.parametrize("D", [256, 384, 768, 1024, 1152])
def test_ln_modulate(dev, D, T, B, mod, kind, down):
    if B == "sms":
        B = tk.num_sms()
    M, L = B * T, 2
    g = gen(D + T + M + down)
    x = ln_rows(kind, M, D, g)
    table = modulation_table(B if mod == "sample" else 1, D, L, g)
    stride = table.shape[1] if mod == "sample" else 0
    shift, scale = table[:, 3 * D:4 * D], table[:, 4 * D:5 * D]     # shift_mlp / scale_mlp of block 0: mb + 3 D, mb + 4 D
    y = nan_like((M, D), torch.bfloat16)
    done(_lib.load().lfm_dbg_ln_modulate(ptr(x), ptr(y), ptr(table, 3 * D), ptr(table, 4 * D), stride, T, M, D, down, None))
    ref, err = layernorm_ref(x, shift, scale, T)
    tk.assert_within(y, ref, tk.bf16_ulp(ref) + err, f"ln_modulate: D {D} T {T} B {B} {mod} {kind} down {down}")


# ------------------------------------------------------------------------------------------------ conditioning


def silu_bound(v):
    return v.abs() * torch.sigmoid(v) * (2.0 ** -21 + 2.0 ** -23 * (v.abs() + 2))


# Label rules (lfm_dbg_condition's max_row / null_row) of the three networks, for a table of n labels: the DiT's null class is its
# last row, which y NULL reads; ADM reads label rows only; EDM's map_label table has one all-zero row after its labels (max_row = n).
LABEL_RULES = {"dit": lambda n: (n - 1, n - 1), "adm": lambda n: (n - 1, -1), "edm": lambda n: (n, -1)}
CONDITION_CASES = [("dit", 256, 384), ("dit", 256, 1152),     # DiT-S / XL widths
                   ("adm", 128, 512), ("adm", 256, 1024),     # UNet model_channels 128 / 256: E = 4 model_channels
                   ("edm", 128, 512), ("edm", 256, 1024),
                   ("adm", 512, 2048), ("edm", 1024, 4096)]   # K > 1152: weights beyond the registers stream from memory


@pytest.mark.parametrize("per_row_t", [False, True])
@pytest.mark.parametrize("labels", [False, True])   # y NULL / labels that include the last table row
@pytest.mark.parametrize("rows", [1, 7, 256])       # 256: CFG doubling of max_batch 128
@pytest.mark.parametrize("net,feat,E", CONDITION_CASES)
def test_condition(dev, net, feat, E, rows, labels, per_row_t):
    g = gen(E + rows + 2 * labels + per_row_t)
    t_numel = rows if per_row_t else 1
    t = torch.rand(t_numel, device="cuda", generator=g)
    max_row, null_row = LABEL_RULES[net](NULL_CLASS)
    y = None
    if labels:
        y = torch.randint(0, max_row, (rows,), device="cuda", generator=g)
        y[::3] = max_row
    w0, b0 = randn(E, feat, g=g) * (2 / math.sqrt(feat)), randn(E, g=g) * 0.5
    w2, b2 = randn(E, E, g=g) * (2 / math.sqrt(E)), randn(E, g=g) * 0.5
    table = randn(max_row + 1, E, g=g)
    tf, h1, c = nan_like((rows, feat)), nan_like((rows, E)), nan_like((rows, E), torch.bfloat16)
    done(_lib.load().lfm_dbg_condition(ptr(t), t_numel, tk.P(y), rows, feat, E, ptr(w0), ptr(b0), ptr(w2), ptr(b2), ptr(table),
                                       max_row, null_row, ptr(tf), ptr(h1), ptr(c), None))
    what = f"{net} {feat} -> {E} rows {rows} labels {labels} t_numel {t_numel}"
    # timestep features [cos | sin](t f_k)
    half = feat // 2
    k = torch.arange(half, device="cuda", dtype=torch.float64)
    a = t.double().expand(rows)[:, None] * torch.exp(-math.log(1e4) * k / half)
    a = torch.cat([a, a], 1)
    tf_ref = torch.cat([torch.cos(a[:, :half]), torch.sin(a[:, half:])], 1)
    tk.assert_within(tf, tf_ref, U * (32 * a.abs() + 4), f"condition tf: {what}")
    # h1 = SiLU(w0 tf + b0), from the kernel's tf
    v = tf.double() @ w0.double().t() + b0.double()
    va = tf.double().abs() @ w0.double().abs().t() + b0.double().abs()
    tk.assert_within(h1, v * torch.sigmoid(v), 1.1 * (feat / 32 + 8) * U * va + silu_bound(v), f"condition h1: {what}")
    # c = bf16(SiLU(w2 h1 + b2 + table[row])), from the kernel's h1
    v = h1.double() @ w2.double().t() + b2.double()
    va = h1.double().abs() @ w2.double().abs().t() + b2.double().abs()
    if y is not None or null_row >= 0:
        row = y if y is not None else torch.full((rows,), null_row, device="cuda")
        v, va = v + table.double()[row], va + table.double()[row].abs()
    ref = v * torch.sigmoid(v)
    tk.assert_within(c, ref, tk.bf16_ulp(ref) + 1.1 * (E / 32 + 8) * U * va + silu_bound(v), f"condition c: {what}")


# ------------------------------------------------------------------------------------------------ patch embed


@pytest.mark.parametrize("D,x_rows,rows", [(1152, 2, 4), (384, 3, 3)])   # 1152: D / 4 > 256 threads, the feature loop runs twice;
@pytest.mark.parametrize("G", [4, 8, 16, 32])                            # rows = 2 x_rows: the CFG duplication
@pytest.mark.parametrize("p", [2, 4, 8])                                 # 2: the specialised kernel; 4, 8: the generic one
def test_patch_embed(dev, p, G, D, x_rows, rows):
    Cc, T = 4, G * G
    M, Pn, side = rows * T, Cc * p * p, p * G
    g = gen(p * 100 + G + D + rows)
    # `rows` latents, of which the kernel may read only the first x_rows: the others differ and must never reach the output
    x = randn(rows, Cc, side, side, g=g)
    Wt, bias, pos = randn(Pn, D, g=g) * Pn ** -0.5, randn(D, g=g) * 0.1, randn(T, D, g=g) * 0.5
    tok = nan_like((M, D))
    done(_lib.load().lfm_dbg_patch_embed(ptr(x), x_rows, ptr(Wt), ptr(bias), ptr(pos), ptr(tok), D, G, Cc, p, M, None))
    src = x[:x_rows].double()[torch.arange(rows, device="cuda") % x_rows]
    patch = src.reshape(rows, Cc, G, p, G, p).permute(0, 2, 4, 1, 3, 5).reshape(M, Pn)     # patch vector order (c, pp, q)
    posr = pos.double().repeat(rows, 1)
    ref = patch @ Wt.double() + bias.double() + posr
    absref = patch.abs() @ Wt.double().abs() + bias.double().abs() + posr.abs()
    tk.assert_within(tok, ref, tk.dot_c(Pn) * absref, f"patch_embed: p {p} G {G} D {D} x_rows {x_rows} rows {rows}")
    if rows == 2 * x_rows:
        assert torch.equal(tok[:M // 2], tok[M // 2:]), "the CFG half differs from the rows it duplicates"


# ------------------------------------------------------------------------------------------------ FinalLayer + unpatchify


# (p, G, B, D, modulation): every case with M > 16 x SMs rows makes each warp of the 2-blocks-per-SM grid loop
FINAL_CASES = [
    (2, 16, 16, 1152, "sample"), (2, 16, 3, 384, "shared"), (2, 32, 3, 1024, "sample"), (2, 4, 150, 768, "sample"),
    (4, 8, 40, 768, "sample"), (4, 16, 3, 1152, "shared"), (4, 32, 3, 384, "sample"),     # 64 outputs: two 32-output chunks
    (8, 4, 150, 1152, "sample"), (8, 8, 2, 384, "shared"), (8, 32, 3, 768, "sample"),     # 256 outputs: eight chunks
]


@pytest.mark.parametrize("p,G,B,D,mod", FINAL_CASES)
def test_final_layer(dev, p, G, B, D, mod):
    Cc, T, L = 4, G * G, 2
    M, Pout, side = B * T, p * p * Cc, p * G
    g = gen(p * 1000 + G + B + D)
    x = randn(M, D, g=g) * torch.exp(randn(M, 1, g=g) * 0.5) + randn(M, 1, g=g)   # distinct rows: no two tokens alike
    table = modulation_table(B if mod == "sample" else 1, D, L, g)
    stride = table.shape[1] if mod == "sample" else 0
    mf = 6 * L * D                                                                  # final_layer's shift | scale
    W, bias = randn(Pout, D, g=g) * D ** -0.5, randn(Pout, g=g) * 0.1
    v_net = nan_like((B, Cc, side, side))
    done(_lib.load().lfm_dbg_final_layer(ptr(x), ptr(table, mf), ptr(table, mf + D), stride, ptr(W), ptr(bias), ptr(v_net), M, D, G,
                                         Cc, p, None))
    yn, ey = layernorm_ref(x, table[:, mf:mf + D], table[:, mf + D:mf + 2 * D], T)
    Wd = W.double()
    out = yn @ Wd.t() + bias.double()
    bound = (D / 32 + 8) * U * (yn.abs() @ Wd.abs().t() + bias.double().abs()) + ey @ Wd.abs().t()

    def unpatchify(o):   # out-feature (pp p + q) C + c of token (gh, gw) -> pixel (c, p gh + pp, p gw + q)
        return o.reshape(B, G, G, p, p, Cc).permute(0, 5, 1, 3, 2, 4).reshape(B, Cc, side, side)

    tk.assert_within(v_net, unpatchify(out), unpatchify(bound), f"final_layer: p {p} G {G} B {B} D {D} {mod}")


# ------------------------------------------------------------------------------------------------ GEMM at the DiT's shapes


def gemm_ref(a, w, bias):
    """fp64 A W^T + b on the bf16 operands, and |A| |W|^T + |b|."""
    ad, wd = a.double(), w.double()
    acc, absacc = ad @ wd.t(), ad.abs() @ wd.abs().t()
    if bias is not None:
        acc, absacc = acc + bias.double(), absacc + bias.double().abs()
    return acc, absacc


def gemm_expect(epi, acc, absacc, K, x0=None, gate=None):
    """The reference output of epilogue `epi` and its elementwise bound (see the header).  gate: [M, N] rows of the gate, or None
    (gate 1: the plain residual add)."""
    err = tk.dot_c(K) * absacc
    if epi == 3:
        return acc, err
    if epi == 2:
        gd = gate.double() if gate is not None else torch.ones_like(acc)
        return x0.double() + gd * acc, gd.abs() * err + tk.dot_c(K) * x0.double().abs()
    if epi == 0:
        return acc, tk.bf16_ulp(acc) + err
    inner = acc * (0.7978845608028654 * (1 + 0.044715 * acc * acc))
    th = torch.tanh(inner)
    ref = 0.5 * acc * (1 + th)
    gelu_err = 1.13 * err + 0.5 * acc.abs() * th.abs() * TANH_REL + 2.0 ** -21 * acc.abs() * inner.abs() + 2.0 ** -23 * ref.abs()
    return ref, tk.bf16_ulp(ref) + gelu_err


def run_gemm(a, w, bias, out, gate_ptr, gate_stride, rows_per_sample, M, N, K, epi, block_n, reversed_m):
    entry = _lib.load().lfm_dbg_gemm_reversed if reversed_m else _lib.load().lfm_dbg_gemm
    done(entry(ptr(a), ptr(w), tk.P(bias), ptr(out), gate_ptr, gate_stride, rows_per_sample, M, N, K, epi, block_n, None))


# preset: (D, Dq, mlp hidden, depth); DiT-XL's 72-channel heads are stored zero-padded to 80 (Dq = 1280)
PRESETS = {"S": (384, 384, 1536, 12), "B": (768, 768, 3072, 12), "L": (1024, 1024, 4096, 24), "XL": (1152, 1280, 4608, 28)}
# (op, epi): qkv bias -> bf16, proj gated residual, fc1 bias + GELU -> bf16, fc2 gated residual
OPS = {"qkv": 0, "proj": 2, "fc1": 1, "fc2": 2}


def op_shape(op, D, Dq, Hd):
    return {"qkv": (3 * Dq, D), "proj": (D, Dq), "fc1": (Hd, D), "fc2": (D, Hd)}[op]


# (T, B): tokens per sample (the gate's rows_per_sample) and batch; T = 16 with an odd batch leaves an M tail in the last tile
TOKEN_BATCHES = [(16, 13), (64, 5), (256, 3), (1024, 2)]


def check_dit_gemm(preset, op, T, B):
    D, Dq, Hd, L = PRESETS[preset]
    N, K = op_shape(op, D, Dq, Hd)
    epi, M = OPS[op], B * T
    g = gen(list(PRESETS).index(preset) * 10000 + list(OPS).index(op) * 2000 + T + B)
    a = (randn(M, K, g=g) * (3.0 if epi == 1 else 1.0)).bfloat16()     # fc1: pre-activations reach GELU's negative tail
    w = (randn(N, K, g=g) * K ** -0.5).bfloat16()
    bias = randn(N, g=g) * 0.1
    acc, absacc = gemm_ref(a, w, bias)
    Nmod = (6 * L + 2) * D
    table = modulation_table(B, D, L, g)
    goff = (2 if op == "proj" else 5) * D                                  # gate_msa / gate_mlp of block 0: mb + 2 D, mb + 5 D
    x0 = randn(M, N, g=g)
    strides = (Nmod, 0) if epi == 2 else (0,)
    for block_n in (128, 256):
        for reversed_m in (False, True):
            for stride in strides:
                what = f"gemm epi {epi}: {preset} {op} T {T} B {B} bn {block_n} reversed {reversed_m} gate stride {stride}"
                if epi == 2:
                    out = x0.clone()
                    gate = table[torch.arange(M, device="cuda") // T if stride else torch.zeros(M, dtype=torch.long, device="cuda"),
                                 goff:goff + D]
                    ref, bound = gemm_expect(epi, acc, absacc, K, x0, gate)
                    run_gemm(a, w, bias, out, ptr(table, goff), stride, T, M, N, K, epi, block_n, reversed_m)
                else:
                    out = nan_like((M, N), torch.bfloat16)
                    ref, bound = gemm_expect(epi, acc, absacc, K)
                    run_gemm(a, w, bias, out, None, 0, T, M, N, K, epi, block_n, reversed_m)
                tk.assert_within(out, ref, bound, what)


@pytest.mark.parametrize("T,B", TOKEN_BATCHES)
@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("preset", list(PRESETS))
def test_dit_gemm(dev, preset, op, T, B):
    check_dit_gemm(preset, op, T, B)


@pytest.mark.parametrize("op", list(OPS))
def test_dit_gemm_dit_l_batch64(dev, op):
    """DiT-L/2 at batch 64 (M = 16384), the benchmark's headline shapes."""
    check_dit_gemm("L", op, 256, 64)


@pytest.mark.parametrize("crows", [1, 37, 74])   # the uniform-c row, B labelled rows, and 2 B under CFG
@pytest.mark.parametrize("preset", list(PRESETS))
def test_dit_adaln_gemm(dev, preset, crows):
    """All adaLN modulation vectors of the network in one GEMM: mod[crows, (6 L + 2) D] = c W^T + b (fp32)."""
    D, _, _, L = PRESETS[preset]
    N, K = (6 * L + 2) * D, D
    g = gen(crows + D)
    a = randn(crows, K, g=g).bfloat16()
    w = (randn(N, K, g=g) * K ** -0.5).bfloat16()
    bias = randn(N, g=g) * 0.1
    ref, bound = gemm_expect(3, *gemm_ref(a, w, bias), K)
    for block_n in (128, 256):
        for reversed_m in (False, True):
            out = nan_like((crows, N))
            run_gemm(a, w, bias, out, None, 0, 1, crows, N, K, 3, block_n, reversed_m)
            tk.assert_within(out, ref, bound, f"gemm epi 3: adaLN {preset} rows {crows} bn {block_n} reversed {reversed_m}")
