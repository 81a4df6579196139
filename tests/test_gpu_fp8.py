"""The DiT's FP8 mode (lfm_set_fp8) on the H100 (`-m gpu`): its three kernels element by element, the forward against the FP8
emulation of the oracle (tests/tools/fp8_oracle.py) and against the plain fp32 oracle, the samplers, the refusals, and the
default (bf16) path's launch count.

Bounds:
  * weight quantiser: bit-exact, codes and scales, against (w / s).to(torch.float8_e4m3fn) with s = amax / 448 (1 for a zero row).
  * ln_modulate with e4m3 output: the row scale is amax / 448 of the kernel's own fp32 row, whose error against the fp64 LayerNorm
    is test_gpu_dit_kernels' bound, so the scale agrees to that bound at the amax element (relative) plus 4 fp32 ulp.  The fp32
    statistics are summed in another order than any reference, so a value within that error of a rounding boundary between two e4m3
    codes may land on either side: at most 1e-3 of the codes differ from e4m3(ref / scale), each by one e4m3 step.
  * GEMM: against the fp64 product of the e4m3 codes times a_scale[m] w_scale[n], then the epilogue.  The products of two e4m3
    values are exact, but the H100's FP8 wgmma does not add them at fp32 precision: each k32 step's sum enters the accumulator
    aligned to the largest magnitude and cut to about 14 significant bits (DeepSeek-V3 technical report, section 3.3.2, measured on
    H800).  Against test_gpu_dit_kernels' bf16 GEMM bound (fp32 summation slack (K + 16) 2^-23 |A||W|, one bf16 ulp, the GELU terms)
    the kernel's error reached 1.0 to 3.1 times that bound at the qkv / fc1 shapes of S, B, L and XL (3.1 at K = 384; an NVIDIA
    H100 80GB HBM3 at 700 W).  So the bound adds (K / 32) 2^-13 |A||W| a_scale w_scale: one 2^-13 cut per k32 step on at most the
    final |A||W|.  That is ~30x the fp32 slack at K = 384 and still ~1e-3 of |A||W|, far below what a wrong row, column, scale or
    slab would cost.
  * forward: rel-L2 against the oracle with FP8 emulation below the bf16 forward's tolerance (test_gpu_parity.TOL_NFE), and against
    the fp32 oracle (the stored fixtures) below 5e-2.
"""
import ctypes as C
import types

import pytest
import torch

import lfm_b200
from lfm_b200 import _lib
from oracle import dit as odit
from tests import test_gpu_dit_kernels as dk
from tests import test_gpu_kernels as tk
from tests._util import T, cfg_from_golden, load_golden, rel_l2
from tests.test_gpu_parity import GEOMETRY, TOL_NFE, make_big, make_net
from tests.tools import fp8_oracle

pytestmark = pytest.mark.gpu

TOL_FP32 = 5e-2     # FP8 forward against the fp32 oracle (rel-L2)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def codes_u8(q):
    return q.view(torch.uint8)


def report(what, value):
    print(f"\n[fp8] {what}: {value}")


# ------------------------------------------------------------------------------------------------ weight quantiser


def padded_qkv(D, heads, dh, dhp, g):
    """An XL-style qkv weight in the stored order: 3 heads dhp rows, rows c >= dh of every head zero."""
    w = torch.zeros(3 * heads, dhp, D, device="cuda")
    w[:, :dh] = dk.randn(3 * heads, dh, D, g=g) * D ** -0.5
    return w.reshape(3 * heads * dhp, D)


@pytest.mark.parametrize("case", ["xl_qkv_padded", "xl_fc1", "s_qkv_zero_rows", "tiny_rows"])
def test_quantize_rows_bit_exact(dev, case):
    g = dk.gen(len(case))
    if case == "xl_qkv_padded":
        w = padded_qkv(1152, 16, 72, 80, g)
    elif case == "xl_fc1":
        w = dk.randn(4608, 1152, g=g) * torch.exp(dk.randn(4608, 1, g=g))
    elif case == "s_qkv_zero_rows":
        w = dk.randn(1152, 384, g=g) * 384 ** -0.5
        w[::7] = 0.0
        w[5, :] = 0.0
        w[5, 100] = -3e-4
    else:
        w = dk.randn(37, 40, g=g) * 2.0 ** -10     # K not a multiple of 32; subnormal codes
    N, K = w.shape
    codes = torch.full((N, K), 0x7F, dtype=torch.uint8, device="cuda")       # NaN codes where nothing is written
    scales = dk.nan_like((N,))
    dk.done(_lib.load().lfm_dbg_quantize_rows_fp8(dk.ptr(w), dk.ptr(codes), dk.ptr(scales), N, K, None))
    q, s = fp8_oracle.quantize_rows(w)
    assert torch.equal(scales, s)
    assert torch.equal(codes, codes_u8(q))
    zero = w.abs().amax(1) == 0
    assert bool((scales[zero] == 1).all()) and not bool(codes[zero].any())


# ------------------------------------------------------------------------------------------------ LayerNorm + modulate -> e4m3


def e4m3_step_apart(a, b):
    """a, b: uint8 e4m3 codes.  True where they are equal or one e4m3 step apart (through zero: +-the smallest subnormal)."""
    sa, sb = a >> 7, b >> 7
    ma, mb = (a & 0x7F).int(), (b & 0x7F).int()
    same = (sa == sb) & ((ma - mb).abs() <= 1)
    through_zero = (ma + mb) <= 1
    return same | through_zero


LN_FP8_SCENARIOS = [(16, "sms", "sample", "normal"), (64, 3, "shared", "normal"), (256, 64, "sample", "normal"),
                    (1024, 5, "sample", "normal"), (256, 4, "sample", "mean50"), (1024, 2, "sample", "small"),
                    (256, 3, "sample", "large")]


@pytest.mark.parametrize("down", [0, 1])
@pytest.mark.parametrize("T,B,mod,kind", LN_FP8_SCENARIOS)
@pytest.mark.parametrize("D", [384, 768, 1024, 1152])
def test_ln_modulate_fp8(dev, D, T, B, mod, kind, down):
    if B == "sms":
        B = tk.num_sms()
    M, L = B * T, 2
    g = dk.gen(D + T + M + down + 7)
    x = dk.ln_rows(kind, M, D, g)
    table = dk.modulation_table(B if mod == "sample" else 1, D, L, g)
    stride = table.shape[1] if mod == "sample" else 0
    shift, scale = table[:, 3 * D:4 * D], table[:, 4 * D:5 * D]
    y = torch.full((M, D), 0x7F, dtype=torch.uint8, device="cuda")
    ys = dk.nan_like((M,))
    dk.done(_lib.load().lfm_dbg_ln_modulate_fp8(dk.ptr(x), dk.ptr(y), dk.ptr(ys), dk.ptr(table, 3 * D), dk.ptr(table, 4 * D), stride,
                                                 T, M, D, down, None))
    ref, err = dk.layernorm_ref(x, shift, scale, T)
    amax = ref.abs().amax(1)
    s_ref = amax / 448.0
    s_tol = err.amax(1) / 448.0 + 4 * 2.0 ** -23 * s_ref
    what = f"ln_modulate_fp8: D {D} T {T} B {B} {mod} {kind} down {down}"
    assert bool(((ys.double() - s_ref).abs() <= s_tol).all()), what
    ref_codes = codes_u8((ref / ys.double()[:, None]).float().to(torch.float8_e4m3fn))
    diff = y != ref_codes
    assert bool(e4m3_step_apart(y, ref_codes).all()), what
    assert float(diff.double().mean()) <= 1e-3, f"{what}: {float(diff.double().mean()):.2e} of the codes differ"


# ------------------------------------------------------------------------------------------------ GEMM


def fp8_operand(rows, K, spread, g):
    v = dk.randn(rows, K, g=g) * torch.exp(dk.randn(rows, 1, g=g) * spread)
    return fp8_oracle.quantize_rows(v)


def check_fp8_gemm(M, N, K, epi, block_n, seed):
    g = dk.gen(seed)
    qa, sa = fp8_operand(M, K, 0.5, g)
    qw, sw = fp8_operand(N, K, 0.3, g)
    sa = sa * (3.0 if epi == 1 else 1.0) * K ** -0.5          # fc1: pre-activations reach GELU's negative tail
    bias = dk.randn(N, g=g) * 0.1
    ad, wd = qa.double(), qw.double()
    scale = sa.double()[:, None] * sw.double()[None, :]
    acc = (ad @ wd.t()) * scale + bias.double()
    absacc = (ad.abs() @ wd.abs().t()) * scale + bias.double().abs()
    slack = tk.dot_c(K) + K / 32 * 2.0 ** -13                     # fp32 roundings + the FP8 wgmma's accumulation (header)
    ref, bound = dk.gemm_expect(epi, acc, absacc * (slack / tk.dot_c(K)), K)
    del ad, wd, scale, absacc
    out = dk.nan_like((M, N), torch.bfloat16)
    dk.done(_lib.load().lfm_dbg_gemm_fp8(dk.ptr(qa), dk.ptr(sa), dk.ptr(qw), dk.ptr(sw), dk.ptr(bias), dk.ptr(out), M, N, K, epi,
                                         block_n, None))
    tk.assert_within(out, ref, bound, f"gemm_fp8 {M}x{N}x{K} epi {epi} bn {block_n}")


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("M", [16384, 13 * 16])                  # DiT-L/2 at batch 64; an M tail (208 rows)
@pytest.mark.parametrize("op", ["qkv", "fc1"])
@pytest.mark.parametrize("preset", list(dk.PRESETS))
def test_fp8_gemm_dit_shapes(dev, preset, op, M, block_n):
    D, Dq, Hd, _ = dk.PRESETS[preset]
    N, K = dk.op_shape(op, D, Dq, Hd)                             # XL qkv: N = 3 x 1280
    check_fp8_gemm(M, N, K, dk.OPS[op], block_n, list(dk.PRESETS).index(preset) * 100 + 10 * (op == "fc1") + M % 7 + block_n)


def test_fp8_gemm_network_tile_pick(dev):
    check_fp8_gemm(300, 1152, 384, 0, 0, 11)                       # block_n 0: the network's pick; an N tail of 128


# ------------------------------------------------------------------------------------------------ forward


def fp8_net(cfg, sd, dev, max_batch=None):
    net = make_net(cfg, sd, dev, max_batch)
    net.fp8 = True
    net.mark_dirty()
    return net


@pytest.mark.parametrize("name", ["mini_uncond", "mini_cond", "mini_d384"] + GEOMETRY)
def test_forward_fixture_fp8(dev, name):
    g = load_golden(name)
    cfg = cfg_from_golden(g)
    sd = odit.synthetic_state_dict(cfg, int(g["weight_seed"]))
    net = fp8_net(cfg, sd, dev)
    x = T(g["x"])
    v = net(T(g["t_vec"]).to(dev), x.to(dev), T(g["y"]).to(dev)).cpu()
    emu = fp8_oracle.dit_forward_fp8(sd, cfg, T(g["t_vec"]), x, T(g["y"]))
    r_emu, r_fp32 = rel_l2(v, emu), rel_l2(v, g["v_vec_y"])
    report(f"forward {name}: rel-L2 vs FP8 emulation / vs fp32 oracle", f"{r_emu:.3e} / {r_fp32:.3e}")
    assert r_emu < TOL_NFE
    assert r_fp32 < TOL_FP32
    if cfg.num_classes > 1:
        x2 = torch.cat([x, x])
        tt = torch.full((4,), 0.4)
        v = net.forward_with_cfg(tt.to(dev), x2.to(dev), T(g["y_cfg"]).to(dev), cfg_scale=1.5).cpu()
        emu = fp8_oracle.dit_forward_with_cfg_fp8(sd, cfg, tt, x2, T(g["y_cfg"]), 1.5)
        assert rel_l2(v, emu) < TOL_NFE
        assert rel_l2(v, g["v_cfg_1p5"]) < TOL_FP32


def big_fp8(model_type, dev, num_classes, label_dropout, max_batch):
    net = make_big(model_type, dev, num_classes, label_dropout, max_batch)
    net.fp8 = True
    net.mark_dirty()
    return net


def test_forward_dit_l2_fp8(dev):
    g = load_golden("dit_l2")
    net = big_fp8("DiT-L/2", dev, 1, 0.0, 2)
    cfg = odit.make_config("DiT-L/2", num_classes=1)
    sd = {k: v.detach().float().cpu() for k, v in net.state_dict().items()}
    x = T(g["x"])
    v = net(T(g["t"]).to(dev), x.to(dev)).cpu()
    emu = fp8_oracle.dit_forward_fp8(sd, cfg, T(g["t"]), x)
    r_emu, r_fp32 = rel_l2(v, emu), rel_l2(v, g["v"])
    report("forward dit_l2: rel-L2 vs FP8 emulation / vs fp32 oracle", f"{r_emu:.3e} / {r_fp32:.3e}")
    assert r_emu < TOL_NFE and r_fp32 < TOL_FP32


def test_forward_dit_b2_cfg_fp8(dev):
    g = load_golden("dit_b2")
    net = big_fp8("DiT-B/2", dev, 1000, 0.1, 4)
    cfg = odit.make_config("DiT-B/2", num_classes=1000, label_dropout=0.1)
    sd = {k: v.detach().float().cpu() for k, v in net.state_dict().items()}
    x2 = torch.cat([T(g["x"])] * 2)
    v = net.forward_with_cfg(T(g["t"]).to(dev), x2.to(dev), T(g["y_cfg"]).to(dev), cfg_scale=1.5).cpu()
    emu = fp8_oracle.dit_forward_with_cfg_fp8(sd, cfg, T(g["t"]), x2, T(g["y_cfg"]), 1.5)
    r_emu, r_fp32 = rel_l2(v, emu), rel_l2(v, g["v_cfg_1p5"])
    report("forward dit_b2 CFG 1.5: rel-L2 vs FP8 emulation / vs fp32 oracle", f"{r_emu:.3e} / {r_fp32:.3e}")
    assert r_emu < TOL_NFE and r_fp32 < TOL_FP32


# ------------------------------------------------------------------------------------------------ sampling


def pair(model_type, dev, num_classes, label_dropout, max_batch):
    return (make_big(model_type, dev, num_classes, label_dropout, max_batch),
            big_fp8(model_type, dev, num_classes, label_dropout, max_batch))


def test_euler10_dit_l2_batch64(dev):
    bf16, fp8 = pair("DiT-L/2", dev, 1, 0.0, 64)
    x = torch.randn(64, 4, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
    args = types.SimpleNamespace(method="euler", step_size=0.1, cfg_scale=1.0)
    a = lfm_b200.sample_from_model(bf16, x, {}, args)[-1]
    b = lfm_b200.sample_from_model(fp8, x, {}, args)[-1]
    r = rel_l2(b.cpu(), a.cpu())
    report("Euler-10 DiT-L/2 batch 64: rel-L2 FP8 vs bf16 final latents", f"{r:.3e}")
    assert torch.isfinite(b).all() and r < TOL_FP32


def test_heun_and_dopri5_dit_b2_cfg(dev):
    bf16, fp8 = pair("DiT-B/2", dev, 1000, 0.1, 8)
    x = torch.randn(4, 4, 32, 32, generator=torch.Generator().manual_seed(4)).to(dev)
    y = torch.tensor([1, 207, 360, 999, 1000, 1000, 1000, 1000], device=dev)
    mk = dict(y=y, cfg_scale=1.5)
    kw = dict(clip_denoised=False, model_kwargs=mk, sigma_min=1e-5, sigma_max=1.0, sampler="heun")
    a = lfm_b200.karras_sample(bf16, torch.cat([x, x]), 10, **kw)
    b = lfm_b200.karras_sample(fp8, torch.cat([x, x]), 10, **kw)
    r = rel_l2(b.cpu(), a.cpu())
    report("Heun-10 DiT-B/2 CFG 1.5: rel-L2 FP8 vs bf16", f"{r:.3e}")
    assert torch.isfinite(b).all() and r < TOL_FP32
    args = types.SimpleNamespace(method="dopri5", atol=1e-5, rtol=1e-5, cfg_scale=1.5, compute_nfe=True)
    (ta, na), (tb, nb) = (lfm_b200.sample_from_model(m, torch.cat([x, x]), mk, args) for m in (bf16, fp8))
    r = rel_l2(tb[-1].cpu(), ta[-1].cpu())
    report("dopri5 DiT-B/2 CFG 1.5: NFE bf16 / FP8, rel-L2 FP8 vs bf16", f"{int(na)} / {int(nb)}, {r:.3e}")
    assert torch.isfinite(tb[-1]).all() and r < TOL_FP32


# ------------------------------------------------------------------------------------------------ refusals and the default path


def test_set_fp8_refusals(dev):
    lib = _lib.load()
    cfg = cfg_from_golden(load_golden("mini_uncond"))
    net = make_net(cfg, odit.synthetic_state_dict(cfg, 1), dev)
    ctx = net.native(2, dev)                                           # finalized
    assert lib.lfm_set_fp8(ctx, 1) != 0 and "finalized" in _lib.last_error(ctx)
    from oracle import unet as ounet
    from tests.test_gpu_parity import make_unet
    from tests.test_oracle_unet import unet_cfg_from_golden
    ucfg = unet_cfg_from_golden(load_golden("unet_mini"))
    uctx = make_unet(ucfg, ounet.synthetic_state_dict(ucfg, 1), dev)._create_ctx(lib, 0)
    try:
        assert lib.lfm_set_fp8(uctx, 1) != 0 and "UNet" in _lib.last_error(uctx)
    finally:
        lib.lfm_destroy(uctx)
    # a weight uploaded in one mode cannot be re-read in the other
    dctx = net._create_ctx(lib, 0)
    try:
        key = "blocks.0.mlp.fc1.weight"
        w = net.state_dict()[key].detach().float().contiguous()
        shape = (C.c_int64 * 2)(*w.shape)
        _lib.check(lib.lfm_set_param(dctx, key.encode(), C.c_void_p(w.data_ptr()), 0, shape, 2), dctx)
        assert lib.lfm_set_fp8(dctx, 1) != 0 and key in _lib.last_error(dctx)
    finally:
        lib.lfm_destroy(dctx)


@pytest.mark.parametrize("name", ["mini_uncond", "mini_xl2"])
def test_launch_count_is_the_same_in_both_modes(dev, name):
    """3 conditioning kernels, the adaLN GEMM, patch embed, 7 launches per block, the final layer - as before the FP8 mode."""
    g = load_golden(name)
    cfg = cfg_from_golden(g)
    sd = odit.synthetic_state_dict(cfg, 1)
    x = T(g["x"]).to(dev)
    for net in (make_net(cfg, sd, dev), fp8_net(cfg, sd, dev)):
        net(0.5, x)
        before = net.launch_count()
        net(0.5, x)
        assert net.launch_count() - before == 6 + 7 * cfg.depth
