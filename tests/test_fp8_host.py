"""CPU checks of the DiT's FP8 mode (lfm_set_fp8): the C-ABI surface, the argument checks of its kernel-level entries, the Python
and command-line switches, and the FP8 emulation the GPU tests compare against (tests/tools/fp8_oracle.py)."""
import ctypes
import types

import pytest
import torch

from lfm_b200 import _lib, cli
from tests.test_lib_symbols import header_symbols
from tests.tools import fp8_oracle

FP8_SYMBOLS = ["lfm_set_fp8", "lfm_dbg_gemm_fp8", "lfm_dbg_ln_modulate_fp8", "lfm_dbg_quantize_rows_fp8"]


@pytest.fixture(scope="module")
def lib():
    from lfm_b200 import build
    build.build()
    return _lib.load()


def refused(rc, word):
    assert rc != 0
    assert word in _lib.last_error(), _lib.last_error()


def test_fp8_entries_in_header_binding_and_library(lib):
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in FP8_SYMBOLS:
        assert n in header_symbols() and n in _lib.SYMBOLS and hasattr(raw, n), n
    assert ctypes.sizeof(_lib.ModelDesc) == 9 * 4       # the mode is a call, not a descriptor field


def test_set_fp8_refuses_a_null_context(lib):
    refused(lib.lfm_set_fp8(None, 1), "null ctx")


def test_gemm_fp8_entry_refuses_bad_arguments(lib):
    p = ctypes.c_void_p(16)   # never dereferenced: every case is refused before the device is touched

    def gemm(M=256, N=1152, K=384, epi=0, block_n=0, a=p, sa=p, w=p, sw=p, out=p):
        return lib.lfm_dbg_gemm_fp8(a, sa, w, sw, None, out, M, N, K, epi, block_n, None)

    refused(gemm(K=320), "K of 128")          # a multiple of 64 but not of 128: one e4m3 slab is 128 elements
    refused(gemm(K=0), "K of 128")
    refused(gemm(N=1156), "N a positive multiple of 8")
    refused(gemm(M=0), "M must be >= 1")
    refused(gemm(epi=2), "epi must be 0")
    refused(gemm(epi=3), "epi must be 0")
    refused(gemm(block_n=64), "block_n")
    for name in ("a", "sa", "w", "sw", "out"):
        refused(gemm(**{name: None}), "must not be NULL")


def test_ln_modulate_fp8_entry_refuses_bad_arguments(lib):
    p = ctypes.c_void_p(256)

    def ln(D=1024, rps=256, M=512, stride=0, down=0, x=p, y=p, ys=p, sh=p, sc=p):
        return lib.lfm_dbg_ln_modulate_fp8(x, y, ys, sh, sc, stride, rps, M, D, down, None)

    refused(ln(D=512), "D must be 128 x")
    refused(ln(D=1000), "D must be 128 x")
    refused(ln(rps=24), "rows_per_sample")
    refused(ln(rps=0), "rows_per_sample")
    refused(ln(M=0), "M must be >= 1")
    refused(ln(stride=6), "mod_stride")
    refused(ln(stride=-4), "mod_stride")
    refused(ln(down=2), "down must be 0 or 1")
    for name in ("x", "y", "ys", "sh", "sc"):
        refused(ln(**{name: None}), "must not be NULL")
    refused(ln(x=ctypes.c_void_p(260)), "16-byte aligned")


def test_quantize_rows_fp8_entry_refuses_bad_arguments(lib):
    p = ctypes.c_void_p(16)
    refused(lib.lfm_dbg_quantize_rows_fp8(p, p, p, 0, 64, None), "N and K must be >= 1")
    refused(lib.lfm_dbg_quantize_rows_fp8(p, p, p, 64, 0, None), "N and K must be >= 1")
    refused(lib.lfm_dbg_quantize_rows_fp8(None, p, p, 4, 4, None), "must not be NULL")
    refused(lib.lfm_dbg_quantize_rows_fp8(p, None, p, 4, 4, None), "must not be NULL")
    refused(lib.lfm_dbg_quantize_rows_fp8(p, p, None, 4, 4, None), "must not be NULL")


def config(**kw):
    base = dict(model_type="DiT-S/2", image_size=256, f=8, num_in_channels=4, label_dropout=0.0, num_classes=1,
                use_origin_adm=False)
    base.update(kw)
    return types.SimpleNamespace(**base)


def test_create_network_passes_fp8_to_the_dit():
    from lfm_b200 import DiT, DiT_models, create_network
    with torch.device("meta"):
        assert create_network(config(fp8=True)).fp8
        assert not create_network(config()).fp8                      # a config without the attribute: off
        assert not create_network(config(fp8=False)).fp8
        assert DiT_models["DiT-XL/2"](fp8=True).fp8 and not DiT_models["DiT-B/4"]().fp8
        assert not DiT(depth=1, hidden_size=256, num_heads=4).fp8


def test_create_network_refuses_fp8_on_the_unets():
    from lfm_b200 import create_network
    with pytest.raises(ValueError, match="DiT models only"):
        create_network(config(model_type="adm", use_origin_adm=True, fp8=True))      # UNetModel
    with pytest.raises(ValueError, match="DiT models only"):
        create_network(config(model_type="adm", fp8=True))                           # DhariwalUNet (EDM)


def test_fp8_flag_parses_and_defaults_off():
    a = cli.build_parser().parse_args([])
    assert a.fp8 is False
    # the reference's defaults (test_flow_latent.py:302-408) are those without the flag
    assert (a.generator, a.seed, a.n_sample, a.model_type, a.method, a.atol, a.rtol) == ("determ", 42, 50000, "adm", "dopri5", 1e-5, 1e-5)
    assert (a.step_size, a.num_steps, a.scale_factor, a.f, a.batch_size, a.cfg_scale) == (0.01, 40, 0.18215, 8, 200, 1.0)
    b = cli.build_parser().parse_args("--model_type DiT-L/2 --fp8 --method euler --num_steps 10".split())
    assert b.fp8 and b.model_type == "DiT-L/2" and b.method == "euler"
    assert {k: v for k, v in vars(b).items() if k not in ("fp8", "model_type", "method", "num_steps")} == \
        {k: v for k, v in vars(a).items() if k not in ("fp8", "model_type", "method", "num_steps")}


def test_cli_builds_an_fp8_dit_and_refuses_an_fp8_unet():
    common = ["--image_size", "256", "--f", "8", "--num_in_channels", "4", "--num_out_channels", "4", "--nf", "128",
              "--synthetic_init", "3", "--no_decode", "--fp8"]
    net = cli.load_model(cli.build_parser().parse_args(common + ["--model_type", "DiT-S/2", "--num_classes", "1"]),
                         torch.device("cpu"))
    assert net.fp8
    with pytest.raises(ValueError, match="DiT models only"):
        cli.load_model(cli.build_parser().parse_args(common + ["--model_type", "adm", "--use_origin_adm", "--ch_mult", "1", "2",
                                                               "--attn_resolutions", "2", "--num_res_blocks", "1"]),
                       torch.device("cpu"))


def e4m3_grid():
    """Every finite e4m3 value (codes 0..126 and their negatives), with the code's mantissa parity."""
    codes = torch.arange(256, dtype=torch.int32)
    vals = codes.to(torch.uint8).view(torch.float8_e4m3fn).double()
    keep = torch.isfinite(vals)
    return vals[keep], (codes[keep] & 1)


def nearest_even_e4m3(x):
    """Round-to-nearest-even onto the e4m3 grid by exhaustive search (fp64), saturating at +-448."""
    vals, odd = e4m3_grid()
    xd = x.double().clamp(-448.0, 448.0).reshape(-1, 1)
    d = (xd - vals.reshape(1, -1)).abs()
    best = d.min(dim=1, keepdim=True).values
    tie = (d == best)
    pick = torch.where(tie & (odd.reshape(1, -1) == 0), 0, 1).to(torch.int64)   # prefer the even code among the nearest
    pick = torch.where(tie, pick, 2)
    idx = pick.argmin(dim=1)
    return vals[idx].reshape(x.shape)


def test_emulated_quantiser_matches_float8_e4m3fn():
    g = torch.Generator().manual_seed(5)
    w = torch.randn(64, 384, generator=g) * torch.exp(torch.randn(64, 1, generator=g) * 3)
    w[3] = 0.0                                                    # zero rows: DiT-XL's padded head channels
    w[7, :] = 0.0
    w[7, 5] = -2.5e-3                                             # one non-zero entry: amax from a negative value
    w[11] = torch.arange(384) * 2.0 ** -12                        # subnormal codes
    q, s = fp8_oracle.quantize_rows(w)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32
    amax = w.abs().amax(1)
    assert torch.equal(s, torch.where(amax > 0, amax / 448.0, torch.ones_like(amax)))
    assert s[3] == 1.0 and torch.equal(q[3].float(), torch.zeros(384))
    assert torch.equal(q.float().abs().amax(1)[amax > 0], torch.full((63,), 448.0))   # every non-zero row spans the range
    assert torch.equal(q.double(), nearest_even_e4m3(w / s[:, None]))
    assert torch.isfinite(q.float()).all()


def test_emulated_fp8_linear_is_the_dequantised_product():
    g = torch.Generator().manual_seed(6)
    x, w, b = torch.randn(5, 256, generator=g), torch.randn(24, 256, generator=g), torch.randn(24, generator=g)
    qx, sx = fp8_oracle.quantize_rows(x)
    qw, sw = fp8_oracle.quantize_rows(w)
    ref = (qx.double() * sx.double()[:, None]) @ (qw.double() * sw.double()[:, None]).t() + b.double()
    out = fp8_oracle.fp8_linear(x, w, b)
    assert float((out.double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    rel = float((out.double() - x.double() @ w.double().t() - b.double()).norm() / (x.double() @ w.double().t()).norm())
    assert rel < 0.1                                              # e4m3 keeps 3 mantissa bits: a few percent


def test_emulated_forward_runs_on_the_cpu():
    import dataclasses
    from oracle import dit as odit
    cfg = dataclasses.replace(odit.make_config("DiT-S/2", img_resolution=8, num_classes=1), depth=2)
    sd = odit.synthetic_state_dict(cfg, 3)
    x = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(1))
    v8 = fp8_oracle.dit_forward_fp8(sd, cfg, torch.tensor(0.3), x)
    v = odit.dit_forward(sd, cfg, torch.tensor(0.3), x, emulate_bf16=True)
    assert v8.shape == v.shape and torch.isfinite(v8).all()
    assert 0 < float((v8 - v).norm() / v.norm()) < 0.1
