"""CPU-side checks of the C-ABI boundary: the library builds, loads, and exports every symbol the header declares.
No compute calls (there is no GPU here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from lfm_b200 import _lib, build
    build.build()
    return _lib.load()


def header_symbols():
    src = open(os.path.join(ROOT, "include", "lfm_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lfm_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree(lib):
    from lfm_b200 import _lib
    names = header_symbols()
    assert len(names) >= 10
    assert sorted(_lib.SYMBOLS) == names
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), f"liblfm_b200.so does not export {n}"


def test_struct_layouts():
    from lfm_b200 import _lib
    assert ctypes.sizeof(_lib.ModelDesc) == 9 * 4
    assert ctypes.sizeof(_lib.OdeStats) == 3 * 8
    assert ctypes.sizeof(_lib.UnetDesc) == 26 * 4
    assert ctypes.sizeof(_lib.EdmDesc) == 24 * 4


def test_create_fails_loudly_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from lfm_b200 import _lib
    desc = _lib.ModelDesc(0, 32, 2, 4, 256, 2, 4, 1024, 1)
    ctx = ctypes.c_void_p()
    rc = lib.lfm_create(ctypes.byref(desc), 0, ctypes.byref(ctx))
    assert rc != 0
    assert "CUDA" in _lib.last_error() or "device" in _lib.last_error()


def test_unsupported_shapes_are_rejected(lib):
    from lfm_b200 import _lib
    ctx = ctypes.c_void_p()
    bad = _lib.ModelDesc(0, 32, 2, 4, 1024, 24, 8, 4096, 1)  # head_dim 128: only 64 and 72 (the reference's size table) are implemented
    assert lib.lfm_create(ctypes.byref(bad), 0, ctypes.byref(ctx)) != 0
    assert "head_dim" in _lib.last_error()
    bad = _lib.ModelDesc(0, 32, 3, 4, 1024, 24, 16, 4096, 1)  # patch 3 (the reference's table has 2, 4, 8)
    assert lib.lfm_create(ctypes.byref(bad), 0, ctypes.byref(ctx)) != 0
    assert "patch_size" in _lib.last_error()
    bad = _lib.ModelDesc(0, 128, 2, 4, 1024, 24, 16, 4096, 1)  # 128 x 128 latents with patch 2: 4096 tokens, not implemented
    assert lib.lfm_create(ctypes.byref(bad), 0, ctypes.byref(ctx)) != 0
    assert "token grid" in _lib.last_error()
    # GEMM tile widths are 128 and 256 (0: the network's pick); anything else is refused before the device is touched
    assert lib.lfm_dbg_gemm(None, None, None, None, None, 0, 1, 128, 128, 64, 3, 640, None) != 0
    assert "block_n" in _lib.last_error()


def test_kernel_entries_refuse_bad_arguments(lib):
    """Every kernel-level entry checks its shape arguments before it touches the device, and names the bad argument."""
    from lfm_b200 import _lib

    def refused(rc, word):
        assert rc != 0
        assert word in _lib.last_error(), _lib.last_error()

    # lfm_dbg_conv(x, w, bias, out, gn_bins, B, side, Cin, Cout, stride, block_n, epi, ksplit, stream)
    conv = lib.lfm_dbg_conv
    refused(conv(None, None, None, None, None, 1, 32, 128, 128, 1, 640, 3, -1, None), "block_n")
    refused(conv(None, None, None, None, None, 1, 32, 128, 128, 3, 0, 3, -1, None), "stride")
    refused(conv(None, None, None, None, None, 1, 2, 128, 128, 1, 0, 3, -1, None), "side")
    refused(conv(None, None, None, None, None, 1, 512, 128, 128, 1, 0, 3, -1, None), "side")
    refused(conv(None, None, None, None, None, 1, 32, 96, 128, 1, 0, 3, -1, None), "Cin")
    refused(conv(None, None, None, None, None, 1, 32, 128, 12, 1, 0, 3, -1, None), "Cout")
    refused(conv(None, None, None, None, None, 1, 32, 128, 128, 1, 0, 1, -1, None), "epi")
    refused(conv(None, None, None, None, None, 1, 32, 128, 128, 1, 0, 3, 9, None), "ksplit")
    refused(conv(None, None, None, None, None, 1, 32, 128, 128, 1, 0, 0, 2, None), "ksplit")
    refused(conv(None, None, None, None, None, 1, 32, 128, 128, 1, 256, 3, 4, None), "ksplit")
    refused(conv(None, None, None, None, None, 0, 32, 128, 128, 1, 0, 3, -1, None), "B")
    dummy = ctypes.c_void_p(64)   # never dereferenced: each call below is refused on its shape arguments
    refused(conv(None, None, None, None, dummy, 1, 32, 128, 128, 1, 0, 2, 1, None), "gn_bins")     # residual epilogue
    refused(conv(None, None, None, None, dummy, 1, 32, 128, 96, 1, 0, 3, 1, None), "gn_bins")      # 3 channels per group
    refused(conv(None, None, None, None, dummy, 1, 4, 128, 128, 1, 0, 3, 1, None), "gn_bins")      # 16 output pixels
    refused(conv(None, None, None, None, None, 1, 32, 128, 128, 1, 0, 3, -1, None), "NULL")
    # lfm_dbg_gemm_batched(a, a_rows, a_ld, w, w_rows, w_ld, K, N, out, bias, B, out_hw, epi, batch_m, a_mod, b_batch_rows, stream)
    bat = lib.lfm_dbg_gemm_batched
    refused(bat(None, 256, 512, None, 256, 512, 512, 128, None, None, 1, 256, 3, 256, 0, 256, None), "N")
    refused(bat(None, 256, 512, None, 256, 512, 96, 256, None, None, 1, 256, 3, 256, 0, 256, None), "K")
    refused(bat(None, 256, 256, None, 256, 512, 512, 256, None, None, 1, 256, 3, 256, 0, 256, None), "a_ld")
    refused(bat(None, 256, 512, None, 256, 512, 512, 256, None, None, 1, 256, 3, 200, 0, 256, None), "batch_m")
    refused(bat(None, 256, 512, None, 256, 512, 512, 256, None, None, 1, 256, 3, 256, 64, 256, None), "a_mod")
    refused(bat(None, 256, 512, None, 256, 512, 512, 256, None, None, 1, 256, 3, 256, 0, 128, None), "b_batch_rows")
    refused(bat(None, 256, 512, None, 256, 512, 512, 256, None, None, 1, 384, 3, 256, 0, 256, None), "batch_m")
    refused(bat(None, 256, 512, None, 256, 512, 512, 256, None, None, 1, 256, 2, 256, 0, 256, None), "epi")
    refused(bat(None, 256, 512, None, 256, 512, 512, 256, None, None, 1, 256, 3, 256, 0, 256, None), "NULL")
    # lfm_dbg_groupnorm(a, Ca, b, Cb, src_bf16, bins, max_chunks, gamma, beta, film, film_stride, act, eps, out, copy_out, raw_out,
    #                   B, HW, stream)
    gn = lib.lfm_dbg_groupnorm
    refused(gn(None, 200, None, 0, None, None, 32, None, None, None, 0, 1, 1e-5, None, None, None, 1, 64, None), "Ca + Cb")
    refused(gn(None, 2048, dummy, 256, None, None, 32, None, None, None, 0, 1, 1e-5, None, None, None, 1, 64, None), "Ca + Cb")
    refused(gn(None, 256, None, 512, None, None, 32, None, None, None, 0, 1, 1e-5, None, None, None, 1, 64, None), "Cb")
    refused(gn(None, 256, None, 0, None, None, 0, None, None, None, 0, 1, 1e-5, None, None, None, 1, 64, None), "max_chunks")
    refused(gn(None, 256, None, 0, None, None, 32, None, None, None, 0, 2, 1e-5, None, None, None, 1, 64, None), "act")
    refused(gn(None, 256, None, 0, None, None, 32, None, None, None, 0, 1, 0.0, None, None, None, 1, 64, None), "eps")
    refused(gn(None, 256, None, 0, None, None, 32, None, None, None, 0, 1, 1e-5, None, None, None, 0, 64, None), "B")
    refused(gn(None, 256, None, 0, None, None, 32, None, None, None, 0, 1, 1e-5, None, None, None, 1, 64, None), "NULL")
    # lfm_dbg_gemm_reversed: lfm_dbg_gemm's checks, under its own name
    rev = lib.lfm_dbg_gemm_reversed
    refused(rev(None, None, None, None, None, 0, 1, 128, 128, 64, 3, 640, None), "block_n")
    refused(rev(None, None, None, None, None, 0, 1, 128, 128, 96, 3, 0, None), "lfm_dbg_gemm_reversed: K")
    refused(rev(None, None, None, None, None, 0, 1, 128, 128, 64, 4, 0, None), "epilogue")
    # lfm_dbg_ln_modulate(x, y, shift, scale, mod_stride, rows_per_sample, M, D, down, stream)
    ln = lib.lfm_dbg_ln_modulate
    refused(ln(None, None, None, None, 0, 256, 512, 512, 0, None), "D")         # D / 128 = 4 has no instantiation
    refused(ln(None, None, None, None, 0, 256, 512, 1000, 0, None), "D")
    refused(ln(None, None, None, None, 0, 24, 512, 1024, 0, None), "rows_per_sample")
    refused(ln(None, None, None, None, 0, 0, 512, 1024, 0, None), "rows_per_sample")
    refused(ln(None, None, None, None, 0, 256, 0, 1024, 0, None), "M")
    refused(ln(None, None, None, None, 6, 256, 512, 1024, 0, None), "mod_stride")
    refused(ln(None, None, None, None, 0, 256, 512, 1024, 2, None), "down")
    refused(ln(None, None, None, None, 0, 256, 512, 1024, 0, None), "NULL")
    # lfm_dbg_patch_embed(x, x_rows, Wt, bias, pos, tok, D, G, C, p, M, stream)
    pe = lib.lfm_dbg_patch_embed
    refused(pe(None, 1, None, None, None, None, 384, 16, 4, 3, 256, None), "p")
    refused(pe(None, 1, None, None, None, None, 384, 16, 3, 2, 256, None), "C")
    refused(pe(None, 1, None, None, None, None, 384, 16, 32, 8, 256, None), "C")        # 8 x 2048 floats: 64 KB of shared memory
    refused(pe(None, 1, None, None, None, None, 386, 16, 4, 2, 256, None), "D")
    refused(pe(None, 0, None, None, None, None, 384, 16, 4, 2, 256, None), "x_rows")
    refused(pe(None, 1, None, None, None, None, 384, 16, 4, 2, 256, None), "NULL")
    # lfm_dbg_final_layer(x, shift, scale, mod_stride, W, bias, v_net, M, D, G, C, p, stream)
    fl = lib.lfm_dbg_final_layer
    refused(fl(None, None, None, 0, None, None, None, 256, 384, 16, 4, 6, None), "p")
    refused(fl(None, None, None, 0, None, None, None, 256, 384, 16, 3, 2, None), "C")    # the p = 2 kernel computes 16 outputs
    refused(fl(None, None, None, 0, None, None, None, 256, 1664, 16, 4, 2, None), "D")   # > 1536
    refused(fl(None, None, None, 0, None, None, None, 256, 320, 16, 4, 4, None), "D")
    refused(fl(None, None, None, 2, None, None, None, 256, 384, 16, 4, 2, None), "mod_stride")
    refused(fl(None, None, None, 0, None, None, None, 0, 384, 16, 4, 2, None), "M")
    refused(fl(None, None, None, 0, None, None, None, 256, 384, 16, 4, 2, None), "NULL")


def test_condition_entry_refuses_bad_arguments(lib):
    """lfm_dbg_condition checks its shapes, its label rule and its pointers before it touches the device, and names the bad
    argument: the K of both MLP layers (feat and E) is a multiple of 128 up to 4096."""
    from lfm_b200 import _lib

    def refused(rc, word):
        assert rc != 0
        assert word in _lib.last_error(), _lib.last_error()

    d = ctypes.c_void_p(64)   # never dereferenced: each call below is refused before the device is touched
    # lfm_dbg_condition(t, t_numel, y, rows, feat, E, w0, b0, w2, b2, table, max_row, null_row, tf, h1, c, stream)
    cond = lib.lfm_dbg_condition
    refused(cond(d, 1, None, 0, 256, 384, d, d, d, d, d, 10, 10, d, d, d, None), "rows")
    refused(cond(d, 3, None, 4, 256, 384, d, d, d, d, d, 10, 10, d, d, d, None), "t_numel")
    refused(cond(d, 1, None, 4, 256, 4224, d, d, d, d, d, 10, 10, d, d, d, None), "E 4224")      # beyond 4096
    refused(cond(d, 1, None, 4, 256, 200, d, d, d, d, d, 10, 10, d, d, d, None), "E 200")       # not a multiple of 128
    refused(cond(d, 1, None, 4, 192, 384, d, d, d, d, d, 10, 10, d, d, d, None), "feat 192")
    refused(cond(d, 1, None, 4, 8192, 1024, d, d, d, d, d, 10, 10, d, d, d, None), "feat 8192")
    refused(cond(d, 1, None, 4, 256, 384, d, d, d, d, d, -1, -1, d, d, d, None), "max_row must be >= 0 and null_row in [-1, max_row] (got -1, -1)")
    refused(cond(d, 1, None, 4, 256, 384, d, d, d, d, d, 10, 11, d, d, d, None), "(got 10, 11)")
    refused(cond(d, 1, None, 4, 256, 384, d, d, d, d, d, 10, -2, d, d, d, None), "(got 10, -2)")
    refused(cond(d, 4, None, 4, 256, 384, None, d, d, d, d, 10, 10, d, d, d, None), "NULL")
    refused(cond(d, 4, None, 4, 256, 384, d, d, d, d, d, 10, 10, d, None, d, None), "NULL")
    refused(cond(d, 4, None, 4, 256, 384, d, d, d, d, None, 10, 10, d, d, d, None), "NULL")   # the null row reads the table
    refused(cond(d, 4, d, 4, 256, 384, d, d, d, d, None, 10, -1, d, d, d, None), "NULL")      # so do labels


def test_attention_entry_refuses_bad_arguments(lib):
    """lfm_dbg_attention checks its arguments against the attention route table before it touches the device, and names the
    bad argument: shapes without a route, then bad layouts, head widths, counts and pointers."""
    from lfm_b200 import _lib

    def refused(rc, word):
        assert rc != 0
        assert word in _lib.last_error(), _lib.last_error()

    # lfm_dbg_attention(qkv, out, B, T, heads, ch, head_dim, layout, stream)
    att = lib.lfm_dbg_attention
    TIMM, HM = _lib.QKV_TIMM, _lib.QKV_HEAD_MAJOR
    refused(att(None, None, 1, 1024, 1, 128, 128, HM, None), "1024 tokens")
    refused(att(None, None, 1, 64, 1, 384, 384, HM, None), "384 channels")
    refused(att(None, None, 1, 64, 32, 12, 12, HM, None), "12 channels")
    refused(att(None, None, 1, 1024, 4, 64, 64, TIMM, None), "1024 tokens")   # the timm layout: 256 tokens with 64 channels only
    refused(att(None, None, 1, 256, 4, 80, 80, TIMM, None), "80 channels")
    refused(att(None, None, 1, 256, 2, 96, 72, HM, None), "head_dim")         # padded heads on the SIMT kernels
    refused(att(None, None, 1, 256, 4, 64, 32, TIMM, None), "head_dim")       # ... and on the wgmma kernel
    refused(att(None, None, 1, 64, 1, 64, 72, HM, None), "head_dim")
    refused(att(None, None, 1, 64, 1, 64, 0, HM, None), "head_dim")
    refused(att(None, None, 1, 64, 1, 64, 64, 2, None), "layout")
    refused(att(None, None, 0, 64, 1, 64, 64, HM, None), "B")
    refused(att(None, None, 1, 64, 0, 64, 64, HM, None), "heads")
    refused(att(None, None, 1, 64, 2, 64, 64, HM, None), "NULL")


def _unet_desc(cfg):
    from lfm_b200 import _lib
    ar, cm = cfg.attention_resolutions, cfg.channel_mult
    return _lib.UnetDesc(cfg.image_size, cfg.in_channels, cfg.model_channels, cfg.out_channels, cfg.num_res_blocks, len(ar),
                         (ctypes.c_int32 * 8)(*ar), len(cm), (ctypes.c_int32 * 8)(*cm), cfg.num_heads, cfg.num_head_channels,
                         cfg.num_classes or 0)


@pytest.mark.parametrize("kw,words", [
    # 32 x 32 = 1024 tokens with one 128-channel head (in the input, output and middle blocks)
    (dict(image_size=32, model_channels=128, channel_mult=(1, 2), attention_resolutions=(1,), num_heads=1), ("1024 tokens", "128")),
    # the middle block alone: 8 x 8 = 64 tokens with one 384-channel head
    (dict(image_size=8, model_channels=384, channel_mult=(1,), attention_resolutions=(), num_heads=1), ("64 tokens", "384")),
    # 12-channel heads (16-byte loads need multiples of 8)
    (dict(image_size=8, model_channels=384, channel_mult=(1,), attention_resolutions=(), num_heads=32), ("64 tokens", "12 channels")),
    # 128 channels do not split into 3 heads
    (dict(image_size=8, model_channels=128, channel_mult=(1,), attention_resolutions=(), num_heads=3), ("128 channels", "3 heads")),
    (dict(image_size=8, model_channels=128, channel_mult=(1,), attention_resolutions=(), num_heads=1, num_head_channels=0),
     ("num_head_channels",)),
])
def test_unet_attention_shapes_without_a_kernel_are_refused(lib, kw, words):
    """UNetModel shapes whose attention no kernel covers are refused by the constructor, before it looks for a device."""
    from lfm_b200 import _lib
    from oracle import unet as ounet
    ctx = ctypes.c_void_p()
    assert lib.lfm_create_unet(ctypes.byref(_unet_desc(ounet.UNetConfig(**kw))), 0, ctypes.byref(ctx)) != 0
    msg = _lib.last_error()
    assert "lfm_create_unet" in msg and "device" not in msg, msg
    for w in words:
        assert w in msg, msg


def test_fixture_unet_configurations_pass_the_attention_check(lib):
    """Every UNetModel configuration the tests and the benchmark build gets past the attention check: without a GPU the
    constructor then fails on the missing device; with one it succeeds."""
    from lfm_b200 import _lib
    from oracle import unet as ounet
    from tests._util import load_golden
    from tests.test_oracle_unet import unet_cfg_from_golden
    cfgs = [unet_cfg_from_golden(load_golden("unet_mini")), unet_cfg_from_golden(load_golden("unet_mini_cond")),
            ounet.UNetConfig(image_size=32, channel_mult=(1, 2, 2, 2)),   # celeb256
            ounet.UNetConfig()]                                           # celeb512 (BASELINE cfg4)
    for cfg in cfgs:
        ctx = ctypes.c_void_p()
        rc = lib.lfm_create_unet(ctypes.byref(_unet_desc(cfg)), 0, ctypes.byref(ctx))
        if rc == 0:
            lib.lfm_destroy(ctx)
        else:
            assert "device" in _lib.last_error(), (cfg, _lib.last_error())
