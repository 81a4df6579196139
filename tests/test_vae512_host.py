"""CPU-side checks of the 512 x 512 VAE decode (64 x 64 latents): lfm_create_vae's size rule, the argument checks of
lfm_dbg_conv_wide (made before the device is touched), and AutoencoderKL's decode chunk.  No compute calls."""
import ctypes

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from lfm_b200 import _lib, build
    build.build()
    return _lib.load()


def vae_desc(latent_size, boc=(128, 256, 512, 512)):
    from lfm_b200 import _lib
    return _lib.VaeDesc(latent_size, 4, 3, len(boc), (ctypes.c_int32 * 8)(*boc), 2, 32)


def test_create_vae_accepts_the_512_decode(lib):
    """Latent 64 with the SD decoder's four blocks (output side 512) passes every size check: without a GPU the refusal is the
    missing device, not the size; with one, a context is created."""
    from lfm_b200 import _lib
    ctx = ctypes.c_void_p()
    rc = lib.lfm_create_vae(ctypes.byref(vae_desc(64)), 0, ctypes.byref(ctx))
    if torch.cuda.is_available():
        assert rc == 0, _lib.last_error()
        lib.lfm_destroy(ctx)
    else:
        assert rc != 0
        assert "no CUDA device" in _lib.last_error(), _lib.last_error()


@pytest.mark.parametrize("latent,boc,side", [(128, (128, 256, 512, 512), 1024), (64, (128, 128, 256, 512, 512), 1024),
                                             (32, (128, 128, 128, 256, 512, 512), 1024)])
def test_create_vae_refuses_sides_above_512(lib, latent, boc, side):
    from lfm_b200 import _lib
    ctx = ctypes.c_void_p()
    assert lib.lfm_create_vae(ctypes.byref(vae_desc(latent, boc)), 0, ctypes.byref(ctx)) != 0
    assert f"output side {side}" in _lib.last_error(), _lib.last_error()


def test_dbg_conv_wide_refuses_bad_arguments(lib):
    """lfm_dbg_conv_wide(x, w, bias, out, gn_bins, B, side, Cin, Cout, stride, block_n, epi, ksplit, stream): each bad argument is
    refused by name before the device is touched."""
    from lfm_b200 import _lib

    def refused(rc, word):
        assert rc != 0
        assert word in _lib.last_error(), _lib.last_error()

    conv = lib.lfm_dbg_conv_wide
    dummy = ctypes.c_void_p(64)   # never dereferenced: each call below is refused on its arguments
    refused(conv(None, None, None, None, None, 1, 384, 128, 128, 1, 0, 3, 1, None), "side")   # three segments: not a decoder size
    refused(conv(None, None, None, None, None, 1, 64, 128, 128, 1, 0, 3, 1, None), "side")    # whole rows: lfm_dbg_conv's ground
    refused(conv(None, None, None, None, None, 1, 1024, 128, 128, 1, 0, 3, 1, None), "side")
    refused(conv(None, None, None, None, None, 1, 512, 128, 128, 2, 0, 3, 1, None), "stride")
    refused(conv(None, None, None, None, None, 1, 512, 128, 128, 1, 0, 3, -1, None), "ksplit")
    refused(conv(None, None, None, None, None, 1, 512, 128, 128, 1, 0, 3, 2, None), "ksplit")
    refused(conv(None, None, None, None, None, 0, 512, 128, 128, 1, 0, 3, 1, None), "B")
    refused(conv(None, None, None, None, None, 8192, 512, 128, 128, 1, 0, 3, 1, None), "B")   # 2^31 output pixels
    refused(conv(None, None, None, None, None, 1, 512, 96, 128, 1, 0, 3, 1, None), "Cin")
    refused(conv(None, None, None, None, None, 1, 512, 128, 12, 1, 0, 3, 1, None), "Cout")
    refused(conv(None, None, None, None, None, 1, 512, 128, 128, 1, 64, 3, 1, None), "block_n")
    refused(conv(None, None, None, None, None, 1, 512, 128, 128, 1, 0, 1, 1, None), "epi")
    refused(conv(None, None, None, None, dummy, 1, 512, 128, 128, 1, 0, 2, 1, None), "gn_bins")    # residual epilogue
    refused(conv(None, None, None, None, dummy, 1, 512, 128, 96, 1, 0, 3, 1, None), "gn_bins")     # 3 channels per group
    refused(conv(None, None, None, None, None, 1, 512, 128, 128, 1, 0, 3, 1, None), "NULL")
    refused(conv(dummy, dummy, None, dummy, None, 1, 256, 128, 128, 1, 0, 3, 1, None), "NULL")


def test_decode_chunk_rule():
    """A 512 x 512 image needs four times the workspace of a 256 x 256 one: at latent 64 the decode chunk (and the batch the native
    workspace is sized for) is max_batch // 4, at least 1; latents up to 32 keep max_batch."""
    import lfm_b200
    vae = lfm_b200.AutoencoderKL(max_batch=16)
    assert [vae.decode_chunk(s) for s in (16, 32, 64)] == [16, 16, 4]
    assert lfm_b200.AutoencoderKL(max_batch=2).decode_chunk(64) == 1
    assert lfm_b200.AutoencoderKL(max_batch=2).decode_chunk(32) == 2
    assert lfm_b200.AutoencoderKL(max_batch=8).decode_chunk(64) == 2
    vae._latent_size = 64
    assert vae._finalize_rows(1) == 4 and vae._finalize_rows(6) == 6
    vae._latent_size = 32
    assert vae._finalize_rows(1) == 16
