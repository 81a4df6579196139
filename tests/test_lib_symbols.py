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
