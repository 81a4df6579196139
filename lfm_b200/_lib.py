"""ctypes binding of liblfm_b200.so (include/lfm_b200.h).  Fails loudly: there is no CPU or eager fallback."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblfm_b200.so")


class ModelDesc(C.Structure):
    _fields_ = [("arch", C.c_int32), ("img_resolution", C.c_int32), ("patch_size", C.c_int32),
                ("in_channels", C.c_int32), ("hidden_size", C.c_int32), ("depth", C.c_int32),
                ("num_heads", C.c_int32), ("mlp_hidden", C.c_int32), ("table_rows", C.c_int32)]


class UnetDesc(C.Structure):
    _fields_ = [("image_size", C.c_int32), ("in_channels", C.c_int32), ("model_channels", C.c_int32),
                ("out_channels", C.c_int32), ("num_res_blocks", C.c_int32), ("n_attn_res", C.c_int32),
                ("attention_resolutions", C.c_int32 * 8), ("n_mult", C.c_int32), ("channel_mult", C.c_int32 * 8),
                ("num_heads", C.c_int32), ("num_head_channels", C.c_int32), ("num_classes", C.c_int32)]


class EdmDesc(C.Structure):
    _fields_ = [("img_resolution", C.c_int32), ("in_channels", C.c_int32), ("out_channels", C.c_int32),
                ("label_dim", C.c_int32), ("model_channels", C.c_int32), ("n_mult", C.c_int32),
                ("channel_mult", C.c_int32 * 8), ("num_blocks", C.c_int32), ("n_attn_res", C.c_int32),
                ("attn_resolutions", C.c_int32 * 8)]


class VaeDesc(C.Structure):
    _fields_ = [("latent_size", C.c_int32), ("latent_channels", C.c_int32), ("out_channels", C.c_int32),
                ("n_blocks", C.c_int32), ("block_out_channels", C.c_int32 * 8), ("layers_per_block", C.c_int32),
                ("norm_num_groups", C.c_int32)]


class OdeStats(C.Structure):
    _fields_ = [("nfe", C.c_int64), ("accepted", C.c_int64), ("rejected", C.c_int64)]


# every symbol include/lfm_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "lfm_create": (C.c_int, [C.POINTER(ModelDesc), C.c_int, C.POINTER(_P)]),
    "lfm_create_unet": (C.c_int, [C.POINTER(UnetDesc), C.c_int, C.POINTER(_P)]),
    "lfm_create_edm": (C.c_int, [C.POINTER(EdmDesc), C.c_int, C.POINTER(_P)]),
    "lfm_create_vae": (C.c_int, [C.POINTER(VaeDesc), C.c_int, C.POINTER(_P)]),
    "lfm_decode": (C.c_int, [_P, _P, C.c_int, _P, _P, _P]),
    "lfm_set_param": (C.c_int, [_P, C.c_char_p, _P, C.c_int, C.POINTER(C.c_int64), C.c_int]),
    "lfm_finalize": (C.c_int, [_P, C.c_int]),
    "lfm_forward": (C.c_int, [_P, _P, C.c_int, _P, _P, C.c_int, C.c_float, _P, _P]),
    "lfm_sample_fixed": (C.c_int, [_P, C.c_int, _P, _P, C.c_int, C.c_int, C.c_int, _P, C.c_int, C.c_float,
                                   C.POINTER(OdeStats), _P]),
    "lfm_sample_dopri5": (C.c_int, [_P, _P, C.c_double, C.c_double, C.c_double, C.c_double, _P, C.c_int, C.c_float,
                                    C.POINTER(OdeStats), _P]),
    "lfm_sample_adaptive": (C.c_int, [_P, C.c_int, _P, C.c_double, C.c_double, C.c_double, C.c_double, _P, C.c_int, C.c_float,
                                      C.POINTER(OdeStats), _P]),
    "lfm_last_error": (C.c_char_p, [_P]),
    "lfm_destroy": (None, [_P]),
    "lfm_launch_count": (C.c_int64, [_P]),
    "lfm_dbg_gemm": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "lfm_dbg_attention": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "lfm_dbg_attention_mma": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "lfm_dbg_tokens": (C.c_int, [_P, _P, C.c_int]),
}

_lib = None


def load():
    """Load the shared library (once).  Raises if it has not been built - never falls back."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m lfm_b200.build` (nvcc, sm_90a). "
            "lfm_b200 has no CPU / eager fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error(ctx=None) -> str:
    msg = load().lfm_last_error(ctx)
    return msg.decode() if msg else ""


def check(rc: int, ctx=None):
    if rc != 0:
        raise RuntimeError("liblfm_b200: " + last_error(ctx))
