"""ctypes loader for libsutro_b200.so (the C-ABI declared in include/sutro_b200.h).

The product path has no CPU fallback: if the shared library is missing or fails
to load, importing anything that needs it raises immediately.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SB200_LIB: load another build of the same library (e.g. one compiled with different flags)
LIB_PATH = os.environ.get("SB200_LIB") or os.path.join(_HERE, "libsutro_b200.so")

_lib = None

c_void_p, c_int, c_float, c_size_t = C.c_void_p, C.c_int, C.c_float, C.c_size_t

# name -> (restype, argtypes); mirrors include/sutro_b200.h one to one.
_SIGNATURES = {
    "sb200_last_error": (C.c_char_p, []),
    "sb200_abi_version": (c_int, []),
    "sb200_device_info": (c_int, [C.POINTER(c_int)] * 3 + [C.POINTER(c_size_t)]),
    "sb200_gemm_bf16_tn": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                   c_int, c_int, c_int, c_int, c_void_p]),
    "sb200_gemm_qkv_rope": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int] +
                            [c_void_p] * 7 + [c_int, c_void_p, c_int, c_int, c_float, c_void_p]),
    "sb200_rmsnorm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "sb200_embed_gather": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "sb200_l2_normalize_rows": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "sb200_rope_kv_write": (c_int, [c_void_p] * 8 + [c_int, c_void_p, c_int, c_int, c_int,
                                                     c_float, c_void_p]),
    "sb200_attn_decode": (c_int, [c_void_p] * 4 + [c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                                   c_float, c_void_p]),
    "sb200_attn_decode_force_variant": (None, [c_int]),
    "sb200_attn_prefill": (c_int, [c_void_p] * 4 + [c_int, c_void_p, c_int] + [c_void_p] * 4 +
                           [c_int, c_int, c_float, c_void_p]),
    "sb200_attn_prefill_q_tile": (c_int, [c_int, c_int]),
    "sb200_attn_prefill_dense": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                         c_int, c_float, c_void_p]),
    "sb200_attn_prefill_chunked": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int,
                                           c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                           c_int, c_int, c_float, c_void_p, c_void_p, c_int,
                                           c_void_p, c_void_p, c_void_p]),
    "sb200_attn_prefill_hist_align": (c_int, [c_int, c_int]),
    "sb200_fsm_build_mask": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int,
                                     c_void_p, c_int, c_void_p]),
}


class Sb200Error(RuntimeError):
    pass


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Sb200Error(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (there is no CPU fallback)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)  # AttributeError here == header/library mismatch
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def exported_symbols() -> list[str]:
    return sorted(_SIGNATURES)


def register(name: str, restype, argtypes) -> None:
    """Used by engine.py to add the engine-level entry points to the table."""
    _SIGNATURES[name] = (restype, argtypes)
    if _lib is not None:
        fn = getattr(_lib, name)
        fn.restype, fn.argtypes = restype, argtypes


def check(status: int) -> None:
    if status != 0:
        raise Sb200Error(lib().sb200_last_error().decode("utf-8", "replace"))


def ptr(t) -> int:
    """Device (or host) address of a torch tensor / None."""
    return 0 if t is None else t.data_ptr()


def current_stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
