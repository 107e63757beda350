"""ctypes binding of libvlo_b200.so (the C ABI declared in include/vlo_b200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails the
caller gets an exception.  Nothing in the product path ever imports `oracle/`.
"""
from __future__ import annotations

import ctypes as C
import os
import pathlib
import threading

PKG = pathlib.Path(__file__).resolve().parent
LIB_PATH = pathlib.Path(os.environ.get("VLO_LIB") or PKG / "libvlo_b200.so")   # VLO_LIB: A/B a second build


class VloError(RuntimeError):
    pass


class VloConfig(C.Structure):
    _fields_ = [
        ("hidden_size", C.c_int32), ("num_layers", C.c_int32), ("num_heads", C.c_int32),
        ("num_kv_heads", C.c_int32), ("head_dim", C.c_int32), ("intermediate_size", C.c_int32),
        ("vocab_size", C.c_int32), ("rms_norm_eps", C.c_float),
        ("vit_hidden", C.c_int32), ("vit_layers", C.c_int32), ("vit_heads", C.c_int32),
        ("vit_mlp", C.c_int32), ("image_size", C.c_int32), ("patch_size", C.c_int32),
        ("vit_ln_eps", C.c_float),
        ("frame_token_cls", C.c_int32), ("pool_h", C.c_int32), ("pool_w", C.c_int32),
        ("max_streams", C.c_int32), ("max_kv_tokens", C.c_int32), ("max_step_tokens", C.c_int32),
        ("max_vit_batch", C.c_int32),
    ]


class VloDecision(C.Structure):
    _fields_ = [
        ("argmax_id", C.c_int32), ("argmax_excl_id", C.c_int32), ("p_interval", C.c_float),
        ("max_logit", C.c_float), ("top2_margin", C.c_float), ("lse", C.c_float),
        ("argmax_prob_id", C.c_int32), ("reserved1", C.c_int32),
    ]


class VloSampleRow(C.Structure):
    _fields_ = [
        ("seed", C.c_uint64), ("position", C.c_int32), ("temperature", C.c_float), ("top_k", C.c_int32),
        ("top_p", C.c_float), ("repetition_penalty", C.c_float), ("penalty_offset", C.c_int32),
        ("penalty_count", C.c_int32), ("reserved", C.c_int32),
    ]


_P = C.c_void_p
_I = C.c_int
_LL = C.c_longlong

# name -> (restype, argtypes); mirrors include/vlo_b200.h one to one.
SIGNATURES = {
    "vlo_last_error": (C.c_char_p, []),
    "vlo_launch_count": (_LL, []),
    "vlo_device_supported": (_I, [_I]),
    "vlo_profile_enable": (_I, [_I]),
    "vlo_profile_read": (_I, [C.POINTER(C.c_double), C.POINTER(_LL), C.POINTER(C.c_double), _I]),
    "vlo_engine_create": (_I, [C.POINTER(VloConfig), _I, C.POINTER(_P)]),
    "vlo_engine_create_pooled": (_I, [C.POINTER(VloConfig), C.c_int64, _I, C.POINTER(_P)]),
    "vlo_kv_pool_info": (_I, [_P, C.POINTER(_I), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "vlo_engine_destroy": (_I, [_P]),
    "vlo_load_tensor": (_I, [_P, C.c_char_p, _P, C.c_int64]),
    "vlo_finalize_weights": (_I, [_P]),
    "vlo_engine_device_bytes": (C.c_int64, [_P]),
    "vlo_stream_open": (_I, [_P, C.POINTER(_I)]),
    "vlo_stream_reset": (_I, [_P, _I]),
    "vlo_stream_close": (_I, [_P, _I]),
    "vlo_kv_len": (_I, [_P, _I, C.POINTER(_I)]),
    "vlo_kv_truncate": (_I, [_P, _I, _I]),
    "vlo_kv_copy_prefix": (_I, [_P, _I, _I, _I, _P]),
    "vlo_kv_evict": (_I, [_P, _I, _I, _I, C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "vlo_kv_compact": (_I, [_P, _I, _I, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_float), _P]),
    "vlo_kv_fill_synthetic": (_I, [_P, _I, _I, C.c_uint64, _P]),
    "vlo_kv_read": (_I, [_P, _I, _I, _I, _P, _P]),
    "vlo_kv_write": (_I, [_P, _I, _I, _I, _P, _I, _P]),
    "vlo_kv_image_bytes": (C.c_int64, [_P, _I]),
    "vlo_kv_swap_out": (_I, [_P, _I, _P, C.c_int64, _P]),
    "vlo_kv_swap_in": (_I, [_P, _I, _P, _I, _P]),
    "vlo_vit_encode": (_I, [_P, _P, _I, _P, _P, _P]),
    "vlo_connector": (_I, [_P, _P, _I, _P, _P]),
    "vlo_embed_tokens": (_I, [_P, _P, _I, _P, _P]),
    "vlo_step": (_I, [_P, _I, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _P, _P, _P, _I, _P]),
    "vlo_step_ids": (_I, [_P, _I, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _P, _P, _P, _P, _I, _P]),
    "vlo_step_segments": (_I, [_P, _I, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), _P, _P, _P, _P,
                               _I, _P]),
    "vlo_sample": (_I, [_P, _P, _I, C.POINTER(VloSampleRow), _P, _I, _P, _P]),
    "vlo_last_step_logits": (_I, [_P, _P, _P]),
    "vlo_last_step_hidden": (_I, [_P, _P, _P]),
    "vlo_bench_attn": (_I, [_P, _I, C.POINTER(C.c_int32), _I, _I, _I, C.POINTER(C.c_double), _P]),
    "vlo_bench_gemm": (_I, [_P, _I, _I, C.POINTER(C.c_double), C.POINTER(_I), _P]),
    "vlo_op_gemm": (_I, [_I, _I, _P, _I, _P, _I, _I, _P, _I, _P, _P, _I, _I, _P]),
    "vlo_op_gemm_ws": (_I, [_I, _I, _P, _I, _P, _I, _I, _P, _I, _LL, _P, _I, _I, _I, C.POINTER(_I), _P]),
    "vlo_op_gemm_ws_f8": (_I, [_P, _P, _I, _P, _I, _I, _P, _LL, _I, C.POINTER(_I), _P]),
    "vlo_op_gemm_vit": (_I, [_P, _I, _P, _I, _I, _P, _I, _P, _I, _I, _P]),
    "vlo_op_attn_ws_bytes": (C.c_int64, [_I, _I, _I, _I]),
    "vlo_op_attn_kvappend": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _LL, _P]),
    "vlo_op_attn_kvappend_paged": (_I, [_P, _P, _P, _P, _I, _P, _P, _I, _I, _I, _I, _I, _P]),
    "vlo_op_attn_kvappend_segments": (_I, [_P, _P, _P, _P, _I, _P, _I, C.POINTER(C.c_int32), _I, _I, _I, _I, _P]),
    "vlo_op_attn_plan_counts": (_I, [_I, C.POINTER(C.c_int32), _I, _I, _I, _I, C.POINTER(C.c_int32)]),
    "vlo_op_vit_attn": (_I, [_P, _P, _I, _I, _I, _P]),
    "vlo_op_probe_attn": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "vlo_op_resid_rmsnorm": (_I, [_P, _I, _I, _P, _P, _P, _P, _P, _I, _I, C.c_float, _P]),
    "vlo_op_qkv_rope_append": (_I, [_P, _I, _I, _P, _P, _I, C.POINTER(C.c_int32), C.POINTER(C.c_int64), _I, _P, _P, _P,
                                    _I, _I, _I, _P]),
    "vlo_op_gemm_swiglu": (_I, [_P, _I, _P, _I, _I, _P, _P, C.c_int64, _P, _I, _P]),
    "vlo_op_gemm_swiglu_f8": (_I, [_P, _P, _I, _P, _I, _I, _P, _P, C.c_int64, _P, _I, _P]),
    "vlo_op_decision": (_I, [_P, _I, _I, _I, _P, _P]),
    "vlo_op_sample": (_I, [_P, _I, _I, C.POINTER(VloSampleRow), _P, _I, _P, _P, _P]),
    "vlo_op_attn_bench": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _LL, _I, _LL, _I, _I, C.POINTER(C.c_double), _P]),
}

_lock = threading.Lock()
_lib = None


def load() -> C.CDLL:
    """Load the shared library (once) and type its entry points.  Raises if it is missing."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not LIB_PATH.exists():
            raise VloError(
                f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback for the hot path)")
        lib = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the header and the library diverge
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().vlo_last_error()
        raise VloError(f"{what or 'libvlo_b200'} failed ({rc}): {msg.decode() if msg else '?'}")
