"""ctypes binding of the C-ABI (include/effort_b200.h).  Fails loudly when the CUDA extension is
missing: there is no CPU or PyTorch fallback for any operator in this package."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

_lib = None

vp, fp, u32p = C.c_void_p, C.c_void_p, C.c_void_p


class MulArgs(C.Structure):
    _fields_ = [("v_dev", C.c_void_p), ("w", C.c_void_p), ("exp_no_dev", C.c_void_p),
                ("out_dev", C.c_void_p), ("effort", C.c_double), ("v_cutoff_dev", C.c_void_p)]


class FusedArgs(C.Structure):
    """effort_fused_args_t"""
    _fields_ = [("v_dev", C.c_void_p), ("x3_dev", C.c_void_p), ("norm_w_dev", C.c_void_p), ("norm_eps", C.c_float),
                ("w", C.c_void_p), ("exp_no_dev", C.c_void_p), ("out_scale_dev", C.c_void_p), ("out_dev", C.c_void_p),
                ("effort", C.c_double), ("accumulate", C.c_int)]


# name -> (restype, argtypes); every symbol include/effort_b200.h declares
SIGNATURES = {
    "effort_version": (C.c_int, []),
    "effort_strerror": (C.c_char_p, [C.c_int]),
    "effort_last_cuda_error": (C.c_char_p, []),
    "effort_ctx_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "effort_ctx_destroy": (C.c_int, [C.c_void_p]),
    "effort_ctx_set_cutoff_mode": (C.c_int, [C.c_void_p, C.c_int]),
    "effort_ctx_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "effort_ctx_error_flag": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint), vp]),
    "effort_weights_create": (C.c_int, [vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_uint, vp, C.POINTER(C.c_void_p)]),
    "effort_weights_destroy": (C.c_int, [C.c_void_p]),
    "effort_weights_owned_bytes": (C.c_size_t, [C.c_void_p]),
    "effort_weights_hint": (C.c_void_p, [C.c_void_p]),
    "effort_pdl_enabled": (C.c_int, []),
    "effort_bucket_mul": (C.c_int, [vp, fp, vp, u32p, fp, C.c_double, vp]),
    "effort_bucket_mul_q4": (C.c_int, [vp, fp, vp, u32p, fp, C.c_double, vp]),
    "effort_expert_mul": (C.c_int, [vp, fp, vp, u32p, fp, C.c_double, vp]),
    "effort_basic_mul": (C.c_int, [vp, fp, vp, C.c_int, C.c_int, fp, vp]),
    "effort_expert_mul_batch": (C.c_int, [vp, C.POINTER(MulArgs), C.c_int, vp]),
    "effort_calc_dispatch": (C.c_int, [vp, fp, vp, u32p, C.c_double, vp]),
    "effort_mul": (C.c_int, [vp, vp, fp, vp]),
    "effort_find_cutoff": (C.c_int, [vp, fp, vp, u32p, C.c_double, vp]),
    "effort_read_dispatch": (C.c_int, [vp, vp, C.c_size_t, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                       C.POINTER(C.c_float), C.POINTER(C.c_int), vp]),
    "effort_bucketize": (C.c_int, [vp, C.c_int, C.c_int, vp, vp, vp, vp]),
    "effort_q4_bucketize": (C.c_int, [vp, C.c_int, C.c_int, vp, vp, vp, vp]),
    "effort_comm_unique_id": (C.c_int, [vp]),
    "effort_comm_init": (C.c_int, [vp, vp, C.c_int, C.c_int]),
    "effort_comm_destroy": (C.c_int, [vp]),
    "effort_comm_p2p_local_handle": (C.c_int, [vp, vp]),
    "effort_comm_p2p_disable": (C.c_int, [vp]),
    "effort_comm_p2p_connect": (C.c_int, [vp, vp, C.c_int, C.c_int]),
    "effort_comm_p2p_collective": (C.c_int, [vp, C.c_int, C.c_int, vp, vp, C.c_size_t, vp]),
    "effort_comm_all_reduce": (C.c_int, [vp, vp, C.c_size_t, vp]),
    "effort_comm_all_gather": (C.c_int, [vp, vp, vp, C.c_size_t, vp]),
    "effort_model_create": (C.c_int, [vp, vp, C.POINTER(C.c_void_p)]),
    "effort_model_destroy": (C.c_int, [vp]),
    "effort_model_set_layer": (C.c_int, [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "effort_model_set_moe": (C.c_int, [vp, C.c_int, vp, C.c_int]),
    "effort_model_set_head": (C.c_int, [vp, vp, vp, vp]),
    "effort_model_reset": (C.c_int, [vp, vp]),
    "effort_model_rewind": (C.c_int, [vp, C.c_int, vp]),
    "effort_model_step": (C.c_int, [vp, vp, C.c_double, vp]),
    "effort_model_prefill": (C.c_int, [vp, vp, C.c_int, C.c_double, vp]),
    "effort_bucket_mul_multi": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_double, vp, vp, vp]),
    "effort_batch_create": (C.c_int, [vp, C.c_int, C.POINTER(C.c_void_p)]),
    "effort_batch_destroy": (C.c_int, [vp]),
    "effort_batch_reset": (C.c_int, [vp, C.c_int, vp]),
    "effort_batch_fork": (C.c_int, [vp, C.c_int, vp]),
    "effort_batch_step": (C.c_int, [vp, vp, C.c_double, vp]),
    "effort_batch_set_sampler": (C.c_int, [vp, C.c_int, vp]),
    "effort_batch_set_scoring": (C.c_int, [vp, C.c_int]),
    "effort_batch_set_score_targets": (C.c_int, [vp, C.c_int, vp, C.c_int, vp]),
    "effort_batch_logits": (C.c_void_p, [vp]),
    "effort_batch_next_tokens": (C.c_void_p, [vp]),
    "effort_batch_scores": (C.c_void_p, [vp]),
    "effort_batch_buffer": (C.c_void_p, [vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "effort_model_step_host": (C.c_int, [vp, C.POINTER(C.c_int32), C.c_double, C.POINTER(C.c_int32), vp, vp]),
    "effort_model_logits": (C.c_void_p, [vp]),
    "effort_model_next_token": (C.c_void_p, [vp]),
    "effort_model_bucket_bytes": (C.c_size_t, [vp]),
    "effort_model_set_graphs": (C.c_int, [vp, C.c_int]),
    "effort_model_set_fused_glue": (C.c_int, [vp, C.c_int]),
    "effort_model_set_chain": (C.c_int, [vp, C.c_int]),
    "effort_model_set_sampler": (C.c_int, [vp, vp]),
    "effort_sample": (C.c_int, [vp, vp, C.c_int, vp, C.c_uint32, vp, vp]),
    "effort_score": (C.c_int, [vp, vp, C.c_int, vp, C.c_int, vp, vp]),
    "effort_model_set_scoring": (C.c_int, [vp, C.c_int]),
    "effort_model_set_score_targets": (C.c_int, [vp, vp, C.c_int, vp]),
    "effort_model_scores": (C.c_void_p, [vp]),
    "effort_model_buffer": (C.c_void_p, [vp, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "effort_fused_mul_batch": (C.c_int, [vp, C.POINTER(FusedArgs), C.c_int, vp]),
    "effort_last_problem": (C.c_int, [vp, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_uint32), vp]),
    "effort_launch_count": (C.c_uint64, []),
    "effort_last_selected": (C.c_int, [vp, C.POINTER(C.c_uint32), vp]),
    "effort_loader_open": (C.c_int, [C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "effort_loader_close": (None, [vp]),
    "effort_loader_count": (C.c_int, [vp]),
    "effort_loader_name": (C.c_char_p, [vp, C.c_int]),
    "effort_loader_has": (C.c_int, [vp, C.c_char_p]),
    "effort_loader_tensor": (C.c_int, [vp, C.c_char_p, vp]),
    "effort_bf16_to_f16": (C.c_int, [vp, vp, C.c_size_t]),
    "effort_saver_open": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "effort_saver_add": (C.c_int, [vp, C.c_int, C.c_char_p, C.c_int, C.c_int, C.POINTER(C.c_int64), vp, C.c_size_t]),
    "effort_saver_save": (C.c_int, [vp]),
    "effort_saver_close": (None, [vp]),
}


class TensorInfo(C.Structure):
    _fields_ = [("dtype", C.c_int), ("ndim", C.c_int), ("shape", C.c_int64 * 8), ("data", C.c_void_p),
                ("nbytes", C.c_size_t)]


class ModelConfig(C.Structure):
    _fields_ = [("dim", C.c_int), ("hidden_dim", C.c_int), ("n_layers", C.c_int), ("n_heads", C.c_int),
                ("n_kv_heads", C.c_int), ("head_dim", C.c_int), ("vocab", C.c_int), ("max_seq", C.c_int),
                ("rope_theta", C.c_float), ("norm_eps", C.c_float), ("tp_rank", C.c_int), ("tp_size", C.c_int)]


class Sampler(C.Structure):
    """effort_sampler_t"""
    _fields_ = [("temperature", C.c_float), ("top_k", C.c_int), ("top_p", C.c_float), ("seed", C.c_uint64)]


class EffortError(RuntimeError):
    pass


def lib_path() -> str:
    return _build.LIB


def load():
    """Load (building if stale and nvcc is present) the native library.  Raises if unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    alt = os.environ.get("EFFORT_LIB")  # A/B experiments against an older build of the library (tools only)
    if alt:
        L = C.CDLL(alt)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name, None)
            if fn is not None:
                fn.restype, fn.argtypes = res, args
        _lib = L
        return L
    if _build.needs_build():
        try:
            _build.build()
        except Exception as e:  # no nvcc on the GPU box is fine iff the prebuilt .so travelled
            if not os.path.exists(path):
                raise EffortError(f"libeffort_b200.so is missing and cannot be built: {e}") from e
    L = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def check(rc: int, what: str = ""):
    if rc != 0:
        L = load()
        msg = L.effort_strerror(rc).decode()
        cu = L.effort_last_cuda_error().decode()
        raise EffortError(f"{what}: {msg} (code {rc}){' [' + cu + ']' if cu and rc == -2 else ''}")
