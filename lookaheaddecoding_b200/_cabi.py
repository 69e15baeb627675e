"""ctypes binding of include/lade_sm100.h (the only way the product path reaches CUDA).

Fails loudly when the library is missing or cannot be loaded: there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

c_i32 = C.c_int32
c_p = C.c_void_p

# indices mirrored from the header (LADE_M_*, LADE_R_*)
M_Q_LEN, M_KV_LEN, M_N_INPUT, M_LEVEL_OFFSET, M_ALL_OFFSET, M_TINY, M_N_LEVELS, M_N_GUESS_TOK, \
    M_IS_PREFILL, M_PHASE, M_Q_PAD, M_DONE, M_STEP = range(13)
META_INTS = 16
R_N_EMIT, R_MAX_HIT, R_MAX_HIT_IDX, R_KV_SRC, R_KV_DST, R_KV_LEN, R_DONE, R_N_OUT, R_STEPS, R_N_GUESS = range(10)
R_HITS = 16
RES_INTS = 48
LADE_OK, LADE_EINVAL, LADE_ECUDA, LADE_ENOMEM, LADE_EUNSUPPORTED, LADE_ESTATE = 0, -1, -2, -3, -4, -5
ROW_PREFIX, ROW_WINDOW, ROW_GUESS, ROW_PAD = 0, 1, 2, 3


class LadeConfig(C.Structure):
    _fields_ = [
        ("window_size", c_i32), ("level", c_i32), ("guess_set_size", c_i32), ("pool_from_prompt", c_i32),
        ("vocab_size", c_i32), ("max_total_len", c_i32), ("n_eos", c_i32), ("eos_token_id", c_i32 * 4),
        ("dist_workers", c_i32), ("rank", c_i32),
    ]


PROC_REPETITION_PENALTY, PROC_NO_REPEAT_NGRAM, PROC_MIN_LENGTH = 1, 2, 4
PROC_MAX_NGRAM, PROC_MAX_EOS = 64, 8


class LadeProcessors(C.Structure):
    _fields_ = [
        ("flags", c_i32), ("penalty_bits", C.c_uint32), ("prompt_ignore_length", c_i32), ("ngram_size", c_i32),
        ("eos_bound", c_i32), ("n_eos", c_i32), ("eos_token_id", c_i32 * PROC_MAX_EOS),
    ]


class LadeWarpers(C.Structure):
    _fields_ = [("temperature", C.c_float), ("top_k", c_i32), ("top_p", C.c_float), ("min_p", C.c_float),
                ("epsilon", C.c_float), ("eta", C.c_float)]


class LadeError(RuntimeError):
    pass


_SIGNATURES = {
    "lade_ctx_create": (C.c_int, [C.POINTER(LadeConfig), C.POINTER(c_p)]),
    "lade_ctx_destroy": (C.c_int, [c_p]),
    "lade_ctx_reset": (C.c_int, [c_p, c_p, c_p, c_i32, c_p, c_i32, c_i32]),
    "lade_step_layout": (C.c_int, [c_p, c_p, c_i32, c_p, c_p, c_p, c_p, c_p, c_p, c_i32]),
    "lade_step_rows_bound": (C.c_int, [C.POINTER(LadeConfig), c_i32, c_i32]),
    "lade_rmsnorm": (C.c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_i32, c_i32, C.c_float]),
    "lade_rmsnorm_gather": (C.c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_i32, c_i32, C.c_float]),
    "lade_rope_append": (C.c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p] + [c_i32] * 7),
    "lade_rope_append_qknorm": (C.c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p] + [c_i32] * 7 + [c_p, c_p, C.c_float]),
    "lade_rope_append_bias": (C.c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p] + [c_i32] * 7 + [c_p]),
    "lade_attn_fwd": (C.c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_i32, c_p, c_p] + [c_i32] * 8),
    "lade_attn_scratch_bytes": (C.c_int64, [c_i32, c_i32, c_i32, c_i32]),
    "lade_debug_attn_timing": (C.c_int, [c_p]),
    "lade_debug_attn_pdl": (C.c_int, [c_i32]),
    "lade_gemm_bf16": (C.c_int, [c_p, c_p, c_p, c_p, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "lade_gemm_fp8": (C.c_int, [c_p, c_p, c_p, c_p, c_p, c_p] + [c_i32] * 7),
    "lade_rmsnorm_quant_fp8": (C.c_int, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_i32, c_i32, C.c_float]),
    "lade_swiglu_quant_fp8": (C.c_int, [c_p, c_p, c_p, c_p, c_i32, c_i32]),
    "lade_quant_rows_fp8": (C.c_int, [c_p, c_p, c_p, c_p, c_i32, c_i32]),
    "lade_debug_gemm_timing": (C.c_int, [c_p]),
    "lade_swiglu": (C.c_int, [c_p, c_p, c_p, c_i32, c_i32]),
    "lade_argmax_rows": (C.c_int, [c_p, c_p, c_i32, c_i32, c_i32, c_p]),
    "lade_argmax_processed": (C.c_int, [c_p, c_p, c_p, c_i32, c_i32, c_i32, c_p, c_p]),
    "lade_processors_upload": (C.c_int, [c_p, C.POINTER(LadeProcessors), c_p]),
    "lade_accept_update": (C.c_int, [c_p, c_p, c_p, c_p, c_p]),
    "lade_commit_decision": (C.c_int, [c_p, c_p, c_p, c_p, c_p]),
    "lade_sample_verify": (C.c_int, [c_p, c_p, c_p, c_i32, c_i32, c_p, c_p, C.c_float, c_i32, C.c_float, c_p, c_p, c_p]),
    "lade_sample_verify_warped": (C.c_int, [c_p, c_p, c_p, c_i32, c_i32, c_p, c_p, C.POINTER(LadeWarpers), c_p, c_p, c_p,
                                            c_p]),
    "lade_capture_rows": (C.c_int, [c_p, c_p, c_p, c_i32, c_i32, c_p, c_p, c_p, c_p, c_i32, c_p, c_i32, c_i32]),
    "lade_kv_compact": (C.c_int, [c_p, c_p, c_p, c_p, C.c_int64, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "lade_ctx_output_ids": (C.c_int, [c_p, c_p, c_p, c_i32]),
    "lade_ctx_pool_snapshot": (C.c_int, [c_p, c_p, c_p, c_p]),
    "lade_ctx_window_snapshot": (C.c_int, [c_p, c_p, c_p, c_p]),
    "lade_lp_record_ints": (C.c_int, [C.POINTER(LadeConfig)]),
    "lade_lp_verify": (C.c_int, [c_p, c_p, c_p, c_p, c_p]),
    "lade_lp_commit": (C.c_int, [c_p, c_p, c_p, c_p, c_p]),
    "lade_nccl_available": (C.c_int, []),
    "lade_nccl_unique_id": (C.c_int, [c_p]),
    "lade_nccl_comm_create": (C.c_int, [c_p, c_i32, c_i32, C.POINTER(c_p)]),
    "lade_nccl_comm_destroy": (C.c_int, [c_p]),
    "lade_lp_exchange": (C.c_int, [c_p, c_p, c_p, c_p, c_p]),
    "lade_strerror": (C.c_char_p, [C.c_int]),
    "lade_last_cuda_error": (C.c_char_p, []),
    "lade_version": (C.c_int, []),
}

# fp16 twins: same signatures as the bf16 entry points
for _name in ("lade_rmsnorm", "lade_rmsnorm_gather", "lade_rope_append", "lade_rope_append_qknorm",
              "lade_rope_append_bias", "lade_swiglu",
              "lade_argmax_rows", "lade_attn_fwd", "lade_sample_verify", "lade_argmax_processed", "lade_sample_verify_warped",
              "lade_gemm_fp8", "lade_rmsnorm_quant_fp8", "lade_swiglu_quant_fp8", "lade_quant_rows_fp8",
              "lade_capture_rows"):
    _SIGNATURES[_name + "_f16"] = _SIGNATURES[_name]

EXPORTED_SYMBOLS = tuple(_SIGNATURES)
_lib = None


def lib_path() -> str:
    return _build.LIB_PATH


def load(build_if_missing: bool = True):
    """Load liblade_sm100.so (building it in-tree first when the sources are newer)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    if build_if_missing and not _build.is_fresh():
        try:
            _build.build()
        except Exception as e:  # no nvcc on the box: use the shipped .so if there is one
            if not os.path.isfile(path):
                raise LadeError(f"liblade_sm100.so is missing and could not be built: {e}") from e
    if not os.path.isfile(path):
        raise LadeError(f"{path} not found: run `python -m lookaheaddecoding_b200.build` (no CPU fallback)")
    lib = C.CDLL(path)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError == missing export: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        lib = load()
        msg = lib.lade_strerror(rc).decode()
        cuda = lib.lade_last_cuda_error().decode()
        raise LadeError(f"{what or 'lade call'} failed: {msg} (rc={rc})" + (f" [{cuda}]" if cuda and rc == -2 else ""))
