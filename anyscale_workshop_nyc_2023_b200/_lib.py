"""ctypes binding of libb200t5.so (the C ABI declared in include/b200t5.h).

The library is built in-tree (``csrc/Makefile`` -> ``libb200t5.so`` next to this file) so it
travels with the repository snapshot. The same sources are compiled a second time into
``libb200t5_f16.so``: identical entry points, the fp16 numerics contract (torch_dtype=float16 with
transformers' fp32 `wo`) instead of the bf16 one - ``load("fp16")``. There is no fallback: if the shared object is missing or a
symbol cannot be resolved, importing callers get a loud ``RuntimeError``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libb200t5.so"
LIB_PATHS = {"bf16": LIB_PATH, "fp16": _HERE / "libb200t5_f16.so"}
CSRC = _HERE / "csrc"

OK, EINVAL, ENODEV, ECUDA, ESTATE, ENOMEM = 0, -1, -2, -3, -4, -5
DTYPE_BF16, DTYPE_F16, DTYPE_F32 = 0, 1, 2


class Config(C.Structure):
    _fields_ = [
        ("vocab_size", C.c_int32),
        ("d_model", C.c_int32),
        ("d_kv", C.c_int32),
        ("d_ff", C.c_int32),
        ("num_heads", C.c_int32),
        ("num_layers", C.c_int32),
        ("num_decoder_layers", C.c_int32),
        ("relative_attention_num_buckets", C.c_int32),
        ("relative_attention_max_distance", C.c_int32),
        ("layer_norm_epsilon", C.c_float),
        ("pad_token_id", C.c_int32),
        ("eos_token_id", C.c_int32),
        ("decoder_start_token_id", C.c_int32),
        ("is_gated_gelu", C.c_int32),
        ("scale_decoder_outputs", C.c_int32),
    ]


class GenParams(C.Structure):
    _fields_ = [
        ("max_new_tokens", C.c_int32),
        ("min_new_tokens", C.c_int32),
        ("eos_token_id", C.c_int32),
        ("pad_token_id", C.c_int32),
        ("decoder_start_token_id", C.c_int32),
        ("poll_interval", C.c_int32),
    ]


class LogitsParams(C.Structure):
    _fields_ = [
        ("repetition_penalty", C.c_double),
        ("encoder_repetition_penalty", C.c_double),
        ("no_repeat_ngram_size", C.c_int32),
        ("encoder_no_repeat_ngram_size", C.c_int32),
        ("suppress_tokens", C.c_void_p),
        ("n_suppress_tokens", C.c_int32),
        ("begin_suppress_tokens", C.c_void_p),
        ("n_begin_suppress_tokens", C.c_int32),
        ("eos_token_ids", C.c_void_p),
        ("n_eos_token_ids", C.c_int32),
        ("bad_words_ids", C.c_void_p),
        ("bad_words_offsets", C.c_void_p),
        ("n_bad_words", C.c_int32),
    ]


class ScoreIO(C.Structure):
    _fields_ = [
        ("token_logprobs", C.c_void_p),
        ("token_logits", C.c_void_p),
        ("forced_ids", C.c_void_p),
        ("forced_len", C.c_int32),
    ]


class BeamParams(C.Structure):
    _fields_ = [
        ("num_beams", C.c_int32),
        ("num_return_sequences", C.c_int32),
        ("length_penalty", C.c_double),
        ("early_stopping", C.c_int32),
    ]


class BeamIO(C.Structure):
    _fields_ = [
        ("sequences", C.c_void_p),
        ("lengths", C.c_void_p),
        ("sequences_scores", C.c_void_p),
        ("beam_indices", C.c_void_p),
        ("token_logprobs", C.c_void_p),
    ]


class ForwardIO(C.Structure):
    _fields_ = [
        ("logits", C.c_void_p),
        ("token_logprobs", C.c_void_p),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("encoder_ms", C.c_float),
        ("decode_ms", C.c_float),
        ("decode_steps", C.c_int32),
        ("kernel_launches", C.c_int64),
        ("decode_algo_bytes", C.c_double),
        ("encoder_flops", C.c_double),
        ("xattn_kernel", C.c_int32),
        ("row_chains", C.c_int32),
    ]


_vp, _i, _i64p, _i32p = C.c_void_p, C.c_int, C.c_void_p, C.c_void_p

# name -> (restype, argtypes); must list every symbol include/b200t5.h declares
SIGNATURES = {
    "b200t5_create": (_i, [C.POINTER(Config), _i, C.POINTER(_vp)]),
    "b200t5_set_weight": (_i, [_vp, C.c_char_p, _vp, _i, C.POINTER(C.c_int64), _i]),
    "b200t5_finalize": (_i, [_vp]),
    "b200t5_destroy": (_i, [_vp]),
    "b200t5_last_error": (C.c_char_p, [_vp]),
    "b200t5_last_global_error": (C.c_char_p, []),
    "b200t5_generate": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), _i64p, _i32p, _vp]),
    "b200t5_generate_host": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), _i64p, _i32p]),
    "b200t5_generate_stream": (_i, [_vp, _i64p, _i64p, C.c_int64, _i, C.POINTER(GenParams), _i, _i, _i64p, _i32p]),
    "b200t5_generate_ex": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), C.POINTER(LogitsParams), _i64p, _i32p, _vp]),
    "b200t5_generate_host_ex": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), C.POINTER(LogitsParams), _i64p, _i32p]),
    "b200t5_generate_stream_ex": (_i, [_vp, _i64p, _i64p, C.c_int64, _i, C.POINTER(GenParams), C.POINTER(LogitsParams), _i, _i,
                                       _i64p, _i32p]),
    "b200t5_generate_scored": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), C.POINTER(LogitsParams), _i64p, _i32p,
                                    C.POINTER(ScoreIO), _vp]),
    "b200t5_generate_host_scored": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), C.POINTER(LogitsParams), _i64p, _i32p,
                                         C.POINTER(ScoreIO)]),
    "b200t5_generate_stream_scored": (_i, [_vp, _i64p, _i64p, C.c_int64, _i, C.POINTER(GenParams), C.POINTER(LogitsParams), _i, _i,
                                           _i64p, _i32p, C.POINTER(ScoreIO)]),
    "b200t5_generate_prefixed": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), C.POINTER(LogitsParams), _i64p, _i32p,
                                      C.POINTER(ScoreIO), _i64p, _i, _vp]),
    "b200t5_generate_host_prefixed": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), C.POINTER(LogitsParams), _i64p,
                                           _i32p, C.POINTER(ScoreIO), _i64p, _i]),
    "b200t5_generate_beam": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), C.POINTER(BeamParams), C.POINTER(BeamIO), _vp]),
    "b200t5_generate_host_beam": (_i, [_vp, _i64p, _i64p, _i, _i, C.POINTER(GenParams), C.POINTER(BeamParams), C.POINTER(BeamIO)]),
    "b200t5_get_beam_stats": (_i, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_int32)]),
    "b200t5_test_beam_step": (_i, [_i, _vp, _i, _i, _i, _i, _i, _i, _i, C.c_double, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                   _vp]),
    "b200t5_test_beam_reorder": (_i, [_i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "b200t5_test_beam_replicate": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200t5_test_beam_search": (_i, [_i, _vp, _i, _i, _i, _i, _i, _i, C.c_double, _i, _i, C.c_int64, C.c_int64, C.POINTER(BeamIO),
                                     C.POINTER(C.c_int32), _vp, _vp, _vp]),
    "b200t5_get_stats": (_i, [_vp, C.POINTER(Stats)]),
    "b200t5_bench_cross_attn": (_i, [_vp, _i, _i, C.POINTER(C.c_float), C.POINTER(C.c_double), _vp]),
    "b200t5_set_option": (_i, [_vp, C.c_char_p, _i]),
    "b200t5_get_xattn_profile": (_i, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "b200t5_test_lm_argmax": (_i, [_i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "b200t5_test_lm_process": (_i, [_i, _vp, _vp, _i, _i, _i, _i, _i, _i, C.POINTER(LogitsParams), _i64p, _i64p, _i, _i64p,
                                    _vp, _vp]),
    "b200t5_test_lm_score": (_i, [_i, _vp, _vp, _i, _i, _i, _i, _i, _i, C.POINTER(LogitsParams), _i64p, _i64p, _i, _i64p, _i64p,
                                  _vp, _vp, _vp, _vp]),
    "b200t5_encode": (_i, [_vp, _i64p, _i64p, _i, _i, _vp, _vp]),
    "b200t5_decode_logits": (_i, [_vp, _i64p, _i64p, _i, _i, _i64p, _i, _vp, _vp]),
    "b200t5_test_prefill_cache": (_i, [_vp, _i, _vp, _vp]),
    "b200t5_forward": (_i, [_vp, _i64p, _i64p, _i, _i, _i64p, _i64p, _i, C.POINTER(ForwardIO), _vp]),
    "b200t5_forward_choices": (_i, [_vp, _i64p, _i64p, _i, _i, _vp, _i64p, _i, C.POINTER(ForwardIO), _vp]),
    "b200t5_relative_bucket": (_i, [_i, _i, _i, _i]),
    "b200t5_test_gemm": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200t5_test_enc_gemm": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _i, _vp]),
    "b200t5_test_gemm_splitk": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i, _i, _vp]),
    "b200t5_test_ffo": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200t5_test_rmsnorm": (_i, [_i, _vp, _vp, _vp, _i, _i, C.c_float, _vp]),
    "b200t5_test_rmsnorm_scaled": (_i, [_i, _vp, _vp, _vp, _i, _i, C.c_float, C.c_float, _vp]),
    "b200t5_test_attn_decode": (_i, [_i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "b200t5_test_encoder_attn": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "b200t5_test_decoder_self_attn": (_i, [_i, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "b200t5_test_decoder_cross_attn": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "b200t5_test_decoder_cross_attn_packed": (_i, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "b200t5_test_geglu": (_i, [_i, _vp, _vp, _vp, C.c_int64, _i, _vp]),
    "b200t5_version": (C.c_char_p, []),
}

_libs = {}


def build(force: bool = False) -> Path:
    """Compile libb200t5.so and libb200t5_f16.so for sm_90a with nvcc (cross-compiles without a GPU)."""
    for path in LIB_PATHS.values():
        if force and path.exists():
            path.unlink()
    proc = subprocess.run(["make", "-j2", "-C", str(CSRC)], capture_output=True, text=True)
    if proc.returncode != 0 or not all(path.exists() for path in LIB_PATHS.values()):
        raise RuntimeError(f"building libb200t5.so / libb200t5_f16.so failed:\n{proc.stdout}\n{proc.stderr}")
    return LIB_PATH


def load(flavour: str = "bf16") -> C.CDLL:
    """Load the shared library of one numerics contract ("bf16" | "fp16") and bind every declared entry point
    (raises if anything is missing)."""
    if flavour in _libs:
        return _libs[flavour]
    path = LIB_PATHS[flavour]
    if not path.exists():
        raise RuntimeError(
            f"{path} is missing: run `make -C {CSRC}` (or __graft_entry__.build()). "
            "There is no CPU or PyTorch fallback for the CUDA path."
        )
    # RTLD_LOCAL (the ctypes default): both flavours export the same names and must not see each other
    lib = C.CDLL(str(path), mode=getattr(os, "RTLD_NOW", 2))
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:  # pragma: no cover
            raise RuntimeError(f"{path.name} does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    _libs[flavour] = lib
    return lib


def last_error(handle=None, lib=None) -> str:
    lib = lib or load()
    msg = lib.b200t5_last_error(handle) if handle else lib.b200t5_last_global_error()
    return (msg or b"").decode("utf-8", "replace")


class B200T5Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libb200t5 error {code}: {msg}")
        self.code = code


def check(rc: int, handle=None, lib=None) -> None:
    if rc != OK:
        raise B200T5Error(rc, last_error(handle, lib))
