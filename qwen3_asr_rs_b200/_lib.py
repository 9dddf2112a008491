"""ctypes binding of libasr_b200.so (include/asr_b200.h).  There is NO fallback: if the
CUDA library is missing or a call fails, an exception is raised."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libasr_b200.so")

# every symbol include/asr_b200.h declares (checked by tests/test_abi.py)
SYMBOLS = [
    "asrb_init", "asrb_ctx_free", "asrb_last_error", "asrb_version", "asrb_dims_default",
    "asrb_model_load", "asrb_model_create", "asrb_model_set_tensor", "asrb_model_finalize",
    "asrb_model_dims", "asrb_model_free", "asrb_session_create", "asrb_session_free",
    "asrb_transcribe_ids", "asrb_mel", "asrb_mel_read", "asrb_encode", "asrb_encode_read",
    "asrb_prefill", "asrb_decode_step", "asrb_generate", "asrb_last_timings", "asrb_session_set_option",
    "asrb_debug_mega_timeline", "asrb_session_stats", "asrb_session_device_ids", "asrb_model_lossy_tensors", "asrb_ingest_pcm", "asrb_ingested_read", "asrb_transcribe_ingested",
    "asrb_last_logprobs", "asrb_last_top_logprobs", "asrb_last_nbest", "asrb_last_beam_stats",
    "asrb_session_create_ex", "asrb_session_set_context", "asrb_last_prefill_stats",
    "asrb_ingest_long", "asrb_long_read", "asrb_segment_long", "asrb_transcribe_segments",
    "asrb_score_ids", "asrb_score_ingested",
    "asrb_align_ids", "asrb_align_ingested", "asrb_align_segments", "asrb_last_align_dims", "asrb_align_matrix_read",
    "asrb_stream_open", "asrb_stream_reset", "asrb_stream_push", "asrb_stream_mel_read", "asrb_stream_encode_read",
    "asrb_last_stream_stats",
]


class AsrbDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "d_model", "encoder_layers", "encoder_attention_heads", "encoder_ffn_dim", "num_mel_bins",
        "max_source_positions", "n_window", "n_window_infer", "downsample_hidden_size", "output_dim",
        "vocab_size", "hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads",
        "num_key_value_heads", "head_dim", "tie_word_embeddings")] + [("rms_norm_eps", C.c_double),
                                                                       ("rope_theta", C.c_double)]


class AsrbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"asr_b200 error {code}: {msg}")
        self.code = code


_lib = None


def load_library() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m qwen3_asr_rs_b200.build` "
            "(or __graft_entry__.build()).  This package has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    P = C.POINTER
    lib.asrb_last_error.restype = C.c_char_p
    lib.asrb_version.restype = C.c_char_p
    sig = {
        "asrb_init": [C.c_int, P(vp)],
        "asrb_ctx_free": [vp],
        "asrb_dims_default": [P(AsrbDims)],
        "asrb_model_load": [vp, C.c_char_p, P(vp)],
        "asrb_model_create": [vp, P(AsrbDims), P(vp)],
        "asrb_model_set_tensor": [vp, C.c_char_p, C.c_int, P(i64), C.c_int, vp],
        "asrb_model_finalize": [vp],
        "asrb_model_dims": [vp, P(AsrbDims)],
        "asrb_model_free": [vp],
        "asrb_model_lossy_tensors": [vp, P(C.c_int)],
        "asrb_session_create": [vp, C.c_int, i64, C.c_int, C.c_int, P(vp)],
        "asrb_session_free": [vp],
        "asrb_transcribe_ids": [vp, P(P(C.c_float)), P(i64), C.c_int, P(P(i64)), P(i32), C.c_int, P(i32), P(i32)],
        "asrb_mel": [vp, P(P(C.c_float)), P(i64), C.c_int, P(i64)],
        "asrb_mel_read": [vp, C.c_int, P(C.c_float)],
        "asrb_encode": [vp, P(i64)],
        "asrb_encode_read": [vp, C.c_int, P(C.c_float)],
        "asrb_prefill": [vp, P(P(i64)), P(i32), P(i64), P(C.c_float)],
        "asrb_decode_step": [vp, P(i64), P(C.c_float)],
        "asrb_generate": [vp, C.c_int, P(i32), P(i32)],
        "asrb_last_timings": [vp, P(C.c_float), P(i64), P(i64)],
        "asrb_session_set_option": [vp, C.c_char_p, C.c_char_p],
        "asrb_debug_mega_timeline": [P(C.c_longlong), C.c_int],
        "asrb_session_stats": [vp, P(i64), C.c_int],
        "asrb_session_device_ids": [vp, P(vp), P(vp), P(C.c_int), P(C.c_int)],
        "asrb_ingest_pcm": [vp, P(vp), P(i64), P(i32), P(i32), P(i32), C.c_int, P(i64)],
        "asrb_ingested_read": [vp, C.c_int, P(C.c_float)],
        "asrb_transcribe_ingested": [vp, P(P(i64)), P(i32), C.c_int, P(i32), P(i32)],
        "asrb_last_logprobs": [vp, C.c_int, P(C.c_float), P(C.c_float)],
        "asrb_last_top_logprobs": [vp, C.c_int, C.c_int, P(i32), P(C.c_float), P(i32), P(C.c_float)],
        "asrb_last_nbest": [vp, C.c_int, C.c_int, P(i32), P(i32), P(C.c_float), P(C.c_float), P(i32)],
        "asrb_last_beam_stats": [vp, P(i64), C.c_int],
        "asrb_session_create_ex": [vp, C.c_int, i64, C.c_int, C.c_int, C.c_int, P(vp)],
        "asrb_session_set_context": [vp, C.c_int, P(P(i64)), P(i32)],
        "asrb_last_prefill_stats": [vp, P(i64), C.c_int],
        "asrb_ingest_long": [vp, P(vp), P(i64), P(i32), P(i32), P(i32), C.c_int, P(i64)],
        "asrb_long_read": [vp, C.c_int, P(C.c_float)],
        "asrb_segment_long": [vp, i64, i64, C.c_int, P(i32), P(i64), P(i64)],
        "asrb_transcribe_segments": [vp, C.c_int, P(i32), P(i64), P(i64), P(P(i64)), P(i32), C.c_int, P(i32), P(i32)],
        "asrb_score_ids": [vp, P(P(C.c_float)), P(i64), C.c_int, P(P(i64)), P(i32), P(i32), P(P(i64)), P(i32), C.c_int,
                           P(C.c_float), P(i32), P(C.c_float)],
        "asrb_score_ingested": [vp, P(P(i64)), P(i32), P(i32), P(P(i64)), P(i32), C.c_int, P(C.c_float), P(i32), P(C.c_float)],
        "asrb_align_ids": [vp, P(P(C.c_float)), P(i64), C.c_int, P(P(i64)), P(i32), P(P(i64)), P(i32), P(i32), P(i32),
                           C.c_int, C.c_int, P(i32), P(i32)],
        "asrb_align_ingested": [vp, P(P(i64)), P(i32), P(P(i64)), P(i32), P(i32), P(i32), C.c_int, C.c_int, P(i32), P(i32)],
        "asrb_align_segments": [vp, C.c_int, P(i32), P(i64), P(i64), P(P(i64)), P(i32), P(P(i64)), P(i32), P(i32), P(i32),
                                C.c_int, C.c_int, P(i32), P(i32)],
        "asrb_last_align_dims": [vp, C.c_int, P(i32), P(i32)],
        "asrb_align_matrix_read": [vp, C.c_int, P(C.c_float)],
        "asrb_stream_open": [vp, C.c_int, C.c_int, C.c_int],
        "asrb_stream_reset": [vp, C.c_int],
        "asrb_stream_push": [vp, C.c_int, P(P(C.c_float)), P(i64), P(i32), P(P(i64)), P(i32), C.c_int, C.c_int, P(i32), P(i32),
                             P(i32)],
        "asrb_stream_mel_read": [vp, C.c_int, P(C.c_float)],
        "asrb_stream_encode_read": [vp, C.c_int, P(C.c_float)],
        "asrb_last_stream_stats": [vp, P(i64), C.c_int],
    }
    for name, args in sig.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int
    _lib = lib
    return lib


def check(code: int) -> None:
    if code != 0:
        raise AsrbError(code, load_library().asrb_last_error().decode("utf-8", "replace"))
