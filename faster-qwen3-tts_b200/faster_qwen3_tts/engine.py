"""ctypes binding of the H100-native decode engine (include/fq3_engine.h).

Python stays a thin host: every tensor crossing this boundary is a torch CUDA tensor whose ``data_ptr()`` is
handed to the C ABI; all arithmetic of the decode loop happens inside ``libfq3_engine.so`` (hand-written
sm_90a CUDA, csrc/).  There is NO fallback: if the shared library is missing or no CUDA device is present the
constructors raise.
"""
from __future__ import annotations

import ctypes as C
import operator
import os
import subprocess
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.normpath(os.path.join(_HERE, "..", "csrc"))
LIB_PATH = os.path.join(CSRC, "libfq3_engine.so")
INCLUDE = os.path.normpath(os.path.join(_HERE, "..", "..", "include"))

FQ3_F32, FQ3_BF16 = 0, 1
FQ3_RUNNING, FQ3_FIN_MAX_NEW, FQ3_FIN_EOS, FQ3_FIN_MAX_SEQ = 0, 1, 2, 3   # enum fq3_finish
FINISH_NAMES = {FQ3_RUNNING: "running", FQ3_FIN_MAX_NEW: "max_new_tokens", FQ3_FIN_EOS: "eos",
                FQ3_FIN_MAX_SEQ: "max_seq_len"}


class StackConfig(C.Structure):
    _fields_ = [("hidden_size", C.c_int32), ("intermediate_size", C.c_int32), ("num_hidden_layers", C.c_int32),
                ("num_attention_heads", C.c_int32), ("num_key_value_heads", C.c_int32), ("vocab_size", C.c_int32),
                ("rms_norm_eps", C.c_float)]


class Config(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("device", C.c_int32), ("max_seq_len", C.c_int32),
                ("num_code_groups", C.c_int32), ("codec_eos_token_id", C.c_int32),
                ("has_mtp_projection", C.c_int32), ("num_ctas", C.c_int32), ("rope_positions", C.c_int32),
                ("talker", StackConfig), ("predictor", StackConfig), ("kv_pages", C.c_int32), ("max_batch", C.c_int32),
                ("max_slots", C.c_int32)]


class Tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("dev_ptr", C.c_void_p), ("numel", C.c_int64)]


class Sampling(C.Structure):
    _fields_ = [("do_sample", C.c_int32), ("top_k", C.c_int32), ("temperature", C.c_float), ("top_p", C.c_float),
                ("repetition_penalty", C.c_float)]


class Request(C.Structure):
    _fields_ = [("first_token", C.c_int32), ("prefill_len", C.c_int32), ("gen_step", C.c_int32),
                ("rope_delta", C.c_int32), ("n_left_pad", C.c_int32), ("max_new_tokens", C.c_int32),
                ("min_new_tokens", C.c_int32), ("trailing_len", C.c_int32)]


class ConvProbe(C.Structure):
    _fields_ = [("X", C.c_void_p), ("W", C.c_void_p), ("bias", C.c_void_p), ("R", C.c_void_p), ("Yraw", C.c_void_p),
                ("Yact", C.c_void_p), ("ea", C.c_void_p), ("ib", C.c_void_p), ("scale", C.c_void_p),
                ("T", C.c_int32), ("Cin", C.c_int32), ("N", C.c_int32), ("taps", C.c_int32), ("dil", C.c_int32),
                ("mode", C.c_int32), ("bias_mod", C.c_int32), ("act_mod", C.c_int32), ("scale_mod", C.c_int32),
                ("x_row0", C.c_int32), ("x_rows", C.c_int32), ("batch", C.c_int32)]


class ChunkResult(C.Structure):
    _fields_ = [("frames_emitted", C.c_int32), ("finished", C.c_int32), ("total_frames", C.c_int32),
                ("next_token", C.c_int32)]


EXPORTS = [
    "fq3_engine_create", "fq3_engine_load_weights", "fq3_engine_destroy", "fq3_import_kv", "fq3_export_kv",
    "fq3_set_generation_state", "fq3_talker_step", "fq3_predictor_run", "fq3_sample_logits", "fq3_sample_logits_lp",
    "fq3_begin_request", "fq3_decode_chunk", "fq3_decode_chunk_lp", "fq3_decode_chunk_n", "fq3_max_slots", "fq3_slot_bytes", "fq3_set_text_rows", "fq3_get_past_hidden", "fq3_debug_enable", "fq3_debug_read", "fq3_tape_bytes",
    "fq3_num_ctas", "fq3_launch_count", "fq3_last_error", "fq3_version", "fq3_engine_set_prefill_weights", "fq3_prefill", "fq3_prefill_batch", "fq3_max_batch", "fq3_debug_gemv",
    "fq3_debug_conv_gemm", "fq3_kv_page_bytes", "fq3_map_kv_pages", "fq3_slot_kv_rows", "fq3_kv_pool_pages",
    "fq3_kv_pages_to", "fq3_kv_pages_from",
    "fq3_codec_create", "fq3_codec_load_weights", "fq3_codec_flops",
    "fq3_codec_load_frontend", "fq3_codec_decode_codes", "fq3_codec_frontend_flops",
    "fq3_codec_stream_create", "fq3_codec_stream_reset", "fq3_codec_stream_destroy", "fq3_codec_stream_frames",
    "fq3_codec_stream_decode", "fq3_codec_stream_copy", "fq3_codec_launch_count",
    "fq3_codec_destroy", "fq3_codec_last_error",
    "fq3_tempo_create", "fq3_tempo_reset", "fq3_tempo_destroy", "fq3_tempo_released", "fq3_tempo_process",
    "fq3_tempo_last_error",
    "fq3_resample_create", "fq3_resample_reset", "fq3_resample_destroy", "fq3_resample_released", "fq3_resample_taps",
    "fq3_resample_process", "fq3_resample_last_error", "fq3_resample_create_pitch", "fq3_resample_set_gain",
    "fq3_resample_released_pitch", "fq3_resample_taps_pitch", "fq3_resample_table_bytes",
    "fq3_flac_create", "fq3_flac_reset", "fq3_flac_destroy", "fq3_flac_max_bytes", "fq3_flac_process",
    "fq3_flac_last_error",
    "fq3_join_create", "fq3_join_reset", "fq3_join_destroy", "fq3_join_released", "fq3_join_total", "fq3_join_process",
    "fq3_join_last_error", "fq3_join_create_pauses", "fq3_join_reset_pauses",
]


def build_extension(verbose: bool = False) -> str:
    """Compile csrc/*.cu into libfq3_engine.so for sm_90a (cross-compiles without a GPU)."""
    srcs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + \
        [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    if os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps):
        return LIB_PATH
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-shared",
           "-Xcompiler", "-fPIC", "-I", INCLUDE, "-o", LIB_PATH] + srcs
    if verbose:
        print(" ".join(cmd))
    subprocess.run(cmd, check=True)
    return LIB_PATH


_lib = None


def load_library() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU / PyTorch fallback for the decode path.")
    lib = C.CDLL(LIB_PATH)
    lib.fq3_last_error.restype = C.c_char_p
    lib.fq3_version.restype = C.c_char_p
    lib.fq3_launch_count.restype = C.c_int64
    lib.fq3_launch_count.argtypes = [C.c_void_p]
    lib.fq3_engine_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
    lib.fq3_engine_load_weights.argtypes = [C.c_void_p, C.POINTER(Tensor), C.c_int32, C.c_void_p]
    lib.fq3_engine_destroy.argtypes = [C.c_void_p]
    lib.fq3_engine_destroy.restype = None
    lib.fq3_import_kv.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.fq3_export_kv.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.fq3_set_generation_state.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    lib.fq3_talker_step.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.fq3_predictor_run.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(Sampling), C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    lib.fq3_sample_logits.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(Sampling), C.c_float, C.c_void_p,
                                      C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.fq3_sample_logits_lp.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(Sampling), C.c_float, C.c_void_p,
                                         C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fq3_begin_request.argtypes = [C.c_void_p, C.c_int32, C.POINTER(Request), C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.POINTER(Sampling), C.POINTER(Sampling), C.c_void_p]
    lib.fq3_decode_chunk.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p,
                                     C.POINTER(ChunkResult), C.c_void_p]
    lib.fq3_decode_chunk_lp.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                        C.POINTER(ChunkResult), C.c_void_p]
    lib.fq3_decode_chunk_n.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_int32), C.c_void_p,
                                       C.c_void_p, C.POINTER(ChunkResult), C.c_void_p]
    lib.fq3_max_slots.argtypes = [C.c_void_p]
    lib.fq3_slot_bytes.argtypes = [C.POINTER(Config)]
    lib.fq3_slot_bytes.restype = C.c_int64
    lib.fq3_kv_page_bytes.argtypes = [C.POINTER(Config)]
    lib.fq3_kv_page_bytes.restype = C.c_int64
    lib.fq3_map_kv_pages.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32]
    lib.fq3_slot_kv_rows.argtypes = [C.c_void_p, C.c_int32]
    lib.fq3_kv_pool_pages.argtypes = [C.c_void_p]
    lib.fq3_kv_pages_to.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_void_p, C.c_void_p]
    lib.fq3_kv_pages_from.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_void_p, C.c_void_p]
    lib.fq3_set_text_rows.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32]
    lib.fq3_get_past_hidden.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.fq3_max_batch.argtypes = [C.c_void_p]
    lib.fq3_debug_gemv.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fq3_debug_conv_gemm.argtypes = [C.POINTER(ConvProbe), C.c_void_p]
    lib.fq3_debug_enable.argtypes = [C.c_void_p, C.c_int32]
    lib.fq3_debug_read.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
    lib.fq3_tape_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.fq3_num_ctas.argtypes = [C.c_void_p]
    lib.fq3_engine_set_prefill_weights.argtypes = [C.c_void_p, C.POINTER(Tensor), C.c_int32]
    lib.fq3_prefill.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                C.c_void_p]
    lib.fq3_prefill_batch.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_void_p, C.POINTER(C.c_int32),
                                      C.POINTER(C.c_int32), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fq3_codec_create.argtypes = [C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_void_p)]
    lib.fq3_codec_destroy.argtypes = [C.c_void_p]
    lib.fq3_codec_destroy.restype = None
    lib.fq3_codec_load_weights.argtypes = [C.c_void_p, C.POINTER(Tensor), C.c_int32, C.c_void_p]
    lib.fq3_codec_load_frontend.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_float), C.c_int32,
                                            C.POINTER(Tensor), C.c_int32, C.c_void_p]
    lib.fq3_codec_decode_codes.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.fq3_codec_stream_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    lib.fq3_codec_stream_reset.argtypes = [C.c_void_p, C.c_void_p]
    lib.fq3_codec_stream_destroy.argtypes = [C.c_void_p]
    lib.fq3_codec_stream_destroy.restype = None
    lib.fq3_codec_stream_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.fq3_codec_stream_frames.argtypes = [C.c_void_p]
    lib.fq3_codec_stream_frames.restype = C.c_int64
    lib.fq3_codec_stream_decode.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                            C.c_void_p]
    lib.fq3_codec_frontend_flops.argtypes = [C.c_void_p, C.c_int32]
    lib.fq3_codec_frontend_flops.restype = C.c_double
    lib.fq3_codec_flops.argtypes = [C.c_void_p, C.c_int32]
    lib.fq3_codec_flops.restype = C.c_double
    lib.fq3_codec_launch_count.argtypes = [C.c_void_p]
    lib.fq3_codec_launch_count.restype = C.c_int64
    lib.fq3_codec_last_error.restype = C.c_char_p
    lib.fq3_tempo_create.argtypes = [C.c_int32, C.c_double, C.POINTER(C.c_void_p)]
    lib.fq3_tempo_reset.argtypes = [C.c_void_p]
    lib.fq3_tempo_destroy.argtypes = [C.c_void_p]
    lib.fq3_tempo_destroy.restype = None
    lib.fq3_tempo_released.argtypes = [C.c_int32, C.c_int64, C.c_int64, C.c_int32]
    lib.fq3_tempo_released.restype = C.c_int64
    lib.fq3_tempo_process.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                      C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    lib.fq3_tempo_last_error.restype = C.c_char_p
    lib.fq3_resample_create.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
    lib.fq3_resample_reset.argtypes = [C.c_void_p]
    lib.fq3_resample_destroy.argtypes = [C.c_void_p]
    lib.fq3_resample_destroy.restype = None
    lib.fq3_resample_released.argtypes = [C.c_int32, C.c_int64, C.c_int64, C.c_int32]
    lib.fq3_resample_released.restype = C.c_int64
    lib.fq3_resample_taps.argtypes = [C.c_int32, C.POINTER(C.c_double), C.c_int32]
    lib.fq3_resample_taps.restype = C.c_int32
    lib.fq3_resample_process.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int64),
                                         C.POINTER(C.c_int32), C.c_void_p, C.c_int64, C.c_void_p]
    lib.fq3_resample_last_error.restype = C.c_char_p
    lib.fq3_resample_create_pitch.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
    lib.fq3_resample_set_gain.argtypes = [C.c_void_p, C.c_float]
    lib.fq3_resample_released_pitch.argtypes = [C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_int32]
    lib.fq3_resample_released_pitch.restype = C.c_int64
    lib.fq3_resample_taps_pitch.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_double), C.c_int32]
    lib.fq3_resample_taps_pitch.restype = C.c_int32
    lib.fq3_resample_table_bytes.argtypes = [C.c_int32]
    lib.fq3_resample_table_bytes.restype = C.c_int64
    lib.fq3_flac_create.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
    lib.fq3_flac_reset.argtypes = [C.c_void_p]
    lib.fq3_flac_destroy.argtypes = [C.c_void_p]
    lib.fq3_flac_destroy.restype = None
    lib.fq3_flac_max_bytes.argtypes = [C.c_int64, C.c_int64, C.c_int32]
    lib.fq3_flac_max_bytes.restype = C.c_int64
    lib.fq3_flac_process.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                     C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.fq3_flac_last_error.restype = C.c_char_p
    lib.fq3_join_create.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
    lib.fq3_join_reset.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    lib.fq3_join_create_pauses.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]
    lib.fq3_join_reset_pauses.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
    lib.fq3_join_destroy.argtypes = [C.c_void_p]
    lib.fq3_join_destroy.restype = None
    lib.fq3_join_released.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                      C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
    lib.fq3_join_total.argtypes = [C.c_void_p]
    lib.fq3_join_total.restype = C.c_int64
    lib.fq3_join_process.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                     C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.c_void_p, C.c_void_p, C.c_int64,
                                     C.c_void_p]
    lib.fq3_join_last_error.restype = C.c_char_p
    _lib = lib
    return lib


class EngineError(RuntimeError):
    pass


def _check(lib, rc: int):
    if rc != 0:
        msg = lib.fq3_last_error().decode()
        if rc == -4:
            raise RuntimeError(msg)  # same type/message as talker_graph.py:163-167
        raise EngineError(f"fq3 error {rc}: {msg}")


def debug_conv_gemm(X: torch.Tensor, W: torch.Tensor, *, mode: int = 0, dil: int = 1, T: Optional[int] = None,
                    bias: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None,
                    R: Optional[torch.Tensor] = None, ea: Optional[torch.Tensor] = None, ib: Optional[torch.Tensor] = None,
                    raw: bool = True, act: bool = False, x_row0: int = 0,
                    history: bool = False) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """One launch of the dense-layer GEMM of the prefill and the codec (numerics probe, fq3_debug_conv_gemm).
    X bf16 [batch, rows, Cin] (or [rows, Cin]); W bf16 [N, taps, Cin]; bias / scale / ea / ib float32 (column n reads
    element n % numel); R bf16 [batch, T, N].  With ``history`` the rows of X are [history ; new]: output row m reads
    input rows x_row0 + m - shift and ``T`` new rows are produced; otherwise T = rows.  Returns (Yraw, Yact) as bf16
    [batch, T, N] (Yraw [batch, T, N/2] in mode 1), None where not requested.  Operands are passed as they are, so an
    unaligned view reaches the kernel's own check; they must be contiguous CUDA tensors of the stated dtype."""
    def ptr(t, dtype, name):
        if t is None:
            return None
        if not (t.is_cuda and t.dtype == dtype and t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous CUDA {dtype} tensor")
        return t.data_ptr()
    lib = load_library()
    X3 = X if X.dim() == 3 else X[None]
    batch, rows, Cin = X3.shape
    N, taps = W.shape[0], W.shape[1]
    if W.shape[2] != Cin:
        raise ValueError("W must be [N, taps, Cin]")
    T = rows if T is None else int(T)
    dev = X.device
    Yraw = torch.empty(batch, T, N // 2 if mode == 1 else N, dtype=torch.bfloat16, device=dev) if raw else None
    Yact = torch.empty(batch, T, N, dtype=torch.bfloat16, device=dev) if act else None
    p = ConvProbe(ptr(X, torch.bfloat16, "X"), ptr(W, torch.bfloat16, "W"), ptr(bias, torch.float32, "bias"),
                  ptr(R, torch.bfloat16, "R"), ptr(Yraw, torch.bfloat16, "Yraw"), ptr(Yact, torch.bfloat16, "Yact"),
                  ptr(ea, torch.float32, "ea"), ptr(ib, torch.float32, "ib"), ptr(scale, torch.float32, "scale"),
                  T, Cin, N, taps, int(dil), int(mode), bias.numel() if bias is not None else 1,
                  ea.numel() if ea is not None else 1, scale.numel() if scale is not None else 1,
                  int(x_row0), rows if history else 0, batch)
    with torch.cuda.device(dev):
        _check(lib, lib.fq3_debug_conv_gemm(C.byref(p), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return Yraw, Yact


@dataclass
class SamplingParams:
    do_sample: bool = True
    top_k: int = 50
    temperature: float = 0.9
    top_p: float = 1.0
    repetition_penalty: float = 1.0

    def c(self) -> Sampling:
        return Sampling(int(bool(self.do_sample)), int(self.top_k), float(self.temperature), float(self.top_p),
                        float(self.repetition_penalty))


def _stack_config(d: dict) -> StackConfig:
    return StackConfig(d["hidden_size"], d["intermediate_size"], d["num_hidden_layers"], d["num_attention_heads"],
                       d["num_key_value_heads"], d["vocab_size"], float(d.get("rms_norm_eps", 1e-6)))


def slot_bytes(talker: dict, predictor: dict, dtype: torch.dtype, max_seq_len: int) -> int:
    """Device bytes one resident request slot costs (fq3_slot_bytes): what ``max_slots`` multiplies.  Needs no GPU."""
    lib = load_library()
    cfg = Config(dtype=FQ3_BF16 if dtype == torch.bfloat16 else FQ3_F32, max_seq_len=int(max_seq_len),
                 talker=_stack_config(talker), predictor=_stack_config(predictor))
    n = lib.fq3_slot_bytes(C.byref(cfg))
    if n < 0:
        _check(lib, int(n))
    return int(n)


def kv_page_bytes(talker: dict, predictor: dict, dtype: torch.dtype) -> int:
    """Device bytes of one talker KV page (fq3_kv_page_bytes): 64 cache rows of every layer and kv head, K and V.
    Needs no GPU."""
    lib = load_library()
    cfg = Config(dtype=FQ3_BF16 if dtype == torch.bfloat16 else FQ3_F32, max_seq_len=64,
                 talker=_stack_config(talker), predictor=_stack_config(predictor))
    n = lib.fq3_kv_page_bytes(C.byref(cfg))
    if n < 0:
        _check(lib, int(n))
    return int(n)


KV_PAGE = 64   # cache rows per talker KV page


class Engine:
    """One engine per device: packed weights, KV caches and the persistent decode kernel.  ``max_batch`` is the number
    of slots one launch may carry (<= 32), ``max_slots`` (default: ``max_batch``) the number of request slots that
    exist; with more slots than columns the caller chooses which ones each launch advances.  ``kv_pages`` (default 0:
    every slot owns ceil(max_seq_len / 64) pages for good) makes the talker cache a pool of that many 64-row pages that
    slots map with ``map_kv_pages`` as their rows are written."""

    def __init__(self, *, talker: dict, predictor: dict, dtype: torch.dtype, device="cuda", max_seq_len: int = 2048,
                 num_code_groups: int = 16, codec_eos_token_id: int = 2150, has_mtp_projection: bool = True,
                 num_ctas: int = 0, rope_positions: Optional[int] = None, max_batch: int = 1,
                 max_slots: Optional[int] = None, kv_pages: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("fq3 engine needs a CUDA device (sm_90a); no CPU fallback exists")
        self.lib = load_library()
        dev = torch.device(device)
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        if dtype not in (torch.float32, torch.bfloat16):
            raise ValueError("engine dtype must be torch.float32 or torch.bfloat16")
        self.dtype = dtype
        self.max_seq_len = int(max_seq_len)
        self.talker_cfg, self.pred_cfg = dict(talker), dict(predictor)
        self.num_code_groups = num_code_groups
        self.eos = codec_eos_token_id
        self.rope_positions = int(rope_positions or (self.max_seq_len + 64))

        cfg = Config(FQ3_BF16 if dtype == torch.bfloat16 else FQ3_F32, self.device.index, self.max_seq_len,
                     num_code_groups, codec_eos_token_id, int(bool(has_mtp_projection)), int(num_ctas),
                     self.rope_positions, _stack_config(talker), _stack_config(predictor), kv_pages=int(kv_pages),
                     max_batch=int(max_batch), max_slots=int(max_slots or 0))
        self.max_batch = int(max_batch)
        h = C.c_void_p()
        _check(self.lib, self.lib.fq3_engine_create(C.byref(cfg), C.byref(h)))
        self.h = h
        self.max_slots = int(self.lib.fq3_max_slots(h))
        self.kv_pages = int(self.lib.fq3_kv_pool_pages(h))   # pages in the pool
        self.paged = int(kv_pages) > 0                       # slots start unmapped: the caller maps their pages
        self.kv_page_bytes = kv_page_bytes(talker, predictor, dtype)
        self.H = talker["hidden_size"]
        self._keep = {}  # slot -> tensors borrowed by the engine for the duration of that slot's request
        self.gen_step0 = {}  # slot -> generation_step latched by begin_request (frame s reads trailing row gen_step0 + s)
        self.loaded = False
        self.has_prefill = False
        self._prefill_keep = None
        self.time_kernels = False   # bench: CUDA-event time of every decode_chunk launch
        self.last_kernel_ms = None

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.fq3_engine_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # -- helpers ---------------------------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _t(self, x: torch.Tensor, dtype=None) -> torch.Tensor:
        x = x.to(device=self.device, dtype=dtype or self.dtype)
        return x if x.is_contiguous() else x.contiguous()

    # -- weights ----------------------------------------------------------------------------------------
    def load_weights(self, tensors: Dict[str, torch.Tensor]):
        keep, arr = [], (Tensor * len(tensors))()
        for i, (name, t) in enumerate(tensors.items()):
            want = torch.float32 if name.split(".")[-1] in ("cos", "sin") else self.dtype
            t = self._t(t, want)
            keep.append(t)
            arr[i] = Tensor(name.encode(), t.data_ptr(), t.numel())
        with torch.cuda.device(self.device):
            _check(self.lib, self.lib.fq3_engine_load_weights(self.h, arr, len(tensors), self._stream()))
        self.loaded = True

    # -- K3 prefill -------------------------------------------------------------------------------------
    def set_prefill_weights(self, tensors: Dict[str, torch.Tensor]):
        """Row-major bf16 weights borrowed by the hand-written prefill (kept alive here)."""
        keep = {k: self._t(v) for k, v in tensors.items()}
        arr = (Tensor * len(keep))()
        for i, (k, v) in enumerate(keep.items()):
            arr[i] = Tensor(k.encode(), v.data_ptr(), v.numel())
        _check(self.lib, self.lib.fq3_engine_set_prefill_weights(self.h, arr, len(keep)))
        self._prefill_keep = keep
        self.has_prefill = True

    def prefill(self, embeds: torch.Tensor, n_left_pad: int = 0, slot: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """embeds [P,H] -> (logits [V], past_hidden [H]); cache rows [0,P) of request slot `slot` are written."""
        x = self._t(embeds.reshape(-1, self.H))
        logits = torch.empty(self.talker_cfg["vocab_size"], dtype=self.dtype, device=self.device)
        hidden = torch.empty(self.H, dtype=self.dtype, device=self.device)
        _check(self.lib, self.lib.fq3_prefill(self.h, int(slot), x.data_ptr(), x.shape[0], int(n_left_pad), logits.data_ptr(),
                                              hidden.data_ptr(), self._stream()))
        return logits, hidden

    def prefill_batch(self, rows, pads, slots) -> Tuple[torch.Tensor, torch.Tensor]:
        """Several prompts into distinct request slots with one chain of launches: ``rows`` is a list of [P_b,H]
        prompts (packed into one [sum P_b, H] tensor) or a left-padded [B,P,H] batch (packed by a reshape); ``pads[b]``
        is the left pad of prompt b, ``slots[b]`` its slot.  Returns (logits [n,V], past_hidden [n,H]); row b and the
        cache of ``slots[b]`` are bit-identical to ``prefill(rows[b], pads[b], slot=slots[b])``."""
        if isinstance(rows, torch.Tensor):
            x = self._t(rows.reshape(-1, self.H))
            lens = [int(rows.shape[1])] * int(rows.shape[0])
        else:
            parts = [r.reshape(-1, self.H) for r in rows]
            if len(parts) == 1:   # one prompt needs no packing copy
                x = self._t(parts[0])
            else:
                x = self._t(torch.cat(parts)) if parts else torch.empty(0, self.H, dtype=self.dtype, device=self.device)
            lens = [int(r.shape[0]) for r in parts]
        n = len(lens)
        if len(pads) != n or len(slots) != n:
            raise ValueError(f"{n} prompts but {len(pads)} pads and {len(slots)} slots")
        logits = torch.empty(n, self.talker_cfg["vocab_size"], dtype=self.dtype, device=self.device)
        hidden = torch.empty(n, self.H, dtype=self.dtype, device=self.device)
        arr = C.c_int32 * n
        _check(self.lib, self.lib.fq3_prefill_batch(self.h, n, arr(*[int(s) for s in slots]), x.data_ptr(), arr(*lens),
                                                    arr(*[int(p) for p in pads]), logits.data_ptr(), hidden.data_ptr(),
                                                    self._stream()))
        return logits, hidden

    # -- paged talker KV cache --------------------------------------------------------------------------------
    def map_kv_pages(self, slot: int, pages):
        """Set slot's page table: ``pages[i]`` holds its cache rows [64 i, 64 i + 64); an empty list unmaps it."""
        pages = [int(p) for p in pages]
        arr = (C.c_int32 * max(len(pages), 1))(*pages)
        _check(self.lib, self.lib.fq3_map_kv_pages(self.h, int(slot), arr, len(pages)))

    def slot_kv_rows(self, slot: int) -> int:
        """cache rows slot's pages map"""
        n = self.lib.fq3_slot_kv_rows(self.h, int(slot))
        if n < 0:
            _check(self.lib, n)
        return n

    def kv_pages_to(self, pages, dst: torch.Tensor):
        """copy whole pages into ``dst`` (uint8 [len(pages), kv_page_bytes], device or pinned host), stream-ordered"""
        self._page_copy(self.lib.fq3_kv_pages_to, pages, dst)

    def kv_pages_from(self, pages, src: torch.Tensor):
        """copy ``src`` (uint8 [len(pages), kv_page_bytes], device or pinned host) into whole pages, stream-ordered"""
        self._page_copy(self.lib.fq3_kv_pages_from, pages, src)

    def _page_copy(self, fn, pages, mem: torch.Tensor):
        pages = [int(p) for p in pages]
        if not (mem.dtype == torch.uint8 and mem.is_contiguous() and mem.numel() == len(pages) * self.kv_page_bytes
                and (mem.is_cuda or mem.is_pinned())):
            raise ValueError(f"page memory must be a contiguous uint8 tensor of {len(pages)} x {self.kv_page_bytes} bytes "
                             "on the device or in pinned host memory")
        arr = (C.c_int32 * max(len(pages), 1))(*pages)
        _check(self.lib, fn(self.h, arr, len(pages), mem.data_ptr(), self._stream()))

    # -- duck-type path ----------------------------------------------------------------------------------
    def import_kv(self, layer: int, k: torch.Tensor, v: torch.Tensor, slot: int = 0):
        """k, v: [1, n_kv, P, 128] (HF cache layout) or [n_kv, P, 128]."""
        k, v = self._t(k.reshape(-1, k.shape[-2], k.shape[-1])), self._t(v.reshape(-1, v.shape[-2], v.shape[-1]))
        _check(self.lib, self.lib.fq3_import_kv(self.h, int(slot), layer, k.data_ptr(), v.data_ptr(), k.shape[1],
                                                self._stream()))
        return k.shape[1]

    def export_kv(self, layer: int, P: int, slot: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
        """cache rows [0,P) of one layer as (k, v) [n_kv, P, 128]"""
        nkv = self.talker_cfg["num_key_value_heads"]
        k = torch.empty(nkv, P, 128, dtype=self.dtype, device=self.device)
        v = torch.empty_like(k)
        _check(self.lib, self.lib.fq3_export_kv(self.h, int(slot), int(layer), k.data_ptr(), v.data_ptr(), int(P),
                                                self._stream()))
        return k, v

    def set_generation_state(self, n_left_pad: int, rope_delta: int, slot: int = 0):
        _check(self.lib, self.lib.fq3_set_generation_state(self.h, int(slot), int(n_left_pad), int(rope_delta)))

    def talker_step(self, embeds: torch.Tensor, position: int, out: Optional[torch.Tensor] = None,
                    slot: int = 0) -> torch.Tensor:
        x = self._t(embeds.reshape(-1))
        if out is None:
            out = torch.empty(self.H, dtype=self.dtype, device=self.device)
        _check(self.lib, self.lib.fq3_talker_step(self.h, int(slot), x.data_ptr(), int(position), out.data_ptr(),
                                                  self._stream()))
        return out

    def predictor_run(self, pred_input: torch.Tensor, sp: SamplingParams,
                      uniforms: Optional[torch.Tensor] = None, slot: int = 0) -> torch.Tensor:
        x = self._t(pred_input.reshape(2, -1))
        out = torch.empty(self.num_code_groups - 1, dtype=torch.long, device=self.device)
        u = None
        if sp.do_sample:
            if uniforms is None:
                uniforms = torch.rand(self.num_code_groups - 1, device=self.device)
            u = self._t(uniforms, torch.float32)
        s = sp.c()
        _check(self.lib, self.lib.fq3_predictor_run(self.h, int(slot), x.data_ptr(), C.byref(s), u.data_ptr() if u is not None else None,
                                                     out.data_ptr(), self._stream()))
        return out

    def sample_logits(self, logits: torch.Tensor, sp: SamplingParams, u: float = 0.0,
                      history: Optional[torch.Tensor] = None, suppress_special: bool = False, eos_id: int = -1,
                      suppress_eos: bool = False, return_logprob: bool = False):
        """token [1] (device); with ``return_logprob``: (token [1], float32 [1] log-probability of the draw,
        fq3_decode_chunk_lp's definition)."""
        lg = self._t(logits.reshape(-1))
        out = torch.empty(1, dtype=torch.long, device=self.device)
        lp = torch.empty(1, dtype=torch.float32, device=self.device) if return_logprob else None
        h = self._t(history.reshape(-1), torch.long) if history is not None and history.numel() else None
        s = sp.c()
        _check(self.lib, self.lib.fq3_sample_logits_lp(self.h, lg.data_ptr(), lg.numel(), C.byref(s), float(u),
                                                        h.data_ptr() if h is not None else None,
                                                        h.numel() if h is not None else 0, int(suppress_special),
                                                        int(eos_id), int(suppress_eos), out.data_ptr(),
                                                        lp.data_ptr() if lp is not None else None, self._stream()))
        return (out, lp) if return_logprob else out

    # -- fused path ----------------------------------------------------------------------------------------
    def begin_request(self, *, first_token: int, prefill_len: int, gen_step: int, past_hidden: torch.Tensor,
                      trailing_text: torch.Tensor, tts_pad: torch.Tensor, max_new_tokens: int, min_new_tokens: int,
                      sp_talker: SamplingParams, sp_predictor: SamplingParams, uniforms: Optional[torch.Tensor],
                      rope_delta: int = 0, n_left_pad: int = 0, slot: int = 0, trailing_len: Optional[int] = None):
        """``trailing_len``: rows of ``trailing_text`` valid now (default: all of them); the rest of the buffer is for rows
        announced later through ``set_text_rows``."""
        ph = self._t(past_hidden.reshape(-1))
        tt = self._t(trailing_text.reshape(-1, self.H)) if trailing_text is not None and trailing_text.numel() else None
        tp = self._t(tts_pad.reshape(-1))
        need_u = sp_talker.do_sample or sp_predictor.do_sample
        if need_u and uniforms is None:
            uniforms = torch.rand(max_new_tokens + 1, 16, device=self.device)
        u = self._t(uniforms, torch.float32) if uniforms is not None else None
        if u is not None and u.numel() < (max_new_tokens + 1) * 16:
            raise ValueError("uniforms must have (max_new_tokens + 1) * 16 elements")
        self._keep[int(slot)] = dict(ph=ph, tt=tt, tp=tp, u=u)
        cap = 0 if tt is None else tt.shape[0]
        if trailing_len is not None and tt is not None and tt.data_ptr() != trailing_text.data_ptr():
            # rows written after the latch must reach the kernel: the engine has to borrow the caller's buffer itself
            raise ValueError("a trailing text buffer filled later must be a contiguous tensor of the engine's dtype on "
                             "its device (it would be copied)")
        n_rows = cap if trailing_len is None else int(trailing_len)
        if not 0 <= n_rows <= cap:
            raise ValueError(f"trailing_len {n_rows} outside the {cap} rows of trailing_text")
        rq = Request(int(first_token), int(prefill_len), int(gen_step), int(rope_delta), int(n_left_pad),
                     int(max_new_tokens), int(min_new_tokens), n_rows)
        st, spd = sp_talker.c(), sp_predictor.c()
        _check(self.lib, self.lib.fq3_begin_request(
            self.h, int(slot), C.byref(rq), ph.data_ptr(), tt.data_ptr() if tt is not None else None, tp.data_ptr(),
            u.data_ptr() if u is not None else None, C.byref(st), C.byref(spd), self._stream()))
        self.gen_step0[int(slot)] = int(gen_step)

    def set_text_rows(self, slot: int, trailing_len: int, open: bool):
        """Rows [0, trailing_len) of the slot's latched trailing buffer are valid; ``open``: more may follow, and a frame
        that would need a missing row waits for it (the launch stops the slot unfinished)."""
        tt = self._keep.get(int(slot), {}).get("tt")
        cap = 0 if tt is None else tt.shape[0]
        if trailing_len > cap:
            raise ValueError(f"trailing_len {trailing_len} exceeds the {cap} rows latched for slot {slot}")
        _check(self.lib, self.lib.fq3_set_text_rows(self.h, int(slot), int(trailing_len), int(bool(open))))

    def _logprob_buf(self, logprobs, shape):
        """float32 device buffer for fq3_decode_chunk_lp: None = off, True = a new one, or the caller's tensor"""
        if logprobs is None or logprobs is False:
            return None
        if logprobs is True:
            return torch.empty(*shape, dtype=torch.float32, device=self.device)
        if not (logprobs.device == self.device and logprobs.dtype == torch.float32 and logprobs.is_contiguous()
                and tuple(logprobs.shape) == tuple(shape)):
            raise ValueError(f"logprobs must be a contiguous float32 tensor of shape {tuple(shape)} on {self.device}")
        return logprobs

    def decode_chunk(self, n_frames: int, out: Optional[torch.Tensor] = None, slot: int = 0, logprobs=None):
        """Single-sequence launch on one slot: (codes [frames_emitted,16], result).  ``logprobs`` (True or a float32
        [n_frames,16] device tensor): also return the log-probability of every draw, (codes, logprobs
        [frames_emitted,16], result) -- column 0 of a row is the cb0 sampled after that frame (fq3_decode_chunk_lp)."""
        if out is None:
            out = torch.empty(n_frames, 16, dtype=torch.long, device=self.device)
        lp = self._logprob_buf(logprobs, (n_frames, 16))
        res = ChunkResult()
        sl = (C.c_int32 * 1)(int(slot))
        if self.time_kernels:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        _check(self.lib, self.lib.fq3_decode_chunk_lp(self.h, sl, 1, int(n_frames), out.data_ptr(),
                                                       lp.data_ptr() if lp is not None else None, C.byref(res),
                                                       self._stream()))
        if self.time_kernels:
            e1.record()
            e1.synchronize()
            self.last_kernel_ms = e0.elapsed_time(e1)
        if lp is not None:
            return out[: res.frames_emitted], lp[: res.frames_emitted], res
        return out[: res.frames_emitted], res

    def decode_chunk_batch(self, slots, n_frames, out: Optional[torch.Tensor] = None, logprobs=None):
        """All listed slots (at most ``max_batch`` of the ``max_slots`` resident ones) advance up to n_frames frames in
        ONE launch sharing every pass over the weights; ``n_frames`` is an int or one budget per slot (below, n_frames
        then stands for the largest).  Returns (codes [n_slots, n_frames, 16] -- row j valid up to
        results[j].frames_emitted --, [ChunkResult]).  ``logprobs`` (True or a float32 [n_slots,n_frames,16] device
        tensor): (codes, logprobs, results), valid as the codes are."""
        slots = [int(x) for x in slots]
        n = len(slots)
        budgets = None
        try:
            n_frames = operator.index(n_frames)   # any integer scalar (int, numpy, 0-d torch): one budget for all
        except TypeError:
            budgets = [int(x) for x in n_frames]
            if len(budgets) != n:
                raise ValueError(f"{n} slots but {len(budgets)} frame budgets")
            n_frames = max(max(budgets, default=0), 1)   # a budget <= 0 is the engine's to refuse
        if out is None:
            out = torch.empty(n, n_frames, 16, dtype=torch.long, device=self.device)
        lp = self._logprob_buf(logprobs, (n, n_frames, 16))
        res = (ChunkResult * n)()
        sl = (C.c_int32 * n)(*slots)
        if self.time_kernels:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        nf = int(n_frames) if budgets is None else (C.c_int32 * n)(*budgets)
        call = self.lib.fq3_decode_chunk_lp if budgets is None else self.lib.fq3_decode_chunk_n
        _check(self.lib, call(self.h, sl, n, nf, out.data_ptr(), lp.data_ptr() if lp is not None else None, res,
                              self._stream()))
        if self.time_kernels:
            e1.record()
            e1.synchronize()
            self.last_kernel_ms = e0.elapsed_time(e1)
        if lp is not None:
            return out, lp, list(res)
        return out, list(res)

    def past_hidden(self, slot: int = 0) -> torch.Tensor:
        out = torch.empty(self.H, dtype=self.dtype, device=self.device)
        _check(self.lib, self.lib.fq3_get_past_hidden(self.h, int(slot), out.data_ptr(), self._stream()))
        return out

    def debug_gemv(self, stack: int, layer: int, which: int, x: torch.Tensor) -> torch.Tensor:
        """One batched GEMV over a weight segment (numerics probe): x [ncols,K] -> [ncols, rows] fp32
        (which == 2: model dtype [ncols, I] = silu(gate) * up)."""
        x = self._t(x)
        d = self.talker_cfg if stack == 0 else self.pred_cfg
        H, I = d["hidden_size"], d["intermediate_size"]
        rows = {0: (d["num_attention_heads"] + 2 * d["num_key_value_heads"]) * 128, 1: H, 2: I, 3: H, 4: d["vocab_size"]}[which]
        out = torch.empty(x.shape[0], rows, dtype=self.dtype if which == 2 else torch.float32, device=self.device)
        _check(self.lib, self.lib.fq3_debug_gemv(self.h, int(stack), int(layer), int(which), x.shape[0], x.data_ptr(),
                                                 out.data_ptr(), self._stream()))
        return out

    # -- introspection ----------------------------------------------------------------------------------------
    def debug_enable(self, on):
        """bit 0: dump per-layer intermediates; bit 1: clock64 probes of CTA 0 (tools/microbench.py)."""
        _check(self.lib, self.lib.fq3_debug_enable(self.h, int(on)))

    def debug_layers(self, which: str, nt: int) -> Dict[str, torch.Tensor]:
        """Intermediates of the last talker step (which='t') / predictor pass 0 (which='p') as float32 CPU tensors."""
        d = self.talker_cfg if which == "t" else self.pred_cfg
        H, I, L = d["hidden_size"], d["intermediate_size"], d["num_hidden_layers"]
        qd, kd = d["num_attention_heads"] * 128, d["num_key_value_heads"] * 128
        strides = []
        for dd in (self.talker_cfg, self.pred_cfg):
            strides.append(2 * (dd["num_attention_heads"] + 2 * dd["num_key_value_heads"]) * 128 +
                           2 * dd["num_attention_heads"] * 128 + 4 * dd["hidden_size"] + 2 * dd["intermediate_size"])
        stride = max(strides)
        buf = torch.empty(stride * L, dtype=torch.float32)
        _check(self.lib, self.lib.fq3_debug_read(self.h, 0, buf.numel(), buf.data_ptr()))
        out = {}
        for l in range(L):
            r = buf[l * stride:(l + 1) * stride]
            o = 0
            out[f"L{l}.qkv"] = r[o:o + 2 * (qd + 2 * kd)].view(2, qd + 2 * kd)[:nt]; o += 2 * (qd + 2 * kd)
            out[f"L{l}.attn"] = r[o:o + nt * qd].view(nt, qd); o += 2 * qd
            out[f"L{l}.x1"] = r[o:o + 2 * H].view(2, H)[:nt]; o += 2 * H
            out[f"L{l}.act"] = r[o:o + nt * I].view(nt, I); o += 2 * I
            out[f"L{l}.x"] = r[o:o + 2 * H].view(2, H)[:nt]
        return out

    def probe_timestamps(self, n: int) -> torch.Tensor:
        buf = torch.empty(2 * n, dtype=torch.float32)
        _check(self.lib, self.lib.fq3_debug_read(self.h, 0, buf.numel(), buf.data_ptr()))
        return buf.view(torch.int64)

    def tape_bytes(self) -> Tuple[int, int]:
        a, b = C.c_int64(), C.c_int64()
        _check(self.lib, self.lib.fq3_tape_bytes(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    @property
    def num_ctas(self) -> int:
        return self.lib.fq3_num_ctas(self.h)

    @property
    def launch_count(self) -> int:
        return self.lib.fq3_launch_count(self.h)
