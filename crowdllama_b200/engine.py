"""ctypes binding of libclengine.so — the same C-ABI a Go cgo shim binds (include/clengine.h).

There is no CPU fallback anywhere in this package: if the shared library is missing the import
of the binding fails loudly, and if no sm_90 device is visible `Engine(...)` raises
`EngineError(CL_ERR_NO_DEVICE)`.
"""
from __future__ import annotations

import ctypes as C
import os
import time
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "lib" / "libclengine.so"

CL_OK = 0
CL_ERR_INVALID_ARG, CL_ERR_NO_DEVICE, CL_ERR_CUDA, CL_ERR_OOM, CL_ERR_UNKNOWN_MODEL, CL_ERR_TOO_LONG, \
    CL_ERR_BAD_SEQ, CL_ERR_SHUTDOWN, CL_ERR_IO, CL_ERR_INTERNAL, CL_ERR_BAD_MESSAGE = range(-1, -12, -1)

KINDS = dict(EMBED=0, LM_HEAD=1, FINAL_NORM=2, ATTN_NORM=3, WQ=4, WK=5, WV=6, WO=7, FFN_NORM=8, WGATE=9, WUP=10,
             WDOWN=11)


class ModelConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_layers", "d_model", "n_heads", "n_kv_heads", "head_dim", "d_ff",
                                         "vocab_size", "max_seq_len")] + \
               [("rope_theta", C.c_float), ("rms_eps", C.c_float), ("rope_factor", C.c_float), ("rope_low_freq_factor", C.c_float),
                ("rope_high_freq_factor", C.c_float), ("rope_original_max_pos", C.c_int32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class EngineConfig(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("device", C.c_int32), ("model_name", C.c_char_p), ("preset", C.c_char_p),
                ("model", ModelConfig), ("weights_path", C.c_char_p), ("weights_seed", C.c_uint64),
                ("kv_pool_bytes", C.c_int64), ("page_size", C.c_int32), ("max_batch", C.c_int32),
                ("max_seqs", C.c_int32), ("use_cuda_graph", C.c_int32), ("decode_path", C.c_int32),
                ("start_scheduler", C.c_int32), ("prefix_cache", C.c_int32), ("speculate", C.c_int32),
                ("reserved", C.c_int32 * 6)]   # reserved[0] .. [3]: the C struct's context_shift, num_keep, context_length, deterministic


class Sampling(C.Structure):
    _fields_ = [("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float), ("repeat_penalty", C.c_float),
                ("repeat_last_n", C.c_int32), ("seed", C.c_uint64), ("max_new_tokens", C.c_int32),
                ("ignore_eos", C.c_int32)]


class SamplingExt(C.Structure):
    """cl_sampling_ext: min_p, presence / frequency penalties and stop strings; all zero = cl_sampling alone."""
    _fields_ = [("min_p", C.c_float), ("presence_penalty", C.c_float), ("frequency_penalty", C.c_float), ("n_stop", C.c_int32),
                ("stop", C.POINTER(C.c_char_p)), ("reserved", C.c_int32 * 8)]


def sampling_ext(min_p: float = 0.0, presence_penalty: float = 0.0, frequency_penalty: float = 0.0, stop=()) -> SamplingExt:
    """A SamplingExt; stop: str or bytes items.  The ctypes array of the strings stays alive on the returned object."""
    x = SamplingExt(min_p=min_p, presence_penalty=presence_penalty, frequency_penalty=frequency_penalty)
    stop = [t.encode("utf-8") if isinstance(t, str) else bytes(t) for t in (stop or ())]
    if stop:
        x._stop_arr = (C.c_char_p * len(stop))(*stop)
        x.stop = C.cast(x._stop_arr, C.POINTER(C.c_char_p))
        x.n_stop = len(stop)
    return x


class Result(C.Structure):
    _fields_ = [("text", C.c_void_p), ("text_len", C.c_size_t), ("done_reason", C.c_void_p),
                ("token_ids", C.POINTER(C.c_int32)), ("n_prompt", C.c_int32), ("n_generated", C.c_int32),
                ("prefill_ns", C.c_int64), ("decode_ns", C.c_int64), ("total_ns", C.c_int64),
                ("n_preempted", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("tokens_per_sec", C.c_double), ("load", C.c_double), ("queue_depth", C.c_int32),
                ("active_seqs", C.c_int32), ("kv_pages_total", C.c_int32), ("kv_pages_used", C.c_int32),
                ("tokens_generated", C.c_int64), ("requests_completed", C.c_int64), ("preemptions", C.c_int64),
                ("vram_gb", C.c_int32), ("gpu_model", C.c_char * 64), ("kernel_launches", C.c_int64),
                ("measured_tokens_per_sec", C.c_double), ("sched_decode_steps", C.c_int64), ("sched_decode_ns", C.c_int64),
                ("sched_prefill_calls", C.c_int64), ("sched_prefill_tokens", C.c_int64), ("sched_prefill_ns", C.c_int64)]


class PrefixStats(C.Structure):
    _fields_ = [("enabled", C.c_int32), ("cached_pages", C.c_int32), ("lookups", C.c_int64), ("tokens_looked_up", C.c_int64),
                ("tokens_reused", C.c_int64), ("pages_evicted", C.c_int64), ("host_pages", C.c_int64), ("host_pages_cached", C.c_int64),
                ("pages_to_host", C.c_int64), ("pages_from_host", C.c_int64)]


class SpecStats(C.Structure):
    _fields_ = [("enabled", C.c_int32), ("max_draft", C.c_int32), ("verify_passes", C.c_int64), ("tokens_drafted", C.c_int64),
                ("tokens_accepted", C.c_int64), ("tokens_emitted", C.c_int64), ("multi_passes", C.c_int64),
                ("reserved", C.c_int64 * 3)]   # the C struct's draft_rows, draft_ns, draft_pages_used (Engine.draft_stats)


# cl_token_logprob (include/clengine.h): one record of the step tail's log-probabilities, 172 bytes
MAX_TOP_LOGPROBS = 20
TOKEN_LOGPROB = np.dtype([("id", np.int32), ("logprob", np.float32), ("n_top", np.int32),
                          ("top_ids", np.int32, (MAX_TOP_LOGPROBS,)), ("top_logprobs", np.float32, (MAX_TOP_LOGPROBS,))])
assert TOKEN_LOGPROB.itemsize == 172

# every symbol include/clengine.h declares (tests check the library exports all of them)
EXPORTS = [
    "cl_abi_version", "cl_strerror", "cl_last_error", "cl_default_engine_config", "cl_default_sampling",
    "cl_greedy_sampling", "cl_sample_token", "cl_model_preset", "cl_engine_create", "cl_engine_destroy", "cl_engine_model_config",
    "cl_engine_stats", "cl_engine_prefix_stats", "cl_engine_spec_stats", "cl_engine_set_speculate_batch", "cl_engine_set_prefix_host_cache", "cl_draft_ngram", "cl_engine_create_with_draft", "cl_draft_model", "cl_decode_verify", "cl_decode_verify_batch", "cl_engine_set_tensor", "cl_checkpoint_info", "cl_generate", "cl_generate_ids", "cl_generate_stream", "cl_result_free",
    "cl_handle_message", "cl_handle_message_stream", "cl_buffer_free", "cl_tokenize", "cl_detokenize", "cl_seq_create", "cl_seq_free",
    "cl_seq_len", "cl_seq_attach_prefix", "cl_prefill", "cl_prefill_batch", "cl_decode_step", "cl_decode_greedy", "cl_decode_greedy_batch", "cl_decode_sample_batch", "cl_decode_step_batch", "cl_seq_fake_fill",
    "cl_time_dominant_kernel", "cl_debug_kv", "cl_debug_hidden", "cl_debug_seq_hidden", "cl_debug_pass_info",
    "cl_debug_pass_rows", "cl_debug_timeline",
    "cl_op_gemv", "cl_op_gemv_residual", "cl_op_rmsnorm_gemv", "cl_op_rmsnorm_gateup", "cl_op_qkv_rope_append", "cl_op_attn_decode",
    "cl_op_attn_decode_batch", "cl_op_attn_verify", "cl_op_gemm_bf16", "cl_op_gemm_bf16_epi", "cl_op_attn_prefill", "cl_op_attn_prefill_variant",
    "cl_op_attn_prefill_cached", "cl_op_attn_prefill_long", "cl_attn_prefill_long_plan", "cl_gemm_split_plan", "cl_resolve_model_config", "cl_op_kv_host_roundtrip", "cl_op_sample", "cl_op_synth_weights", "cl_kvpool_create", "cl_kvpool_destroy",
    "cl_kvpool_reserve", "cl_kvpool_release", "cl_kvpool_pages_of", "cl_kvpool_free_pages", "cl_kvpool_used_pages",
    "cl_kvpool_attach", "cl_kvpool_publish", "cl_kvpool_cached_pages", "cl_kvpool_set_host_pages", "cl_kvpool_take_moves",
    "cl_kvpool_host_cached_pages", "cl_kvpool_shift", "cl_seq_shift", "cl_op_kv_shift", "cl_seq_set_logprobs", "cl_seq_take_logprobs", "cl_generate_ids_logprobs", "cl_op_sample_logprobs",
    "cl_sample_token_ext", "cl_op_sample_ext", "cl_seq_set_sampling_ext", "cl_generate_ids_ext",
    "cl_tokenizer_load", "cl_tokenizer_free", "cl_tokenizer_encode", "cl_tokenizer_decode", "cl_tokenizer_info", "cl_engine_load_tokenizer",
]

_lib = None


# callback types of the streaming entry points (include/clengine.h: cl_token_cb, cl_frame_cb)
TOKEN_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_int32), C.c_int32)
FRAME_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise ImportError(f"{LIB_PATH} is missing: run `python -m crowdllama_b200.build` "
                          "(there is no CPU fallback for the CUDA extension)")
    L = C.CDLL(str(LIB_PATH))
    vp, i32, i64, u64, f32, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_float, C.c_size_t
    P = C.POINTER
    sig = {
        "cl_abi_version": (C.c_int, []),
        "cl_strerror": (C.c_char_p, [C.c_int]),
        "cl_last_error": (C.c_char_p, []),
        "cl_default_engine_config": (None, [P(EngineConfig)]),
        "cl_default_sampling": (None, [P(Sampling)]),
        "cl_greedy_sampling": (None, [P(Sampling), i32]),
        "cl_model_preset": (C.c_int, [C.c_char_p, P(ModelConfig)]),
        "cl_engine_create": (C.c_int, [P(EngineConfig), P(vp)]),
        "cl_engine_destroy": (None, [vp]),
        "cl_engine_model_config": (C.c_int, [vp, P(ModelConfig)]),
        "cl_engine_stats": (C.c_int, [vp, P(Stats)]),
        "cl_engine_prefix_stats": (C.c_int, [vp, P(PrefixStats)]),
        "cl_engine_spec_stats": (C.c_int, [vp, P(SpecStats)]),
        "cl_draft_ngram": (C.c_int, [vp, i32, i32, vp, P(i32)]),
        "cl_engine_create_with_draft": (C.c_int, [P(EngineConfig), P(EngineConfig), P(vp)]),
        "cl_draft_model": (C.c_int, [vp, vp, i32, vp, vp, vp, vp, vp, vp, vp]),
        "cl_decode_verify": (C.c_int, [vp, i32, i32, vp, i32, P(Sampling), u64, vp, P(i32), vp]),
        "cl_engine_set_speculate_batch": (C.c_int, [vp, i32]),
        "cl_engine_set_prefix_host_cache": (C.c_int, [vp, i64]),
        "cl_decode_verify_batch": (C.c_int, [vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
        "cl_engine_set_tensor": (C.c_int, [vp, i32, i32, vp, i64]),
        "cl_checkpoint_info": (C.c_int, [C.c_char_p, P(ModelConfig), P(i32), P(i64)]),
        "cl_generate": (C.c_int, [vp, C.c_char_p, C.c_char_p, sz, P(Sampling), P(Result)]),
        "cl_generate_ids": (C.c_int, [vp, vp, i32, P(Sampling), P(Result)]),
        "cl_generate_stream": (C.c_int, [vp, C.c_char_p, C.c_char_p, sz, P(Sampling), TOKEN_CB, vp, P(Result)]),
        "cl_handle_message_stream": (C.c_int, [vp, C.c_char_p, sz, P(Sampling), FRAME_CB, vp]),
        "cl_result_free": (None, [P(Result)]),
        "cl_handle_message": (C.c_int, [vp, C.c_char_p, sz, P(Sampling), P(vp), P(sz)]),
        "cl_buffer_free": (None, [vp]),
        "cl_tokenize": (C.c_int, [vp, C.c_char_p, sz, vp, i32, P(i32)]),
        "cl_detokenize": (C.c_int, [vp, vp, i32, vp, sz, P(sz)]),
        "cl_seq_create": (C.c_int, [vp, P(i32)]),
        "cl_sample_token": (C.c_int, [vp, i32, vp, vp, i32, C.c_uint64, P(i32)]),
        "cl_seq_free": (C.c_int, [vp, i32]),
        "cl_seq_len": (C.c_int, [vp, i32, P(i32)]),
        "cl_seq_attach_prefix": (C.c_int, [vp, i32, vp, i32, P(i32)]),
        "cl_prefill": (C.c_int, [vp, i32, vp, i32, vp]),
        "cl_prefill_batch": (C.c_int, [vp, vp, i32, vp, vp, vp]),
        "cl_decode_step": (C.c_int, [vp, i32, i32, vp, P(i32)]),
        "cl_decode_greedy": (C.c_int, [vp, i32, i32, i32, vp, P(f32)]),
        "cl_decode_greedy_batch": (C.c_int, [vp, vp, i32, vp, i32, vp, P(f32)]),
        "cl_decode_sample_batch": (C.c_int, [vp, vp, i32, vp, P(Sampling), vp, i32, vp, P(f32)]),
        "cl_decode_step_batch": (C.c_int, [vp, vp, i32, vp, vp, vp]),
        "cl_seq_fake_fill": (C.c_int, [vp, i32, i32]),
        "cl_time_dominant_kernel": (C.c_int, [vp, i32, i32, i32, P(f32), P(f32)]),
        "cl_debug_kv": (C.c_int, [vp, i32, i32, i32, i32, i32, vp]),
        "cl_debug_hidden": (C.c_int, [vp, vp, i32]),
        "cl_debug_seq_hidden": (C.c_int, [vp, i32, i32, vp, i32, P(i32)]),
        "cl_debug_pass_info": (C.c_int, [vp, vp, vp, i32]),
        "cl_debug_pass_rows": (C.c_int, [vp, i32, i32, i32, vp]),
        "cl_debug_timeline": (C.c_int, [vp, vp, i32]),
        "cl_op_gemv": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, i32, i32, i32, P(f32)]),
        "cl_op_gemv_residual": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, vp, i32, i32]),
        "cl_op_rmsnorm_gemv": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, f32, vp, i32, i32]),
        "cl_op_rmsnorm_gateup": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, f32, vp, i32, i32]),
        "cl_op_attn_decode": (C.c_int, [C.c_int, vp, vp, vp, i32, i32, i32, i32, i32, vp]),
        "cl_op_qkv_rope_append": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, f32, i32, i32, i32, i32, i32, f32, vp, vp, vp]),
        "cl_op_attn_decode_batch": (C.c_int, [C.c_int, C.c_int, i32, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp,
                                              P(i32), P(i32)]),
        "cl_op_attn_verify": (C.c_int, [C.c_int, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp, P(i32)]),
        "cl_op_attn_prefill_long": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp, P(f32),
                                              P(i32), P(i32)]),
        "cl_attn_prefill_long_plan": (C.c_int, [i32, i32, i32, i32, i32, P(i32), P(i64)]),
        "cl_gemm_split_plan": (C.c_int, [i32, i32, i32, i32, P(i32)]),
        "cl_resolve_model_config": (C.c_int, [P(EngineConfig), P(ModelConfig)]),
        "cl_op_gemm_bf16": (C.c_int, [C.c_int, vp, vp, vp, i32, i32, i32, i32, P(f32)]),
        "cl_op_gemm_bf16_epi": (C.c_int, [C.c_int, C.c_int, i32, C.c_int, vp, vp, vp, vp, vp, i32, i32, i32, P(i32)]),
        "cl_op_attn_prefill": (C.c_int, [C.c_int, vp, vp, vp, i32, i32, i32, i32, vp]),
        "cl_op_attn_prefill_variant": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, i32, i32, i32, i32, vp, i32, P(f32)]),
        "cl_op_attn_prefill_cached": (C.c_int, [C.c_int, C.c_int, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]),
        "cl_op_kv_host_roundtrip": (C.c_int, [C.c_int, i32, i32, i32, i32, i32, i32, P(f32)]),
        "cl_op_sample": (C.c_int, [C.c_int, vp, i32, i32, P(Sampling), vp, vp, i32, vp, vp]),
        "cl_op_sample_logprobs": (C.c_int, [C.c_int, vp, i32, i32, P(Sampling), vp, vp, i32, vp, i32, vp, vp]),
        "cl_seq_set_logprobs": (C.c_int, [vp, i32, i32]),
        "cl_seq_shift": (C.c_int, [vp, i32, i32, i32]),
        "cl_kvpool_shift": (C.c_int, [vp, i32, i32, i32, i32, vp, i32, P(i32)]),
        "cl_op_kv_shift": (C.c_int, [C.c_int, i32, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, i32, P(f32)]),
        "cl_seq_take_logprobs": (C.c_int, [vp, i32, vp, i32, P(i32)]),
        "cl_generate_ids_logprobs": (C.c_int, [vp, vp, i32, P(Sampling), i32, P(Result), P(vp)]),
        "cl_op_synth_weights": (C.c_int, [C.c_int, u64, i32, i64, f32, vp]),
        "cl_sample_token_ext": (C.c_int, [vp, i32, P(Sampling), P(SamplingExt), vp, i32, u64, P(i32)]),
        "cl_op_sample_ext": (C.c_int, [C.c_int, vp, i32, i32, P(Sampling), P(SamplingExt), vp, vp, i32, vp, vp]),
        "cl_seq_set_sampling_ext": (C.c_int, [vp, i32, P(SamplingExt)]),
        "cl_generate_ids_ext": (C.c_int, [vp, vp, i32, P(Sampling), P(SamplingExt), i32, TOKEN_CB, vp, P(Result), P(vp)]),
        "cl_tokenizer_load": (C.c_int, [C.c_char_p, C.c_char_p, P(vp)]),
        "cl_tokenizer_free": (None, [vp]),
        "cl_tokenizer_encode": (C.c_int, [vp, C.c_char_p, sz, i32, i32, vp, i32, P(i32)]),
        "cl_tokenizer_decode": (C.c_int, [vp, vp, i32, vp, sz, P(sz)]),
        "cl_tokenizer_info": (C.c_int, [vp, P(i32), P(i32), P(i32)]),
        "cl_engine_load_tokenizer": (C.c_int, [vp, C.c_char_p, C.c_char_p]),
        "cl_kvpool_create": (C.c_int, [i32, i32, P(vp)]),
        "cl_kvpool_destroy": (None, [vp]),
        "cl_kvpool_reserve": (C.c_int, [vp, i32, i32]),
        "cl_kvpool_release": (C.c_int, [vp, i32]),
        "cl_kvpool_pages_of": (C.c_int, [vp, i32, vp, i32, P(i32)]),
        "cl_kvpool_free_pages": (C.c_int, [vp]),
        "cl_kvpool_used_pages": (C.c_int, [vp]),
        "cl_kvpool_attach": (C.c_int, [vp, i32, vp, i32, P(i32)]),
        "cl_kvpool_publish": (C.c_int, [vp, i32, vp, i32]),
        "cl_kvpool_cached_pages": (C.c_int, [vp]),
        "cl_kvpool_set_host_pages": (C.c_int, [vp, i32]),
        "cl_kvpool_take_moves": (C.c_int, [vp, vp, i32, P(i32)]),
        "cl_kvpool_host_cached_pages": (C.c_int, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


class EngineError(RuntimeError):
    def __init__(self, status: int, where: str):
        L = lib()
        self.status = status
        self.detail = L.cl_last_error().decode(errors="replace")
        super().__init__(f"{where}: {L.cl_strerror(status).decode()} ({status}) {self.detail}")


def _check(rc: int, where: str):
    if rc != CL_OK:
        raise EngineError(rc, where)


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def device_count() -> int:
    """Number of visible CUDA devices according to the driver (no torch involved)."""
    try:
        cuda = C.CDLL("libcuda.so.1")
    except OSError:
        return 0
    if cuda.cuInit(0) != 0:
        return 0
    n = C.c_int(0)
    if cuda.cuDeviceGetCount(C.byref(n)) != 0:
        return 0
    return n.value


def model_preset(name: str) -> dict:
    mc = ModelConfig()
    _check(lib().cl_model_preset(name.encode(), C.byref(mc)), "cl_model_preset")
    return mc.as_dict()


def checkpoint_info(path, model: dict | None = None):
    """cl_checkpoint_info: (model config, tensors, parameters) of an HF safetensors checkpoint; host-only validation."""
    mc = ModelConfig(**model) if model else ModelConfig()
    nt, npar = C.c_int32(0), C.c_int64(0)
    _check(lib().cl_checkpoint_info(str(path).encode(), C.byref(mc), C.byref(nt), C.byref(npar)), "cl_checkpoint_info")
    return mc.as_dict(), nt.value, npar.value


def greedy(max_new_tokens: int, ignore_eos: bool = False) -> Sampling:
    s = Sampling()
    lib().cl_greedy_sampling(C.byref(s), max_new_tokens)
    s.ignore_eos = 1 if ignore_eos else 0
    return s


def sample_token(logits, sampling: Sampling, history=(), step: int = 0) -> int:
    """The engine's host-side sampler on caller-provided logits (cl_sample_token; no GPU involved)."""
    lg = np.ascontiguousarray(logits, dtype=np.float32)
    h = np.ascontiguousarray(list(history), dtype=np.int32)
    out = C.c_int32()
    _check(lib().cl_sample_token(_ptr(lg), lg.size, C.byref(sampling), _ptr(h) if h.size else None, h.size, step, C.byref(out)), "cl_sample_token")
    return int(out.value)


def sample_token_ext(logits, sampling: Sampling, ext: SamplingExt | None, history=(), step: int = 0) -> int:
    """cl_sample_token_ext: sample_token with min_p and the presence / frequency penalties of ext (None: all zero)."""
    lg = np.ascontiguousarray(logits, dtype=np.float32)
    h = np.ascontiguousarray(list(history), dtype=np.int32)
    out = C.c_int32()
    _check(lib().cl_sample_token_ext(_ptr(lg), lg.size, C.byref(sampling), C.byref(ext) if ext is not None else None,
                                     _ptr(h) if h.size else None, h.size, step, C.byref(out)), "cl_sample_token_ext")
    return int(out.value)


def draft_ngram(hist, k: int) -> np.ndarray:
    """The prompt-lookup drafter of speculative decoding (cl_draft_ngram; no GPU involved): the up to k ids that followed
    the most recent earlier occurrence of hist's last 3 (else 2) ids; empty when there is none."""
    h = np.ascontiguousarray(hist, dtype=np.int32)
    out = np.empty(max(k, 1), np.int32)
    n = C.c_int32(0)
    _check(lib().cl_draft_ngram(_ptr(h) if h.size else None, h.size, k, _ptr(out), C.byref(n)), "cl_draft_ngram")
    return out[:n.value].copy()


def ollama_default_sampling(seed: int = 0, max_new_tokens: int = -1) -> Sampling:
    s = Sampling()
    lib().cl_default_sampling(C.byref(s))
    s.seed = seed
    s.max_new_tokens = max_new_tokens
    return s


def draft_engine_config(preset: str | None, model: dict | None, weights_path: str | None, seed: int, keep: list):
    """The draft config cl_engine_create_with_draft reads (preset / model / weights_path / weights_seed), or None when no
    draft model is asked for.  keep: a list that holds the encoded strings alive as long as the engine."""
    if preset is None and model is None and weights_path is None:
        return None
    d = EngineConfig()
    lib().cl_default_engine_config(C.byref(d))
    if preset is not None:
        keep.append(preset.encode())
        d.preset = keep[-1]
    else:
        d.preset = None
    if model is not None:
        d.model = ModelConfig(**model)
    if weights_path is not None:
        keep.append(str(weights_path).encode())
        d.weights_path = keep[-1]
    d.weights_seed = seed
    return d


class GenerateResult:
    def __init__(self, r: Result):
        self.text = C.string_at(r.text, r.text_len).decode("utf-8", errors="replace") if r.text else ""
        self.done_reason = C.string_at(r.done_reason).decode() if r.done_reason else ""
        self.token_ids = np.ctypeslib.as_array(r.token_ids, shape=(max(r.n_generated, 1),))[:r.n_generated].copy() \
            if r.n_generated else np.zeros(0, np.int32)
        self.n_prompt, self.n_generated = r.n_prompt, r.n_generated
        self.prefill_ns, self.decode_ns, self.total_ns = r.prefill_ns, r.decode_ns, r.total_ns
        self.n_preempted = r.n_preempted

    @classmethod
    def from_response(cls, text: str, done_reason: str) -> "GenerateResult":
        """A result answered over the wire (GenerateResponse): text and done_reason, no ids or timings."""
        g = cls.__new__(cls)
        g.text, g.done_reason, g.token_ids = text, done_reason, np.zeros(0, np.int32)
        g.n_prompt = g.n_generated = g.prefill_ns = g.decode_ns = g.total_ns = g.n_preempted = 0
        return g


def _ext_kwargs(stop=None, min_p=None, presence_penalty=None, frequency_penalty=None) -> dict:
    return {k: v for k, v in dict(stop=stop, min_p=min_p, presence_penalty=presence_penalty, frequency_penalty=frequency_penalty).items()
            if v is not None}


class Engine:
    """One engine per GPU process (independent replicas; no NCCL on the decode path)."""

    def __init__(self, preset: str | None = None, model: dict | None = None, model_name: str | None = None,
                 device: int = 0, seed: int = 1234, max_batch: int = 8, max_seqs: int | None = None,
                 page_size: int = 32, kv_pool_bytes: int = 0, use_cuda_graph: bool = True, decode_path: int = 0,
                 start_scheduler: bool = False, weights_path: str | None = None, prefix_cache: bool = False,
                 speculate: int = 0, speculate_batch: int = 1, prefix_cache_host_bytes: int = 0, context_shift: bool = False,
                 num_keep: int = 4, context_length: int = 0, draft_preset: str | None = None, draft_model: dict | None = None,
                 draft_weights_path: str | None = None, draft_seed: int | None = None, deterministic: bool = False):
        L = lib()
        cfg = EngineConfig()
        L.cl_default_engine_config(C.byref(cfg))
        cfg.device = device
        self._keep = [(model_name or preset or "model").encode(), preset.encode() if preset else None]
        cfg.model_name = self._keep[0]
        cfg.preset = self._keep[1]
        if model is not None:
            cfg.preset = None
            cfg.model = ModelConfig(**model)
        cfg.weights_seed = seed
        if weights_path is not None:
            self._keep.append(str(weights_path).encode())
            cfg.weights_path = self._keep[-1]
        cfg.max_batch = max_batch
        cfg.max_seqs = max_seqs or max_batch
        cfg.page_size = page_size
        cfg.kv_pool_bytes = kv_pool_bytes
        cfg.use_cuda_graph = 1 if use_cuda_graph else -1
        cfg.decode_path = decode_path
        cfg.start_scheduler = 1 if start_scheduler else 0
        cfg.prefix_cache = 1 if prefix_cache else 0     # env CL_PREFIX_CACHE=0|1 overrides
        cfg.speculate = speculate                       # 0 off, 1..15 drafted tokens per verify pass; env CL_SPECULATE overrides
        cfg.reserved[0] = 1 if context_shift else 0     # cl_engine_config.context_shift; env CL_CONTEXT_SHIFT=0|1 overrides
        cfg.reserved[1] = num_keep                      # cl_engine_config.num_keep (Ollama's documented default 4); env CL_NUM_KEEP overrides
        cfg.reserved[2] = context_length                # cl_engine_config.context_length (0: the model's window); env CL_CONTEXT_LENGTH overrides
        cfg.reserved[3] = 1 if deterministic else 0     # cl_engine_config.deterministic; env CL_DETERMINISTIC=0|1 overrides
        h = C.c_void_p()
        dcfg = draft_engine_config(draft_preset, draft_model, draft_weights_path, seed if draft_seed is None else draft_seed,
                                   self._keep)
        if dcfg is None:
            _check(L.cl_engine_create(C.byref(cfg), C.byref(h)), "cl_engine_create")
        else:   # speculative decoding with a draft model (cl_engine_create_with_draft); env CL_DRAFT_MODEL is for plain creates
            _check(L.cl_engine_create_with_draft(C.byref(cfg), C.byref(dcfg), C.byref(h)), "cl_engine_create_with_draft")
        self._h = h
        # requests verified in one pass; env CL_SPECULATE_BATCH overrides the argument, as CL_SPECULATE does `speculate`
        if speculate_batch != 1 and "CL_SPECULATE_BATCH" not in os.environ:
            self.set_speculate_batch(speculate_batch)
        # host tier of the prefix cache; env CL_PREFIX_CACHE_HOST_MIB sizes it at create and overrides the argument
        if prefix_cache_host_bytes and "CL_PREFIX_CACHE_HOST_MIB" not in os.environ:
            self.set_prefix_host_cache(prefix_cache_host_bytes)
        mc = ModelConfig()
        _check(L.cl_engine_model_config(self._h, C.byref(mc)), "cl_engine_model_config")
        self.cfg = mc.as_dict()
        self.model_name = self._keep[0].decode()

    def close(self):
        if getattr(self, "_h", None):
            lib().cl_engine_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights ---------------------------------------------------------------------------------
    def set_tensor(self, layer: int, kind: str, bf16: np.ndarray):
        a = np.ascontiguousarray(bf16, dtype=np.uint16)
        _check(lib().cl_engine_set_tensor(self._h, layer, KINDS[kind], _ptr(a), a.size), f"set_tensor({kind})")

    # ---- token level -----------------------------------------------------------------------------
    def seq_create(self) -> int:
        s = C.c_int32(-1)
        _check(lib().cl_seq_create(self._h, C.byref(s)), "cl_seq_create")
        return s.value

    def seq_free(self, s: int):
        _check(lib().cl_seq_free(self._h, s), "cl_seq_free")

    def set_logprobs(self, s: int, top_n: int):
        """cl_seq_set_logprobs: -1 off, 0..20 = every later step tail of s leaves a record with top_n alternatives."""
        _check(lib().cl_seq_set_logprobs(self._h, s, top_n), "cl_seq_set_logprobs")

    def set_sampling_ext(self, s: int, ext: SamplingExt | None):
        """cl_seq_set_sampling_ext: min_p and the presence / frequency penalties for every later draw of s (None: all zero)."""
        _check(lib().cl_seq_set_sampling_ext(self._h, s, C.byref(ext) if ext is not None else None), "cl_seq_set_sampling_ext")

    def take_logprobs(self, s: int) -> np.ndarray:
        """cl_seq_take_logprobs: the records of the ids chosen for s since the last take (a TOKEN_LOGPROB array)."""
        n = C.c_int32()
        _check(lib().cl_seq_take_logprobs(self._h, s, None, 0, C.byref(n)), "cl_seq_take_logprobs")
        out = np.zeros(n.value, TOKEN_LOGPROB)
        _check(lib().cl_seq_take_logprobs(self._h, s, out.ctypes.data, n.value, C.byref(n)), "cl_seq_take_logprobs")
        return out[:n.value]

    def seq_len(self, s: int) -> int:
        n = C.c_int32()
        _check(lib().cl_seq_len(self._h, s, C.byref(n)), "cl_seq_len")
        return n.value

    def attach_prefix(self, s: int, ids) -> int:
        """cl_seq_attach_prefix: a new sequence takes the cached K/V of the longest page-aligned prefix of ids (at most
        len(ids) - 1 tokens); returns the tokens reused, after which the caller prefills ids[reused:].  0 with the cache off."""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        n = C.c_int32(0)
        _check(lib().cl_seq_attach_prefix(self._h, s, _ptr(ids), len(ids), C.byref(n)), "cl_seq_attach_prefix")
        return n.value

    def seq_shift(self, s: int, n_keep: int, n_discard: int):
        """cl_seq_shift: cached tokens [n_keep, n_keep + n_discard) leave the sequence (n_discard a multiple of page_size); the
        kept K after them is rotated to its new position, len drops by n_discard."""
        _check(lib().cl_seq_shift(self._h, s, n_keep, n_discard), "cl_seq_shift")

    def prefill(self, s: int, ids, want_logits: bool = True):
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        out = np.empty(self.cfg["vocab_size"], np.float32) if want_logits else None
        _check(lib().cl_prefill(self._h, s, _ptr(ids), len(ids), _ptr(out) if want_logits else None), "cl_prefill")
        return out

    def prefill_batch(self, seqs, prompts, want_logits: bool = True):
        """cl_prefill_batch: several prompts in one pass; returns [n_seqs][vocab] logits of the last positions (or None)."""
        ss = np.ascontiguousarray(seqs, dtype=np.int32)
        lens = np.ascontiguousarray([len(p) for p in prompts], dtype=np.int32)
        ids = np.ascontiguousarray(np.concatenate([np.asarray(p, np.int32) for p in prompts]), dtype=np.int32)
        out = np.empty((len(ss), self.cfg["vocab_size"]), np.float32) if want_logits else None
        _check(lib().cl_prefill_batch(self._h, _ptr(ss), len(ss), _ptr(ids), _ptr(lens), _ptr(out) if want_logits else None), "cl_prefill_batch")
        return out

    def decode_step(self, s: int, tok: int, want_logits: bool = True):
        out = np.empty(self.cfg["vocab_size"], np.float32) if want_logits else None
        am = C.c_int32(-1)
        _check(lib().cl_decode_step(self._h, s, int(tok), _ptr(out) if want_logits else None, C.byref(am)),
               "cl_decode_step")
        return out, am.value

    def decode_greedy(self, s: int, first_id: int, n_steps: int):
        ids = np.empty(n_steps, np.int32)
        ms = C.c_float(0)
        _check(lib().cl_decode_greedy(self._h, s, int(first_id), n_steps, _ptr(ids), C.byref(ms)), "cl_decode_greedy")
        return ids, ms.value

    def decode_greedy_batch(self, seqs, first_ids, n_steps: int):
        seqs = np.ascontiguousarray(seqs, dtype=np.int32)
        first = np.ascontiguousarray(first_ids, dtype=np.int32)
        ids = np.empty((n_steps, len(seqs)), np.int32)
        ms = C.c_float(0)
        _check(lib().cl_decode_greedy_batch(self._h, _ptr(seqs), len(seqs), _ptr(first), n_steps, _ptr(ids),
                                            C.byref(ms)), "cl_decode_greedy_batch")
        return ids, ms.value

    def decode_sample_batch(self, seqs, first_ids, samplings, n_steps: int, step0=None):
        """cl_decode_sample_batch: like decode_greedy_batch, sequence b drawing with samplings[b] on the device (greedy where
        its temperature is 0); draw i of sequence b uses RNG step step0[b] + i.  Returns (ids [n_steps][B], device ms)."""
        seqs = np.ascontiguousarray(seqs, dtype=np.int32)
        first = np.ascontiguousarray(first_ids, dtype=np.int32)
        sp = (Sampling * len(seqs))(*samplings)
        st = np.ascontiguousarray(step0 if step0 is not None else np.zeros(len(seqs)), dtype=np.uint64)
        ids = np.empty((n_steps, len(seqs)), np.int32)
        ms = C.c_float(0)
        _check(lib().cl_decode_sample_batch(self._h, _ptr(seqs), len(seqs), _ptr(first), sp, _ptr(st), n_steps, _ptr(ids),
                                            C.byref(ms)), "cl_decode_sample_batch")
        return ids, ms.value

    def decode_step_batch(self, seqs, toks, want_logits: bool = True):
        """One batched step with caller-chosen tokens; returns (logits [B][V] or None, greedy next ids [B])."""
        seqs = np.ascontiguousarray(seqs, dtype=np.int32)
        toks = np.ascontiguousarray(toks, dtype=np.int32)
        out = np.empty((len(seqs), self.cfg["vocab_size"]), np.float32) if want_logits else None
        am = np.empty(len(seqs), np.int32)
        _check(lib().cl_decode_step_batch(self._h, _ptr(seqs), len(seqs), _ptr(toks), _ptr(out) if want_logits else None, _ptr(am)),
               "cl_decode_step_batch")
        return out, am

    def decode_verify(self, s: int, input_id: int, draft, sampling: Sampling | None = None, step0: int = 0,
                      want_logits: bool = False):
        """cl_decode_verify: one verify pass of input_id (the next input) and the drafted ids after it.  Returns (emitted ids
        y_1 .. y_{a+1}, logits [k + 1][vocab] or None); the sequence advances by a + 1 tokens."""
        d = np.ascontiguousarray(draft, dtype=np.int32)
        ids = np.empty(max(len(d), 0) + 1, np.int32)
        n = C.c_int32(0)
        out = np.empty((len(d) + 1, self.cfg["vocab_size"]), np.float32) if want_logits else None
        _check(lib().cl_decode_verify(self._h, s, int(input_id), _ptr(d), len(d), C.byref(sampling) if sampling else None, step0,
                                      _ptr(ids), C.byref(n), _ptr(out) if want_logits else None), "cl_decode_verify")
        return ids[:n.value].copy(), out

    def decode_verify_batch(self, seqs, input_ids, drafts, samplings=None, step0=None, want_logits: bool = False):
        """cl_decode_verify_batch: one verify pass over several sequences; drafts[i] (0..15 ids) follow input_ids[i].
        samplings (None, or one Sampling or None per sequence: greedy) and step0 as in decode_verify.  Returns (a list of the
        emitted ids of every sequence, logits [sum(k_i + 1)][vocab] or None)."""
        seqs = np.ascontiguousarray(seqs, dtype=np.int32)
        x0 = np.ascontiguousarray(input_ids, dtype=np.int32)
        ks = np.array([len(d) for d in drafts], np.int32)
        flat = np.ascontiguousarray(np.concatenate([np.asarray(d, np.int64) for d in drafts] + [np.zeros(1, np.int64)]), dtype=np.int32)
        rows = int(ks.sum()) + len(seqs)
        sp = None
        if samplings is not None:
            sp = (Sampling * len(seqs))(*[s if s is not None else greedy(-1) for s in samplings])
        st = np.ascontiguousarray(step0 if step0 is not None else np.zeros(len(seqs)), dtype=np.uint64)
        ids = np.empty(rows, np.int32)
        n = np.zeros(len(seqs), np.int32)
        out = np.empty((rows, self.cfg["vocab_size"]), np.float32) if want_logits else None
        _check(lib().cl_decode_verify_batch(self._h, _ptr(seqs), len(seqs), _ptr(x0), _ptr(flat), _ptr(ks), sp, _ptr(st), _ptr(ids),
                                            _ptr(n), _ptr(out) if want_logits else None), "cl_decode_verify_batch")
        r0 = np.concatenate([[0], np.cumsum(ks + 1)])
        return [ids[r0[i]:r0[i] + n[i]].copy() for i in range(len(seqs))], out

    def draft_model(self, seqs, hists, ks, samplings=None, step0=None):
        """cl_draft_model: the draft model's drafter.  For target sequence seqs[i], its mirror catches up with hists[i] (the
        window ending with the next input) and drafts ks[i] ids (0..15), greedy or with samplings[i] (None, or one Sampling
        or None per sequence) at RNG steps step0[i] + j.  Returns the list of every sequence's drafted ids."""
        seqs = np.ascontiguousarray(seqs, dtype=np.int32)
        hs = [np.ascontiguousarray(h, dtype=np.int32) for h in hists]
        ptrs = (C.c_void_p * len(hs))(*[h.ctypes.data for h in hs])
        lens = np.array([len(h) for h in hs], np.int32)
        ks = np.ascontiguousarray(ks, dtype=np.int32)
        sp = None
        if samplings is not None:
            sp = (Sampling * len(seqs))(*[s if s is not None else greedy(-1) for s in samplings])
        st = np.ascontiguousarray(step0 if step0 is not None else np.zeros(len(seqs)), dtype=np.uint64)
        out = np.zeros(max(int(ks.sum()), 1), np.int32)
        n = np.zeros(len(seqs), np.int32)
        _check(lib().cl_draft_model(self._h, _ptr(seqs), len(seqs), ptrs, _ptr(lens), _ptr(ks), sp, _ptr(st), _ptr(out), _ptr(n)),
               "cl_draft_model")
        off = np.concatenate([[0], np.cumsum(ks)])
        return [out[off[i]:off[i] + n[i]].copy() for i in range(len(seqs))]

    def set_speculate_batch(self, n: int):
        """cl_engine_set_speculate_batch: how many running requests the scheduler may verify in one pass (1 = only a
        request running alone)."""
        _check(lib().cl_engine_set_speculate_batch(self._h, n), "cl_engine_set_speculate_batch")

    def set_prefix_host_cache(self, nbytes: int):
        """cl_engine_set_prefix_host_cache: pinned host memory behind the prefix cache (whole pages; 0 frees it).  Only with
        the prefix cache on and no sequence live or queued."""
        _check(lib().cl_engine_set_prefix_host_cache(self._h, nbytes), "cl_engine_set_prefix_host_cache")

    def seq_fake_fill(self, s: int, n_tokens: int):
        """Fill the sequence's paged KV (all layers) with the synthetic cache pattern the parity tests' CPU checker also
        generates (include/clengine.h: cl_seq_fake_fill) — a parity aid."""
        _check(lib().cl_seq_fake_fill(self._h, s, n_tokens), "cl_seq_fake_fill")

    def debug_kv(self, s: int, layer: int, which: int, t0: int, n: int) -> np.ndarray:
        """Cached K (which=0) / V (which=1) rows of `layer` for tokens t0..t0+n-1: [n][n_kv*head_dim] fp32.  which 2 / 3:
        K / V up to the end of the pages the sequence holds, where a verify pass leaves its rejected rows (valid until the
        sequence's next pass or step)."""
        out = np.empty((n, self.cfg["n_kv_heads"] * self.cfg["head_dim"]), np.float32)
        _check(lib().cl_debug_kv(self._h, s, layer, which, t0, n, _ptr(out)), "cl_debug_kv")
        return out

    def time_dominant_kernel(self, s: int, first_id: int, n_steps: int):
        """(kernel_ms, step_ms): mean CUDA-event time of the dominant kernel / of the whole eagerly launched step."""
        k, t = C.c_float(0), C.c_float(0)
        _check(lib().cl_time_dominant_kernel(self._h, s, int(first_id), n_steps, C.byref(k), C.byref(t)), "cl_time_dominant_kernel")
        return k.value, t.value

    def debug_hidden(self) -> np.ndarray:
        out = np.empty(self.cfg["d_model"], np.float32)
        _check(lib().cl_debug_hidden(self._h, _ptr(out), out.size), "cl_debug_hidden")
        return out

    def debug_seq_hidden(self, s: int, what: str) -> np.ndarray:
        """cl_debug_seq_hidden: one buffer of sequence s after the latest decode step that contained it.  what: "h" (residual
        stream), "q" (roped q), "attn" (attention output, fp32), "act" (SwiGLU activation of a single-sequence step),
        "attn_bf16" / "act_bf16" (the rows the batched step's o / down projections read)."""
        i = ("h", "q", "attn", "act", "attn_bf16", "act_bf16").index(what)
        n = self.cfg["d_model"] if i == 0 else self.cfg["d_ff"] if i in (3, 5) else self.cfg["n_heads"] * self.cfg["head_dim"]
        out = np.empty(n, np.float32)
        _check(lib().cl_debug_seq_hidden(self._h, s, i, _ptr(out), n, None), "cl_debug_seq_hidden")
        return out

    PASS_PATHS = ("split-k", "tile")
    PASS_ATTN = ("mma", "wgmma", "verify", "mixed", "long")

    def debug_pass_info(self) -> dict:
        """cl_debug_pass_info: the latest multi-row pass.  {"path": "split-k" | "tile", "attn": "mma" | "wgmma" | "verify" |
        "mixed" | "long" (the split-KV wgmma kernel), "T": rows, "segs": [(seq, row0, n, pos0), ...]}.  EngineError when none is recorded (a token-wise prefill
        or a failed pass since)."""
        info = np.zeros(4, np.int32)
        _check(lib().cl_debug_pass_info(self._h, _ptr(info), None, 0), "cl_debug_pass_info")
        segs = np.zeros((max(int(info[3]), 1), 4), np.int32)
        _check(lib().cl_debug_pass_info(self._h, _ptr(info), _ptr(segs), int(info[3])), "cl_debug_pass_info")
        return dict(path=self.PASS_PATHS[info[0]], attn=self.PASS_ATTN[info[1]], T=int(info[2]),
                    segs=[tuple(int(v) for v in g) for g in segs[:int(info[3])]])

    def debug_pass_rows(self, what: str, row0: int = 0, n: int = None) -> np.ndarray:
        """cl_debug_pass_rows: rows row0 .. row0 + n - 1 (n None: to the last row) of the latest multi-row pass after its
        last layer.  what: "h" (fp32 residual stream), "q" (roped), "attn", "act" (bf16 values as float32)."""
        i = ("h", "q", "attn", "act").index(what)
        if n is None:
            n = self.debug_pass_info()["T"] - row0
        w = self.cfg["d_model"] if i == 0 else self.cfg["d_ff"] if i == 3 else self.cfg["n_heads"] * self.cfg["head_dim"]
        out = np.empty((max(n, 0), w), np.float32)
        _check(lib().cl_debug_pass_rows(self._h, i, row0, n, _ptr(out) if n > 0 else None), "cl_debug_pass_rows")
        return out

    def runs_mega_kernel(self) -> bool:
        """Whether single-sequence steps of this engine run decode_mega_kernel (else the per-op kernels)."""
        m = C.c_int32(-1)
        _check(lib().cl_debug_seq_hidden(self._h, 0, 0, None, 0, C.byref(m)), "cl_debug_seq_hidden")
        return m.value == 1

    def debug_timeline(self) -> np.ndarray:
        n = (self.cfg["n_layers"] * 5 + 1) * 4
        out = np.zeros(n, np.int64)
        rc = lib().cl_debug_timeline(self._h, _ptr(out), n)
        if rc < 0:
            raise EngineError(rc, "cl_debug_timeline")
        return out.reshape(-1, 4)

    # ---- request level ---------------------------------------------------------------------------
    def generate_ids(self, prompt_ids, sampling: Sampling, stop=None, min_p=None, presence_penalty=None,
                     frequency_penalty=None) -> GenerateResult:
        """cl_generate_ids; with any of stop / min_p / presence_penalty / frequency_penalty, cl_generate_ids_ext."""
        ext = _ext_kwargs(stop, min_p, presence_penalty, frequency_penalty)
        if ext:
            return self.generate_ids_ext(prompt_ids, sampling, sampling_ext(**ext))[0]
        ids = np.ascontiguousarray(prompt_ids, dtype=np.int32)
        r = Result()
        _check(lib().cl_generate_ids(self._h, _ptr(ids), len(ids), C.byref(sampling), C.byref(r)), "cl_generate_ids")
        try:
            return GenerateResult(r)
        finally:
            lib().cl_result_free(C.byref(r))

    def generate_ids_ext(self, prompt_ids, sampling: Sampling, ext: SamplingExt | None, top_n: int = -1, on_text=None):
        """cl_generate_ids_ext: (GenerateResult, records or None).  on_text(text_delta: str, ids: list[int]) streams the
        text as cl_generate_stream does (a truthy return cancels); records: a TOKEN_LOGPROB array when top_n >= 0."""
        ids = np.ascontiguousarray(prompt_ids, dtype=np.int32)
        r = Result()
        lp = C.c_void_p()

        def cb(user, text, text_len, cids, n_ids):
            try:
                delta = C.string_at(text, text_len).decode("utf-8", "replace") if text_len else ""
                return 1 if on_text(delta, [cids[i] for i in range(n_ids)] if n_ids else []) else 0
            except Exception:       # never unwind through the C frames
                return 1

        cfn = TOKEN_CB(cb) if on_text else TOKEN_CB()
        _check(lib().cl_generate_ids_ext(self._h, _ptr(ids), len(ids), C.byref(sampling), C.byref(ext) if ext is not None else None,
                                         top_n, cfn, None, C.byref(r), C.byref(lp) if top_n >= 0 else None), "cl_generate_ids_ext")
        try:
            res = GenerateResult(r)
            recs = np.frombuffer(C.string_at(lp, res.n_generated * TOKEN_LOGPROB.itemsize), TOKEN_LOGPROB).copy() if top_n >= 0 else None
            return res, recs
        finally:
            lib().cl_result_free(C.byref(r))
            if top_n >= 0:
                lib().cl_buffer_free(lp)

    def _generate_wire(self, model: str, prompt: str, sampling: Sampling | None, ext: dict, on_text=None) -> GenerateResult:
        """generate / generate_stream with Ollama's stop, min_p or penalties: the request goes through cl_handle_message[_stream]
        with every cl_sampling field as an explicit option, so the chat template and the stop rule are libclengine's."""
        from .pb import BaseMessage, GenerateOptions, GenerateRequest
        s = sampling if sampling is not None else ollama_default_sampling(seed=time.time_ns() & 0xFFFFFFFF)
        opts = GenerateOptions(seed=s.seed, temperature=s.temperature, top_k=s.top_k, top_p=s.top_p, repeat_penalty=s.repeat_penalty,
                               repeat_last_n=s.repeat_last_n, num_predict=s.max_new_tokens, **ext)
        req = BaseMessage(generate_request=GenerateRequest(model=model, prompt=prompt, stream=on_text is not None, options=opts)).encode()
        if on_text is None:
            g = BaseMessage.decode(self.handle_message(req)).generate_response
            return GenerateResult.from_response(g.response, g.done_reason)
        last = {}

        def on_frame(msg):
            g = BaseMessage.decode(msg).generate_response
            if g.done:
                last["g"] = g
            return bool(g.response) and bool(on_text(g.response, []))

        self.handle_message_stream(req, None, on_frame)
        return GenerateResult.from_response("", last["g"].done_reason)

    def generate_ids_logprobs(self, prompt_ids, sampling: Sampling, top_n: int):
        """cl_generate_ids_logprobs: (GenerateResult, records), records a TOKEN_LOGPROB array with one entry per generated id."""
        ids = np.ascontiguousarray(prompt_ids, dtype=np.int32)
        r = Result()
        lp = C.c_void_p()
        _check(lib().cl_generate_ids_logprobs(self._h, _ptr(ids), len(ids), C.byref(sampling), top_n, C.byref(r), C.byref(lp)),
               "cl_generate_ids_logprobs")
        try:
            res = GenerateResult(r)
            recs = np.frombuffer(C.string_at(lp, res.n_generated * TOKEN_LOGPROB.itemsize), TOKEN_LOGPROB).copy()
            return res, recs
        finally:
            lib().cl_result_free(C.byref(r))
            lib().cl_buffer_free(lp)

    def generate(self, model: str, prompt: str, sampling: Sampling | None = None, stop=None, min_p=None, presence_penalty=None,
                 frequency_penalty=None) -> GenerateResult:
        """cl_generate.  With stop / min_p / presence_penalty / frequency_penalty the request goes over the byte-level
        handler (_generate_wire): the result then has text and done_reason only."""
        ext = _ext_kwargs(stop, min_p, presence_penalty, frequency_penalty)
        if ext:
            return self._generate_wire(model, prompt, sampling, ext)
        r = Result()
        p = prompt.encode("utf-8")
        _check(lib().cl_generate(self._h, model.encode(), p, len(p), C.byref(sampling) if sampling else None,
                                 C.byref(r)), "cl_generate")
        try:
            return GenerateResult(r)
        finally:
            lib().cl_result_free(C.byref(r))

    def generate_stream(self, model: str, prompt: str, sampling: Sampling | None = None, on_text=None, stop=None, min_p=None,
                        presence_penalty=None, frequency_penalty=None) -> GenerateResult:
        """cl_generate_stream: on_text(text_delta: str, ids: list[int]) is called on this thread as tokens arrive;
        a truthy return cancels the request.  With stop / min_p / presence_penalty / frequency_penalty the request goes over
        the byte-level handler (_generate_wire): ids are then [] and the result has done_reason only."""
        ext = _ext_kwargs(stop, min_p, presence_penalty, frequency_penalty)
        if ext:
            return self._generate_wire(model, prompt, sampling, ext, on_text or (lambda d, i: False))
        r = Result()
        p = prompt.encode("utf-8")

        def cb(user, text, text_len, ids, n_ids):
            try:
                delta = C.string_at(text, text_len).decode("utf-8", "replace") if text_len else ""
                new = [ids[i] for i in range(n_ids)] if n_ids else []
                return 1 if (on_text and on_text(delta, new)) else 0
            except Exception:       # never unwind through the C frames
                return 1

        cfn = TOKEN_CB(cb)
        _check(lib().cl_generate_stream(self._h, model.encode(), p, len(p), C.byref(sampling) if sampling else None, cfn, None,
                                        C.byref(r)), "cl_generate_stream")
        try:
            return GenerateResult(r)
        finally:
            lib().cl_result_free(C.byref(r))

    def handle_message_stream(self, req: bytes, sampling: Sampling | None = None, on_frame=None) -> int:
        """cl_handle_message_stream: on_frame(serialised BaseMessage) per response frame; returns the frame count."""
        n = [0]

        def cb(user, msg, length):
            try:
                n[0] += 1
                return 1 if (on_frame and on_frame(C.string_at(msg, length))) else 0
            except Exception:
                return 1

        cfn = FRAME_CB(cb)
        _check(lib().cl_handle_message_stream(self._h, req, len(req), C.byref(sampling) if sampling else None, cfn, None),
               "cl_handle_message_stream")
        return n[0]

    def handle_message(self, req: bytes, sampling: Sampling | None = None) -> bytes:
        out, n = C.c_void_p(), C.c_size_t()
        _check(lib().cl_handle_message(self._h, req, len(req), C.byref(sampling) if sampling else None,
                                       C.byref(out), C.byref(n)), "cl_handle_message")
        try:
            return C.string_at(out, n.value)
        finally:
            lib().cl_buffer_free(out)

    def load_tokenizer(self, tokenizer_json_path: str, chat_family: str | None = None) -> None:
        """Replace the byte-level fallback by an HF tokenizer.json (cl_engine_load_tokenizer)."""
        _check(lib().cl_engine_load_tokenizer(self._h, str(tokenizer_json_path).encode(), chat_family.encode() if chat_family else None),
               "cl_engine_load_tokenizer")

    def tokenize(self, text: str) -> np.ndarray:
        b = text.encode("utf-8")
        n = C.c_int32()
        _check(lib().cl_tokenize(self._h, b, len(b), None, 0, C.byref(n)), "cl_tokenize")
        ids = np.empty(n.value, np.int32)
        _check(lib().cl_tokenize(self._h, b, len(b), _ptr(ids), n.value, C.byref(n)), "cl_tokenize")
        return ids

    def detokenize(self, ids) -> str:
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        n = C.c_size_t()
        _check(lib().cl_detokenize(self._h, _ptr(ids), len(ids), None, 0, C.byref(n)), "cl_detokenize")
        buf = C.create_string_buffer(n.value + 1)
        _check(lib().cl_detokenize(self._h, _ptr(ids), len(ids), buf, n.value + 1, C.byref(n)), "cl_detokenize")
        return buf.value.decode("utf-8", errors="replace")

    def stats(self) -> dict:
        st = Stats()
        _check(lib().cl_engine_stats(self._h, C.byref(st)), "cl_engine_stats")
        d = {n: getattr(st, n) for n, _ in st._fields_}
        d["gpu_model"] = st.gpu_model.decode(errors="replace")
        return d

    def spec_stats(self) -> dict:
        """cl_engine_spec_stats: enabled, max_draft, verify_passes, tokens_drafted, tokens_accepted, tokens_emitted."""
        st = SpecStats()
        _check(lib().cl_engine_spec_stats(self._h, C.byref(st)), "cl_engine_spec_stats")
        return {n: getattr(st, n) for n, _ in st._fields_ if n not in ("reserved", "multi_passes")}

    def draft_stats(self) -> dict:
        """cl_spec_stats.draft_rows, draft_ns, draft_pages_used (the struct's last three fields; all zero without a draft)."""
        st = SpecStats()
        _check(lib().cl_engine_spec_stats(self._h, C.byref(st)), "cl_engine_spec_stats")
        return dict(zip(("draft_rows", "draft_ns", "draft_pages_used"), st.reserved))

    def spec_multi_passes(self) -> int:
        """cl_spec_stats.multi_passes: verify passes that checked two or more sequences at once."""
        st = SpecStats()
        _check(lib().cl_engine_spec_stats(self._h, C.byref(st)), "cl_engine_spec_stats")
        return st.multi_passes

    def prefix_stats(self, host: bool = False) -> dict:
        """cl_engine_prefix_stats: enabled, cached_pages, lookups, tokens_looked_up, tokens_reused, pages_evicted; with
        host=True also the host tier's host_pages, host_pages_cached, pages_to_host and pages_from_host."""
        st = PrefixStats()
        _check(lib().cl_engine_prefix_stats(self._h, C.byref(st)), "cl_engine_prefix_stats")
        return {n: getattr(st, n) for n, _ in st._fields_[:None if host else 6]}


# ---- single-op wrappers (host numpy in / out) -----------------------------------------------------
def op_gemv(w_bf16, x, variant=0, iters=0, device=0):
    w = np.ascontiguousarray(w_bf16, dtype=np.uint16)
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.empty(w.shape[0], np.float32)
    ms = C.c_float(0)
    _check(lib().cl_op_gemv(device, variant, _ptr(w), _ptr(x), _ptr(y), w.shape[0], w.shape[1], iters, C.byref(ms)),
           "cl_op_gemv")
    return (y, ms.value) if iters else y


def op_gemv_residual(w_bf16, x, resid, variant=0, device=0):
    w = np.ascontiguousarray(w_bf16, dtype=np.uint16)
    x = np.ascontiguousarray(x, dtype=np.float32)
    r = np.ascontiguousarray(resid, dtype=np.float32)
    y = np.empty(w.shape[0], np.float32)
    _check(lib().cl_op_gemv_residual(device, variant, _ptr(w), _ptr(x), _ptr(r), _ptr(y), w.shape[0], w.shape[1]),
           "cl_op_gemv_residual")
    return y


def op_rmsnorm_gemv(w_bf16, h, gain, eps, variant=0, device=0):
    w = np.ascontiguousarray(w_bf16, dtype=np.uint16)
    h = np.ascontiguousarray(h, dtype=np.float32)
    g = np.ascontiguousarray(gain, dtype=np.float32)
    y = np.empty(w.shape[0], np.float32)
    _check(lib().cl_op_rmsnorm_gemv(device, variant, _ptr(w), _ptr(h), _ptr(g), eps, _ptr(y), w.shape[0], w.shape[1]),
           "cl_op_rmsnorm_gemv")
    return y


def op_rmsnorm_gateup(w_gu_bf16, h, gain, eps, variant=0, device=0):
    w = np.ascontiguousarray(w_gu_bf16, dtype=np.uint16)
    h = np.ascontiguousarray(h, dtype=np.float32)
    g = np.ascontiguousarray(gain, dtype=np.float32)
    act = np.empty(w.shape[0] // 2, np.float32)
    _check(lib().cl_op_rmsnorm_gateup(device, variant, _ptr(w), _ptr(h), _ptr(g), eps, _ptr(act), w.shape[0] // 2,
                                      w.shape[1]), "cl_op_rmsnorm_gateup")
    return act


def op_attn_decode(q_roped, k_cache_bf16, v_cache_bf16, n_heads, n_kv, head_dim, page_size=32, device=0):
    q = np.ascontiguousarray(q_roped, dtype=np.float32)
    kc = np.ascontiguousarray(k_cache_bf16, dtype=np.uint16)
    vc = np.ascontiguousarray(v_cache_bf16, dtype=np.uint16)
    out = np.empty(n_heads * head_dim, np.float32)
    _check(lib().cl_op_attn_decode(device, _ptr(q), _ptr(kc), _ptr(vc), kc.shape[0], n_heads, n_kv, head_dim, page_size,
                                   _ptr(out)), "cl_op_attn_decode")
    return out


def op_attn_decode_batch(q, k_cache_bf16, v_cache_bf16, ctx_lens, n_heads, n_kv, head_dim, page_size=32, slots=None, n_slots=None,
                         out_init=None, variant=-1, nsplit=0, tc_small=-1, with_bf16=True, device=0):
    """cl_op_attn_decode_batch: decode attention of the batched step.  q [B][H*D] fp32; k/v caches [sum(ctx_lens)][n_kv][D] bf16,
    the sequences back to back.  Returns (out [n_slots][H*D] fp32 (starts as out_init, NaN when None), out_bf16 [B][H*D] uint16
    or None, nsplit used, tc_small used (-1: the CUDA-core kernel ran))."""
    q = np.ascontiguousarray(q, dtype=np.float32)
    kc = np.ascontiguousarray(k_cache_bf16, dtype=np.uint16)
    vc = np.ascontiguousarray(v_cache_bf16, dtype=np.uint16)
    lens = np.ascontiguousarray(ctx_lens, dtype=np.int32)
    B = len(lens)
    n_slots = n_slots or B
    sl = None if slots is None else np.ascontiguousarray(slots, dtype=np.int32)
    out = np.full((n_slots, n_heads * head_dim), np.nan, np.float32) if out_init is None else \
        np.array(out_init, dtype=np.float32, order="C", copy=True)
    ob = np.empty((B, n_heads * head_dim), np.uint16) if with_bf16 else None
    ns, small = C.c_int32(), C.c_int32()
    _check(lib().cl_op_attn_decode_batch(device, variant, nsplit, tc_small, _ptr(q), _ptr(kc), _ptr(vc), _ptr(lens),
                                         None if sl is None else _ptr(sl), B, n_slots, n_heads, n_kv, head_dim, page_size, _ptr(out),
                                         None if ob is None else _ptr(ob), C.byref(ns), C.byref(small)), "cl_op_attn_decode_batch")
    return out, ob, ns.value, small.value


def op_attn_verify(q_bf16, k_cache_bf16, v_cache_bf16, ctx_lens, rows, n_heads, n_kv, head_dim, page_size=32, nsplit=0, device=0):
    """cl_op_attn_verify: the multi-row split-KV attention of a verify pass.  q [sum(rows)][H*D] bf16; k/v caches
    [sum(ctx_lens + rows)][n_kv][D] bf16, the segments back to back.  Returns (out [sum(rows)][H*D] bf16 as uint16, splits)."""
    q = np.ascontiguousarray(q_bf16, dtype=np.uint16)
    kc = np.ascontiguousarray(k_cache_bf16, dtype=np.uint16)
    vc = np.ascontiguousarray(v_cache_bf16, dtype=np.uint16)
    lens = np.ascontiguousarray(ctx_lens, dtype=np.int32)
    rw = np.ascontiguousarray(rows, dtype=np.int32)
    out = np.empty((int(rw.sum()), n_heads * head_dim), np.uint16)
    ns = C.c_int32()
    _check(lib().cl_op_attn_verify(device, _ptr(q), _ptr(kc), _ptr(vc), _ptr(lens), _ptr(rw), len(lens), n_heads, n_kv, head_dim,
                                   page_size, nsplit, _ptr(out), C.byref(ns)), "cl_op_attn_verify")
    return out, ns.value


def op_qkv_rope_append(w_qkv_bf16, h, gain, eps, n_heads, n_kv, head_dim, pos, rope_theta, variant=0, device=0):
    w = np.ascontiguousarray(w_qkv_bf16, dtype=np.uint16)
    h = np.ascontiguousarray(h, dtype=np.float32)
    g = np.ascontiguousarray(gain, dtype=np.float32)
    q = np.empty(n_heads * head_dim, np.float32)
    k = np.empty(n_kv * head_dim, np.uint16)
    v = np.empty(n_kv * head_dim, np.uint16)
    _check(lib().cl_op_qkv_rope_append(device, variant, _ptr(w), _ptr(h), _ptr(g), eps, w.shape[1], n_heads, n_kv, head_dim, pos,
                                       rope_theta, _ptr(q), _ptr(k), _ptr(v)), "cl_op_qkv_rope_append")
    return q, k, v


def op_gemm_bf16(x_bf16, w_bf16, iters=0, device=0):
    x = np.ascontiguousarray(x_bf16, dtype=np.uint16)
    w = np.ascontiguousarray(w_bf16, dtype=np.uint16)
    y = np.empty((x.shape[0], w.shape[0]), np.float32)
    ms = C.c_float(0)
    _check(lib().cl_op_gemm_bf16(device, _ptr(x), _ptr(w), _ptr(y), x.shape[0], w.shape[0], w.shape[1], iters,
                                 C.byref(ms)), "cl_op_gemm_bf16")
    return (y, ms.value) if iters else y


def op_gemm_bf16_epi(x_bf16, w_bf16, epi=0, k_splits=0, pdl=False, resid=None, device=0):
    """cl_op_gemm_bf16_epi.  epi 0: (partials [k_splits][T][N] fp32, k_splits used); epi 1: (resid + X W^T [T][N] fp32, 1);
    epi 2: (bf16(silu(gate) * up) [T][N/2] as uint16, 1) of interleaved gate|up rows of W."""
    x = np.ascontiguousarray(x_bf16, dtype=np.uint16)
    w = np.ascontiguousarray(w_bf16, dtype=np.uint16)
    t, n, k = x.shape[0], w.shape[0], w.shape[1]
    ks = C.c_int32()
    L = lib()
    if epi == 0:
        _check(L.cl_op_gemm_bf16_epi(device, 0, k_splits, int(pdl), _ptr(x), _ptr(w), None, None, None, t, n, k, C.byref(ks)),
               "cl_op_gemm_bf16_epi")
        y, act, r = np.empty((ks.value, t, n), np.float32), None, None
    elif epi == 1:
        r = np.ascontiguousarray(resid, dtype=np.float32)
        y, act = np.empty((t, n), np.float32), None
    else:
        y, act, r = None, np.empty((t, n // 2), np.uint16), None
    _check(L.cl_op_gemm_bf16_epi(device, epi, k_splits, int(pdl), _ptr(x), _ptr(w), None if r is None else _ptr(r),
                                 None if y is None else _ptr(y), None if act is None else _ptr(act), t, n, k, C.byref(ks)),
           "cl_op_gemm_bf16_epi")
    return (act if epi == 2 else y), ks.value


def op_attn_prefill_cached(q_bf16, k_bf16, v_bf16, pos0, n_heads, n_kv, head_dim, page_size=32, variant=-1, device=0):
    """cl_op_attn_prefill_cached: causal attention of q [T][H*D] (positions pos0 .. pos0+T-1) over k, v [pos0+T][n_kv][D]."""
    q = np.ascontiguousarray(q_bf16, dtype=np.uint16)
    k = np.ascontiguousarray(k_bf16, dtype=np.uint16)
    v = np.ascontiguousarray(v_bf16, dtype=np.uint16)
    t = q.shape[0]
    out = np.empty((t, n_heads * head_dim), np.float32)
    _check(lib().cl_op_attn_prefill_cached(device, variant, _ptr(q), _ptr(k), _ptr(v), pos0, t, n_heads, n_kv, head_dim, page_size,
                                           _ptr(out)), "cl_op_attn_prefill_cached")
    return out


def op_attn_prefill_long(q_bf16, k_bf16, v_bf16, pos0, n_heads, n_kv, head_dim, page_size=32, variant=2, nsplit=0, iters=0,
                         device=0):
    """cl_op_attn_prefill_long: cl_op_attn_prefill_cached with variant 2's split count (0: its plan, > 0: forced) and a
    timing loop.  Returns (out [T][H*D] fp32, splits used, kernel that ran: "mma" | "wgmma" | "long", ms per launch or None)."""
    q = np.ascontiguousarray(q_bf16, dtype=np.uint16)
    k = np.ascontiguousarray(k_bf16, dtype=np.uint16)
    v = np.ascontiguousarray(v_bf16, dtype=np.uint16)
    t = q.shape[0]
    out = np.empty((t, n_heads * head_dim), np.float32)
    ms, ns, kind = C.c_float(0.0), C.c_int32(0), C.c_int32(-1)
    _check(lib().cl_op_attn_prefill_long(device, variant, _ptr(q), _ptr(k), _ptr(v), pos0, t, n_heads, n_kv, head_dim, page_size,
                                         nsplit, iters, _ptr(out), C.byref(ms), C.byref(ns), C.byref(kind)), "cl_op_attn_prefill_long")
    return out, ns.value, Engine.PASS_ATTN[kind.value], (ms.value if iters > 0 else None)


def op_attn_prefill(q_bf16, k_bf16, v_bf16, n_heads, n_kv, head_dim, device=0):
    q = np.ascontiguousarray(q_bf16, dtype=np.uint16)
    k = np.ascontiguousarray(k_bf16, dtype=np.uint16)
    v = np.ascontiguousarray(v_bf16, dtype=np.uint16)
    t = q.shape[0]
    out = np.empty((t, n_heads * head_dim), np.float32)
    _check(lib().cl_op_attn_prefill(device, _ptr(q), _ptr(k), _ptr(v), t, n_heads, n_kv, head_dim, _ptr(out)),
           "cl_op_attn_prefill")
    return out


def op_attn_prefill_variant(q_bf16, k_bf16, v_bf16, n_heads, n_kv, head_dim, variant, iters=0, device=0):
    """variant 0: mma.sync kernel, 1: wgmma kernel, -1: auto.  Returns (out, ms per launch or None)."""
    q = np.ascontiguousarray(q_bf16, dtype=np.uint16)
    k = np.ascontiguousarray(k_bf16, dtype=np.uint16)
    v = np.ascontiguousarray(v_bf16, dtype=np.uint16)
    t = q.shape[0]
    out = np.empty((t, n_heads * head_dim), np.float32)
    ms = C.c_float(0)
    _check(lib().cl_op_attn_prefill_variant(device, variant, _ptr(q), _ptr(k), _ptr(v), t, n_heads, n_kv, head_dim, _ptr(out), iters,
                                            C.byref(ms)), "cl_op_attn_prefill_variant")
    return out, (ms.value if iters > 0 else None)


def op_sample(logits, samplings, histories, steps, device=0):
    """cl_op_sample: the step tail's device sampler on host logits [n_rows][vocab]; row r draws with samplings[r], history
    histories[r] (a sequence of ids) at RNG step steps[r].  Returns the ids [n_rows]."""
    lg = np.ascontiguousarray(np.atleast_2d(logits), dtype=np.float32)
    rows = lg.shape[0]
    stride = max(1, max(len(h) for h in histories))
    hist = np.zeros((rows, stride), np.int32)
    for r, h in enumerate(histories):
        hist[r, :len(h)] = np.asarray(h, np.int32)
    nh = np.ascontiguousarray([len(h) for h in histories], dtype=np.int32)
    st = np.ascontiguousarray(steps, dtype=np.uint64)
    sp = (Sampling * rows)(*samplings)
    out = np.empty(rows, np.int32)
    _check(lib().cl_op_sample(device, _ptr(lg), rows, lg.shape[1], sp, _ptr(hist), _ptr(nh), stride, _ptr(st), _ptr(out)),
           "cl_op_sample")
    return out


def op_sample_ext(logits, samplings, exts, histories, steps, device=0):
    """cl_op_sample_ext: op_sample where row r also applies exts[r] (a SamplingExt, or None for all zero)."""
    lg = np.ascontiguousarray(np.atleast_2d(logits), dtype=np.float32)
    rows = lg.shape[0]
    stride = max(1, max(len(h) for h in histories))
    hist = np.zeros((rows, stride), np.int32)
    for r, h in enumerate(histories):
        hist[r, :len(h)] = np.asarray(h, np.int32)
    nh = np.ascontiguousarray([len(h) for h in histories], dtype=np.int32)
    st = np.ascontiguousarray(steps, dtype=np.uint64)
    sp = (Sampling * rows)(*samplings)
    xs = (SamplingExt * rows)(*[x if x is not None else SamplingExt() for x in exts])
    out = np.empty(rows, np.int32)
    _check(lib().cl_op_sample_ext(device, _ptr(lg), rows, lg.shape[1], sp, xs, _ptr(hist), _ptr(nh), stride, _ptr(st), _ptr(out)),
           "cl_op_sample_ext")
    return out


def op_sample_logprobs(logits, samplings, histories, steps, top_n, device=0):
    """cl_op_sample_logprobs: op_sample with every row's logprobs on (a row with temperature <= 0 takes the greedy choice).
    Returns (ids [n_rows], records: a TOKEN_LOGPROB array [n_rows])."""
    lg = np.ascontiguousarray(np.atleast_2d(logits), dtype=np.float32)
    rows = lg.shape[0]
    stride = max(1, max(len(h) for h in histories))
    hist = np.zeros((rows, stride), np.int32)
    for r, h in enumerate(histories):
        hist[r, :len(h)] = np.asarray(h, np.int32)
    nh = np.ascontiguousarray([len(h) for h in histories], dtype=np.int32)
    st = np.ascontiguousarray(steps, dtype=np.uint64)
    sp = (Sampling * rows)(*samplings)
    out = np.empty(rows, np.int32)
    recs = np.zeros(rows, TOKEN_LOGPROB)
    _check(lib().cl_op_sample_logprobs(device, _ptr(lg), rows, lg.shape[1], sp, _ptr(hist), _ptr(nh), stride, _ptr(st), top_n,
                                       _ptr(out), recs.ctypes.data), "cl_op_sample_logprobs")
    return out, recs


def op_kv_host_roundtrip(n_layers, n_kv, head_dim, page_size, n_moves, iters=0, device=0):
    """cl_op_kv_host_roundtrip: spill n_moves pages of a scrambled pool to host pages and fill them into other pages; raises
    unless the round trip is bit-exact and no other page changed.  Returns (spill ms, fill ms) per launch over `iters` timed
    launches of each, or None when iters is 0."""
    ms = (C.c_float * 2)()
    _check(lib().cl_op_kv_host_roundtrip(device, n_layers, n_kv, head_dim, page_size, n_moves, iters, ms if iters else None),
           "cl_op_kv_host_roundtrip")
    return (ms[0], ms[1]) if iters else None


def op_kv_shift(k, v, page_size, n_keep, n_discard, rope_row, iters=0, device=0):
    """cl_op_kv_shift: k, v uint16 (bf16) [n_layers][len][n_kv][head_dim] paged into a scattered pool, shifted by one
    kv_shift_kernel launch with rope_row [head_dim / 2][2] (cos, sin); raises if anything outside the sequence's rows changed.
    Returns (k_out, v_out) [n_layers][len - n_discard][n_kv][head_dim], and the ms of one launch over `iters` timed launches
    (None when iters is 0)."""
    k = np.ascontiguousarray(k, dtype=np.uint16)
    v = np.ascontiguousarray(v, dtype=np.uint16)
    L, T, KV, D = k.shape
    cs = np.ascontiguousarray(rope_row, dtype=np.float32)
    ko = np.zeros((L, max(T - n_discard, 0), KV, D), np.uint16)
    vo = np.zeros_like(ko)
    ms = C.c_float(0.0)
    _check(lib().cl_op_kv_shift(device, L, KV, D, page_size, T, n_keep, n_discard, _ptr(cs), _ptr(k), _ptr(v), _ptr(ko), _ptr(vo),
                                iters, C.byref(ms) if iters else None), "cl_op_kv_shift")
    return ko, vo, (ms.value if iters else None)


def op_synth_weights(seed, key, n, scale, device=0):
    out = np.empty(n, np.uint16)
    _check(lib().cl_op_synth_weights(device, seed, key, n, scale, _ptr(out)), "cl_op_synth_weights")
    return out


class HfTokenizer:
    """Native tokenizer.json loader (csrc/tokenizer.cpp) — host logic, works without a GPU."""

    def __init__(self, tokenizer_json_path, chat_family: str | None = None):
        h = C.c_void_p()
        _check(lib().cl_tokenizer_load(str(tokenizer_json_path).encode(), chat_family.encode() if chat_family else None, C.byref(h)),
               "cl_tokenizer_load")
        self._h = h
        v, b, e = C.c_int32(), C.c_int32(), C.c_int32()
        _check(lib().cl_tokenizer_info(self._h, C.byref(v), C.byref(b), C.byref(e)), "cl_tokenizer_info")
        self.vocab_size, self.bos, self.eos = v.value, b.value, e.value

    def encode(self, text: str, add_bos: bool = False, chat: bool = False) -> list:
        b = text.encode("utf-8")
        n = C.c_int32()
        _check(lib().cl_tokenizer_encode(self._h, b, len(b), int(add_bos), int(chat), None, 0, C.byref(n)), "cl_tokenizer_encode")
        ids = np.zeros(max(n.value, 1), np.int32)
        _check(lib().cl_tokenizer_encode(self._h, b, len(b), int(add_bos), int(chat), _ptr(ids), n.value, C.byref(n)), "cl_tokenizer_encode")
        return ids[:n.value].tolist()

    def decode(self, ids) -> str:
        a = np.ascontiguousarray(ids, dtype=np.int32)
        n = C.c_size_t()
        _check(lib().cl_tokenizer_decode(self._h, _ptr(a), len(a), None, 0, C.byref(n)), "cl_tokenizer_decode")
        buf = C.create_string_buffer(n.value + 1)
        _check(lib().cl_tokenizer_decode(self._h, _ptr(a), len(a), buf, n.value, C.byref(n)), "cl_tokenizer_decode")
        return buf.raw[:n.value].decode("utf-8", errors="replace")

    def close(self):
        if getattr(self, "_h", None):
            lib().cl_tokenizer_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class KvPool:
    """Host-side paged-KV allocator (usable without a GPU)."""

    def __init__(self, n_pages: int, page_size: int):
        h = C.c_void_p()
        _check(lib().cl_kvpool_create(n_pages, page_size, C.byref(h)), "cl_kvpool_create")
        self._h = h

    def close(self):
        if self._h:
            lib().cl_kvpool_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reserve(self, owner: int, n_tokens: int) -> int:
        return lib().cl_kvpool_reserve(self._h, owner, n_tokens)

    def release(self, owner: int) -> int:
        return lib().cl_kvpool_release(self._h, owner)

    def pages_of(self, owner: int):
        n = C.c_int32()
        lib().cl_kvpool_pages_of(self._h, owner, None, 0, C.byref(n))
        a = np.empty(max(n.value, 1), np.int32)
        _check(lib().cl_kvpool_pages_of(self._h, owner, _ptr(a), a.size, C.byref(n)), "cl_kvpool_pages_of")
        return a[:n.value].tolist()

    @property
    def free_pages(self) -> int:
        return lib().cl_kvpool_free_pages(self._h)

    @property
    def used_pages(self) -> int:
        return lib().cl_kvpool_used_pages(self._h)

    def attach(self, owner: int, ids) -> int:
        """Take the longest published page chain matching ids (owner must hold no pages); returns the tokens reused."""
        a = np.ascontiguousarray(ids, dtype=np.int32)
        n = C.c_int32(0)
        _check(lib().cl_kvpool_attach(self._h, owner, _ptr(a), len(a), C.byref(n)), "cl_kvpool_attach")
        return n.value

    def publish(self, owner: int, ids, n_known: int | None = None) -> int:
        """Index the owner's full pages covering ids[:n_known] (default: all of ids)."""
        a = np.ascontiguousarray(ids, dtype=np.int32)
        return lib().cl_kvpool_publish(self._h, owner, _ptr(a), len(a) if n_known is None else min(n_known, len(a)))

    @property
    def cached_pages(self) -> int:
        return lib().cl_kvpool_cached_pages(self._h)

    def set_host_pages(self, n: int):
        """Host tier of n pages (0: off); drops every entry it held."""
        _check(lib().cl_kvpool_set_host_pages(self._h, n), "cl_kvpool_set_host_pages")

    def take_moves(self):
        """The spills (kind 0) and fills (kind 1) recorded since the last call, in order: a list of (kind, device page,
        host page)."""
        n = C.c_int32()
        _check(lib().cl_kvpool_take_moves(self._h, None, 0, C.byref(n)), "cl_kvpool_take_moves")
        a = np.empty((max(n.value, 1), 3), np.int32)
        _check(lib().cl_kvpool_take_moves(self._h, _ptr(a), n.value, C.byref(n)), "cl_kvpool_take_moves")
        return [tuple(int(x) for x in r) for r in a[:n.value]]

    @property
    def host_cached_pages(self) -> int:
        return lib().cl_kvpool_host_cached_pages(self._h)

    def shift(self, owner: int, length: int, n_keep: int, n_discard: int):
        """Context shift of an owner holding `length` tokens (cl_kvpool_shift): returns (status, work items as a list of
        (source page, destination page, first row, end row, rotate))."""
        cap = len(self.pages_of(owner)) + 1
        a = np.zeros((cap, 5), np.int32)
        n = C.c_int32(0)
        rc = lib().cl_kvpool_shift(self._h, owner, length, n_keep, n_discard, _ptr(a), cap, C.byref(n))
        return rc, [tuple(int(x) for x in r) for r in a[:n.value]] if rc == 0 else []
