"""ctypes binding of libb200engine.so (include/b200engine.h).  No compute lives in Python."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_LIB = None
LIB_PATH = Path(__file__).resolve().parent / "lib" / "libb200engine.so"
MAX_SPEC_TOKENS = 3   # B200_MAX_SPEC_TOKENS


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200engine error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [
        ("device", C.c_int32),
        ("num_layers", C.c_int32), ("hidden", C.c_int32), ("q_heads", C.c_int32), ("kv_heads", C.c_int32),
        ("intermediate", C.c_int32), ("vocab", C.c_int32),
        ("rms_eps", C.c_float), ("rope_theta", C.c_float),
        ("max_model_len", C.c_int32), ("max_num_seqs", C.c_int32), ("max_batched_tokens", C.c_int32),
        ("num_kv_blocks", C.c_int64), ("kv_fraction", C.c_float),
        ("enable_prefix_caching", C.c_int32), ("eos_token_id", C.c_int32),
        ("seed", C.c_uint64), ("init_scale", C.c_float),
        ("manual_step", C.c_int32), ("record_steps", C.c_int32),
        ("rope_scaling_type", C.c_int32), ("rope_factor", C.c_float), ("rope_low_freq_factor", C.c_float),
        ("rope_high_freq_factor", C.c_float), ("rope_original_max_pos", C.c_int32),
        ("num_speculative_tokens", C.c_int32), ("prompt_lookup_min", C.c_int32), ("prompt_lookup_max", C.c_int32),
        ("head_dim", C.c_int32), ("runner", C.c_int32), ("sliding_window", C.c_int32),
        ("num_labels", C.c_int32), ("score_activation", C.c_int32), ("score_join_pair", C.c_int32),
    ]


class Gemm3Args(C.Structure):
    _fields_ = [("N", C.c_int32), ("T", C.c_int32), ("K", C.c_int32), ("x_rows", C.c_int32),
                ("pro", C.c_int32), ("epi", C.c_int32), ("force", C.c_int32),
                ("w", C.c_void_p), ("x", C.c_void_p), ("ssq_in", C.c_void_p), ("ssq_slabs", C.c_int32),
                ("norm_w", C.c_void_p), ("eps", C.c_float), ("out", C.c_void_p), ("ldo", C.c_int32),
                ("ssq_out", C.c_void_p), ("positions", C.c_void_p), ("slots", C.c_void_p), ("cos_sin", C.c_void_p),
                ("kv_layer", C.c_void_p), ("q_heads", C.c_int32), ("kv_heads", C.c_int32), ("max_pos", C.c_int32),
                ("argmax_out", C.c_void_p), ("n_valid", C.c_int32), ("normed_out", C.c_void_p), ("norm_w_out", C.c_void_p),
                ("head_dim", C.c_int32)]


class Sampling(C.Structure):
    _fields_ = [("max_tokens", C.c_int32), ("temperature", C.c_float), ("ignore_eos", C.c_int32),
                ("num_stop_ids", C.c_int32), ("stop_ids", C.POINTER(C.c_int32)),
                ("top_p", C.c_float), ("top_k", C.c_int32), ("has_seed", C.c_int32), ("seed", C.c_uint64),
                ("logprobs", C.c_int32), ("top_logprobs", C.c_int32),
                ("presence_penalty", C.c_float), ("frequency_penalty", C.c_float), ("repetition_penalty", C.c_float),
                ("min_p", C.c_float), ("min_tokens", C.c_int32), ("num_logit_bias", C.c_int32),
                ("logit_bias_ids", C.POINTER(C.c_int32)), ("logit_bias_values", C.POINTER(C.c_float)),
                ("prompt_logprobs", C.c_int32), ("top_prompt_logprobs", C.c_int32)]


class SampleRow(C.Structure):
    _fields_ = [("temperature", C.c_float), ("top_k", C.c_int32), ("top_p", C.c_float),
                ("seed_lo", C.c_uint32), ("seed_hi", C.c_uint32), ("n", C.c_int32), ("min_p", C.c_float)]


class PenaltyRow(C.Structure):
    _fields_ = [("presence_penalty", C.c_float), ("frequency_penalty", C.c_float), ("repetition_penalty", C.c_float),
                ("min_tokens", C.c_int32), ("num_prompt", C.c_int32), ("prompt", C.POINTER(C.c_int32)),
                ("num_output", C.c_int32), ("output", C.POINTER(C.c_int32)), ("num_logit_bias", C.c_int32),
                ("logit_bias_ids", C.POINTER(C.c_int32)), ("logit_bias_values", C.POINTER(C.c_float)),
                ("num_stop_ids", C.c_int32), ("stop_ids", C.POINTER(C.c_int32))]


class Usage(C.Structure):
    _fields_ = [("prompt_tokens", C.c_int32), ("cached_tokens", C.c_int32), ("completion_tokens", C.c_int32)]


class Stats(C.Structure):
    _fields_ = [("steps", C.c_int64), ("running", C.c_int32), ("waiting", C.c_int32),
                ("kv_blocks_total", C.c_int64), ("kv_blocks_free", C.c_int64),
                ("prompt_tokens", C.c_int64), ("cached_prompt_tokens", C.c_int64), ("generated_tokens", C.c_int64),
                ("preemptions", C.c_int64), ("last_step_device_us", C.c_double), ("total_device_us", C.c_double),
                ("last_step_tokens", C.c_int64), ("kernel_launches", C.c_int64),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("spec_drafts", C.c_int64), ("spec_draft_tokens", C.c_int64), ("spec_accepted_tokens", C.c_int64),
                ("spec_accepted_per_pos", C.c_int64 * MAX_SPEC_TOKENS)]


class StepInfo(C.Structure):
    _fields_ = [("tokens", C.c_int32), ("decode_seqs", C.c_int32), ("prefill_seqs", C.c_int32),
                ("sampled", C.c_int32), ("kv_tokens_read", C.c_int64), ("device_us", C.c_double),
                ("draft_tokens", C.c_int32), ("accepted_tokens", C.c_int32)]


BEGIN_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_char_p)
WRITE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_char), C.c_size_t)


class ResponseWriter(C.Structure):
    _fields_ = [("ud", C.c_void_p), ("begin", BEGIN_FN), ("write", WRITE_FN)]


class ServerConfig(C.Structure):
    _fields_ = [("model", C.c_char_p), ("adapters", C.c_char_p), ("strategy", C.c_int32),
                ("mean_load_pct", C.c_int32), ("replication", C.c_int32), ("prefix_char_length", C.c_int32),
                ("max_retries", C.c_int32), ("default_max_tokens", C.c_int32), ("vocab", C.c_int32),
                ("max_model_len", C.c_int32), ("enable_sampling", C.c_int32), ("enable_logprobs", C.c_int32),
                ("enable_logits_processors", C.c_int32), ("enable_prompt_logprobs", C.c_int32), ("max_n", C.c_int32)]


class HarnessConfig(C.Structure):
    _fields_ = [("request_model", C.c_char_p), ("max_concurrent_threads", C.c_int32),
                ("max_completion_tokens", C.c_int32), ("temperature", C.c_float), ("thread_count", C.c_int32),
                ("seed", C.c_int64), ("request_timeout_s", C.c_double), ("synth_threads", C.c_int32),
                ("synth_mean_msgs", C.c_double), ("synth_mean_words", C.c_int32), ("vocab", C.c_int32)]


class HarnessResult(C.Structure):
    _fields_ = [("input_thread_count", C.c_int32), ("input_messages_per_thread_mean", C.c_double),
                ("duration_s", C.c_double), ("request_count", C.c_int32), ("failed_threads", C.c_int32),
                ("request_duration_mean_s", C.c_double), ("chunks_per_request_mean", C.c_double),
                ("run_output_throughput", C.c_double), ("run_total_throughput", C.c_double),
                ("ttft_mean_s", C.c_double), ("itl_mean_s", C.c_double),
                ("ttft_p50_s", C.c_double), ("ttft_p90_s", C.c_double), ("ttft_p99_s", C.c_double),
                ("itl_p50_s", C.c_double), ("itl_p99_s", C.c_double),
                ("prompt_tokens", C.c_int64), ("cached_prompt_tokens", C.c_int64),
                ("completion_tokens", C.c_int64), ("total_tokens", C.c_int64), ("first_error", C.c_char * 256)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_}
        d["first_error"] = d["first_error"].decode("utf-8", "replace")
        return d


# every symbol include/b200engine.h declares: name -> (restype, argtypes)
_vp, _i32, _i64, _u64, _f = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_float
_pi32 = C.POINTER(C.c_int32)
SYMBOLS = {
    "b200_last_error": (C.c_char_p, []),
    "b200_version": (C.c_char_p, []),
    "b200_config_default": (None, [C.POINTER(Config)]),
    "b200_engine_create": (C.c_int, [C.POINTER(Config), C.POINTER(_vp)]),
    "b200_engine_destroy": (None, [_vp]),
    "b200_submit": (C.c_int, [_vp, _pi32, _i32, C.POINTER(Sampling), C.POINTER(_u64)]),
    "b200_poll": (C.c_int, [_vp, _u64, _pi32, _i32, _pi32, _pi32, C.POINTER(Usage)]),
    "b200_poll_logprobs": (C.c_int, [_vp, _u64, _pi32, _vp, _pi32, _vp, _i32, _pi32, _pi32, C.POINTER(Usage)]),
    "b200_poll_prompt_logprobs": (C.c_int, [_vp, _u64, _vp, _pi32, _pi32, _vp, _i32, _pi32]),
    "b200_submit_embed": (C.c_int, [_vp, _pi32, _i32, _i32, C.POINTER(_u64)]),
    "b200_poll_embedding": (C.c_int, [_vp, _u64, _vp, _i32, _pi32, C.POINTER(Usage)]),
    "b200_submit_score": (C.c_int, [_vp, _pi32, _i32, _i32, C.POINTER(_u64)]),
    "b200_poll_score": (C.c_int, [_vp, _u64, _vp, _i32, _pi32, C.POINTER(Usage)]),
    "b200_submit_n": (C.c_int, [_vp, _pi32, _i32, C.POINTER(Sampling), _i32, C.POINTER(_u64)]),
    "b200_wait": (C.c_int, [_vp, _u64, _i64]),
    "b200_wait_any": (C.c_int, [_vp, C.POINTER(_u64), _i32, _i64]),
    "b200_abort": (C.c_int, [_vp, _u64]),
    "b200_release": (C.c_int, [_vp, _u64]),
    "b200_stats_get": (C.c_int, [_vp, C.POINTER(Stats)]),
    "b200_engine_is_failed": (C.c_int, [_vp]),
    "b200_engine_step": (C.c_int, [_vp, C.POINTER(StepInfo)]),
    "b200_engine_unfinished": (C.c_int32, [_vp]),
    "b200_engine_set_fixed_admission": (C.c_int, [_vp, _i32]),
    "b200_harness_expected_inflight": (C.c_int64, []),
    "b200_engine_run": (C.c_int, [_vp, _i32, _i64, C.POINTER(StepInfo), C.POINTER(_i32)]),
    "b200_engine_replay": (C.c_int, [_vp, _i32, _i32, C.POINTER(C.c_double), C.POINTER(_i64), C.POINTER(_i64),
                                      C.POINTER(_i64), C.POINTER(_i64)]),
    "b200_engine_reset_prefix_cache": (C.c_int, [_vp]),
    "b200_engine_set_skip_mask": (C.c_int, [_vp, C.c_uint32]),
    "b200_engine_set_recording": (C.c_int, [_vp, _i32]),
    "b200_engine_profile": (C.c_int, [_vp, _i32, C.POINTER(C.c_double), C.POINTER(_i64), _i32]),
    "b200_engine_profile_range": (C.c_int, [_vp, _i32, _i32, _i32, C.POINTER(C.c_double), C.POINTER(_i64), _i32,
                                            C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64)]),
    "b200_engine_tensor_info": (C.c_int, [_vp, C.c_char_p, C.POINTER(_u64), C.POINTER(_vp)]),
    "b200_engine_tensor_read": (C.c_int, [_vp, C.c_char_p, _vp, _u64]),
    "b200_engine_tensor_write": (C.c_int, [_vp, C.c_char_p, _vp, _u64]),
    "b200_engine_forward_logits": (C.c_int, [_vp, _pi32, _i32, _vp]),
    "b200_engine_set_keep_logits": (C.c_int, [_vp, _i32]),
    "b200_engine_read_logits": (C.c_int, [_vp, _vp, _i32]),
    "b200_config_from_hf": (C.c_int, [C.c_char_p, C.POINTER(Config)]),
    "b200_engine_load_safetensors": (C.c_int, [_vp, C.c_char_p]),
    "b200_safetensors_list": (C.c_int64, [C.c_char_p, C.c_char_p, C.c_size_t]),
    "b200_router_create": (C.c_int, [_i32, C.POINTER(_vp)]),
    "b200_router_destroy": (None, [_vp]),
    "b200_router_set_endpoints": (C.c_int, [_vp, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p),
                                             C.POINTER(C.c_char_p), _i32]),
    "b200_router_pick": (C.c_int, [_vp, _i32, C.c_char_p, C.c_char_p, _i32, _i32, _i64, C.c_char_p, _i32,
                                    C.POINTER(_u64)]),
    "b200_router_done": (C.c_int, [_vp, _u64]),
    "b200_router_add_inflight": (C.c_int, [_vp, C.c_char_p, _i64]),
    "b200_router_inflight": (C.c_int, [_vp, C.c_char_p, C.POINTER(_i64), C.POINTER(_i64)]),
    "b200_router_metrics": (C.c_int64, [_vp, C.c_char_p, C.c_size_t]),
    "b200_xxh64": (_u64, [_vp, C.c_size_t]),
    "b200_server_create": (C.c_int, [C.POINTER(ServerConfig), C.POINTER(_vp), _i32, C.POINTER(_vp)]),
    "b200_server_destroy": (None, [_vp]),
    "b200_server_handle": (C.c_int, [_vp, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t,
                                      C.POINTER(ResponseWriter)]),
    "b200_server_parse_request": (C.c_int, [_vp, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t, _i32, C.c_char_p,
                                            C.c_size_t]),
    "b200_server_listen": (C.c_int, [_vp, C.c_char_p, _i32, _pi32]),
    "b200_server_metrics": (C.c_int, [_vp, C.c_char_p, C.c_size_t]),
    "b200_speculative_config_parse": (C.c_int, [C.c_char_p, _vp]),
    "b200_server_inject_fault": (C.c_int, [_vp, _i32, _i32]),
    "b200_tokenize": (C.c_int, [_i32, C.c_char_p, C.c_size_t, _pi32, _i32]),
    "b200_detokenize": (C.c_int, [_i32, _pi32, _i32, C.c_char_p, C.c_size_t]),
    "b200_harness_config_default": (None, [C.POINTER(HarnessConfig)]),
    "b200_harness_synth_threads": (C.c_int64, [C.POINTER(HarnessConfig), C.c_char_p, C.c_size_t]),
    "b200_harness_run": (C.c_int, [_vp, C.c_char_p, _i32, C.POINTER(HarnessConfig), C.c_char_p, C.c_size_t,
                                    C.POINTER(HarnessResult)]),
    "b200_set_gemm_variant": (C.c_int, [_i32]),
    "b200_op_gemm_trace": (C.c_int, [_vp]),
    "b200_op_gemm_deferred": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "b200_op_gemm": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "b200_op_gemm3": (C.c_int, [C.POINTER(Gemm3Args), _vp, _pi32]),
    "b200_op_embed": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "b200_op_rmsnorm": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _f, _vp]),
    "b200_op_pool_rows": (C.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _f, _vp, _vp]),
    "b200_op_score_rows": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _f, _vp, _vp]),
    "b200_op_rope_kvwrite": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "b200_op_rope_kvwrite_hd": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b200_op_silu_mul": (C.c_int, [_vp, _vp, _i32, _i32, _vp]),
    "b200_op_silu_mul_il": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp]),
    "b200_op_argmax": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp]),
    "b200_op_sample": (C.c_int, [_vp, _i32, _vp, _i32, _i32, _vp, _vp]),
    "b200_op_penalize": (C.c_int, [_vp, _i32, _i32, _i32, C.POINTER(PenaltyRow), _vp, _vp]),
    "b200_op_penalty_list": (C.c_int, [C.POINTER(PenaltyRow), _i32, _vp, _vp, _i32, _i32, _i32, _vp]),
    "b200_op_penalize_update": (C.c_int, [_vp, _i32, _pi32, _i32, _i32, _vp, _vp, _i32, _i32, _vp]),
    "b200_op_penalize_slots": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _i32, _vp, _vp, _i32, _i32, _vp, _vp]),
    "b200_op_logprobs": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_op_logprobs_rank": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_op_paged_attn": (C.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _f, _i32, _vp]),
    "b200_op_paged_attn_hd": (C.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _f, _i32, _i32, _vp]),
    "b200_server_set_tokenizer": (C.c_int, [C.c_void_p, C.c_void_p]),
    "b200_server_render_prompt": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t, _vp, C.c_size_t]),
    "b200_tokenizer_load": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "b200_tokenizer_destroy": (None, [C.c_void_p]),
    "b200_tokenizer_vocab_size": (C.c_int32, [C.c_void_p]),
    "b200_tokenizer_token_id": (C.c_int32, [C.c_void_p, C.c_char_p]),
    "b200_tokenizer_encode": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_size_t, _i32, _vp, C.c_size_t]),
    "b200_tokenizer_decode": (C.c_int64, [C.c_void_p, _vp, C.c_size_t, _i32, C.c_char_p, C.c_size_t]),
    "b200_tokenizer_encode_pair": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, _i32, _i32, _vp,
                                               C.c_size_t]),
    "b200_tokenizer_stream_new": (C.c_void_p, [C.c_void_p, _i32]),
    "b200_tokenizer_stream_free": (None, [C.c_void_p]),
    "b200_tokenizer_stream_push": (C.c_int64, [C.c_void_p, _i32, C.c_char_p, C.c_size_t]),
    "b200_tokenizer_chat_llama3": (C.c_int64, [C.c_void_p, _vp, _vp, _i32, _i32, _vp, C.c_size_t]),
    "b200_schedule_query": (C.c_int, [_i32, _i32, _i32, _i32, _vp]),
    "b200_attn_split_query": (C.c_int, [_i32, _i32, _i32, _i32]),
    "b200_ngram_propose": (C.c_int32, [_pi32, _i32, _i32, _i32, _i32, _i32, _pi32]),
    "b200_op_paged_attn_decode_split": (C.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _f, _i32, _vp]),
    "b200_op_paged_attn_decode_split_hd": (C.c_int, [_vp, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _f, _i32,
                                                     _i32, _vp]),
    "b200_op_paged_attn_prefill_tc": (C.c_int, [_vp, _i32, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _f, _vp]),
    "b200_op_paged_attn_prefill_tc_hd": (C.c_int, [_vp, _i32, _i32, _vp, _i32, _vp, _vp, _i32, _vp, _i32, _i32, _i32, _f,
                                                   _i32, _vp]),
    "b200_op_init_uniform": (C.c_int, [_vp, _u64, C.c_uint32, _f, _f, _vp]),
    "b200_op_kv_copy_blocks": (C.c_int, [_vp, _i32, _i64, _i64, _vp, _vp, _i32, _vp]),
}


def lib() -> C.CDLL:
    """Load the engine library, building it in-tree first if it is missing.  Fails loudly."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not LIB_PATH.exists():
        from . import _build
        _build.build()
    if not LIB_PATH.exists():
        raise ImportError(f"{LIB_PATH} is missing and could not be built: the CUDA engine is required")
    l = C.CDLL(str(LIB_PATH), mode=os.RTLD_GLOBAL if hasattr(os, "RTLD_GLOBAL") else C.DEFAULT_MODE)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(l, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _LIB = l
    return l


def check(rc: int) -> int:
    if rc < 0:
        raise B200Error(rc, lib().b200_last_error().decode("utf-8", "replace"))
    return rc
