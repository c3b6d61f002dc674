"""Python driver for the engine part of the C ABI (tests, bench, smoke).  Mirrors the calls a cgo
shim would make (INTEGRATION.md); holds no model logic."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._lib import Config, Sampling, Stats, StepInfo, Usage, check, lib

FINISH = {0: None, 1: "stop", 2: "length", 3: "aborted", 4: "error"}
MAX_LOGPROBS = 20   # B200_MAX_LOGPROBS
_PI32 = C.POINTER(C.c_int32)


def default_config(**kw) -> Config:
    cfg = Config()
    lib().b200_config_default(C.byref(cfg))
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise AttributeError(k)
        setattr(cfg, k, v)
    return cfg


def config_from_hf(model_dir: str, **kw) -> Config:
    """Engine config whose architecture comes from an HF config.json (SURVEY.md §8f-2)."""
    cfg = default_config(**kw)
    check(lib().b200_config_from_hf(str(model_dir).encode(), C.byref(cfg)))
    return cfg


def safetensors_list(path: str) -> dict:
    import json
    n = check(lib().b200_safetensors_list(str(path).encode(), None, 0))
    buf = C.create_string_buffer(n + 1)
    lib().b200_safetensors_list(str(path).encode(), buf, n + 1)
    return json.loads(buf.value)


def mini_config(**kw) -> Config:
    """The 2-layer test model of oracle/weights.py ModelCfg()."""
    base = dict(num_layers=2, hidden=512, q_heads=4, kv_heads=1, intermediate=1024, vocab=512,
                max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=128,
                manual_step=1, seed=0)
    base.update(kw)
    return default_config(**base)


@dataclass
class PollResult:
    tokens: list
    finished: str | None
    usage: tuple


@dataclass
class LogprobsPollResult(PollResult):
    lp: np.ndarray        # float32 [n]: each token's own log-probability
    top_ids: np.ndarray   # int32 [n, N]
    top_lp: np.ndarray    # float32 [n, N]


class Engine:
    def __init__(self, cfg: Config):
        self._l = lib()
        self._h = C.c_void_p()
        self.cfg = cfg
        check(self._l.b200_engine_create(C.byref(cfg), C.byref(self._h)))

    def close(self):
        if self._h:
            self._l.b200_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def submit(self, prompt_ids, max_tokens=16, ignore_eos=True, stop_ids=(), temperature=0.0, top_p=1.0, top_k=0,
               seed=None, logprobs=False, top_logprobs=0, min_p=0.0, presence_penalty=0.0, frequency_penalty=0.0,
               repetition_penalty=1.0, min_tokens=0, logit_bias=None, prompt_logprobs=None) -> int:
        """temperature < 1e-5 is greedy; top_k 0 / -1 and top_p 1 are off; seed None = one drawn by the engine.
        logprobs: keep each generated token's log-probability and its top_logprobs (0..20) most likely tokens, read with
        poll_logprobs.  min_p 0, the penalties 0 (repetition 1), min_tokens 0 and logit_bias None ({id: bias}) are off.
        prompt_logprobs N (0..20): keep each prompt token's log-probability, rank and its position's top N, read with
        poll_prompt_logprobs; None is off."""
        return self.submit_n(prompt_ids, 1, max_tokens, ignore_eos, stop_ids, temperature, top_p, top_k, seed, logprobs,
                             top_logprobs, min_p, presence_penalty, frequency_penalty, repetition_penalty, min_tokens,
                             logit_bias, prompt_logprobs, _single=True)

    def submit_n(self, prompt_ids, n, max_tokens=16, ignore_eos=True, stop_ids=(), temperature=0.0, top_p=1.0, top_k=0,
                 seed=None, logprobs=False, top_logprobs=0, min_p=0.0, presence_penalty=0.0, frequency_penalty=0.0,
                 repetition_penalty=1.0, min_tokens=0, logit_bias=None, prompt_logprobs=None, _single=False):
        """Parallel sampling (b200_submit_n): n request ids sharing one prefill; member i uses seed + i (seed None: one
        drawn per member).  The parameters are submit()'s; n > 1 needs temperature >= 1e-5."""
        ids = np.ascontiguousarray(prompt_ids, dtype=np.int32)
        stops = np.ascontiguousarray(stop_ids, dtype=np.int32)
        bias = dict(logit_bias or {})
        bias_ids = np.ascontiguousarray(list(bias.keys()), dtype=np.int32)
        bias_vals = np.ascontiguousarray(list(bias.values()), dtype=np.float32)
        sp = Sampling(max_tokens=max_tokens, temperature=temperature, ignore_eos=1 if ignore_eos else 0,
                      num_stop_ids=len(stops),
                      stop_ids=stops.ctypes.data_as(C.POINTER(C.c_int32)) if len(stops) else None,
                      top_p=top_p, top_k=top_k, has_seed=0 if seed is None else 1,
                      seed=0 if seed is None else seed & 0xFFFFFFFFFFFFFFFF,
                      logprobs=1 if logprobs else 0, top_logprobs=top_logprobs,
                      presence_penalty=presence_penalty, frequency_penalty=frequency_penalty,
                      repetition_penalty=repetition_penalty, min_p=min_p, min_tokens=min_tokens,
                      num_logit_bias=len(bias_ids),
                      logit_bias_ids=bias_ids.ctypes.data_as(C.POINTER(C.c_int32)) if len(bias_ids) else None,
                      logit_bias_values=bias_vals.ctypes.data_as(C.POINTER(C.c_float)) if len(bias_ids) else None,
                      prompt_logprobs=0 if prompt_logprobs is None else 1,
                      top_prompt_logprobs=0 if prompt_logprobs is None else prompt_logprobs)
        if _single:
            rid = C.c_uint64()
            check(self._l.b200_submit(self._h, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(ids), C.byref(sp),
                                      C.byref(rid)))
            return rid.value
        rids = (C.c_uint64 * max(n, 1))()
        check(self._l.b200_submit_n(self._h, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(ids), C.byref(sp), n, rids))
        return list(rids[:n])

    def submit_embed(self, prompt_ids, normalize: bool = True) -> int:
        """One embedding request (pooling runner, b200_submit_embed): the last prompt position's final-normed hidden state,
        L2-normalised in fp32 when normalize."""
        ids = np.ascontiguousarray(prompt_ids, dtype=np.int32)
        rid = C.c_uint64()
        check(self._l.b200_submit_embed(self._h, ids.ctypes.data_as(_PI32), len(ids), 1 if normalize else 0, C.byref(rid)))
        return rid.value

    def poll_embedding(self, rid: int):
        """(vector float32 [hidden] or None until finished, finish reason, usage) of an embedding request."""
        out = np.zeros(self.cfg.hidden, dtype=np.float32)
        fin, u = C.c_int32(), Usage()
        check(self._l.b200_poll_embedding(self._h, rid, out.ctypes.data_as(C.c_void_p), self.cfg.hidden, C.byref(fin),
                                          C.byref(u)))
        return (out if fin.value == 1 else None), FINISH[fin.value], (u.prompt_tokens, u.cached_tokens, u.completion_tokens)

    def submit_score(self, prompt_ids, use_activation: bool = True) -> int:
        """One score request (score head, b200_submit_score): the score logits of the last prompt position, with the
        engine's activation when use_activation."""
        ids = np.ascontiguousarray(prompt_ids, dtype=np.int32)
        rid = C.c_uint64()
        check(self._l.b200_submit_score(self._h, ids.ctypes.data_as(_PI32), len(ids), 1 if use_activation else 0,
                                        C.byref(rid)))
        return rid.value

    def poll_score(self, rid: int):
        """(scores float32 [num_labels] or None until finished, finish reason, usage) of a score request."""
        out = np.zeros(max(self.cfg.num_labels, 1), dtype=np.float32)
        fin, u = C.c_int32(), Usage()
        check(self._l.b200_poll_score(self._h, rid, out.ctypes.data_as(C.c_void_p), self.cfg.num_labels, C.byref(fin),
                                      C.byref(u)))
        return (out if fin.value == 1 else None), FINISH[fin.value], (u.prompt_tokens, u.cached_tokens, u.completion_tokens)

    def score(self, prompts, use_activation: bool = True, max_steps: int = 100000):
        """Manual-step helper: submit every prompt as a score request, step until all are finished, return float32
        [len(prompts), num_labels]."""
        return self._run_pooled([self.submit_score(p, use_activation) for p in prompts], self.poll_score, max_steps)

    def embed(self, prompts, normalize: bool = True, max_steps: int = 100000):
        """Manual-step helper: submit every prompt, step until all are finished, return float32 [len(prompts), hidden]."""
        return self._run_pooled([self.submit_embed(p, normalize) for p in prompts], self.poll_embedding, max_steps)

    def _run_pooled(self, rids, poll, max_steps):
        vecs = [None] * len(rids)
        for _ in range(max_steps):
            ran, _info = self.step()
            for i, r in enumerate(rids):
                if vecs[i] is None:
                    v, fin, _u = poll(r)
                    if fin is not None and v is None:
                        raise RuntimeError(f"pooled request finished with {fin}")
                    vecs[i] = v
            if all(v is not None for v in vecs):
                break
            if not ran:
                raise RuntimeError("engine idle with unfinished requests")
        for r in rids:
            self.release(r)
        return np.stack(vecs)

    def wait_any(self, rids, timeout_s: float = -1.0) -> bool:
        """Block until any of rids (one submit_n group, or a single id) has undrained tokens or is finished."""
        arr = (C.c_uint64 * len(rids))(*rids)
        rc = self._l.b200_wait_any(self._h, arr, len(rids), int(timeout_s * 1e6) if timeout_s >= 0 else -1)
        if rc == -7:
            return False
        check(rc)
        return True

    def poll(self, rid: int, cap: int = 4096) -> PollResult:
        buf = (C.c_int32 * cap)()
        n, fin, u = C.c_int32(), C.c_int32(), Usage()
        check(self._l.b200_poll(self._h, rid, buf, cap, C.byref(n), C.byref(fin), C.byref(u)))
        return PollResult(list(buf[: n.value]), FINISH[fin.value],
                          (u.prompt_tokens, u.cached_tokens, u.completion_tokens))

    def poll_logprobs(self, rid: int, top_logprobs: int, cap: int = 4096) -> LogprobsPollResult:
        """poll() with the records of the drained tokens: lp float32 [n], top_ids int32 [n, top_logprobs] and
        top_lp float32 [n, top_logprobs] (top_logprobs = the request's)."""
        ids = (C.c_int32 * cap)()
        lp = np.zeros(cap, dtype=np.float32)
        tid = np.zeros((cap, MAX_LOGPROBS), dtype=np.int32)
        tlp = np.zeros((cap, MAX_LOGPROBS), dtype=np.float32)
        n, fin, u = C.c_int32(), C.c_int32(), Usage()
        check(self._l.b200_poll_logprobs(self._h, rid, ids, lp.ctypes.data_as(C.c_void_p), tid.ctypes.data_as(_PI32),
                                         tlp.ctypes.data_as(C.c_void_p), cap, C.byref(n), C.byref(fin), C.byref(u)))
        k = n.value
        return LogprobsPollResult(list(ids[:k]), FINISH[fin.value],
                                  (u.prompt_tokens, u.cached_tokens, u.completion_tokens), lp[:k].copy(),
                                  tid[:k, :top_logprobs].copy(), tlp[:k, :top_logprobs].copy())

    def poll_prompt_logprobs(self, rid: int, n_prompt: int, top_n: int):
        """The prompt records of a request submitted with prompt_logprobs=top_n, or None until they all exist: (lp
        float32 [n_prompt - 1], rank int32 [n_prompt - 1], top_ids int32 [n_prompt - 1, top_n], top_lp float32
        [n_prompt - 1, top_n]); record k is prompt token k + 1's.  Does not drain any token."""
        cap = max(n_prompt - 1, 0)
        lp = np.zeros(max(cap, 1), dtype=np.float32)
        rank = np.zeros(max(cap, 1), dtype=np.int32)
        tid = np.zeros((max(cap, 1), MAX_LOGPROBS), dtype=np.int32)
        tlp = np.zeros((max(cap, 1), MAX_LOGPROBS), dtype=np.float32)
        n = C.c_int32()
        check(self._l.b200_poll_prompt_logprobs(self._h, rid, lp.ctypes.data_as(C.c_void_p), rank.ctypes.data_as(_PI32),
                                                tid.ctypes.data_as(_PI32), tlp.ctypes.data_as(C.c_void_p), cap,
                                                C.byref(n)))
        if n.value != cap:
            return None
        return lp[:cap].copy(), rank[:cap].copy(), tid[:cap, :top_n].copy(), tlp[:cap, :top_n].copy()

    def wait(self, rid: int, timeout_s: float = -1.0) -> bool:
        rc = self._l.b200_wait(self._h, rid, int(timeout_s * 1e6) if timeout_s >= 0 else -1)
        if rc == -7:
            return False
        check(rc)
        return True

    def abort(self, rid: int):
        check(self._l.b200_abort(self._h, rid))

    def release(self, rid: int):
        check(self._l.b200_release(self._h, rid))

    def step(self):
        info = StepInfo()
        rc = check(self._l.b200_engine_step(self._h, C.byref(info)))
        return rc == 1, info

    def run(self, max_steps: int, idle_timeout_us: int = 20000):
        """Up to max_steps pipelined iterations (b200_engine_run); returns the StepInfo of every step that ran."""
        infos = (StepInfo * max_steps)()
        n = C.c_int32()
        check(self._l.b200_engine_run(self._h, max_steps, idle_timeout_us, infos, C.byref(n)))
        return [infos[i] for i in range(n.value)]

    def stats(self) -> Stats:
        s = Stats()
        check(self._l.b200_stats_get(self._h, C.byref(s)))
        return s

    def replay(self, n: int, repeat: int = 1):
        ms, tok, smp, kvt, ln = C.c_double(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        check(self._l.b200_engine_replay(self._h, n, repeat, C.byref(ms), C.byref(tok), C.byref(smp), C.byref(kvt),
                                         C.byref(ln)))
        return dict(ms=ms.value, tokens=tok.value, sampled=smp.value, kv_tokens=kvt.value, launches=ln.value)

    KERNEL_CLASSES = ["embed", "rmsnorm", "gemm_qkv", "rope_kvwrite", "attn_decode", "attn_prefill", "gemm_o",
                      "gemm_gate_up", "silu_mul", "gemm_down", "gemm_lm_head", "argmax"]

    def set_skip_mask(self, classes=()):
        mask = 0
        for c in classes:
            mask |= 1 << self.KERNEL_CLASSES.index(c)
        check(self._l.b200_engine_set_skip_mask(self._h, mask))

    def set_recording(self, on: bool):
        check(self._l.b200_engine_set_recording(self._h, 1 if on else 0))

    def profile(self, n: int) -> dict:
        """Per-kernel-class device time (us) and launch counts over the last n recorded steps."""
        k = len(self.KERNEL_CLASSES)
        us, ln = (C.c_double * k)(), (C.c_int64 * k)()
        check(self._l.b200_engine_profile(self._h, n, us, ln, k))
        return {name: dict(us=us[i], launches=ln[i]) for i, name in enumerate(self.KERNEL_CLASSES)}

    def profile_range(self, n: int, min_tokens: int, max_tokens: int):
        """profile() over the recorded steps with min_tokens <= T <= max_tokens; returns (per-class dict, totals dict)."""
        k = len(self.KERNEL_CLASSES)
        us, ln = (C.c_double * k)(), (C.c_int64 * k)()
        st, tk, sm, kv = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        check(self._l.b200_engine_profile_range(self._h, n, min_tokens, max_tokens, us, ln, k, C.byref(st), C.byref(tk),
                                                C.byref(sm), C.byref(kv)))
        return ({name: dict(us=us[i], launches=ln[i]) for i, name in enumerate(self.KERNEL_CLASSES)},
                dict(steps=st.value, tokens=tk.value, sampled=sm.value, kv_tokens=kv.value))

    def reset_prefix_cache(self):
        check(self._l.b200_engine_reset_prefix_cache(self._h))

    def tensor(self, name: str) -> np.ndarray:
        """bf16 bit patterns (uint16) of a named weight, copied to host."""
        nb, p = C.c_uint64(), C.c_void_p()
        check(self._l.b200_engine_tensor_info(self._h, name.encode(), C.byref(nb), C.byref(p)))
        out = np.empty(nb.value // 2, dtype=np.uint16)
        check(self._l.b200_engine_tensor_read(self._h, name.encode(), out.ctypes.data_as(C.c_void_p), nb.value))
        return out

    def tensor_write(self, name: str, bits: np.ndarray):
        bits = np.ascontiguousarray(bits, dtype=np.uint16)
        check(self._l.b200_engine_tensor_write(self._h, name.encode(), bits.ctypes.data_as(C.c_void_p), bits.nbytes))

    def load_safetensors(self, path: str):
        check(self._l.b200_engine_load_safetensors(self._h, str(path).encode()))

    def forward_logits(self, ids) -> np.ndarray:
        """fp32 array [n, vocab] of the bf16 logits for one sequence (debug/parity)."""
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        out = np.empty((len(ids), self.cfg.vocab), dtype=np.uint16)
        check(self._l.b200_engine_forward_logits(self._h, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(ids),
                                                 out.ctypes.data_as(C.c_void_p)))
        return (out.astype(np.uint32) << 16).view(np.float32)

    def set_keep_logits(self, on: bool):
        check(self._l.b200_engine_set_keep_logits(self._h, 1 if on else 0))

    def read_logits(self, rows: int) -> np.ndarray:
        """fp32 array [rows, vocab] of the bf16 logits the last step sampled from (after set_keep_logits(True))."""
        out = np.empty((rows, self.cfg.vocab), dtype=np.uint16)
        check(self._l.b200_engine_read_logits(self._h, out.ctypes.data_as(C.c_void_p), rows))
        return (out.astype(np.uint32) << 16).view(np.float32)

    def generate(self, prompts, max_tokens=16, max_steps=100000):
        """Manual-step helper: run all prompts to completion, return the list of token lists."""
        rids = [self.submit(p, max_tokens=max_tokens) for p in prompts]
        outs = [[] for _ in rids]
        done = [False] * len(rids)
        for _ in range(max_steps):
            ran, _info = self.step()
            for i, r in enumerate(rids):
                if not done[i]:
                    pr = self.poll(r)
                    outs[i] += pr.tokens
                    done[i] = pr.finished is not None
            if all(done):
                break
            if not ran:
                raise RuntimeError("engine idle with unfinished requests")
        for r in rids:
            self.release(r)
        return outs
