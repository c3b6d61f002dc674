"""Reference of the engine's logits edits (kubeai_b200/csrc/penalties.cu) and of min_p in its sampler
(kubeai_b200/csrc/sampling.cu), in numpy: test infrastructure, never imported by the package.

Edits (vLLM V1's order: LogitBiasLogitsProcessor, MinTokensLogitsProcessor, then apply_penalties), in float32 for each token
v that the request names (a bias id, a stop id while fewer than min_tokens tokens exist, a prompt or an output token):
    l = float32(bf16 logit);  l += bias[v];  l = -inf (stop id);  l *= (l > 0 ? float32(1 / r) : r) (in prompt or output);
    l -= float32(frequency * count[v]);  l -= presence * (count[v] > 0)
then rounded to bf16 (RNE).  Every other token keeps its value: vLLM's arithmetic is the identity there.

min_p (sampled rows, after temperature): keep v iff float64(float32(z_v - z_max)) >= log(min_p), a fixed form of vLLM's
p_v >= min_p * p_max; top-k and top-p then run over the kept tokens (oracle/sampling.py).
"""
from __future__ import annotations

import numpy as np

from oracle.sampling import SAMPLING_EPS, filter_mask, scaled, uniforms


def bf16_round(x):
    """float32 -> the nearest bf16 (ties to even), as float32; inf and -inf stay."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + np.uint64(0x7FFF) + ((b >> np.uint64(16)) & np.uint64(1))) >> np.uint64(16)) << np.uint64(16)
    return r.astype(np.uint32).view(np.float32)


def edit_f32(logits, prompt=(), output=(), presence=0.0, frequency=0.0, repetition=1.0, min_tokens=0, stop_ids=(),
             logit_bias=None):
    """One row's edited logits in float32, before the bf16 rounding.  repetition 0 means 1 (off); min_tokens counts
    `output`; stop_ids are the stops (EOS included)."""
    l = np.array(logits, dtype=np.float32)
    V = l.shape[0]
    prompt = np.asarray(prompt, dtype=np.int64)
    output = np.asarray(output, dtype=np.int64)
    r = np.float32(repetition if repetition > 0 else 1.0)
    history = presence != 0 or frequency != 0 or r != 1
    for t, b in (logit_bias or {}).items():
        l[t] = l[t] + np.float32(min(100.0, max(-100.0, b)))
    if len(output) < min_tokens:
        for t in stop_ids:
            l[t] = -np.inf
    if history:
        count = np.bincount(output, minlength=V).astype(np.int64)
        in_prompt = np.zeros(V, dtype=bool)
        in_prompt[prompt] = True
        touched = in_prompt | (count > 0)
        inv = np.float32(1.0) / r
        with np.errstate(invalid="ignore"):
            scale = np.where(touched, np.where(l > 0, inv, r), np.float32(1.0)).astype(np.float32)
            l = (l * scale).astype(np.float32)
            l = (l - np.float32(frequency) * count.astype(np.float32)).astype(np.float32)
            l = (l - np.float32(presence) * (count > 0).astype(np.float32)).astype(np.float32)
    return l


def edit(logits, **kw):
    """edit_f32 rounded to bf16, as the engine writes the row (float32 values)."""
    return bf16_round(edit_f32(logits, **kw))


def named(V, prompt=(), output=(), presence=0.0, frequency=0.0, repetition=1.0, min_tokens=0, stop_ids=(),
          logit_bias=None):
    """Mask of the tokens the engine's record list names (the only entries it may write)."""
    m = np.zeros(V, dtype=bool)
    r = repetition if repetition > 0 else 1.0
    if presence != 0 or frequency != 0 or r != 1:
        m[np.asarray(prompt, dtype=np.int64)] = True
        m[np.asarray(output, dtype=np.int64)] = True
    if len(output) < min_tokens:
        m[np.asarray(stop_ids, dtype=np.int64)] = True
    for t in (logit_bias or {}):
        m[t] = True
    return m


PEN_PROMPT, PEN_STOP, PEN_BIAS = 1, 2, 4   # kPen* of kubeai_b200/csrc/kernels.h


def records(prompt=(), output=(), history=True, logit_bias=None, stop_ids=(), min_tokens=0):
    """The record list penalty_records builds (kubeai_b200/csrc/penalties.cu), as int32 [n, 4] rows (id, count, bias as
    float32 bits, flags), sorted by id: one record per distinct id; the prompt (PEN_PROMPT) and the output (count) only
    with `history`; the stop ids (PEN_STOP) only while len(output) < min_tokens; the last bias of an id, clamped to
    [-100, 100] in float32 (PEN_BIAS).  penalize_update keeps a list equal to this with each sampled token appended to
    `output` (the stop records stay while the list lives: pass the min_tokens the list was built under)."""
    prompt = np.asarray(prompt, dtype=np.int64).ravel() if history else np.zeros(0, np.int64)
    output_h = np.asarray(output, dtype=np.int64).ravel() if history else np.zeros(0, np.int64)
    stops = np.asarray(stop_ids, dtype=np.int64).ravel() if len(output) < min_tokens else np.zeros(0, np.int64)
    bias = {int(t): np.float32(min(np.float32(100.0), max(np.float32(-100.0), np.float32(b))))
            for t, b in (logit_bias or {}).items()}
    bid = np.array(sorted(bias), dtype=np.int64)
    ids = np.unique(np.concatenate([prompt, output_h, stops, bid]))
    out = np.zeros((ids.size, 4), dtype=np.int32)
    out[:, 0] = ids
    if output_h.size:
        u, c = np.unique(output_h, return_counts=True)
        out[np.searchsorted(ids, u), 1] = c
    flags = np.zeros(ids.size, dtype=np.int32)
    flags[np.searchsorted(ids, np.unique(prompt))] |= PEN_PROMPT
    flags[np.searchsorted(ids, np.unique(stops))] |= PEN_STOP
    if bid.size:
        pos = np.searchsorted(ids, bid)
        flags[pos] |= PEN_BIAS
        out[pos, 2] = np.array([bias[int(t)] for t in bid], dtype=np.float32).view(np.int32)
    out[:, 3] = flags
    return out


def min_p_keep(z, min_p):
    """(kept mask, boundary slack) of min_p over one row of scaled logits z (float32 values): the slack is the distance in
    log space between log(min_p) and the nearest d_v = z_v - z_max."""
    z32 = np.asarray(z, dtype=np.float32)
    if not min_p > 0:
        return np.ones(z32.shape[0], dtype=bool), np.inf
    d = (z32 - z32.max()).astype(np.float32).astype(np.float64)
    lm = np.log(np.float64(np.float32(min_p)))
    fin = np.isfinite(d)
    slack = float(np.min(np.abs(d[fin] - lm))) if fin.any() else np.inf
    return d >= lm, slack


def sample_ref(logits, temperature, top_k=0, top_p=1.0, seed=0, n=0, min_p=0.0):
    """oracle/sampling.py sample_ref with min_p: (token, race margin, top-p slack, min_p slack)."""
    l = np.asarray(logits, dtype=np.float32)
    V = l.shape[0]
    if not np.float32(temperature) >= SAMPLING_EPS:
        top2 = np.sort(l.astype(np.float64))[-2:]
        return int(np.argmax(l)), float(top2[1] - top2[0]) if V > 1 else np.inf, np.inf, np.inf
    z = scaled(l, temperature)
    mkeep, mslack = min_p_keep(z.astype(np.float32), min_p)
    keep, slack = filter_mask(np.where(mkeep, z, -np.inf), top_k, top_p)
    keep &= mkeep
    e = -np.log(uniforms(seed, n, V))
    score = np.where(keep, z - np.log(e), -np.inf)
    tok = int(np.argmax(score))
    kept = np.sort(score[keep])
    margin = float(kept[-1] - kept[-2]) if kept.size > 1 else np.inf
    return tok, margin, slack, mslack
