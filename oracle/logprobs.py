"""Numpy oracle of the logprobs the engine serves (csrc/sampling.cu logprobs_rows; vLLM V1's raw_logprobs,
vllm/v1/sample/sampler.py compute_logprobs / gather_logprobs) and of vLLM 0.22's OpenAI response shapes built from them
(vllm/v1/engine/logprobs.py, chat_completion/serving.py _create_chat_logprobs, completion/serving.py
_create_completion_logprobs)."""
from __future__ import annotations

import numpy as np

MAX_LOGPROBS = 20


def logprobs_ref(row, n):
    """float64 log-softmax of one row of bf16 logits (given as their exact float32 values) and its n most likely ids:
    descending logit, lowest id among equal logits (-0 and +0 are equal)."""
    x = np.asarray(row, dtype=np.float64)
    m = x.max()
    lp = (x - m) - np.log(np.exp(x - m).sum())
    order = np.lexsort((np.arange(len(x)), -x))
    return lp, order[:n]


def position_entries(token, lp, top_ids, top_lp):
    """vLLM's Logprob dict of one position: the sampled token first, then the top N, one entry per id."""
    d = {}
    for i, v in zip([int(token)] + [int(t) for t in top_ids], [float(lp)] + [float(v) for v in top_lp]):
        d[i] = v
    return d


def _clamp(v):
    return max(v, -9999.0)


def chat_logprobs(records, n, token_str):
    """The "logprobs" object of a chat choice (or of one stream chunk) for records [(token, lp, top_ids, top_lp)]."""
    content = []
    for tok, lp, top_ids, top_lp in records:
        d = position_entries(tok, lp, top_ids, top_lp)
        s = token_str(int(tok))
        top = [dict(token=token_str(t), logprob=_clamp(v), bytes=list(token_str(t).encode("utf-8", "replace")))
               for i, (t, v) in enumerate(d.items()) if n and i < n]
        content.append(dict(token=s, logprob=_clamp(d[int(tok)]), bytes=list(s.encode("utf-8", "replace")),
                            top_logprobs=top))
    return dict(content=content)


def completion_logprobs(records, n, token_str, initial_text_offset=0):
    """The "logprobs" object of a completions choice (or of one stream chunk): the first n + 1 entries per position."""
    out = dict(text_offset=[], token_logprobs=[], tokens=[], top_logprobs=[])
    last = 0
    for tok, lp, top_ids, top_lp in records:
        d = position_entries(tok, lp, top_ids, top_lp)
        s = token_str(int(tok))
        out["tokens"].append(s)
        out["token_logprobs"].append(_clamp(d[int(tok)]))
        out["top_logprobs"].append({token_str(t): _clamp(v) for i, (t, v) in enumerate(d.items()) if n >= i})
        out["text_offset"].append(initial_text_offset if not out["text_offset"] else out["text_offset"][-1] + last)
        last = len(s)
    return out
