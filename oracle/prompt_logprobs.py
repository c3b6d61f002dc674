"""Numpy oracle of the prompt logprobs the engine serves (csrc/sampling.cu logprobs_rows with ranks; vLLM V1's
Sampler.gather_logprobs on prompt rows) and of vLLM 0.22's response shapes built from them: the prompt_logprobs list
(vllm/logprobs.py append_logprobs_for_next_position, clamp_prompt_logprobs) and the completions logprobs of an echo
(completion/serving.py _create_completion_logprobs over the prompt's records, led by a null entry, and the output's)."""
from __future__ import annotations

import math

import numpy as np

from oracle.logprobs import completion_logprobs


def rank_ref(row, token):
    """vLLM's batched_count_greater_than: how many entries of the row are >= the token's (equal logits count, -0 == +0)."""
    x = np.asarray(row, dtype=np.float64)
    return int((x >= x[int(token)]).sum())


def prompt_entry(token, lp, rank, top_ids, top_lp):
    """vLLM's {id: (logprob, rank)} dict of one prompt position: the prompt token with its rank first, then the top N with
    ranks 1..N; a repeated id keeps its first place and takes the later entry."""
    d = {}
    for i, v, r in zip([int(token)] + [int(t) for t in top_ids], [float(lp)] + [float(v) for v in top_lp],
                       [int(rank)] + list(range(1, len(top_ids) + 1))):
        d[i] = (v, r)
    return d


def _clamp_inf(v):
    return -9999.0 if v == -math.inf else v


def prompt_logprobs_json(records, token_str):
    """The "prompt_logprobs" list for records [(token, lp, rank, top_ids, top_lp)] of prompt positions 1..n-1, as vLLM's
    pydantic model_dump writes it (JSON object keys are strings)."""
    out = [None]
    for tok, lp, rank, top_ids, top_lp in records:
        d = prompt_entry(tok, lp, rank, top_ids, top_lp)
        out.append({str(t): dict(logprob=_clamp_inf(v), rank=r, decoded_token=token_str(t)) for t, (v, r) in d.items()})
    return out


def echo_completion_logprobs(prompt_ids, prompt_records, n, token_str, output_records=()):
    """The completions "logprobs" of an echo: the first prompt token (null entries), the prompt records (token, lp, rank,
    top_ids, top_lp), then the output records (token, lp, top_ids, top_lp) of vLLM's generated tokens; the first n + 1
    entries per position."""
    head = token_str(int(prompt_ids[0]))
    rest = completion_logprobs([(t, lp, ids, lps) for t, lp, _r, ids, lps in prompt_records] + list(output_records), n,
                               token_str, len(head))
    return dict(text_offset=[0] + rest["text_offset"], token_logprobs=[None] + rest["token_logprobs"],
                tokens=[head] + rest["tokens"], top_logprobs=[None] + rest["top_logprobs"])

