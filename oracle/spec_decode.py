"""Reference of n-gram speculative decoding (kubeai_b200/csrc/engine.cu ngram_propose, Engine::complete): test
infrastructure, never imported by the package.

- propose: vLLM's prompt-lookup proposer (vllm/v1/spec_decode/ngram_proposer.py
  _find_longest_matched_ngram_and_propose_tokens) restated by brute force: the longest suffix n-gram of the context with
  min_n <= length <= max_n that occurred earlier, at its earliest occurrence among the longest ones (vLLM's tie rule), and
  up to k tokens that followed it, never past max_model_len.
- accept: the tokens a verify step emits, given the drafts and the token each kept row draws (the sampler's token at index
  n_generated + j after the row's edits, oracle/penalties.py).
"""
from __future__ import annotations

import numpy as np

from oracle import penalties


def propose(toks, min_n: int, max_n: int, k: int, max_model_len: int) -> list:
    toks = [int(t) for t in toks]
    n = len(toks)
    if n < min_n:
        return []
    k = min(k, max_model_len - n)
    if k <= 0:
        return []
    best_len, best_start = 0, -1
    for length in range(1, min(max_n, n - 1) + 1):
        suffix = toks[n - length:]
        # occurrences that end before the context's last token (the suffix itself excluded), earliest first
        for s in range(0, n - length):
            if toks[s:s + length] == suffix:
                if length > best_len:
                    best_len, best_start = length, s
                break
    if best_len < min_n:
        return []
    start = best_start + best_len
    return toks[start:start + min(k, n - start)]


def row_token(row, temperature=0.0, top_k=0, top_p=1.0, seed=0, n=0, min_p=0.0, **edits):
    """The token the engine draws from one raw bf16 row (float32 values) with the request's edits (penalties.edit keyword
    arguments, output = the tokens generated before it) at token index n: (token, race margin)."""
    row = np.asarray(row, dtype=np.float32)
    if edits:
        row = penalties.edit(row, **edits)
    tok, margin, *_ = penalties.sample_ref(row, temperature, top_k, top_p, seed, n, min_p)
    return tok, margin


def accept(drafts, row_tokens, finishes=lambda j, t: False) -> list:
    """Emitted tokens of a verify: t_j = row_tokens[j] for j = 0..len(drafts), stopping after t_j at the last row, when
    t_j differs from drafts[j], or when finishes(j, t_j) (EOS, a stop id, max_tokens or max_model_len)."""
    out = []
    for j, t in enumerate(row_tokens[:len(drafts) + 1]):
        out.append(int(t))
        if j == len(drafts) or finishes(j, t) or t != drafts[j]:
            break
    return out
