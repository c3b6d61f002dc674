"""Rerank at Llama-3-8B's shape (H100 only): a score-head engine with seeded weights (32 layers, hidden 4096, 32:8 heads
of 128, intermediate 14336, vocab 128 256, one label) scores 1 query x 64 documents of about 256 tokens each.

    python -m scripts.rerank_step [--reps 3]

Prints one JSON line with the card name and power limit read in the same call, and for each case ("distinct": 64 prompts
with nothing in common; "shared_prefix": the same 64 prompts behind one 128-token query, prefix cache on, the query
computed once first) the prompt tokens submitted, the tokens computed and prompt tokens/s over the wall time from submit
to the last score (manual steps, pipelined by b200_engine_run).  The score tail is timed with CUDA events around
b200_op_score_rows over 256 rows of a [16384, 4096] residual stream, against b200_op_pool_rows on the same rows (the
tail an embedding engine runs).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import time

import numpy as np

from kubeai_b200.engine import Engine, default_config

SHAPE = dict(num_layers=32, hidden=4096, q_heads=32, kv_heads=8, intermediate=14336, vocab=128256, max_model_len=1024,
             max_num_seqs=64, max_batched_tokens=8192, num_kv_blocks=4096, manual_step=1, runner=1, num_labels=1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def serve(e, prompts):
    t0 = time.perf_counter()
    rids = [e.submit_score(p) for p in prompts]
    st0 = e.stats()
    while e._l.b200_engine_unfinished(e._h) > 0:
        e.run(64, 2000)
    dt = time.perf_counter() - t0
    out = [e.poll_score(r)[0][0] for r in rids]
    for r in rids:
        e.release(r)
    st = e.stats()
    computed = (st.prompt_tokens - st0.prompt_tokens) - (st.cached_prompt_tokens - st0.cached_prompt_tokens)
    return dt, computed, out


def case(prompts, prefix, reps):
    rates, computed = [], 0
    with Engine(default_config(enable_prefix_caching=1 if prefix else 0, **SHAPE)) as e:
        for r in range(reps + 1):   # the first round warms up
            e.reset_prefix_cache()
            if prefix:
                serve(e, [prefix])
            dt, computed, _ = serve(e, prompts)
            if r:
                rates.append(sum(map(len, prompts)) / dt)
    return dict(prompt_tokens=sum(map(len, prompts)), computed_tokens=int(computed),
                prompt_tokens_per_s=float(np.median(rates)))


def tail_us(fn_name, rows=256, T=16384, H=4096, reps=200):
    import torch

    from kubeai_b200 import lib
    hid = torch.randn(T, H, device="cuda").to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(H, device="cuda")).to(torch.bfloat16)
    sw = (torch.randn(1, H, device="cuda") / 64).to(torch.bfloat16)
    idx = (torch.arange(rows, dtype=torch.int32, device="cuda") + 1) * (T // rows) - 1
    flags = torch.ones(rows, dtype=torch.int32, device="cuda")
    out = torch.empty(rows, H, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())
    if fn_name == "score":
        call = lambda: lib().b200_op_score_rows(p(hid), p(w), p(sw), p(idx), p(flags), rows, H, 1, 0, C.c_float(1e-5),
                                                p(out), None)
    else:
        call = lambda: lib().b200_op_pool_rows(p(hid), p(w), p(idx), p(flags), rows, H, C.c_float(1e-5), p(out), None)
    for _ in range(10):
        assert call() == 0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        call()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    V = SHAPE["vocab"]
    query = rng.integers(0, V, size=128).tolist()
    docs = [rng.integers(0, V, size=int(n)).tolist() for n in rng.integers(120, 136, size=64)]
    distinct = [rng.integers(0, V, size=128).tolist() + d for d in docs]   # ~256 tokens, no common prefix
    shared = [query + d for d in docs]
    print(json.dumps(dict(card=card(), documents=len(docs),
                          distinct=case(distinct, None, a.reps), shared_prefix=case(shared, query, a.reps),
                          score_tail_us=tail_us("score"), pool_rows_tail_us=tail_us("pool"), tail_rows=256)))


if __name__ == "__main__":
    main()
