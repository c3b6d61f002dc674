#!/usr/bin/env python
"""What n-gram speculative decoding costs and gains in Llama-3-8B decode steps (seeded random weights, full size).

  python scripts/spec_decode_step.py [--seqs 1,8,32,128] [--ctx 1000,2000] [--k 0,1,2,3] [--steps 8] [--repeat 5]
                                     [--json OUT.json]

For each k one engine is created (num_speculative_tokens = k, lookup 1..3).  For each context length and batch size the
prompts are a random context whose tail is a run of one token X, and every request carries logit_bias {X: 100}: the
output is X forever, so every decoding sequence proposes k drafts (X X X, found in the run) and all of them are accepted.
After the prompts are prefilled and every sequence runs a full verify, --steps steps run live and are replayed from their
HBM-resident inputs (b200_engine_replay, CUDA events around --repeat back-to-back passes).  Printed per (k, ctx, seqs):
  - step_ms: replayed device time per step; drafts_per_seq (k unless a full KV pool clipped some), tokens_per_step and
    tok_s at the measured (full) acceptance;
  - attn_decode_us / per class: b200_engine_profile_range, an event pair around every launch of each kernel class;
  - vs_k0: step time and decode-attention time over k = 0 at the same (ctx, seqs);
  - break_even_acceptance: the per-draft acceptance a at which (1 - a^(k+1)) / (1 - a) tokens per verify step give the
    tokens per second of plain decoding;
  - proposer_us_per_step: host time of b200_ngram_propose over the step's contexts (a ctypes call per sequence, so an
    upper bound on the engine's own loop).
The card's name, power limit and max SM clock are read in the same process."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

X = 4242


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def break_even(ratio, k):
    """Per-draft acceptance a with (1 - a^(k+1)) / (1 - a) == ratio (verify step time over decode step time)."""
    if k == 0:
        return None
    if ratio <= 1.0:
        return 0.0
    if ratio >= k + 1:
        return None   # not reachable even at full acceptance
    lo, hi = 0.0, 1.0
    for _ in range(60):
        a = (lo + hi) / 2
        e = sum(a ** j for j in range(k + 1))
        lo, hi = (a, hi) if e < ratio else (lo, a)
    return lo


def proposer_us(contexts, k):
    from kubeai_b200 import _lib
    l = _lib.lib()
    arrs = [(C.c_int32 * len(c))(*c) for c in contexts]
    out = (C.c_int32 * 4)()
    reps = 20
    t0 = time.perf_counter()
    for _ in range(reps):
        for a, c in zip(arrs, contexts):
            l.b200_ngram_propose(a, len(c), 1, 3, max(k, 1), 1 << 30, out)
    return (time.perf_counter() - t0) / reps * 1e6


def measure(eng, k, ctx, S, K, repeat, rng):
    prompts = []
    for _ in range(S):
        p = rng.integers(0, 128256, ctx - 8).tolist()
        p = [t if t != X else X + 1 for t in p] + [X] * 8
        prompts.append(p)
    rids = [eng.submit(p, max_tokens=4096, ignore_eos=True, logit_bias={X: 100.0}) for p in prompts]
    waited = idle = 0
    while True:                                    # prefill everything; then wait for a full verify (drafts take only
        ran, info = eng.step()                     # free pages, so a full pool can clip some)
        idle = 0 if ran else idle + 1              # a step that preempted its only candidate runs nothing
        if idle >= 8:
            st = eng.stats()
            fins = [eng.poll(r).finished for r in rids]
            raise RuntimeError(f"engine idle with unfinished work: running {st.running} waiting {st.waiting} kv free "
                               f"{st.kv_blocks_free}/{st.kv_blocks_total} preemptions {st.preemptions} finished "
                               f"{sum(f is not None for f in fins)} ({set(fins)})")
        if ran and info.decode_seqs == S and info.prefill_seqs == 0:
            waited += 1
            if info.draft_tokens == S * k or waited == 16:
                break
    live, acc, drafts, T = 0.0, 0, 0, []
    for _ in range(K):
        ran, info = eng.step()
        assert ran and info.decode_seqs == S and info.sampled == info.tokens
        live += info.device_us
        acc += info.accepted_tokens
        drafts += info.draft_tokens
        T.append(info.tokens)
    eng.replay(min(K, 4), 1)                       # warm
    r = eng.replay(K, repeat)
    prof, tot = eng.profile_range(K, min(T), max(T))
    assert tot["steps"] == K
    ctxs = [p + [X] * 16 for p in prompts]
    for rid in rids:
        eng.abort(rid)
    while eng.step()[0]:
        pass
    for rid in rids:
        eng.release(rid)
    eng.reset_prefix_cache()                       # the replays overwrote KV pages the cache still points at
    step_ms = r["ms"] / (K * repeat)
    tps = (S * K + acc) / K   # every verify emits its accepted drafts plus one token
    return dict(step_ms=step_ms, live_step_us=live / K, tokens_per_step=tps, tok_s=tps / (step_ms * 1e-3),
                drafts_per_seq=drafts / (K * S), acceptance=acc / drafts if drafts else None,
                classes_us={n: v["us"] / K for n, v in prof.items() if v["launches"]},
                attn_decode_us=prof["attn_decode"]["us"] / K, proposer_us_per_step=proposer_us(ctxs, k) if k else 0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", default="1,8,32,128")
    ap.add_argument("--ctx", default="1000,2000")
    ap.add_argument("--k", default="0,1,2,3")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from kubeai_b200.engine import Engine, default_config

    assert torch.cuda.is_available(), "needs a GPU"
    seqs = [int(x) for x in args.seqs.split(",")]
    ctxs = [int(x) for x in args.ctx.split(",")]
    ks = [int(x) for x in args.k.split(",")]
    res = {"card": card(), "steps": args.steps, "repeat": args.repeat, "runs": {}}
    print(json.dumps(res["card"]), flush=True)
    # max_model_len leaves room for the tokens the first-admitted sequences generate (1 + k per step) while the others
    # are still prefilling: a sequence that reaches it finishes before the batch is all decoding
    for k in ks:
        eng = Engine(default_config(manual_step=1, record_steps=args.steps, max_num_seqs=max(seqs), max_batched_tokens=1536,
                                    max_model_len=max(ctxs) + 1024, kv_fraction=0.80, num_speculative_tokens=k,
                                    prompt_lookup_min=1, prompt_lookup_max=3))
        for ctx in ctxs:
            for S in seqs:
                m = measure(eng, k, ctx, S, args.steps, args.repeat, np.random.default_rng(ctx * 1000 + S))
                res["runs"][f"k{k}_ctx{ctx}_s{S}"] = m
                print(f"k={k} ctx={ctx} seqs={S}", json.dumps({a: b for a, b in m.items() if a != "classes_us"}), flush=True)
        eng.close()
    for key, m in res["runs"].items():
        k = int(key[1:key.index("_")])
        base = res["runs"].get("k0" + key[key.index("_"):])
        if k and base:
            m["step_vs_k0"] = m["step_ms"] / base["step_ms"]
            m["attn_decode_vs_k0"] = m["attn_decode_us"] / base["attn_decode_us"]
            m["break_even_acceptance"] = break_even(m["step_vs_k0"], k)
    summary = {key: {a: m.get(a) for a in ("step_ms", "tok_s", "step_vs_k0", "attn_decode_vs_k0", "break_even_acceptance",
                                          "proposer_us_per_step")} for key, m in res["runs"].items()}
    print(json.dumps(summary), flush=True)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
