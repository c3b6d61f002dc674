#!/usr/bin/env python
"""What the group size G = q_heads / kv_heads costs in decode attention, and a Llama-3.2-3B-shaped engine's steps.

  python scripts/gqa_step.py [--groups 1,3,4,8] [--seqs 1,8,32,128] [--ctx 1000,2000] [--iters 200] [--no-engine]
                             [--json OUT.json]

1. Decode attention (b200_op_paged_attn / _decode_split) at each G with kv_heads fixed at 8, so every G reads the same
   K/V bytes: seqs x ctx x 8 heads x (K + V) x 128 x 2 bytes.  The split is the engine's choice (attn_decode_split:
   about two CTAs per SM, at least two 64-token tiles each, at most 32 parts).  CUDA events around --iters back-to-back
   launches after a warm-up; printed: us per launch and K/V bytes/s.
2. A 28-layer engine at the Llama-3.2-3B shape (hidden 3072, 24:8 heads, intermediate 8192, vocab 128256, llama3 rope
   with factor 32) with seeded random weights: replayed decode steps at 1-128 sequences and verify steps at k = 3
   (scripts/spec_decode_step.py's method: every draft accepted), and one 1536-token prefill step (device time, median
   of 5).
The card's name, power limit and max SM clock are read in the same process."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from scripts.spec_decode_step import card, measure  # noqa: E402

SHAPE_3B = dict(num_layers=28, hidden=3072, q_heads=24, kv_heads=8, intermediate=8192, vocab=128256, rope_scaling_type=2,
                rope_factor=32.0, rope_low_freq_factor=1.0, rope_high_freq_factor=4.0, rope_original_max_pos=8192)
HKV = 8


def engine_split(num_work, Hkv, max_ctx, sms):
    """attention.cu attn_decode_split."""
    ctas = num_work * Hkv
    if ctas >= sms:
        return 1
    p = min((2 * sms + ctas - 1) // ctas, (max_ctx + 127) // 128, 32)
    return max(p, 1)


def attention(G, S, ctx, iters):
    import torch
    from kubeai_b200 import ops
    Hq = G * HKV
    nb = (ctx + 15) // 16
    gen = torch.Generator(device="cuda").manual_seed(G * 1000 + S)
    kv = torch.randn(S * nb, 2, HKV, 16, 128, device="cuda", generator=gen).bfloat16()
    btab = torch.randperm(S * nb, device="cuda", generator=gen).int().reshape(S, nb)
    q = torch.randn(S, Hq * 128, device="cuda", generator=gen).bfloat16()
    work = torch.tensor([(s, 1, ctx - 1, s) for s in range(S)], dtype=torch.int32, device="cuda")
    out = torch.empty(S, Hq * 128, dtype=torch.bfloat16, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    split = engine_split(S, HKV, ctx, sms)
    call = lambda: ops.paged_attn(q, kv, btab, work, Hq, HKV, decode=True, out=out, split=split if split > 1 else 0)
    for _ in range(10):
        call()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        call()
    b.record()
    torch.cuda.synchronize()
    us = a.elapsed_time(b) * 1e3 / iters
    kv_bytes = S * ctx * HKV * 2 * 128 * 2
    return dict(us=us, split=split, kv_bytes=kv_bytes, kv_gb_s=kv_bytes / (us * 1e-6) / 1e9)


def prefill_ms(eng, T, reps=5):
    import numpy as np
    rng = np.random.default_rng(T)
    times = []
    for _ in range(reps + 1):
        rid = eng.submit(rng.integers(0, 128256, T).tolist(), max_tokens=2)
        ran, info = eng.step()
        assert ran and info.prefill_seqs == 1 and info.tokens == T, (info.prefill_seqs, info.tokens)
        times.append(info.device_us / 1e3)
        eng.abort(rid)
        while eng.step()[0]:
            pass
        eng.release(rid)
        eng.reset_prefix_cache()
    return float(np.median(times[1:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", default="1,3,4,8")
    ap.add_argument("--seqs", default="1,8,32,128")
    ap.add_argument("--ctx", default="1000,2000")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--no-engine", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    groups = [int(x) for x in args.groups.split(",")]
    seqs = [int(x) for x in args.seqs.split(",")]
    ctxs = [int(x) for x in args.ctx.split(",")]
    res = {"card": card(), "attention": {}, "engine_3b": {}}
    print(json.dumps(res["card"]), flush=True)
    for ctx in ctxs:
        for S in seqs:
            row = {G: attention(G, S, ctx, args.iters) for G in groups}
            for G, m in row.items():
                if 4 in row:
                    m["kv_bytes_s_vs_g4"] = m["kv_gb_s"] / row[4]["kv_gb_s"]
                res["attention"][f"G{G}_ctx{ctx}_s{S}"] = m
            print(f"attention ctx={ctx} seqs={S}", json.dumps({G: {a: round(b, 3) for a, b in m.items()} for G, m in row.items()}),
                  flush=True)
    if not args.no_engine:
        from kubeai_b200.engine import Engine, default_config
        for k in (0, 3):
            eng = Engine(default_config(manual_step=1, record_steps=args.steps, max_num_seqs=max(seqs), max_batched_tokens=1536,
                                        max_model_len=max(ctxs) + 1024, kv_fraction=0.80, num_speculative_tokens=k,
                                        prompt_lookup_min=1, prompt_lookup_max=3, **SHAPE_3B))
            if k == 0:
                res["engine_3b"]["prefill_1536_ms"] = prefill_ms(eng, 1536)
                print("prefill T=1536 ms", res["engine_3b"]["prefill_1536_ms"], flush=True)
            for ctx in ctxs:
                for S in seqs:
                    m = measure(eng, k, ctx, S, args.steps, args.repeat, np.random.default_rng(ctx * 1000 + S))
                    m.pop("classes_us")
                    res["engine_3b"][f"k{k}_ctx{ctx}_s{S}"] = m
                    print(f"3B k={k} ctx={ctx} seqs={S}", json.dumps(m), flush=True)
            eng.close()
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
