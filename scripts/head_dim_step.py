#!/usr/bin/env python
"""What the head size D costs in decode and chunked-prefill attention, and a Llama-3.2-1B-shaped engine's steps.

  python scripts/head_dim_step.py [--seqs 1,8,32,128] [--ctx 1000,2000] [--iters 200] [--no-engine] [--json OUT.json]

1. Decode attention (b200_op_paged_attn_hd / _decode_split_hd) at D = 64 and 128 with 8 KV heads and G = 4: seqs x ctx x
   8 heads x (K + V) x D x 2 bytes.  The split is the engine's (attn_decode_split).  CUDA events around --iters
   back-to-back launches after a warm-up; printed: us per launch, K/V bytes/s and the D = 64 / D = 128 ratio.
2. Chunked-prefill attention (b200_op_paged_attn_prefill_tc_hd) for one 1536-token prompt, 32:8 heads, at D = 64 and 128:
   us per launch and TFLOP/s of the causal 4 * T^2 / 2 * D * heads multiply-adds.
3. A 16-layer engine at the Llama-3.2-1B shape (hidden 2048, 32:8 heads of 64, intermediate 8192, vocab 128256, llama3
   rope with factor 32) with seeded random weights: replayed decode steps at 1-128 sequences, verify steps at k = 3 and
   one 1536-token prefill step (scripts/gqa_step.py's method).
The card's name, power limit and max SM clock are read in the same process."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from scripts.gqa_step import engine_split, prefill_ms  # noqa: E402
from scripts.spec_decode_step import card, measure  # noqa: E402

SHAPE_1B = dict(num_layers=16, hidden=2048, q_heads=32, kv_heads=8, head_dim=64, intermediate=8192, vocab=128256,
                rope_scaling_type=2, rope_factor=32.0, rope_low_freq_factor=1.0, rope_high_freq_factor=4.0,
                rope_original_max_pos=8192)
HKV, G = 8, 4


def timed(call, iters):
    import torch
    for _ in range(10):
        call()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        call()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def decode_attention(D, S, ctx, iters):
    import torch
    from kubeai_b200 import ops
    Hq = G * HKV
    nb = (ctx + 15) // 16
    gen = torch.Generator(device="cuda").manual_seed(D * 1000 + S)
    kv = torch.randn(S * nb, 2, HKV, 16, D, device="cuda", generator=gen).bfloat16()
    btab = torch.randperm(S * nb, device="cuda", generator=gen).int().reshape(S, nb)
    q = torch.randn(S, Hq * D, device="cuda", generator=gen).bfloat16()
    work = torch.tensor([(s, 1, ctx - 1, s) for s in range(S)], dtype=torch.int32, device="cuda")
    out = torch.empty(S, Hq * D, dtype=torch.bfloat16, device="cuda")
    split = engine_split(S, HKV, ctx, torch.cuda.get_device_properties(0).multi_processor_count)
    us = timed(lambda: ops.paged_attn(q, kv, btab, work, Hq, HKV, decode=True, out=out, split=split if split > 1 else 0,
                                      head_dim=D), iters)
    kv_bytes = S * ctx * HKV * 2 * D * 2
    return dict(us=us, split=split, kv_bytes=kv_bytes, kv_gb_s=kv_bytes / (us * 1e-6) / 1e9)


def prefill_attention(D, T, iters):
    import torch
    from kubeai_b200 import ops
    Hq = G * HKV
    nb = (T + 15) // 16
    gen = torch.Generator(device="cuda").manual_seed(D + T)
    kv = torch.randn(nb, 2, HKV, 16, D, device="cuda", generator=gen).bfloat16()
    btab = torch.randperm(nb, device="cuda", generator=gen).int().reshape(1, nb)
    qkv = torch.randn(T, (Hq + 2 * HKV) * D, device="cuda", generator=gen).bfloat16()
    work = torch.tensor([(t0, min(64, T - t0), t0, 0) for t0 in range(0, T, 64)], dtype=torch.int32, device="cuda")
    out = torch.empty(T, Hq * D, dtype=torch.bfloat16, device="cuda")
    us = timed(lambda: ops.paged_attn_prefill_tc(qkv, kv, btab, work, Hq, HKV, out=out, head_dim=D), iters)
    flops = 4.0 * (T * (T + 1) / 2) * D * Hq        # QK^T and PV over the causal triangle
    return dict(us=us, tflop_s=flops / (us * 1e-6) / 1e12)


def main():
    ap = argparse.ArgumentParser()
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
    seqs = [int(x) for x in args.seqs.split(",")]
    ctxs = [int(x) for x in args.ctx.split(",")]
    res = {"card": card(), "decode_attention": {}, "prefill_attention": {}, "engine_1b": {}}
    print(json.dumps(res["card"]), flush=True)
    for ctx in ctxs:
        for S in seqs:
            row = {D: decode_attention(D, S, ctx, args.iters) for D in (64, 128)}
            row[64]["kv_bytes_s_vs_d128"] = row[64]["kv_gb_s"] / row[128]["kv_gb_s"]
            for D, m in row.items():
                res["decode_attention"][f"D{D}_ctx{ctx}_s{S}"] = m
            print(f"decode attention ctx={ctx} seqs={S}", json.dumps({D: {a: round(b, 3) for a, b in m.items()}
                                                                     for D, m in row.items()}), flush=True)
    for D in (64, 128):
        res["prefill_attention"][f"D{D}_T1536"] = m = prefill_attention(D, 1536, args.iters)
        print(f"prefill attention D={D} T=1536", json.dumps({a: round(b, 3) for a, b in m.items()}), flush=True)
    if not args.no_engine:
        from kubeai_b200.engine import Engine, default_config
        for k in (0, 3):
            eng = Engine(default_config(manual_step=1, record_steps=args.steps, max_num_seqs=max(seqs), max_batched_tokens=1536,
                                        max_model_len=max(ctxs) + 1024, kv_fraction=0.80, num_speculative_tokens=k,
                                        prompt_lookup_min=1, prompt_lookup_max=3, **SHAPE_1B))
            if k == 0:
                res["engine_1b"]["prefill_1536_ms"] = prefill_ms(eng, 1536)
                print("prefill T=1536 ms", res["engine_1b"]["prefill_1536_ms"], flush=True)
            for ctx in ctxs:
                for S in seqs:
                    m = measure(eng, k, ctx, S, args.steps, args.repeat, np.random.default_rng(ctx * 1000 + S))
                    m.pop("classes_us")
                    res["engine_1b"][f"k{k}_ctx{ctx}_s{S}"] = m
                    print(f"1B k={k} ctx={ctx} seqs={S}", json.dumps(m), flush=True)
            eng.close()
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
