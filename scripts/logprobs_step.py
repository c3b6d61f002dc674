#!/usr/bin/env python
"""What logprobs cost in a 128-sequence decode step of Llama-3-8B (seeded random weights, full size).

  python scripts/logprobs_step.py [--steps 16] [--repeat 10] [--prompt 480] [--json OUT.json]

For each mode the same 128 prompts are prefilled, then --steps decode steps of 128 sequences are recorded and replayed
from their HBM-resident inputs (b200_engine_replay, CUDA events around --repeat back-to-back passes).  The modes are greedy
(the lm_head's argmax-candidate epilogue), greedy with logprobs at N = 0, 5 and 20 (plain lm_head + argmax_rows +
logprobs_rows), and temperature 0.8 / top_p 0.95 with N = 5 (sample_rows + logprobs_rows).  Greedy runs first and last, so
clock drift over the run shows as a difference between the two.  Printed per mode: device time per step, and per step the
time of the token-selection class (B200_K_ARGMAX, which counts logprobs_rows too) and of the lm_head from
b200_engine_profile_range (an event pair around every launch, run separately).  Then logprobs_rows alone over 128 rows at
V = 128256, N = 20, by a CUDA event pair around each launch, the rows first read by an argmax so they sit in L2 as they do
after the lm_head.  The card's name, power limit and max SM clock are read in the same process."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

MODES = [("greedy", {}), ("greedy_lp0", dict(logprobs=True)), ("greedy_lp5", dict(logprobs=True, top_logprobs=5)),
         ("greedy_lp20", dict(logprobs=True, top_logprobs=20)),
         ("T0.8_p0.95_lp5", dict(temperature=0.8, top_p=0.95, logprobs=True, top_logprobs=5)), ("greedy_again", {})]


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def run_mode(eng, prompts, sp, K, repeat):
    rids = [eng.submit(p, max_tokens=4096, ignore_eos=True, seed=1000 + i, **sp) for i, p in enumerate(prompts)]
    S = len(prompts)
    while True:                                    # prefill everything; stop once a step is decode-only at full batch
        ran, info = eng.step()
        assert ran
        if info.decode_seqs == S and info.prefill_seqs == 0:
            break
    for _ in range(K):
        ran, info = eng.step()
        assert ran and info.tokens == S and info.sampled == S
    eng.replay(min(K, 4), 1)                       # warm
    r = eng.replay(K, repeat)
    prof, tot = eng.profile_range(K, S, S)
    assert tot["steps"] == K
    for rid in rids:
        eng.abort(rid)
    while eng.step()[0]:
        pass
    for rid in rids:
        eng.release(rid)
    eng.reset_prefix_cache()                       # the replays overwrote KV pages the cache still points at
    return dict(step_ms=r["ms"] / (K * repeat), select_us_per_step=prof["argmax"]["us"] / K,
                select_launches_per_step=prof["argmax"]["launches"] / K,
                lm_head_us_per_step=prof["gemm_lm_head"]["us"] / K, launches_per_step=r["launches"] / (K * repeat))


def kernel_us(n):
    """logprobs_rows over 128 L2-warm rows of V = 128256 at N = 20: median of n event pairs, in us."""
    import numpy as np
    import torch
    from kubeai_b200 import ops
    from kubeai_b200._lib import check, lib
    S, V = 128, 128256
    g = torch.Generator().manual_seed(0)
    logits = (torch.randn(S, V, generator=g) * 3).bfloat16().cuda()
    ns = torch.full((S,), 20, dtype=torch.int32, device="cuda")
    tokens = torch.zeros(S, dtype=torch.int32, device="cuda")
    lp, top_lp = torch.empty(S, device="cuda"), torch.empty(S, 20, device="cuda")
    top_ids = torch.empty(S, 20, dtype=torch.int32, device="cuda")
    args = [ops._p(logits), V, S, V, ops._p(tokens), ops._p(ns), ops._p(lp), ops._p(top_ids), ops._p(top_lp), ops._stream()]
    check(lib().b200_op_logprobs(*args))
    times = []
    for _ in range(n):
        ops.argmax(logits)                          # leaves the rows in L2, as the lm_head does
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        check(lib().b200_op_logprobs(*args))
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1000)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--repeat", type=int, default=10)
    ap.add_argument("--seqs", type=int, default=128)
    ap.add_argument("--prompt", type=int, default=480, help="prompt tokens per sequence")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from kubeai_b200.engine import Engine, default_config

    assert torch.cuda.is_available(), "needs a GPU"
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, 128256, args.prompt).tolist() for _ in range(args.seqs)]
    eng = Engine(default_config(manual_step=1, record_steps=args.steps, max_num_seqs=args.seqs, max_batched_tokens=1536,
                                max_model_len=2048, kv_fraction=0.80))
    res = {"card": card(), "seqs": args.seqs, "prompt_tokens": args.prompt, "steps": args.steps, "repeat": args.repeat}
    for name, sp in MODES:
        res[name] = run_mode(eng, prompts, sp, args.steps, args.repeat)
        print(name, json.dumps(res[name]), flush=True)
    eng.close()
    res["logprobs_rows_128x128256_n20_us"] = kernel_us(args.repeat * 10)
    g = (res["greedy"]["step_ms"] + res["greedy_again"]["step_ms"]) / 2
    for name, _ in MODES[1:-1]:
        res[name]["added_us_per_step_vs_greedy"] = (res[name]["step_ms"] - g) * 1000
    print(json.dumps(res), flush=True)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
