#!/usr/bin/env python
"""What logits edits cost in a 128-sequence decode step of Llama-3-8B (seeded random weights, full size).

  python scripts/penalties_step.py [--steps 16] [--repeat 10] [--prompt 1000] [--json OUT.json]

For each mode the same 128 prompts are prefilled (so each edited row's record list holds about --prompt records), then
--steps decode steps of 128 sequences run live and are replayed from their HBM-resident inputs (b200_engine_replay, CUDA
events around --repeat back-to-back passes).  Modes: greedy; greedy with repetition_penalty 1.1; temperature 0.8 / top_p
0.95, plain and with presence 0.5, frequency 0.5 and a 20-entry logit_bias, and the same with min_p 0.05.  Greedy runs
first and last, so clock drift over the run shows as a difference between the two.  Printed per mode:
  - step_ms: replayed device time per step (the edit pass and the restore run in a replay; the history update does not);
  - live_step_us: device time of the live steps (b200_step_info.device_us), which include the history update;
  - select_us_per_step: the token-selection class (B200_K_ARGMAX) from b200_engine_profile_range, an event pair around
    every launch: for edited modes it holds the edit pass, the selection kernel and the restore, so the edit pass plus the
    restore is its growth over the unedited mode with the same selection kernel (edit_restore_us_per_step).
The card's name, power limit and max SM clock are read in the same process."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

BIAS = {int(t): (-1) ** t * 2.5 for t in range(1000, 21000, 1000)}          # 20 entries
SAMPLED = dict(temperature=0.8, top_p=0.95)
PEN = dict(presence_penalty=0.5, frequency_penalty=0.5, logit_bias=BIAS)
MODES = [("greedy", {}, None), ("greedy_rep1.1", dict(repetition_penalty=1.1), "greedy"),
         ("T0.8_p0.95", SAMPLED, None), ("T0.8_p0.95_pen_bias", {**SAMPLED, **PEN}, "T0.8_p0.95"),
         ("T0.8_p0.95_pen_bias_minp0.05", {**SAMPLED, **PEN, "min_p": 0.05}, "T0.8_p0.95"),
         ("greedy_again", {}, None)]


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
    live = 0.0
    for _ in range(K):
        ran, info = eng.step()
        assert ran and info.tokens == S and info.sampled == S
        live += info.device_us
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
    return dict(step_ms=r["ms"] / (K * repeat), live_step_us=live / K, select_us_per_step=prof["argmax"]["us"] / K,
                select_launches_per_step=prof["argmax"]["launches"] / K, launches_per_step=r["launches"] / (K * repeat))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--repeat", type=int, default=10)
    ap.add_argument("--seqs", type=int, default=128)
    ap.add_argument("--prompt", type=int, default=1000, help="prompt tokens per sequence")
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
    for name, sp, _ in MODES:
        res[name] = run_mode(eng, prompts, sp, args.steps, args.repeat)
        print(name, json.dumps(res[name]), flush=True)
    eng.close()
    g = (res["greedy"]["step_ms"] + res["greedy_again"]["step_ms"]) / 2
    for name, _, base in MODES[1:-1]:
        res[name]["added_us_per_step_vs_greedy"] = (res[name]["step_ms"] - g) * 1000
        if base:
            b = res[base]
            res[name]["added_us_per_step_vs_" + base] = (res[name]["step_ms"] - (g if base == "greedy" else b["step_ms"])) * 1000
            res[name]["edit_restore_us_per_step"] = res[name]["select_us_per_step"] - b["select_us_per_step"]
    print(json.dumps(res), flush=True)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
