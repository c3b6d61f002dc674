#!/usr/bin/env python
"""What prompt logprobs cost in 1536-token prefill steps of Llama-3-8B (seeded random weights, full size).

  python scripts/prompt_logprobs_step.py [--steps 4] [--repeat 10] [--json OUT.json]

For each mode, --steps prompts of 1536 tokens are submitted with max_tokens 1; the engine's budget of 1536 tokens makes each
of them one prefill step with 1535 prompt-logprob rows (three groups of at most 512 through the final norm, the lm_head and
the ranked log-softmax).  Those steps are recorded and replayed from their HBM-resident inputs (b200_engine_replay, CUDA
events around --repeat back-to-back passes).  The modes are prompt logprobs off, then N = 0, 1 and 20, then off again, so
clock drift over the run shows as a difference between the two off runs.  Printed per mode: device time per step, its change
per prompt position against the mean of the off runs, and per step the time of the lm_head class (B200_K_GEMM_LM) and of
the token-selection class (B200_K_ARGMAX, which counts the log-softmax launches) from b200_engine_profile_range (an event
pair around every launch, run separately).  The prefix cache is off, so every mode computes every position.  The card's
name, power limit and max SM clock are read in the same process."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

T = 1536
MODES = [("off", None), ("n0", 0), ("n1", 1), ("n20", 20), ("off_again", None)]


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def run_mode(eng, prompts, n, repeat):
    K = len(prompts)
    rids = [eng.submit(p, max_tokens=1, ignore_eos=True, prompt_logprobs=n) for p in prompts]
    for _ in range(K):
        ran, info = eng.step()
        assert ran and info.tokens == T and info.prefill_seqs == 1, (info.tokens, info.prefill_seqs)
    for rid in rids:
        assert eng.poll(rid).finished
        if n is not None:
            assert eng.poll_prompt_logprobs(rid, T, n) is not None
        eng.release(rid)
    eng.replay(K, 1)                               # warm
    r = eng.replay(K, repeat)
    prof, tot = eng.profile_range(K, T, T)
    assert tot["steps"] == K
    return dict(step_ms=r["ms"] / (K * repeat), launches_per_step=r["launches"] / (K * repeat),
                lm_head_us_per_step=prof["gemm_lm_head"]["us"] / K, select_us_per_step=prof["argmax"]["us"] / K,
                norm_us_per_step=prof["rmsnorm"]["us"] / K)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--repeat", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from kubeai_b200.engine import Engine, default_config

    assert torch.cuda.is_available(), "needs a GPU"
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, 128256, T).tolist() for _ in range(args.steps)]
    eng = Engine(default_config(manual_step=1, record_steps=args.steps, max_num_seqs=8, max_batched_tokens=T,
                                max_model_len=2048, kv_fraction=0.80, enable_prefix_caching=0))
    res = {"card": card(), "step_tokens": T, "prompt_rows_per_step": T - 1, "steps": args.steps, "repeat": args.repeat}
    for name, n in MODES:
        res[name] = run_mode(eng, prompts, n, args.repeat)
        print(name, json.dumps(res[name]), flush=True)
    eng.close()
    off = (res["off"]["step_ms"] + res["off_again"]["step_ms"]) / 2
    for name, n in MODES[1:-1]:
        res[name]["added_us_per_prompt_position"] = (res[name]["step_ms"] - off) * 1000 / (T - 1)
    print(json.dumps(res), flush=True)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
