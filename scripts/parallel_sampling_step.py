#!/usr/bin/env python
"""What parallel sampling (n) costs and saves on Llama-3-8B (seeded random weights, full size).

  python scripts/parallel_sampling_step.py [--groups 16] [--n 8] [--prompt 1000] [--max-tokens 4] [--json OUT.json]

The same work is run four ways on one engine configuration (max_num_seqs 128, a 1536-token step budget): --groups prompts
of --prompt tokens, each sampled --n times, submitted as --groups b200_submit_n groups or as groups * n separate requests,
each with the prefix cache on and off.  Every request generates --max-tokens tokens at temperature 0.8 with its own seed.
Printed per mode: steps, prompt tokens computed, the device time (CUDA events around each step's kernels,
b200_step_info.device_us) summed over the steps that compute prompt tokens, and for the group runs the mean device time of
the steps that fork a group.  Separately, b200_op_kv_copy_blocks is timed alone with CUDA events around --copy-repeat
launches of one n-member fork at the Llama-3-8B page shape: n - 1 pairs of 32 layers x 64 KiB (--copy-only: that
alone).  The card's name, power limit and max SM clock are read in the same process."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def run_mode(prompts, n, grouped, caching, max_tokens):
    from kubeai_b200.engine import Engine, default_config
    eng = Engine(default_config(manual_step=1, max_num_seqs=128, max_batched_tokens=1536, max_model_len=2048,
                                kv_fraction=0.80, enable_prefix_caching=1 if caching else 0))
    rids = []
    for g, p in enumerate(prompts):
        if grouped:
            rids += eng.submit_n(p, n, max_tokens=max_tokens, temperature=0.8, seed=1000 * g)
        else:
            rids += [eng.submit(p, max_tokens=max_tokens, temperature=0.8, seed=1000 * g + i) for i in range(n)]
    steps = prefill_us = prompt_tokens = 0
    fork_us = []
    while True:
        ran, info = eng.step()
        if not ran:
            break
        steps += 1
        if info.prefill_seqs:
            prefill_us += info.device_us
            prompt_tokens += info.tokens - info.decode_seqs
            # a step that forks samples more rows than it has sequences that complete a prompt or decode
            if grouped and info.sampled > info.decode_seqs + info.prefill_seqs:
                fork_us.append(info.device_us)
    for r in rids:
        assert eng.poll(r, cap=max_tokens).finished == "length"
        eng.release(r)
    st = eng.stats()
    eng.close()
    out = dict(steps=steps, prompt_tokens_computed=prompt_tokens, prefill_device_ms=prefill_us / 1000,
               stats_prompt_tokens=st.prompt_tokens, cached_prompt_tokens=st.cached_prompt_tokens,
               generated_tokens=st.generated_tokens)
    if grouped:
        out.update(fork_steps=len(fork_us), fork_step_device_us_mean=sum(fork_us) / max(len(fork_us), 1))
    return out


def time_copy(n, repeat):
    import ctypes as C
    import torch
    from kubeai_b200._lib import check, lib
    layers, block_bytes, nblocks = 32, 2 * 8 * 16 * 128 * 2, 64
    kv = torch.zeros(layers, nblocks, block_bytes // 2, dtype=torch.int16, device="cuda")
    src = torch.full((n - 1,), 5, dtype=torch.int32, device="cuda")
    dst = torch.arange(10, 10 + n - 1, dtype=torch.int32, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = (C.c_void_p(kv.data_ptr()), layers, nblocks * block_bytes, block_bytes, C.c_void_p(src.data_ptr()),
            C.c_void_p(dst.data_ptr()), n - 1, st)
    check(lib().b200_op_kv_copy_blocks(*args))   # warm
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(repeat):   # the page lists stay on the device: the launches queue back to back
        lib().b200_op_kv_copy_blocks(*args)
    b.record()
    torch.cuda.synchronize()
    us = a.elapsed_time(b) * 1000 / repeat
    moved = 2 * (n - 1) * layers * block_bytes   # read + written
    return dict(pairs=n - 1, us_per_fork=us, bytes_read_and_written=moved, achieved_TBps=moved / us / 1e6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=16)
    ap.add_argument("--n", type=int, default=8)
    ap.add_argument("--prompt", type=int, default=1000)
    ap.add_argument("--max-tokens", type=int, default=4)
    ap.add_argument("--copy-repeat", type=int, default=1000)
    ap.add_argument("--copy-only", action="store_true", help="time kv_copy_blocks alone")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, 128256, args.prompt).tolist() for _ in range(args.groups)]
    res = {"card": card(), "groups": args.groups, "n": args.n, "prompt_tokens": args.prompt, "max_tokens": args.max_tokens}
    res["kv_copy_blocks"] = time_copy(args.n, args.copy_repeat)
    print("kv_copy_blocks", json.dumps(res["kv_copy_blocks"]), flush=True)
    for grouped in (() if args.copy_only else (True, False)):
        for caching in (True, False):
            name = f"{'groups' if grouped else 'separate'}_cache_{'on' if caching else 'off'}"
            res[name] = run_mode(prompts, args.n, grouped, caching, args.max_tokens)
            print(name, json.dumps(res[name]), flush=True)
    print(json.dumps(res), flush=True)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
