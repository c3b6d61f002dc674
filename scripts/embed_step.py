"""Embedding step at e5-mistral-7b-instruct's shape (H100 only): a pooling engine with seeded weights (32 layers, hidden
4096, 32:8 heads of 128, intermediate 14336, vocab 32 000) embeds 256 prompts of 128 tokens in one 32 768-token step.

    python -m scripts.embed_step [--reps 5]

Prints one JSON line: prompt tokens/s and device time of the step (replayed), the pooled tail's time, and for comparison
the lm_head + argmax tail a generation engine runs on the same step (its B200_K_GEMM_LM + B200_K_ARGMAX classes), with the
card name and power limit read in the same call.  The pooled tail is the one pool_rows launch of the step (B200_K_NORM
holds the per-layer norms too), timed with CUDA events around b200_op_pool_rows over the same 256 rows of a [32768, 4096]
residual stream.
"""
from __future__ import annotations

import argparse
import json
import subprocess

import numpy as np

from kubeai_b200.engine import Engine, default_config

SHAPE = dict(num_layers=32, hidden=4096, q_heads=32, kv_heads=8, intermediate=14336, vocab=32000, max_model_len=512,
             max_num_seqs=256, max_batched_tokens=32768, num_kv_blocks=4096, manual_step=1, record_steps=1,
             enable_prefix_caching=0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def run(runner: int, prompts, reps: int):
    with Engine(default_config(runner=runner, **SHAPE)) as e:
        if runner:
            for p in prompts:
                e.submit_embed(p)
        else:
            for p in prompts:
                e.submit(p, max_tokens=1)
        ran, info = e.step()
        assert ran and info.tokens == sum(map(len, prompts)), info.tokens
        e.replay(1, 1)   # warm-up
        r = e.replay(1, reps)
        prof = {k: v["us"] for k, v in e.profile(1).items()}
        return r["ms"] / reps, prof


def pool_rows_us(rows: int, T: int, H: int, reps: int = 200) -> float:
    import ctypes as C

    import torch

    from kubeai_b200 import lib
    hid = torch.randn(T, H, device="cuda").to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(H, device="cuda")).to(torch.bfloat16)
    idx = (torch.arange(rows, dtype=torch.int32, device="cuda") + 1) * (T // rows) - 1   # each prompt's last token
    flags = torch.ones(rows, dtype=torch.int32, device="cuda")
    out = torch.empty(rows, H, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())
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
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    prompts = [rng.integers(0, SHAPE["vocab"], size=128).tolist() for _ in range(256)]
    T = sum(map(len, prompts))
    ms_p, _prof_p = run(1, prompts, a.reps)
    ms_g, prof_g = run(0, prompts, a.reps)
    print(json.dumps(dict(
        card=card(), tokens=T, prompts=len(prompts),
        pooling_step_ms=ms_p, prompt_tokens_per_s=T / (ms_p * 1e-3),
        pooled_tail_us=pool_rows_us(len(prompts), T, SHAPE["hidden"]),
        generate_step_ms=ms_g, lm_head_argmax_tail_us=prof_g["gemm_lm_head"] + prof_g["argmax"])))


if __name__ == "__main__":
    main()
