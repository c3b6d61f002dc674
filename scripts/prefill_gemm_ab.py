#!/usr/bin/env python
"""Prefill-step projection GEMMs of Llama-3-8B, one tree at a time: kernel time, TFLOP/s, share of the bf16 peak and a
digest of every output, so that two trees run one after the other can be compared for speed and for identical bits.

  python scripts/prefill_gemm_ab.py --root .            # this tree's kubeai_b200
  python scripts/prefill_gemm_ab.py --root OTHER_TREE   # another checkout, built in place

Each projection runs at every step size in --tokens, with the epilogue the engine fuses into it (qkv: RoPE + KV-cache
write, o / down: residual add, gate_up: SiLU * up) and as the plain product.  Each launch is timed with its own pair of
CUDA events, and L2 is overwritten before each launch: in the engine the 15 GB of weights stream from HBM every step.
Inputs are seeded; the digests come from one launch on fresh inputs before the timed ones."""
from __future__ import annotations

import argparse
import hashlib
import json
import math
import subprocess
import sys
from pathlib import Path

SHAPES = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336)}
HQ, HKV, MAX_POS = 32, 8, 2048


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def peak_tflops(root: Path):
    p = root / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return float(d.get("bf16_tflops_sustained", d.get("bf16_tflops"))), "measured"
    return 989.0, "H100 SXM data sheet (dense BF16)"


def digest(*tensors):
    import torch
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.contiguous().view(-1).view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", required=True, help="repository tree whose kubeai_b200 (built in place) is measured")
    ap.add_argument("--tokens", default="200,384,512,768,1024,1340,1536")
    ap.add_argument("--iters", type=int, default=50, help="timed launches per case (each after an L2 flush)")
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    root = Path(args.root).resolve()
    sys.path.insert(0, str(root))
    import torch
    from kubeai_b200 import ops
    import kubeai_b200
    assert Path(kubeai_b200.__file__).resolve().is_relative_to(root), kubeai_b200.__file__
    assert torch.cuda.is_available(), "this script measures the GPU"

    epi_name = {ops.EPI_PLAIN: "plain", ops.EPI_ROPE_KV: "rope_kv", ops.EPI_RESADD: "resadd", ops.EPI_SILU: "silu"}
    peak, peak_src = peak_tflops(root)
    print(json.dumps({"root": str(root), **card(), "peak_tflops": peak, "peak_source": peak_src}), flush=True)
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g, device=dev) * scale).bfloat16()

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)      # 256 MB: five times the H100's 50 MB L2
    gcpu = torch.Generator().manual_seed(1)
    cos_sin = rnd(MAX_POS, 128)
    weights = {name: rnd(n, k, scale=1 / math.sqrt(k)) for name, (n, k) in SHAPES.items()}
    for T in [int(t) for t in args.tokens.split(",")]:
        positions = torch.randint(0, MAX_POS, (T,), generator=gcpu, dtype=torch.int32).to(dev)
        nblocks = (T + 15) // 16 + 4
        slots = torch.randperm(nblocks * 16, generator=gcpu)[:T].to(torch.int32).to(dev)
        for name, (N, K) in SHAPES.items():
            w = weights[name]
            x = rnd(T, K)
            epi = {"qkv": ops.EPI_ROPE_KV, "o": ops.EPI_RESADD, "gate_up": ops.EPI_SILU, "down": ops.EPI_RESADD}[name]
            res0 = rnd(T, N, scale=2.0) if epi == ops.EPI_RESADD else None
            for e in (ops.EPI_PLAIN, epi):
                if e == ops.EPI_ROPE_KV:
                    out = torch.zeros(T, N, dtype=torch.bfloat16, device=dev)
                    kv = torch.zeros(nblocks, 2, HKV, 16, 128, dtype=torch.bfloat16, device=dev)
                    kw = dict(epi=e, out=out, positions=positions, slots=slots, cos_sin=cos_sin, kv_layer=kv, q_heads=HQ, kv_heads=HKV)
                    outputs = lambda r: (out, kv)      # noqa: E731
                elif e == ops.EPI_RESADD:
                    res, ssq = res0.clone(), torch.zeros(T, N // 128, dtype=torch.float32, device=dev)
                    kw = dict(epi=e, out=res, ssq_out=ssq)
                    outputs = lambda r: r              # noqa: E731  (residual, per-slab sums of squares)
                else:
                    kw = dict(epi=e)
                    outputs = lambda r: (r,)           # noqa: E731
                r, sch = ops.gemm3(x, w, **kw)
                torch.cuda.synchronize()
                dg = digest(*outputs(r))
                for _ in range(args.warmup):
                    ops.gemm3(x, w, **kw)
                evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
                for a, b in evs:
                    flush.add_(1)
                    a.record()
                    ops.gemm3(x, w, **kw)
                    b.record()
                torch.cuda.synchronize()
                us = sorted(a.elapsed_time(b) * 1e3 for a, b in evs)
                mean = sum(us) / len(us)
                tf = 2.0 * T * N * K / (mean * 1e-6) / 1e12
                print(json.dumps({"proj": name, "T": T, "epi": epi_name[e], "schedule": list(sch),
                    "us": round(mean, 2), "us_min": round(us[0], 2), "us_median": round(us[len(us) // 2], 2),
                    "tflops": round(tf, 1), "frac": round(tf / peak, 4), "sha256": dg}), flush=True)


if __name__ == "__main__":
    main()
