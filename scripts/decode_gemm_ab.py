#!/usr/bin/env python
"""Decode-step projection GEMMs of Llama-3-8B, one tree at a time: µs per launch, weight bytes/s, weight + token-tile
bytes/s out of L2, share of the HBM bandwidth and a digest of every output, so that two trees run one after the other can
be compared for speed and for identical bits.  The decode counterpart of prefill_gemm_ab.py.

  python scripts/decode_gemm_ab.py --root .            # this tree's kubeai_b200
  python scripts/decode_gemm_ab.py --root OTHER_TREE   # another checkout, built in place

Each projection runs at every step size in --tokens (all of them one token tile, T <= 128), with the epilogue the engine
fuses into it (qkv: RoPE + KV-cache write, o / down: residual add, gate_up: SiLU * up, lm_head: per-slab argmax) and as
the plain product.  Each launch is timed with its own pair of CUDA events after a read of a buffer five times the size of
L2: in the engine the 15 GB of weights stream from HBM every step, and the read leaves L2 holding clean lines only.  The
read also keeps the device busy while the host prepares the launch, so the events time the kernel alone.
Inputs are seeded; the digests come from one launch on fresh inputs before the timed ones."""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import math
import subprocess
import sys
from pathlib import Path

SHAPES = {"qkv": (6144, 4096), "o": (4096, 4096), "gate_up": (28672, 4096), "down": (4096, 14336), "lm_head": (128256, 4096)}
HQ, HKV, MAX_POS = 32, 8, 2048
HBM_GBS = 3350.0     # H100 SXM data sheet


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def digest(*tensors):
    import torch
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.contiguous().view(-1).view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def schedule(lib, N, K, T, sms):
    """(token-tile width, weight rows per CTA, CTAs) of the automatic schedule; a tree that does not report the rows
    (slot 6 zero) runs 128-row tiles"""
    out = (C.c_int32 * 8)()
    assert lib.b200_schedule_query(N, K, T, sms, out) == 0
    return out[0], out[6] or 128, out[4]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", required=True, help="repository tree whose kubeai_b200 (built in place) is measured")
    ap.add_argument("--tokens", default="1,32,64,128")
    ap.add_argument("--iters", type=int, default=200, help="timed launches per case (each after an L2 flush)")
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    root = Path(args.root).resolve()
    sys.path.insert(0, str(root))
    import torch
    from kubeai_b200 import lib, ops
    import kubeai_b200
    assert Path(kubeai_b200.__file__).resolve().is_relative_to(root), kubeai_b200.__file__
    assert torch.cuda.is_available(), "this script measures the GPU"

    epi_name = {ops.EPI_PLAIN: "plain", ops.EPI_ROPE_KV: "rope_kv", ops.EPI_RESADD: "resadd", ops.EPI_SILU: "silu",
                ops.EPI_ARGMAX: "argmax"}
    fused = {"qkv": ops.EPI_ROPE_KV, "o": ops.EPI_RESADD, "gate_up": ops.EPI_SILU, "down": ops.EPI_RESADD, "lm_head": ops.EPI_ARGMAX}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(json.dumps({"root": str(root), **card(), "sms": sms, "hbm_gbs": HBM_GBS, "hbm_source": "H100 SXM data sheet"}), flush=True)
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g, device=dev) * scale).bfloat16()

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev).fill_(1)   # 256 MB: five times the H100's 50 MB L2
    gcpu = torch.Generator().manual_seed(1)
    cos_sin = rnd(MAX_POS, 128)
    weights = {name: rnd(n, k, scale=1 / math.sqrt(k)) for name, (n, k) in SHAPES.items()}
    for T in [int(t) for t in args.tokens.split(",")]:
        assert 1 <= T <= 128, "decode steps: one token tile"
        positions = torch.randint(0, MAX_POS, (T,), generator=gcpu, dtype=torch.int32).to(dev)
        nblocks = (T + 15) // 16 + 4
        slots = torch.randperm(nblocks * 16, generator=gcpu)[:T].to(torch.int32).to(dev)
        for name, (N, K) in SHAPES.items():
            w = weights[name]
            x = rnd(T, K)
            res0 = rnd(T, N, scale=2.0) if fused[name] == ops.EPI_RESADD else None
            bn, rows, ctas = schedule(lib(), N, K, T, sms)
            w_bytes = 2 * N * K
            # every CTA reads its K range of the token tile; rows past T lie outside the token map and are not read
            x_l2_bytes = 2 * K * min(bn, T) * ((N + rows - 1) // rows)
            for e in (ops.EPI_PLAIN, fused[name]):
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
                sink = torch.zeros((), dtype=torch.int64, device=dev)
                for a, b in evs:
                    sink += flush.sum()
                    a.record()
                    ops.gemm3(x, w, **kw)
                    b.record()
                torch.cuda.synchronize()
                us = sorted(a.elapsed_time(b) * 1e3 for a, b in evs)
                mean = sum(us) / len(us)
                w_gbs = w_bytes / (mean * 1e-6) / 1e9
                l2_gbs = (w_bytes + x_l2_bytes) / (mean * 1e-6) / 1e9
                print(json.dumps({"proj": name, "T": T, "epi": epi_name[e], "schedule": list(sch), "block_n": bn, "rows": rows,
                    "us": round(mean, 2), "us_min": round(us[0], 2), "us_median": round(us[len(us) // 2], 2),
                    "weight_gbs": round(w_gbs, 1), "weight_plus_tile_gbs": round(l2_gbs, 1), "frac": round(w_gbs / HBM_GBS, 4),
                    "sha256": dg}), flush=True)


if __name__ == "__main__":
    main()
