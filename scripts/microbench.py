"""Per-kernel timings on the GPU (CUDA events, L2 flushed between iterations), with cuBLAS /
FlashInfer on the same box as the bars to beat (SURVEY.md Appendix B).  Not a bench.py number."""
import json
import math
import sys
import time

import torch

sys.path.insert(0, ".")
from kubeai_b200 import ops  # noqa: E402

PEAK = json.load(open("MEASURED_PEAKS.json"))["hbm_gbs"] if __import__("os").path.exists("MEASURED_PEAKS.json") else 6490.0
flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def gemm_bench():
    print("== GEMM (wgmma, split-K) vs cuBLAS, us median, L2 flushed")
    shapes = [("qkv", 6144, 4096), ("o", 4096, 4096), ("gate_up", 28672, 4096), ("down", 4096, 14336),
              ("lm_head", 128256, 4096)]
    for T in (16, 128, 256, 512, 2048):
        for name, N, K in shapes:
            if name == "lm_head" and T > 256:
                continue
            x = torch.randn(T, K, device="cuda").bfloat16()
            w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
            t_mine = timeit(lambda: ops.gemm(x, w))
            t_cublas = timeit(lambda: torch.nn.functional.linear(x, w))
            byts = (N * K + T * K + T * N) * 2
            fl = 2.0 * T * N * K
            print(f"T={T:5d} {name:8s} mine {t_mine:8.1f} us ({byts / t_mine / 1e3:7.0f} GB/s {byts / t_mine / 1e3 / PEAK:5.2f} of HBM, "
                  f"{fl / t_mine / 1e6:7.1f} TF/s)   cublas {t_cublas:8.1f} us ({byts / t_cublas / 1e3:7.0f} GB/s)  ratio {t_cublas / t_mine:5.2f}x")
            del x, w


def gemm3_bench():
    """fused GEMM (plain epilogue) vs the engine's op-level form vs cuBLAS, T <= 128"""
    print("== gemm3 (in-kernel split-K, T<=128) vs gemm2 deferred (+reducer) vs cuBLAS, us median, L2 flushed")
    shapes = [("qkv", 6144, 4096), ("o", 4096, 4096), ("gate_up", 28672, 4096), ("down", 4096, 14336), ("lm_head", 128256, 4096)]
    for T in (16, 64, 128):
        for name, N, K in shapes:
            x = torch.randn(T, K, device="cuda").bfloat16()
            w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
            byts = (N * K + T * K + T * N) * 2
            res = {}
            for force in ([0] if N > 16384 else [1, 2, 3]):
                try:
                    sch = ops.gemm3(x, w, force=force)[1]
                    res[f"g3{sch}"] = timeit(lambda: ops.gemm3(x, w, force=force))
                except Exception as ex:  # noqa: BLE001
                    res[f"g3 force {force}"] = float("nan")
            t_def = timeit(lambda: ops.gemm_deferred(x, w))
            t_cublas = timeit(lambda: torch.nn.functional.linear(x, w))
            best = min(v for v in res.values() if v == v)
            print(f"T={T:4d} {name:8s} " + "  ".join(f"{k} {v:6.1f}" for k, v in res.items()) +
                  f" | best {best:6.1f} us = {byts / best / 1e3:6.0f} GB/s ({byts / best / 1e3 / PEAK:4.2f} of HBM) | gemm2+reduce {t_def:6.1f} | cublas {t_cublas:6.1f} "
                  f"ratio {t_cublas / best:4.2f}x")
            del x, w


def large_bench():
    """steps of more than 128 tokens: the wgmma GEMM with its fused epilogue (the engine's gate_up form, plain and
    SiLU epilogue) and with fp32 segments + the generic reducer (an upper bound for the engine's segment form, whose
    consumer does useful work while it sums) vs cuBLAS"""
    print("== large steps: wgmma GEMM (fused epilogue / plain) vs cuBLAS, us median, L2 flushed")
    tf_peak = json.load(open("MEASURED_PEAKS.json")).get("bf16_tflops", 0) if __import__("os").path.exists("MEASURED_PEAKS.json") else 0
    shapes = [("qkv", 6144, 4096), ("o", 4096, 4096), ("gate_up", 28672, 4096), ("down", 4096, 14336)]
    for T in (256, 512, 1408, 2048):
        for name, N, K in shapes:
            x = torch.randn(T, K, device="cuda").bfloat16()
            w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
            fl = 2.0 * T * N * K
            t_f = timeit(lambda: ops.gemm3(x, w))
            t_s = timeit(lambda: ops.gemm3(x, w, epi=ops.EPI_SILU)) if name == "gate_up" else float("nan")
            t_d = timeit(lambda: ops.gemm_deferred(x, w))
            t_c = timeit(lambda: torch.nn.functional.linear(x, w))
            print(f"T={T:5d} {name:8s} fused {t_f:7.1f} us ({fl / t_f / 1e6:6.0f} TF/s)  fused+silu {t_s:7.1f}  segments+reducer {t_d:7.1f}  "
                  f"cublas {t_c:7.1f} us ({fl / t_c / 1e6:6.0f} TF/s)  ratio {t_c / t_f:4.2f}x")
            del x, w


def attn_prefill_bench():
    """chunked-prefill attention (tensor-core kernel, 64-query work items) vs FlashInfer's paged prefill on burst-like shapes:
    (requests, cached prefix, new tokens)"""
    print("== paged prefill attention, Hq=32/Hkv=8: (requests x [cached + new]) mine (wgmma) / mine (mma.sync) / FlashInfer")
    Hq, Hkv, D = 32, 8, 128
    for nreq, cached, new in ((10, 320, 130), (4, 0, 384), (1, 0, 1536), (3, 1500, 500), (24, 400, 64)):
        ctx = cached + new
        pages = (ctx + 15) // 16
        nblk = nreq * pages
        kv = torch.randn(nblk, 2, Hkv, 16, D, device="cuda").bfloat16()
        perm = torch.randperm(nblk, device="cuda").to(torch.int32).reshape(nreq, -1).contiguous()
        T = nreq * new
        qkv = torch.randn(T, (Hq + 2 * Hkv) * D, device="cuda").bfloat16()
        res = {}
        for name, qb, fn in (("tc", 64, ops.paged_attn_prefill_tc), ("mma", 16, None)):
            work = []
            for r in range(nreq):
                for j in range(0, new, qb):
                    work.append([r * new + j, min(qb, new - j), cached + j, r])
            wt = torch.tensor(work, dtype=torch.int32, device="cuda")
            out = torch.zeros(T, Hq * D, dtype=torch.bfloat16, device="cuda")
            if fn is not None:
                res[name] = (timeit(lambda: fn(qkv, kv, perm, wt, Hq, Hkv, out=out)), out)
            else:
                res[name] = (timeit(lambda: ops.paged_attn(qkv, kv, perm, wt, Hq, Hkv, False, out=out)), out)
        line = f"{nreq:3d} x [{cached:4d} + {new:4d}]  wgmma {res['tc'][0]:7.1f} us   mma.sync {res['mma'][0]:7.1f} us"
        try:
            import flashinfer
            ws = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
            wr = flashinfer.BatchPrefillWithPagedKVCacheWrapper(ws, "HND")
            qo_indptr = torch.arange(0, nreq + 1, dtype=torch.int32, device="cuda") * new
            kv_indptr = torch.arange(0, nreq + 1, dtype=torch.int32, device="cuda") * pages
            last = torch.full((nreq,), (ctx - 1) % 16 + 1, dtype=torch.int32, device="cuda")
            wr.plan(qo_indptr, kv_indptr, perm.reshape(-1), last, Hq, Hkv, D, 16, causal=True, q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16)
            q = qkv[:, :Hq * D].reshape(T, Hq, D).contiguous()
            tf = timeit(lambda: wr.run(q, kv))
            o2 = wr.run(q, kv).reshape(T, Hq * D)
            line += f"   flashinfer {tf:7.1f} us   ratio {tf / res['tc'][0]:4.2f}x   max |mine - flashinfer| {float((res['tc'][1].float() - o2.float()).abs().max()):.4f}"
        except Exception as e:  # noqa: BLE001
            line += "   flashinfer unavailable: " + repr(e)[:160]
        print(line, flush=True)
        del kv


def attn_bench():
    print("== paged decode attention, B=128, Hq=32/Hkv=8")
    Hq, Hkv, D = 32, 8, 128
    for ctx in (256, 1024, 2048):
        B = 128
        nblk = B * ((ctx + 15) // 16)
        kv = (torch.randn(nblk, 2, Hkv, 16, D, device="cuda")).bfloat16()
        perm = torch.randperm(nblk, device="cuda").to(torch.int32).reshape(B, -1).contiguous()
        qkv = torch.randn(B, (Hq + 2 * Hkv) * D, device="cuda").bfloat16()
        work = torch.tensor([[i, 1, ctx - 1, i] for i in range(B)], dtype=torch.int32, device="cuda")
        out = torch.zeros(B, Hq * D, dtype=torch.bfloat16, device="cuda")
        t = timeit(lambda: ops.paged_attn(qkv, kv, perm, work, Hq, Hkv, True, out=out))
        byts = B * ctx * 2 * Hkv * D * 2
        print(f"ctx={ctx:5d} mine {t:8.1f} us  {byts / t / 1e3:7.0f} GB/s ({byts / t / 1e3 / PEAK:4.2f} of HBM)")
        try:
            import flashinfer
            ws = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
            wr = flashinfer.BatchDecodeWithPagedKVCacheWrapper(ws, "HND", use_tensor_cores=True)
            indptr = torch.arange(0, B + 1, dtype=torch.int32, device="cuda") * ((ctx + 15) // 16)
            last = torch.full((B,), (ctx - 1) % 16 + 1, dtype=torch.int32, device="cuda")
            wr.plan(indptr, perm.reshape(-1), last, Hq, Hkv, D, 16, q_data_type=torch.bfloat16, kv_data_type=torch.bfloat16)
            q = qkv[:, :Hq * D].reshape(B, Hq, D).contiguous()
            tf = timeit(lambda: wr.run(q, kv))
            print(f"          flashinfer {tf:8.1f} us  {byts / tf / 1e3:7.0f} GB/s   ratio {tf / t:5.2f}x")
            o2 = wr.run(q, kv).reshape(B, Hq * D)
            print("          max |mine - flashinfer| =", float((out.float() - o2.float()).abs().max()))
        except Exception as e:  # noqa: BLE001
            print("          flashinfer unavailable:", repr(e)[:200])
        del kv


def engine_bench():
    print("== Llama-3-8B engine, 128 seqs")
    from kubeai_b200.engine import Engine, default_config
    import numpy as np
    t0 = time.time()
    e = Engine(default_config(manual_step=1, record_steps=64, max_batched_tokens=2048, max_num_seqs=128,
                              max_model_len=2048, kv_fraction=0.5))
    print("engine create %.1fs, kv blocks %d" % (time.time() - t0, e.stats().kv_blocks_total))
    rng = np.random.default_rng(0)
    rids = [e.submit(rng.integers(0, 128000, size=int(rng.integers(300, 500))).tolist(), max_tokens=64) for _ in range(128)]
    groups = {"attention": ["attn_decode", "attn_prefill"], "rmsnorm": ["rmsnorm"], "rope_kvwrite": ["rope_kvwrite"], "silu_mul": ["silu_mul"],
              "gemm_qkv": ["gemm_qkv"], "gemm_o": ["gemm_o"], "gemm_gate_up": ["gemm_gate_up"], "gemm_down": ["gemm_down"],
              "all GEMMs": ["gemm_qkv", "gemm_o", "gemm_gate_up", "gemm_down", "gemm_lm_head"],
              "all elementwise": ["rmsnorm", "rope_kvwrite", "silu_mul", "embed", "argmax"]}

    def marginal(tag, n, rep):
        base = e.replay(n, rep)["ms"] / (n * rep)
        print(f"{tag} {base:.3f} ms; marginal cost when removed:")
        for name, cls in groups.items():
            e.set_skip_mask(cls)
            t = e.replay(n, rep)["ms"] / (n * rep)
            print(f"    {name:18s} {base - t:7.3f} ms")
        e.set_skip_mask(())

    for i in range(60):
        if i == 6:
            marginal("prefill step (T=2048, steps 3-5)", 3, 3)
        ran, info = e.step()
        if i < 30 or i % 10 == 0:
            print(f"step {i:3d} T={info.tokens:5d} dec={info.decode_seqs:4d} pre={info.prefill_seqs:3d} "
                  f"kv_read={info.kv_tokens_read:8d} dev={info.device_us / 1e3:7.3f} ms")
    r = e.replay(8, 3)
    per = r["ms"] / (8 * 3)
    byts = 15.009e9 + r["kv_tokens"] / 24 * 131072
    print(f"replay of last 8 decode steps x3: {per:.3f} ms/step, {r['sampled'] / 24 / per * 1e3:.0f} tok/s, "
          f"alg bytes/step {byts / 1e9:.2f} GB -> {byts / per / 1e6:.0f} GB/s ({byts / per / 1e6 / PEAK:.2f} of HBM), launches/step {r['launches'] / 24:.0f}")
    marginal("decode step", 8, 3)
    toks = e.poll(rids[0]).tokens
    print("first request tokens:", toks[:16])
    e.close()


if __name__ == "__main__":
    which = sys.argv[1:] or ["gemm", "attn", "engine"]
    print("HBM peak (measured):", PEAK)
    for w in which:
        try:
            globals()[w + "_bench"]()
        except Exception as ex:  # noqa: BLE001
            import traceback
            traceback.print_exc()
