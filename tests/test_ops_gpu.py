"""GPU parity: every hand-written kernel, called through the C ABI, against the CPU oracle."""
import math

import numpy as np
import pytest
import torch

from oracle import llama_oracle as O
from oracle.weights import init_uniform as np_init_uniform
from test_attention_exact_gpu import assert_rms_close

pytestmark = pytest.mark.gpu

# vllm/ir/tolerances.py:13-24 — bf16 kernels: atol 1e-3, rtol 1.6e-2
ATOL, RTOL = 1e-3, 1.6e-2


def dev(x):
    return x.to(torch.bfloat16).cuda().contiguous()


def close(got, want, atol=ATOL, rtol=RTOL, what=""):
    got, want = got.float().cpu(), want.float().cpu()
    err = (got - want).abs()
    tol = atol + rtol * want.abs()
    bad = err > tol
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {err.max():.4g} " \
                          f"(at {np.unravel_index(int(err.argmax()), err.shape)}), want there {want.flatten()[err.argmax()]:.4g}"


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return O.r(torch.randn(*shape, generator=g) * scale)


@pytest.fixture(params=[2, 1], ids=["pair", "single"])
def gemm_variant(request):
    """2 = split-K sized to the device (default product path), 1 = every tile over its whole K."""
    from kubeai_b200 import lib
    lib().b200_set_gemm_variant(request.param)
    yield request.param
    lib().b200_set_gemm_variant(2)


@pytest.mark.parametrize("T,N,K", [
    (128, 256, 256),      # single k-range, multiple slabs
    (16, 128, 64),        # one tile, one k-block
    (1, 384, 512),        # decode with one token
    (40, 768, 512),       # mini-model qkv
    (128, 4096, 4096),    # o_proj shape: stream-K splits every tile
    (128, 6144, 4096),    # qkv shape
    (100, 1000, 520),     # ragged N (not /128), K not /64, T not /16
    (300, 512, 1024),     # two token tiles (256 + 44)
    (50, 1004, 256),      # output leading dimension not a multiple of 8: per-thread stores instead of TMA
    (700, 640, 384),      # three token tiles
    (64, 4096, 14336),    # down_proj shape (deep K)
    (33, 130, 72),
    (384, 1024, 512),     # 512-token tile: 256 + 128 (two MMA chunks per k-step in the pair kernel)
    (400, 28672, 4096),   # gate_up at a mixed decode+prefill step
    (512, 768, 1024),
    (1100, 512, 256),     # three 512-token tiles (512 + 512 + 76)
])
def test_gemm_matches_oracle(T, N, K, gemm_variant):
    from kubeai_b200 import ops
    x, w = rnd(T, K, seed=1), rnd(N, K, scale=1 / math.sqrt(K), seed=2)
    got = ops.gemm(dev(x), dev(w))
    torch.cuda.synchronize()
    want = O.gemm(x, w)
    # fp32 accumulation order differs (stream-K partial sums): allow one bf16 ulp on top of vLLM's tolerance
    close(got, want, atol=2e-3, rtol=RTOL, what=f"gemm {T}x{N}x{K}")


@pytest.mark.parametrize("T,N,K", [(128, 4096, 4096), (1, 512, 512), (40, 768, 512), (100, 1000, 520), (384, 2048, 1024),
                                   (512, 28672, 4096), (128, 128256, 4096), (17, 4096, 14336),
                                   (2048, 4096, 4096), (1100, 768, 512), (700, 6144, 4096),
                                   (2048, 6144, 4096), (1800, 28672, 4096)])
def test_gemm_deferred_reduction_matches_oracle(T, N, K):
    """The engine's path: split-K partials summed in-kernel in split order."""
    from kubeai_b200 import ops
    x, w = rnd(T, K, seed=1), rnd(N, K, scale=1 / math.sqrt(K), seed=2)
    got = ops.gemm_deferred(dev(x), dev(w))
    torch.cuda.synchronize()
    close(got, O.gemm(x, w), atol=2e-3, rtol=RTOL, what=f"deferred gemm {T}x{N}x{K}")
    assert torch.equal(got, ops.gemm_deferred(dev(x), dev(w))), "fixed summation order => bit-reproducible"


def test_gemm_repeatable_and_counters_reset(gemm_variant):
    from kubeai_b200 import ops
    x, w = dev(rnd(128, 4096, seed=3)), dev(rnd(4096, 4096, scale=1 / 64, seed=4))
    a = ops.gemm(x, w)
    for _ in range(5):
        b = ops.gemm(x, w)
        assert torch.equal(a, b), "stream-K fix-up must be deterministic and self-resetting"


def test_gemm_deferred_rejects_unaligned_output_rows():
    """Consumers of deferred partials read the dense tiles 16 bytes at a time: N % 8 != 0 is refused, not mis-read."""
    from kubeai_b200 import B200Error, ops
    with pytest.raises(B200Error):
        ops.gemm_deferred(dev(rnd(50, 256, seed=1)), dev(rnd(1004, 256, seed=2)))


def test_embed_silu_argmax():
    from kubeai_b200 import ops
    table = rnd(300, 512, seed=8)
    ids = torch.tensor([0, 299, 5, 5, 17], dtype=torch.int32)
    assert torch.equal(ops.embed(dev(table), ids.cuda()).float().cpu(), table[ids.long()])
    gu = rnd(9, 2 * 1024, scale=2.0, seed=9)
    close(ops.silu_mul(dev(gu)), O.silu_and_mul(gu), what="silu_mul")
    logits = rnd(6, 1000, seed=10)
    logits[2, 77] = logits[2, 500] = 9.0     # tie: lowest index wins
    logits[3, 999] = 11.0                    # tail element (V not /8 handled too)
    got = ops.argmax(dev(logits)).cpu()
    assert got.tolist() == torch.argmax(logits, dim=-1).tolist()
    assert got[2] == 77 and got[3] == 999


def test_init_uniform_matches_numpy_replica():
    from kubeai_b200 import ops
    from oracle.weights import bf16_bits_to_f32
    for n, seed, scale, off in [(1000, 1, 1.0, 0.0), (4096 * 33 + 5, 0xDEADBEEF, 0.0156, 0.0), (777, 5, 0.1, 1.0)]:
        got = ops.init_uniform(n, seed, scale, off).float().cpu().numpy()
        want = bf16_bits_to_f32(np_init_uniform(n, seed, scale, off))
        assert np.array_equal(got, want), (n, seed)


def _paged_setup(seq_lens, q_lens, Hq=4, Hkv=1, seed=0, nblocks=64, want_raw=False):
    """Random q/k/v for several sequences; writes K/V through the rope_kvwrite kernel into a
    shuffled page pool.  Returns everything needed to call paged_attn and the oracle."""
    from kubeai_b200 import ops
    from oracle.weights import ModelCfg, cos_sin_cache
    g = torch.Generator().manual_seed(seed)
    D = 128
    cs = O.r(torch.from_numpy(cos_sin_cache(ModelCfg(max_model_len=max(seq_lens) + 1))))
    perm = torch.randperm(nblocks, generator=g).tolist()
    max_blocks = (max(seq_lens) + 15) // 16
    btab = torch.zeros(len(seq_lens), max_blocks, dtype=torch.int32)
    kv = torch.zeros(nblocks, 2, Hkv, 16, D, dtype=torch.bfloat16).cuda()
    seqs, raws = [], []
    for s, L in enumerate(seq_lens):
        nb = (L + 15) // 16
        blocks = [perm.pop() for _ in range(nb)]
        btab[s, :nb] = torch.tensor(blocks, dtype=torch.int32)
        qkv = O.r(torch.randn(L, (Hq + 2 * Hkv) * D, generator=g))
        pos = torch.arange(L, dtype=torch.int32)
        slots = torch.tensor([blocks[p // 16] * 16 + p % 16 for p in range(L)], dtype=torch.int32)
        dq = dev(qkv)
        raws.append(qkv)
        ops.rope_kvwrite(dq, pos.cuda(), slots.cuda(), dev(cs), kv, Hq, Hkv)
        q = O.rope_neox(qkv[:, :Hq * D].reshape(L, Hq, D), pos.long(), cs)
        k = O.rope_neox(qkv[:, Hq * D:(Hq + Hkv) * D].reshape(L, Hkv, D), pos.long(), cs)
        v = qkv[:, (Hq + Hkv) * D:].reshape(L, Hkv, D)
        # the oracle's attention inputs are the kernel's own rotated q/k (RoPE itself is checked
        # bit-exactly in test_elementwise_exact_gpu.py), so attention parity is not coupled to RoPE rounding
        q_dev = dq[:, :Hq * D].float().cpu().reshape(L, Hq, D)
        k_dev = dq[:, Hq * D:(Hq + Hkv) * D].float().cpu().reshape(L, Hkv, D)
        close(q_dev, q, what="rope(q)")
        close(k_dev, k, what="rope(k)")
        q, k = q_dev, k_dev
        seqs.append((dq, q, k, v, blocks))
    # paged cache content check
    kvc = kv.float().cpu()
    for s, L in enumerate(seq_lens):
        _, _, k, v, blocks = seqs[s]
        for p in (0, L // 2, L - 1):
            assert torch.equal(kvc[blocks[p // 16], 0, :, p % 16], k[p]), "K page write"
            assert torch.equal(kvc[blocks[p // 16], 1, :, p % 16], v[p]), "V page write"
    if want_raw:
        return kv, btab.cuda(), seqs, raws, cs
    return kv, btab.cuda(), seqs


@pytest.mark.parametrize("seq_lens", [[1], [16], [17, 64, 65], [200, 3, 129, 500]])
@pytest.mark.parametrize("Hkv", [1, 2])
def test_paged_attention_decode(seq_lens, Hkv):
    from kubeai_b200 import ops
    Hq = 4 * Hkv
    kv, btab, seqs = _paged_setup(seq_lens, None, Hq, Hkv, seed=11, nblocks=sum((l + 15) // 16 for l in seq_lens) + 5)
    # batch: the LAST token of every sequence is the decode query
    rows = torch.cat([s[0][-1:] for s in seqs], dim=0).contiguous()
    work = torch.tensor([[i, 1, L - 1, i] for i, L in enumerate(seq_lens)], dtype=torch.int32).cuda()
    got = ops.paged_attn(rows, kv, btab, work, Hq, Hkv, decode=True)
    torch.cuda.synchronize()
    for i, L in enumerate(seq_lens):
        _, q, k, v, _ = seqs[i]
        want = O.attention(q[-1:], k, v, torch.tensor([L - 1]), 128 ** -0.5).reshape(1, Hq * 128)
        close(got[i:i + 1], want, atol=4e-3, what=f"decode attn seq {i} len {L}")
        assert_rms_close(got[i:i + 1], want, f"decode attn seq {i} len {L}")


@pytest.mark.parametrize("case", [
    [(40, 40)],                                 # one partial block, no cached prefix
    [(64, 64)],                                 # exactly one block, one kv tile
    [(100, 37), (16, 16)],                      # 37 new tokens on 63 cached; a 16-token prompt
    [(300, 130), (65, 1), (33, 33)],            # three blocks (64 + 64 + 2) on 170 cached; a 1-token chunk
    [(513, 200), (129, 129)],
])
@pytest.mark.parametrize("Hkv", [1, 2])
def test_paged_attention_prefill_tensor_core(case, Hkv):
    """64-query prefill work items of the wgmma kernel, against the oracle."""
    from kubeai_b200 import ops
    Hq = 4 * Hkv
    seq_lens = [c[0] for c in case]
    kv, btab, seqs = _paged_setup(seq_lens, None, Hq, Hkv, seed=13, nblocks=sum((l + 15) // 16 for l in seq_lens) + 3)
    rows, work, spans = [], [], []
    tok = 0
    for i, (L, n) in enumerate(case):
        rows.append(seqs[i][0][L - n:])
        for j in range(0, n, 64):
            work.append([tok + j, min(64, n - j), L - n + j, i])
        spans.append((tok, n))
        tok += n
    rows = torch.cat(rows, dim=0).contiguous()
    got = ops.paged_attn_prefill_tc(rows, kv, btab, torch.tensor(work, dtype=torch.int32).cuda(), Hq, Hkv)
    torch.cuda.synchronize()
    for i, (L, n) in enumerate(case):
        _, q, k, v, _ = seqs[i]
        want = O.attention(q[L - n:], k, v, torch.arange(L - n, L), 128 ** -0.5).reshape(n, Hq * 128)
        t0 = spans[i][0]
        close(got[t0:t0 + n], want, atol=4e-3, what=f"tensor-core prefill attn seq {i} (ctx {L}, new {n})")
        assert_rms_close(got[t0:t0 + n], want, f"tensor-core prefill attn seq {i} (ctx {L}, new {n})")
