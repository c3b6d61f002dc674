"""GPU parity of the fused projection GEMM (kubeai_b200/csrc/gemm_wgmma.cu) through the C ABI (b200_op_gemm3): the plain
product against the oracle's GEMM for every reduction schedule (1..4 K-splits per tile, split counts sized to the device,
chosen split counts; the partials summed in-kernel in split order), then every prologue / epilogue mode
against the oracle's op applied to the kernel's own plain output — bit-exact, because the fused modes must round exactly
where the separate kernels (and the reference backend) round."""
import math

import numpy as np
import pytest
import torch

from oracle import llama_oracle as O

pytestmark = pytest.mark.gpu
ATOL, RTOL = 1e-3, 1.6e-2      # vllm/ir/tolerances.py:13-24 (bf16 kernels)


def dev(x):
    return x.to(torch.bfloat16).cuda().contiguous()


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).bfloat16()


def ref_gemm(x, w):
    """The oracle's GEMM (fp32 accumulate, one bf16 rounding) evaluated with torch fp32 on the GPU (TF32 off)."""
    assert not torch.backends.cuda.matmul.allow_tf32
    return O.gemm(x.float(), w.float())


def close(got, want, what=""):
    got, want = got.float(), want.float()
    err = (got - want).abs()
    tol = ATOL + RTOL * want.abs()
    bad = err > tol
    assert not bool(bad.any()), f"{what}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {float(err.max()):.4g}"
    # a bf16 GEMM output is ONE rounding of the fp32 sum: apart from the fp32 summation order it must be the oracle's value,
    # i.e. within one bf16 ulp — measured against max(|value|, rms / 8): an output near zero is the cancellation of terms
    # of the row's typical size, and its fp32 summation noise is far above its own (tiny) ulp
    floor = want.pow(2).mean().sqrt() / 8
    ulp = torch.exp2(torch.floor(torch.log2(torch.maximum(want.abs(), floor))) - 7)
    assert float((err / ulp).max()) <= 1.0 + 1e-3, f"{what}: more than one bf16 ulp from the oracle ({float((err / ulp).max()):.2f})"


SCHEDULES = [0, 1, 2, 3, 4]


@pytest.mark.parametrize("force", SCHEDULES)
@pytest.mark.parametrize("T,N,K", [
    (128, 512, 512),       # mini-model projections
    (1, 768, 512),
    (17, 768, 512),
    (128, 4096, 4096),     # o_proj
    (100, 6144, 4096),     # qkv, ragged T
    (33, 4096, 14336),     # down_proj, deep K
    (128, 2048, 1024),
    (64, 256, 256),        # one tile, 4 k-blocks
])
def test_plain_product_matches_oracle_for_every_cluster_schedule(T, N, K, force):
    from kubeai_b200 import B200Error, ops
    x, w = rnd(T, K, seed=1), rnd(N, K, scale=1 / math.sqrt(K), seed=2)
    try:
        got, sch = ops.gemm3(x, w, force=force)
    except B200Error:
        if force in (3, 4):       # more splits than k-blocks
            pytest.skip(f"schedule {force} not available for N={N} K={K}")
        raise
    torch.cuda.synchronize()
    if force:
        assert sch[0] == force and sch[1] == 0 and sch[2] == N // 256 * 2 * force
    close(got, ref_gemm(x, w), f"T={T} N={N} K={K} schedule {sch}")


@pytest.mark.parametrize("T,N,K,force", [
    (128, 28672, 4096, 0),      # gate_up: more slabs than SMs, whole-K tiles
    (77, 128256, 4096, 0),      # lm_head
    (128, 20480, 256, -1),      # split count from the device rule, 4 k-blocks per tile
    (50, 20480, 512, -7),       # 7 splits of 8 k-blocks: uneven pieces
    (128, 2560, 1024, -10),     # 10 splits of 16 k-blocks
    (16, 5120, 640, -9),
])
def test_plain_product_matches_oracle_under_stream_k(T, N, K, force):
    """Split-K over many tiles (the name predates the split-K kernel): device-sized and given split counts."""
    from kubeai_b200 import ops
    x, w = rnd(T, K, seed=3), rnd(N, K, scale=1 / math.sqrt(K), seed=4)
    for rep in range(3):          # repeated launches: the split-K arrival counters must reset after every launch
        got, sch = ops.gemm3(x, w, force=force)
        torch.cuda.synchronize()
        assert sch[1] == (1 if force in (0, -1) else 0) and (force in (0, -1) or sch[0] == -force)
        close(got, ref_gemm(x, w), f"T={T} N={N} K={K} schedule {sch} rep {rep}")


def _ssq(res):
    """per (token, 128-column slab) sum of squares, as the RESADD epilogue leaves it"""
    T, H = res.shape
    return res.float().reshape(T, H // 128, 128).pow(2).sum(-1).contiguous()


@pytest.mark.parametrize("force", [0, 1, 4, -1])
@pytest.mark.parametrize("T,N,K", [(128, 6144, 4096), (19, 768, 512), (128, 28672, 4096), (64, 20480, 256)])
def test_norm_prologue_equals_rmsnorm_then_gemm(T, N, K, force):
    """PRO_NORM: the B operand is RMSNorm(residual) computed in shared memory from the per-slab sums of squares."""
    from kubeai_b200 import B200Error, ops
    if (force == -1) != (N >= 20480):
        pytest.skip("the wide shapes with the device-sized split count, the narrow ones with given split counts")
    res = rnd(T, K, scale=2.0, seed=5)
    nw = (1.0 + 0.1 * torch.randn(K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))).bfloat16()
    w = rnd(N, K, scale=1 / math.sqrt(K), seed=7)
    try:
        got, sch = ops.gemm3(res, w, pro=ops.PRO_NORM, ssq_in=_ssq(res), norm_w=nw, eps=1e-5, force=force)
    except B200Error:
        if force == 4:
            pytest.skip("4 splits need at least 4 k-blocks")
        raise
    torch.cuda.synchronize()
    h = O.rms_norm(res.float(), nw.float(), 1e-5)
    # same kernel without the prologue on the oracle's normalised tile: the two must agree bit for bit unless a
    # normalised value sits on a bf16 rounding boundary (rsqrtf vs torch.rsqrt differ in the last fp32 bit)
    want_same_order, _ = ops.gemm3(h.bfloat16().contiguous(), w, force=force)
    torch.cuda.synchronize()
    diff = (got.float() - want_same_order.float()).abs()
    assert float((diff > 0).float().mean()) < 2e-3, f"{float((diff > 0).float().mean()):.4f} of the outputs differ from norm-then-GEMM"
    close(got, ref_gemm(h, w), f"norm prologue T={T} N={N} K={K} {sch}")


@pytest.mark.parametrize("force", [0, 2, 4])
@pytest.mark.parametrize("T,N,K", [(128, 4096, 4096), (128, 4096, 14336), (37, 512, 1024)])
def test_residual_add_epilogue(T, N, K, force):
    from kubeai_b200 import B200Error, ops
    x, w = rnd(T, K, seed=8), rnd(N, K, scale=1 / math.sqrt(K), seed=9)
    res0 = rnd(T, N, scale=2.0, seed=10)
    try:
        plain, _ = ops.gemm3(x, w, force=force)
        res = res0.clone()
        (res, ssq), sch = ops.gemm3(x, w, epi=ops.EPI_RESADD, out=res, force=force)
    except B200Error:
        if force == 4:
            pytest.skip("4 splits need at least 4 k-blocks")
        raise
    torch.cuda.synchronize()
    want = O.r(plain.float() + res0.float())                 # bf16(bf16(acc) + residual): the rounded sum is the new residual
    assert torch.equal(res.float(), want), f"residual differs in {int((res.float() != want).sum())} places ({sch})"
    want_ssq = _ssq(res)
    assert torch.allclose(ssq, want_ssq, rtol=1e-5, atol=1e-6), float((ssq - want_ssq).abs().max())


@pytest.mark.parametrize("force", [0, 1, 2])
@pytest.mark.parametrize("T,N,K", [(128, 4096, 4096), (128, 4096, 14336), (37, 512, 1024), (1, 512, 512)])
def test_residual_add_epilogue_with_the_next_norm_fused(T, N, K, force):
    """EPI_RESADD + fused RMSNorm: the new residual's norm needs every slab's sum of squares, i.e. all clusters of the
    launch (flag exchange at the end of the kernel); result = the oracle's fused_add_rms_norm on the kernel's own product."""
    from kubeai_b200 import ops
    x, w = rnd(T, K, seed=19), rnd(N, K, scale=1 / math.sqrt(K), seed=20)
    res0 = rnd(T, N, scale=2.0, seed=21)
    nw = (1.0 + 0.1 * torch.randn(N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(22))).bfloat16()
    plain, _ = ops.gemm3(x, w, force=force)
    for rep in range(3):
        res = res0.clone()
        (res, ssq, normed), sch = ops.gemm3(x, w, epi=ops.EPI_RESADD, out=res, norm_w_out=nw, force=force)
        torch.cuda.synchronize()
        want_h, want_res = O.fused_add_rms_norm(plain.float(), res0.float(), nw.float(), 1e-5)
        assert torch.equal(res.float(), want_res), f"residual ({sch})"
        bad = normed.float() != want_h
        # rsqrtf on the device vs torch.rsqrt: a few normalised values land on the other side of a bf16 boundary
        assert float(bad.float().mean()) < 2e-3, f"{int(bad.sum())} of {bad.numel()} normalised values differ ({sch}, rep {rep})"
        err = (normed.float() - want_h).abs()
        assert bool((err <= ATOL + RTOL * want_h.abs()).all())


def _interleave64(wg, wu):
    """gate rows and up rows interleaved in 64-row blocks: the engine's physical gate_up layout."""
    I, K = wg.shape
    return torch.stack([wg.reshape(I // 64, 64, K), wu.reshape(I // 64, 64, K)], dim=1).reshape(2 * I, K).contiguous()


@pytest.mark.parametrize("T,I,K,force", [(128, 14336, 4096, 0), (128, 1024, 512, 0), (45, 1024, 512, 2), (128, 10240, 256, -1)])
def test_silu_epilogue(T, I, K, force):
    from kubeai_b200 import ops
    x = rnd(T, K, seed=11)
    wg, wu = rnd(I, K, scale=1 / math.sqrt(K), seed=12), rnd(I, K, scale=1 / math.sqrt(K), seed=13)
    w = _interleave64(wg, wu)
    plain, sch = ops.gemm3(x, w, force=force)
    act, sch2 = ops.gemm3(x, w, epi=ops.EPI_SILU, force=force)
    torch.cuda.synchronize()
    assert sch == sch2
    p = plain.float().reshape(T, I // 64, 2, 64)
    gu = torch.cat([p[:, :, 0].reshape(T, I), p[:, :, 1].reshape(T, I)], dim=1)      # back to [gate | up]
    want = O.silu_and_mul(gu)
    bad = act.float() != want
    # expf on the device vs torch.exp: a handful of silu values may land on the other side of a bf16 boundary
    assert float(bad.float().mean()) < 1e-3, f"{int(bad.sum())} of {bad.numel()} differ"
    err = (act.float() - want).abs()
    assert bool((err <= ATOL + RTOL * want.abs()).all())
    close(plain, ref_gemm(x, w), "plain gate_up")


@pytest.mark.parametrize("T,Hq,Hkv,K,force", [(128, 32, 8, 4096, 0), (128, 4, 1, 512, 0), (50, 8, 2, 512, 2), (1, 4, 1, 512, 1)])
def test_rope_kv_epilogue_is_bit_exact_on_the_kernels_own_product(T, Hq, Hkv, K, force):
    from kubeai_b200 import ops
    from oracle.weights import ModelCfg, cos_sin_cache
    D = 128
    N = (Hq + 2 * Hkv) * D
    x, w = rnd(T, K, seed=14), rnd(N, K, scale=1 / math.sqrt(K), seed=15)
    max_pos = 2048
    cs = O.r(torch.from_numpy(cos_sin_cache(ModelCfg(max_model_len=max_pos)))).cuda()
    g = torch.Generator().manual_seed(16)
    pos = torch.randint(0, max_pos, (T,), generator=g, dtype=torch.int32)
    nblocks = T + 8
    slots = torch.randperm(nblocks * 16, generator=g)[:T].to(torch.int32)
    if T > 3:
        slots[3] = -1                                   # padding token: must not touch the cache
    kv = torch.zeros(nblocks, 2, Hkv, 16, D, dtype=torch.bfloat16, device="cuda")
    qkv = torch.zeros(T, N, dtype=torch.bfloat16, device="cuda")
    plain, sch = ops.gemm3(x, w, force=force)
    _, sch2 = ops.gemm3(x, w, epi=ops.EPI_ROPE_KV, out=qkv, positions=pos.cuda(), slots=slots.cuda(), cos_sin=dev(cs), kv_layer=kv,
                        q_heads=Hq, kv_heads=Hkv, force=force)
    torch.cuda.synchronize()
    assert sch == sch2
    p = plain.float()
    q = O.rope_neox(p[:, :Hq * D].reshape(T, Hq, D), pos.long().cuda(), cs)
    k = O.rope_neox(p[:, Hq * D:(Hq + Hkv) * D].reshape(T, Hkv, D), pos.long().cuda(), cs)
    v = p[:, (Hq + Hkv) * D:].reshape(T, Hkv, D)
    assert torch.equal(qkv[:, :Hq * D].float().reshape(T, Hq, D), q), "rotated q rows of the qkv buffer"
    kvc = kv.float()
    for t in range(T):
        s = int(slots[t])
        if s < 0:
            continue
        assert torch.equal(kvc[s // 16, 0, :, s % 16], k[t]), f"K page row of token {t}"
        assert torch.equal(kvc[s // 16, 1, :, s % 16], v[t]), f"V page row of token {t}"
    used = torch.zeros(nblocks * 16, dtype=torch.bool)
    used[slots[slots >= 0].long()] = True
    untouched = kvc.permute(0, 3, 1, 2, 4).reshape(nblocks * 16, 2, Hkv, D)[~used.cuda()]
    assert not bool(untouched.any()), "only the named slots are written"
    close(plain, ref_gemm(x, w), "plain qkv")


@pytest.mark.parametrize("T,N,K,force,n_valid", [(128, 128256, 4096, 0, 0), (128, 512, 512, 0, 0), (31, 512, 512, 2, 500),
                                                  (128, 20480, 256, -1, 20000)])
def test_argmax_epilogue_equals_argmax_of_the_plain_logits(T, N, K, force, n_valid):
    from kubeai_b200 import ops
    x, w = rnd(T, K, seed=17), rnd(N, K, scale=4 / math.sqrt(K), seed=18)
    plain, sch = ops.gemm3(x, w, force=force)
    ids, _ = ops.gemm3(x, w, epi=ops.EPI_ARGMAX, force=force, n_valid=n_valid)
    torch.cuda.synchronize()
    lg = plain.float()
    if n_valid:
        lg = lg[:, :n_valid]
    mx = lg.max(-1).values
    first = (lg == mx[:, None]).float().argmax(-1)           # the first maximum: lowest index wins ties
    assert torch.equal(ids.long(), first), f"{int((ids.long() != first).sum())} rows differ ({sch})"
    # constructed exact ties (duplicated weight rows): tests/test_sampling_exact_gpu.py


# ---------------------------------------------------------------------------------------------------------------------
# steps of more than 128 tokens: several token tiles per launch (force = requested token-tile size: the largest of
# 64 / 128 / 256 that does not exceed it),
# the same epilogues
LARGE = [
    (300, 4096, 4096, 0),       # two 256-token tiles, the last one ragged (44)
    (1408, 4096, 4096, 0),      # 6 token tiles, the last one ragged (128)
    (1536, 6144, 4096, 0),
    (700, 4096, 14336, 0),      # down_proj, deep K
    (129, 512, 512, 0),         # mini-model shapes
    (513, 768, 512, 0),
    (1000, 2560, 1024, 256),    # 256-token tiles given explicitly
    (2048, 28672, 4096, 0),     # gate_up at the largest step: 1792 tiles
    (1408, 4096, 4096, 384),    # a wider request than the widest tile: 256-token tiles (the largest supported <= 384)
    (1340, 6144, 4096, 384),    # ragged last tile
    (900, 28672, 4096, 384),
]


@pytest.mark.parametrize("T,N,K,bn", LARGE)
def test_large_step_plain_product_matches_oracle(T, N, K, bn):
    from kubeai_b200 import ops
    x, w = rnd(T, K, seed=31), rnd(N, K, scale=1 / math.sqrt(K), seed=32)
    for rep in range(2):
        got, sch = ops.gemm3(x, w, force=bn)
        torch.cuda.synchronize()
        assert sch[1] == 2 and sch[2] % ((N + 127) // 128) == 0
        close(got, ref_gemm(x, w), f"T={T} N={N} K={K} schedule {sch} rep {rep}")


@pytest.mark.parametrize("T,N,K,bn", [c for c in LARGE if c[1] <= 6144])
def test_large_step_residual_add_epilogue(T, N, K, bn):
    from kubeai_b200 import ops
    x, w = rnd(T, K, seed=33), rnd(N, K, scale=1 / math.sqrt(K), seed=34)
    res0 = rnd(T, N, scale=2.0, seed=35)
    plain, _ = ops.gemm3(x, w, force=bn)
    res = res0.clone()
    (res, _), sch = ops.gemm3(x, w, epi=ops.EPI_RESADD, out=res, force=bn)
    torch.cuda.synchronize()
    want = O.r(plain.float() + res0.float())
    assert torch.equal(res.float(), want), f"residual differs in {int((res.float() != want).sum())} places ({sch})"


@pytest.mark.parametrize("T,I,K", [(1408, 14336, 4096), (300, 1024, 512), (640, 2048, 1024)])
def test_large_step_silu_epilogue(T, I, K):
    from kubeai_b200 import ops
    x = rnd(T, K, seed=36)
    wg, wu = rnd(I, K, scale=1 / math.sqrt(K), seed=37), rnd(I, K, scale=1 / math.sqrt(K), seed=38)
    w = _interleave64(wg, wu)
    plain, _ = ops.gemm3(x, w)
    act, sch = ops.gemm3(x, w, epi=ops.EPI_SILU)
    torch.cuda.synchronize()
    p = plain.float().reshape(T, I // 64, 2, 64)
    gu = torch.cat([p[:, :, 0].reshape(T, I), p[:, :, 1].reshape(T, I)], dim=1)
    want = O.silu_and_mul(gu)
    bad = act.float() != want
    assert float(bad.float().mean()) < 1e-3, f"{int(bad.sum())} of {bad.numel()} differ ({sch})"
    err = (act.float() - want).abs()
    assert bool((err <= ATOL + RTOL * want.abs()).all())


@pytest.mark.parametrize("T,Hq,Hkv,K", [(1408, 32, 8, 4096), (200, 4, 1, 512), (777, 8, 2, 512)])
def test_large_step_rope_kv_epilogue(T, Hq, Hkv, K):
    from kubeai_b200 import ops
    from oracle.weights import ModelCfg, cos_sin_cache
    D = 128
    N = (Hq + 2 * Hkv) * D
    x, w = rnd(T, K, seed=39), rnd(N, K, scale=1 / math.sqrt(K), seed=40)
    max_pos = 2048
    cs = O.r(torch.from_numpy(cos_sin_cache(ModelCfg(max_model_len=max_pos)))).cuda()
    g = torch.Generator().manual_seed(41)
    pos = torch.randint(0, max_pos, (T,), generator=g, dtype=torch.int32)
    nblocks = (T + 15) // 16 + 8
    slots = torch.randperm(nblocks * 16, generator=g)[:T].to(torch.int32)
    slots[3] = -1
    kv = torch.zeros(nblocks, 2, Hkv, 16, D, dtype=torch.bfloat16, device="cuda")
    qkv = torch.zeros(T, N, dtype=torch.bfloat16, device="cuda")
    plain, _ = ops.gemm3(x, w)
    ops.gemm3(x, w, epi=ops.EPI_ROPE_KV, out=qkv, positions=pos.cuda(), slots=slots.cuda(), cos_sin=dev(cs), kv_layer=kv, q_heads=Hq, kv_heads=Hkv)
    torch.cuda.synchronize()
    p = plain.float()
    q = O.rope_neox(p[:, :Hq * D].reshape(T, Hq, D), pos.long().cuda(), cs)
    k = O.rope_neox(p[:, Hq * D:(Hq + Hkv) * D].reshape(T, Hkv, D), pos.long().cuda(), cs)
    v = p[:, (Hq + Hkv) * D:].reshape(T, Hkv, D)
    assert torch.equal(qkv[:, :Hq * D].float().reshape(T, Hq, D), q), "rotated q rows of the qkv buffer"
    kvc = kv.float().permute(0, 3, 1, 2, 4).reshape(nblocks * 16, 2, Hkv, D)      # [slot, k|v, head, d]
    ok = slots >= 0
    sl = slots[ok].long().cuda()
    assert torch.equal(kvc[sl, 0], k[ok.cuda()]), "K page rows"
    assert torch.equal(kvc[sl, 1], v[ok.cuda()]), "V page rows"
    used = torch.zeros(nblocks * 16, dtype=torch.bool)
    used[slots[ok].long()] = True
    assert not bool(kvc[~used.cuda()].any()), "only the named slots are written"
