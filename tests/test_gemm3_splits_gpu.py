"""The projection GEMM's split-K tail (kubeai_b200/csrc/gemm_wgmma.cu) at every split count S = 1..16 and step sizes
1 / 37 / 64 / 128: the S pieces of a tile run as clusters, reduce in split order and share the epilogue by token range.
Each fused epilogue must give the bits of the PLAIN launch at the same S followed by the standalone kernel, on capacity
buffers whose rows past T and columns past N carry a sentinel that must survive.  The split order itself is pinned by
inputs whose per-piece partials are exact and whose sum depends on the order the pieces are added in.

Shapes: N = 256 (two slabs) runs every S as one cluster per tile (sum over distributed shared memory); N = 4096 (32
slabs, o_proj's shape) has more clusters of S than a 132-SM H100 keeps resident from S = 4 on, so there the pieces pass
through the L2 workspace and clusters of a divisor of S (or single CTAs) finish the tile."""
import math

import pytest
import torch

from kernel_numerics import bf16_bits
from kubeai_b200 import ops
from oracle import llama_oracle as O
from oracle.weights import ModelCfg, cos_sin_cache

pytestmark = pytest.mark.gpu
ATOL, RTOL = 1e-3, 1.6e-2      # the oracle bound of test_gemm3_gpu.py
SENT = 0x5A5A                  # a bf16 no kernel writes here
PAD = 3                        # sentinel rows past every launch
K = 1024                       # 16 k-blocks: every S up to 16
SPLITS = list(range(1, 17))
STEPS = [1, 37, 64, 128]


def _sentinel(*shape, bits=SENT):
    return torch.full(shape, bits, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _inputs(T, N, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.empty(T + PAD, K, device="cuda")
    x[:T] = torch.randn(T, K, generator=g, device="cuda")
    x[T:] = float("nan")                                     # rows past T are never part of the product
    w = torch.randn(N, K, generator=g, device="cuda") * (scale / math.sqrt(K))
    return x.bfloat16(), w.bfloat16(), g


def _plain(x, w, T, S):
    out = _sentinel(T + PAD, w.shape[0] + 64)
    _, sch = ops.gemm3(x, w, T=T, out=out[:, :w.shape[0]], force=S)
    torch.cuda.synchronize()
    assert sch[0] == S and sch[1] == 0, sch
    assert bool((bf16_bits(out[T:]) == SENT).all()) and bool((bf16_bits(out[:, w.shape[0]:]) == SENT).all()), \
        f"S={S} T={T}: PLAIN wrote past row T or column N"
    return out[:T, :w.shape[0]].clone()


def _close(got, want, what):
    err = (got.float() - want.float()).abs()
    assert bool((err <= ATOL + RTOL * want.float().abs()).all()), f"{what}: max err {float(err.max()):.4g}"


@pytest.mark.parametrize("N", [256, 4096])
@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("S", SPLITS)
def test_plain_is_repeatable_and_within_the_oracle_bound(S, T, N):
    x, w, _ = _inputs(T, N, seed=S * 131 + T + N)
    a = _plain(x, w, T, S)
    b = _plain(x, w, T, S)
    assert torch.equal(bf16_bits(a), bf16_bits(b)), f"S={S} T={T} N={N}: two launches of the same inputs differ"
    _close(a, O.gemm(x[:T].float(), w.float()), f"S={S} T={T} N={N}")


def _warp_ssq(z, fused):
    """the RESADD epilogue's per-slab sum of squares of the bf16 residual z [T, N]: lane l sums rows 4l..4l+3 in order
    (fused: one fma per row), then the __shfl_xor butterfly over the 32 lanes"""
    T, N = z.shape
    v = z.float().reshape(T, N // 128, 32, 4)
    s = torch.zeros(T, N // 128, 32, device=z.device)
    for e in range(4):
        q = v[..., e]
        s = (q.double() * q.double() + s.double()).float() if fused else s + q * q
    lanes = torch.arange(32, device=z.device)
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., lanes ^ o]
    return s[..., 0].contiguous()


@pytest.mark.parametrize("N", [256, 4096])
@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("S", SPLITS)
def test_residual_add_equals_plain_then_add(S, T, N):
    x, w, g = _inputs(T, N, seed=S * 137 + T + N)
    plain = _plain(x, w, T, S)
    res0 = (torch.randn(T, N, generator=g, device="cuda") * 2).bfloat16()
    res = _sentinel(T + PAD, N)
    res[:T] = res0
    ssq = torch.full((T + PAD, N // 128), -7.5, device="cuda")
    ops.gemm3(x, w, T=T, epi=ops.EPI_RESADD, out=res, ssq_out=ssq, force=S)
    torch.cuda.synchronize()
    want = O.r(plain.float() + res0.float())
    assert torch.equal(res[:T].float(), want), f"S={S} T={T} N={N}: residual differs in {int((res[:T].float() != want).sum())}"
    assert bool((bf16_bits(res[T:]) == SENT).all()) and bool((ssq[T:] == -7.5).all()), f"S={S} T={T}: wrote past row T"
    got = ssq[:T].view(torch.int32)
    assert any(torch.equal(got, _warp_ssq(res[:T], f).view(torch.int32)) for f in (True, False)), \
        f"S={S} T={T} N={N}: ssq_out is not the per-slab sum of squares in the epilogue's order"


@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("S", SPLITS)
def test_residual_add_with_the_next_norm(S, T):
    """the fused RMSNorm waits for every slab's sums: the last of the token tile's CTAs to finish its share runs it"""
    N = 4096
    x, w, g = _inputs(T, N, seed=S * 139 + T)
    plain = _plain(x, w, T, S)
    res0 = (torch.randn(T, N, generator=g, device="cuda") * 2).bfloat16()
    nw = (1.0 + 0.1 * torch.randn(N, generator=g, device="cuda")).bfloat16()
    for rep in range(2):                                      # the arrival counters reset after every launch
        res = res0.clone()
        (res, _, normed), _ = ops.gemm3(x, w, T=T, epi=ops.EPI_RESADD, out=res, norm_w_out=nw, force=S)
        torch.cuda.synchronize()
        want_h, want_res = O.fused_add_rms_norm(plain.float(), res0.float(), nw.float(), 1e-5)
        assert torch.equal(res.float(), want_res), f"S={S} T={T} rep {rep}: residual"
        bad = normed.float() != want_h
        # rsqrtf on the device vs torch.rsqrt: a few values land on the other side of a bf16 boundary
        assert float(bad.float().mean()) < 2e-3, f"S={S} T={T} rep {rep}: {int(bad.sum())} normalised values differ"


@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("S", SPLITS)
def test_silu_equals_plain_then_silu_mul(S, T):
    I = 512
    x, w, _ = _inputs(T, 2 * I, seed=S * 149 + T)
    plain = _plain(x, w, T, S)
    act = _sentinel(T + PAD, I)
    ops.gemm3(x, w, T=T, epi=ops.EPI_SILU, out=act, force=S)
    want = ops.silu_mul(plain.contiguous(), interleaved=True)
    torch.cuda.synchronize()
    assert torch.equal(bf16_bits(act[:T]), bf16_bits(want)), f"S={S} T={T}: SiLU·up differs from the standalone kernel"
    assert bool((bf16_bits(act[T:]) == SENT).all()), f"S={S} T={T}: wrote past row T"


@pytest.mark.parametrize("D", [128, 64])
@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("S", SPLITS)
def test_rope_kv_equals_plain_then_rope_kvwrite(S, T, D):
    Hq, Hkv = (4, 2) if D == 128 else (8, 3)                  # D = 64 with an odd kv_heads: a slab holds a k and a v head
    N = (Hq + 2 * Hkv) * D
    x, w, g = _inputs(T, N, seed=S * 151 + T + D)
    plain = _plain(x, w, T, S)
    max_pos = 2048
    cs = O.r(torch.from_numpy(cos_sin_cache(ModelCfg(max_model_len=max_pos, head_dim=D)))).bfloat16().cuda()
    pos = torch.randint(-3, max_pos + 3, (T,), generator=g, device="cuda", dtype=torch.int32)
    nblocks = T // 16 + 4
    slots = torch.randperm(nblocks * 16, generator=g, device="cuda")[:T].to(torch.int32)
    slots[T // 2] = -1                                        # padding token: its page row stays untouched
    qkv = _sentinel(T + PAD, N)
    kv = _sentinel(nblocks, 2, Hkv, 16, D, bits=0x7FA5)      # a NaN
    ops.gemm3(x, w, T=T, epi=ops.EPI_ROPE_KV, out=qkv, positions=pos, slots=slots, cos_sin=cs, kv_layer=kv, q_heads=Hq,
              kv_heads=Hkv, head_dim=D, force=S)
    want_qkv = plain.contiguous()
    want_kv = _sentinel(nblocks, 2, Hkv, 16, D, bits=0x7FA5)
    ops.rope_kvwrite(want_qkv, pos, slots, cs, want_kv, Hq, Hkv, head_dim=D)
    torch.cuda.synchronize()
    assert torch.equal(bf16_bits(qkv[:T, :Hq * D]), bf16_bits(want_qkv[:, :Hq * D])), f"S={S} T={T} D={D}: rotated q rows"
    assert torch.equal(bf16_bits(kv), bf16_bits(want_kv)), f"S={S} T={T} D={D}: the KV pool differs from the standalone write"
    assert bool((bf16_bits(qkv[T:]) == SENT).all()) and bool((bf16_bits(qkv[:, Hq * D:]) == SENT).all()), \
        f"S={S} T={T} D={D}: wrote past row T or into the k / v columns"


@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("S", SPLITS)
def test_argmax_equals_argmax_of_plain(S, T):
    N, n_valid = 1024, 1000
    x, w, _ = _inputs(T, N, seed=S * 157 + T, scale=4.0)
    plain = _plain(x, w, T, S)
    ids = torch.full((T + PAD,), -7, dtype=torch.int32, device="cuda")
    ops.gemm3(x, w, T=T, epi=ops.EPI_ARGMAX, argmax_out=ids, n_valid=n_valid, force=S)
    torch.cuda.synchronize()
    lg = plain.float()[:, :n_valid]
    first = (lg == lg.max(-1).values[:, None]).float().argmax(-1)     # lowest index wins ties
    assert torch.equal(ids[:T].long(), first), f"S={S} T={T}: {int((ids[:T].long() != first).sum())} rows differ"
    assert bool((ids[T:] == -7).all()), f"S={S} T={T}: wrote past row T"


def _order_inputs(T, N, S, seed):
    """x [T, 64 S], w [N, 64 S] in bf16 such that piece s (k-block s, one per split) has an exact fp32 partial: every
    piece sees the same token block of small integers, and w's row n in piece s is small integers times 2^f(n, s).  Each
    row has one pair of pieces at 2^40 that cancel exactly and small pieces elsewhere, so adding the pieces in any order
    but p0 + p1 + .. + p(S-1) absorbs or keeps different small pieces in most rows."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(-3, 4, (T, 64), generator=g).double()
    b = torch.randint(-3, 4, (N, S, 64), generator=g).double()
    f = torch.randint(0, 5, (N, S), generator=g).double()
    pi = torch.randint(0, S, (N,), generator=g)
    pj = (pi + 1 + torch.randint(0, S - 1, (N,), generator=g)) % S
    rows = torch.arange(N)
    b[rows, pj] = -b[rows, pi]
    f[rows, pi] = 40
    f[rows, pj] = 40
    w = (b * torch.exp2(f)[:, :, None]).reshape(N, 64 * S)
    partials = torch.stack([a @ w[:, 64 * s:64 * (s + 1)].T for s in range(S)]).float()   # exact in fp32
    want = partials[0].clone()
    for s in range(1, S):
        want = want + partials[s]                             # fp32, in split order
    return a.repeat(1, S).bfloat16().cuda(), w.bfloat16().cuda(), want.bfloat16().cuda()


@pytest.mark.parametrize("N", [256, 4096])
@pytest.mark.parametrize("T", STEPS)
@pytest.mark.parametrize("S", SPLITS[2:])
def test_pieces_are_summed_in_split_order(S, T, N):
    """one k-block per piece and exact per-piece partials: the output is the fp32 left fold p0 + p1 + .. rounded once to
    bf16, whichever cluster size the launch takes (N = 256: the whole tile in one cluster; N = 4096: L2 shares)"""
    x, w, want = _order_inputs(T, N, S, seed=S * 163 + T + N)
    got = _plain(x, w, T, S)
    bad = bf16_bits(got) != bf16_bits(want)
    assert not bool(bad.any()), f"S={S} T={T} N={N}: {int(bad.sum())} of {bad.numel()} outputs are not the split-order sum"
