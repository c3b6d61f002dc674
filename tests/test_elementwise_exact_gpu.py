"""The per-step elementwise kernels (kubeai_b200/csrc/elementwise.cu) held to exact answers at every launch shape the
engine uses: RMSNorm (rmsnorm_kernel<1..4>) and SiLU·up (silu_mul_kernel<1|2>, both gate_up layouts) against float64
through the checkers of tests/kernel_numerics.py, RoPE / KV write (rope_kv_kernel<64|128>) and the embedding gather bit
for bit; and the projection GEMM on the engine's capacity buffers, where rows past the step's T hold whatever an earlier
step left.  Output buffers are larger than the launch and carry a sentinel past it that must survive."""
import ctypes as C

import pytest
import torch

from kernel_numerics import bf16, bf16_bits, check_rmsnorm, check_silu, f32_bits, norm_launch, rope_expected
from kubeai_b200 import B200Error, lib, ops
from oracle import llama_oracle as O
from oracle.weights import ModelCfg, cos_sin_cache

pytestmark = pytest.mark.gpu
EPS = 1e-5
SENT = 0x5A5A                 # a bf16 no kernel writes here (about 1.5e16)
PAD = 3                       # sentinel rows past every launch


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _sentinel(*shape, bits=SENT):
    return torch.full(shape, bits, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def _untouched(t, bits=SENT):
    return bool((bf16_bits(t) == bits).all())


def _interleave64(g, u):
    """[gate | up] columns -> the engine's gate_up layout: 64 gate columns, their 64 up columns, ..."""
    T, I = g.shape
    return torch.stack([g.reshape(T, I // 64, 64), u.reshape(T, I // 64, 64)], dim=2).reshape(T, 2 * I).contiguous()


# ------------------------------------------------------------------------------------------------------------- RMSNorm
def _norm_rows(H, n, g):
    """n bf16 rows of N(0, 1); the last min(5, n - 1) are the hard rows: zero, eps-dominated (|v| ~ 1e-4), bf16 subnormals,
    constant, and a few massive-activation channels (+-1e4) among N(0, 1)."""
    x = torch.randn(n, H, generator=g, device="cuda")
    massive = torch.randn(H, generator=g, device="cuda")
    massive[torch.randperm(H, generator=g, device="cuda")[:4]] = torch.tensor([1e4, -1e4, 5e3, -2e4], device="cuda")
    hard = [torch.zeros(H, device="cuda"), torch.randn(H, generator=g, device="cuda") * 1e-4,
            torch.randn(H, generator=g, device="cuda") * 2.0 ** -130, torch.full((H,), -0.625, device="cuda"), massive]
    k = min(len(hard), n - 1)
    if k > 0:
        x[n - k:] = torch.stack(hard[:k])
    return x.bfloat16()


def _check_norm(v, w, out, what):
    ok, nonnearest = check_rmsnorm(v, w, out, EPS)
    assert bool(ok.all()), f"{what}: rows {(~ok).nonzero().flatten()[:8].tolist()} are no rounding of a float64 RMSNorm"
    return nonnearest


@pytest.mark.parametrize("rows", [1, 7, 511, 512, 1500])
@pytest.mark.parametrize("H", [256, 512, 1024, 2048, 3072, 4096, 5120, 6144, 8192])
def test_rmsnorm_matches_float64_at_every_launch_shape(H, rows):
    """H / 8 threads of one vector (32 to 1024 threads) and 256 threads of 1 to 4 vectors: plain, fused add, and gathered
    rows with and without a residual."""
    l = lib()
    g = torch.Generator(device="cuda").manual_seed(H * 31 + rows)
    x = _norm_rows(H, rows, g)
    res = (torch.randn(rows, H, generator=g, device="cuda") * 2).bfloat16()
    if rows > 1:
        res[0] = -x[0]                                     # the fused sum of this row is zero
    w = (1 + 0.1 * torch.randn(H, generator=g, device="cuda"))
    w[::97] *= -1
    w = w.bfloat16()
    n_nn = 0

    out = _sentinel(rows + PAD, H)
    assert l.b200_op_rmsnorm(_p(x), None, _p(w), _p(out), None, rows, H, C.c_float(EPS), None) == 0
    torch.cuda.synchronize()
    n_nn += _check_norm(x, w, out[:rows], "plain")
    assert _untouched(out[rows:]), "plain: rows past the launch were written"

    resbuf = _sentinel(rows + PAD, H)
    resbuf[:rows] = res
    out = _sentinel(rows + PAD, H)
    assert l.b200_op_rmsnorm(_p(x), _p(resbuf), _p(w), _p(out), None, rows, H, C.c_float(EPS), None) == 0
    torch.cuda.synchronize()
    z = bf16(x.float() + res.float())
    assert torch.equal(f32_bits(resbuf[:rows]), f32_bits(z)), "fused add: the residual is not bf16(x + res)"
    assert _untouched(resbuf[rows:]) and _untouched(out[rows:]), "fused add: rows past the launch were written"
    if rows > 1:
        assert not bool(z[0].any())
    n_nn += _check_norm(z, w, out[:rows], "fused add")

    idx = torch.randint(0, rows, (rows,), generator=g, device="cuda", dtype=torch.int32)
    idx[0] = rows - 1
    if rows > 2:
        idx[2] = idx[1]                                    # a repeated row
    for with_res in (False, True):
        resbuf = _sentinel(rows + PAD, H)
        resbuf[:rows] = res
        out = _sentinel(rows + PAD, H)
        assert l.b200_op_rmsnorm(_p(x), _p(resbuf) if with_res else None, _p(w), _p(out), _p(idx), rows, H,
                                 C.c_float(EPS), None) == 0
        torch.cuda.synchronize()
        v = (z if with_res else x)[idx.long()]
        n_nn += _check_norm(v, w, out[:rows], f"gathered, residual {with_res}")
        assert _untouched(out[rows:]), "gathered: rows past the launch were written"
        assert torch.equal(bf16_bits(resbuf[:rows]), bf16_bits(res)) and _untouched(resbuf[rows:]), \
            "gathered: the residual must not be written"
    threads, vpt = norm_launch(rows, H)
    print(f"rmsnorm H={H} rows={rows} ({threads} threads x {vpt} vectors): {n_nn} of {4 * rows} rows needed an inv other "
          f"than the fp32 nearest float64")


@pytest.mark.parametrize("H", [264, 16384])
def test_rmsnorm_refuses_unserved_widths(H):
    l = lib()
    x = torch.ones(4, H, dtype=torch.bfloat16, device="cuda")
    out = _sentinel(4, H)
    rc = l.b200_op_rmsnorm(_p(x), None, _p(x[0]), _p(out), None, 4, H, C.c_float(EPS), None)
    assert rc == -1, rc                                    # B200_ERR_INVALID, not a launch error
    assert b"rmsnorm" in l.b200_last_error()
    torch.cuda.synchronize()
    assert _untouched(out)


# ---------------------------------------------------------------------------------------------------------- SiLU * up
SILU_SHAPES = [(T, I) for T in (1, 9, 511, 512, 1500) for I in (64, 1024, 1088, 8192, 14336, 28672)] + [(65536, 64)]


@pytest.mark.parametrize("interleaved", [0, 1])
@pytest.mark.parametrize("T,I", SILU_SHAPES)
def test_silu_mul_matches_float64(T, I, interleaved):
    """silu_mul_kernel<1> below 512 tokens, <2> from 512; I = 1088 clamps the tail loads; T = 65536 is more tokens than
    gridDim.y holds."""
    g = torch.Generator(device="cuda").manual_seed(T * 3 + I + interleaved)
    gate = torch.where(torch.arange(I, device="cuda") % 2 == 0, torch.rand(T, I, generator=g, device="cuda") * 160 - 80,
                       torch.randn(T, I, generator=g, device="cuda") * 4)
    tail = torch.arange(I, device="cuda") % 16 == 5         # the far tail, where __fdividef flushes to 0
    gate = torch.where(tail, -87.5 - torch.rand(T, I, generator=g, device="cuda") * 300, gate).bfloat16()
    up = (torch.randn(T, I, generator=g, device="cuda") * 2).bfloat16()
    gu = _interleave64(gate, up) if interleaved else torch.cat([gate, up], dim=1).contiguous()
    out = _sentinel(T + PAD, I)
    rc = lib().b200_op_silu_mul_il(_p(gu), _p(out), T, I, interleaved, None)
    assert rc == 0, lib().b200_last_error().decode()
    torch.cuda.synchronize()
    ok, straddle = check_silu(gate, up, out[:T])
    if not bool(ok.all()):
        t, i = (~ok).nonzero()[0].tolist()
        raise AssertionError(f"{int((~ok).sum())} elements wrong; first at ({t}, {i}): gate {float(gate[t, i])!r} "
                             f"up {float(up[t, i])!r} got {float(out[t, i])!r}")
    assert _untouched(out[T:]), "rows past the launch were written"
    print(f"silu_mul T={T} I={I} interleaved={interleaved}: {straddle} of {T * I} elements straddle a bf16 boundary")


def test_silu_mul_interleaved_needs_whole_64_column_blocks():
    gu = torch.zeros(2, 2 * 1000, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(B200Error) as ei:
        ops.silu_mul(gu, interleaved=True)
    assert ei.value.code == -1 and "I % 64" in str(ei.value)
    assert ops.silu_mul(gu).shape == (2, 1000)              # the [gate | up] layout takes any I % 8 == 0


# ------------------------------------------------------------------------------------------------------ RoPE / KV write
ROPE_SHAPES = [
    (32, 8, 128),    # Llama-3-8B: 256 threads below 512 tokens
    (64, 8, 128),    # Llama-3-70B: 512 threads and a second rotation pass
    (24, 8, 128),    # Llama-3.2-3B: 256 threads
    (32, 8, 64),     # Llama-3.2-1B: 128 threads
    (6, 3, 64),
    (4, 1, 128),
    (8, 2, 128),
]


@pytest.mark.parametrize("T", [1, 200, 511, 512, 1500])
@pytest.mark.parametrize("Hq,Hkv,D", ROPE_SHAPES)
def test_rope_kv_write_is_bit_exact_at_every_cta_shape(Hq, Hkv, D, T):
    """From 512 tokens every shape runs 128-thread CTAs with several tasks per thread.  Positions outside [0, max_pos)
    are clamped; slot -1 writes no page; the pool starts as NaN and exactly the named (page, offset, head) rows change."""
    max_pos = 2048
    cs = O.r(torch.from_numpy(cos_sin_cache(ModelCfg(max_model_len=max_pos, head_dim=D)))).cuda()
    g = torch.Generator().manual_seed(Hq * 1000 + Hkv * 100 + D + T)
    qkv0 = (torch.randn(T, (Hq + 2 * Hkv) * D, generator=g) * 3).bfloat16().cuda()
    pos = torch.randint(0, max_pos, (T,), generator=g, dtype=torch.int32)
    special = torch.tensor([max_pos + 3, 0, max_pos - 1, -5], dtype=torch.int32)
    pos[:min(T, 4)] = special[:min(T, 4)]
    nblocks = (T + 15) // 16 + 6
    slots = torch.randperm(nblocks * 16, generator=g)[:T].to(torch.int32)
    if T > 1:
        slots[T // 2] = -1
        slots[T - 1] = -1
    kv = _sentinel(nblocks, 2, Hkv, 16, D, bits=0x7FA5)     # a NaN
    qkv = qkv0.clone()
    ops.rope_kvwrite(qkv, pos.cuda(), slots.cuda(), cs.bfloat16(), kv, Hq, Hkv, head_dim=D)
    torch.cuda.synchronize()
    rot = rope_expected(qkv0, pos.cuda(), cs, Hq, Hkv, D)
    got = qkv[:, :(Hq + Hkv) * D].float().reshape(T, Hq + Hkv, D)
    bad = f32_bits(got) != f32_bits(rot)
    assert not bool(bad.any()), f"{int(bad.sum())} rotated q / k values differ, first at {bad.nonzero()[0].tolist()}"
    assert torch.equal(bf16_bits(qkv[:, (Hq + Hkv) * D:]), bf16_bits(qkv0[:, (Hq + Hkv) * D:])), "the v columns changed"
    want = _sentinel(nblocks, 2, Hkv, 16, D, bits=0x7FA5)
    live = (slots >= 0).cuda()
    sl = slots.cuda()[live].long()
    blk, off = sl // 16, sl % 16
    want[blk, torch.zeros_like(blk), :, off, :] = rot[live][:, Hq:].bfloat16()
    want[blk, torch.ones_like(blk), :, off, :] = qkv0[live][:, (Hq + Hkv) * D:].reshape(-1, Hkv, D)
    diff = bf16_bits(kv) != bf16_bits(want)
    assert not bool(diff.any()), f"{int(diff.sum())} KV pool values differ, first at [page, k|v, head, offset, d] = " \
                                 f"{diff.nonzero()[0].tolist()}"


# --------------------------------------------------------------------------------------------------- embedding gather
@pytest.mark.parametrize("T", [1, 2048])
@pytest.mark.parametrize("H", [256, 3072, 8192])
def test_embed_gather_is_exact_and_reads_row_0_for_out_of_range_ids(H, T):
    vocab = 1000
    g = torch.Generator(device="cuda").manual_seed(H + T)
    table = torch.randn(vocab, H, generator=g, device="cuda").bfloat16()
    ids = torch.randint(0, vocab, (T,), generator=g, device="cuda", dtype=torch.int32)
    special = torch.tensor([-1, vocab, 2 ** 31 - 1, vocab - 1, 0, -2 ** 31], dtype=torch.int32, device="cuda")
    ids[:min(T, 6)] = special[:min(T, 6)]
    out = _sentinel(T + PAD, H)
    assert lib().b200_op_embed(_p(table), _p(ids), _p(out), T, H, vocab, None) == 0
    torch.cuda.synchronize()
    want = table[torch.where((ids < 0) | (ids >= vocab), 0, ids).long()]
    assert torch.equal(bf16_bits(out[:T]), bf16_bits(want))
    assert _untouched(out[T:]), "rows past the launch were written"


# --------------------------------------------------------------------------------- the projection GEMM on capacity buffers
CAPACITY = [(1, 64), (63, 128), (65, 128), (129, 512), (300, 512), (700, 1024)]
EPIS = ["plain", "resadd", "silu", "rope128", "rope64", "argmax"]


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("T,Tcap", CAPACITY)
def test_gemm3_on_capacity_buffers_matches_the_clean_launch(T, Tcap, epi):
    """The engine's x maps and outputs span Tcap rows of which a step uses T: rows >= T of x hold NaN / +-Inf, the
    outputs' rows >= T and a PLAIN output's columns past N hold a sentinel, and positions / slots past T name live pages.
    Rows < T must carry the bits of the same launch on a clean [T, K] tensor, and nothing else may change."""
    if epi == "argmax" and T > 128:
        pytest.skip("the argmax epilogue serves T <= 128")
    K = 512
    g = torch.Generator(device="cuda").manual_seed(T * 7 + Tcap)
    x = torch.empty(Tcap, K, device="cuda")
    x[:T] = torch.randn(T, K, generator=g, device="cuda")
    x[T:] = torch.tensor([float("nan"), float("inf"), -float("inf")], device="cuda").repeat((K + 2) // 3)[:K]
    x = x.bfloat16()
    clean = x[:T].clone()
    D = 64 if epi == "rope64" else 128
    Hq, Hkv = (8, 2) if epi == "rope64" else (4, 2)
    N = {"plain": 768, "resadd": 512, "silu": 1024, "argmax": 512}.get(epi, (Hq + 2 * Hkv) * D)
    w = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).bfloat16()
    max_pos = 2048
    cs = O.r(torch.from_numpy(cos_sin_cache(ModelCfg(max_model_len=max_pos, head_dim=D)))).bfloat16().cuda()
    pos = torch.randint(-3, max_pos + 3, (Tcap,), generator=g, device="cuda", dtype=torch.int32)
    nblocks = Tcap // 16 + 4
    slots = torch.randperm(nblocks * 16, generator=g, device="cuda")[:Tcap].to(torch.int32)
    slots[T // 2] = -1
    res0 = (torch.randn(T, N, generator=g, device="cuda") * 2).bfloat16()
    for force in ([0, 1, 2, 3, 4] if T <= 128 else [0]):
        def run(xx, rows):
            """one launch on buffers of `rows` rows (sentinel past T); returns every buffer it may write"""
            bufs = {}
            kw = dict(T=T, force=force)
            if epi == "plain":
                bufs["out"] = _sentinel(rows, N + 64)
                _, sch = ops.gemm3(xx, w, out=bufs["out"][:, :N], **kw)
            elif epi == "resadd":
                bufs["out"] = _sentinel(rows, N)
                bufs["out"][:T] = res0
                bufs["ssq"] = torch.full((rows, N // 128), -7.5, device="cuda")
                _, sch = ops.gemm3(xx, w, epi=ops.EPI_RESADD, out=bufs["out"], ssq_out=bufs["ssq"], **kw)
            elif epi == "silu":
                bufs["out"] = _sentinel(rows, N // 2)
                _, sch = ops.gemm3(xx, w, epi=ops.EPI_SILU, out=bufs["out"], **kw)
            elif epi == "argmax":
                bufs["ids"] = torch.full((rows,), -7, dtype=torch.int32, device="cuda")
                _, sch = ops.gemm3(xx, w, epi=ops.EPI_ARGMAX, argmax_out=bufs["ids"], **kw)
            else:
                bufs["out"] = _sentinel(rows, N)
                bufs["kv"] = _sentinel(nblocks, 2, Hkv, 16, D, bits=0x7FA5)
                _, sch = ops.gemm3(xx, w, epi=ops.EPI_ROPE_KV, out=bufs["out"], positions=pos[:rows].contiguous(),
                                   slots=slots[:rows].contiguous(), cos_sin=cs, kv_layer=bufs["kv"], q_heads=Hq,
                                   kv_heads=Hkv, head_dim=D, **kw)
            torch.cuda.synchronize()
            return bufs, sch
        want, sch_clean = run(clean, T)
        got, sch = run(x, Tcap)
        what = f"{epi} T={T} Tcap={Tcap} force={force} schedule {sch}"
        assert sch == sch_clean, what
        for name, b in got.items():
            ref = want[name]
            if name == "kv":                                    # stale slots past T name pages that must stay NaN
                assert torch.equal(bf16_bits(b), bf16_bits(ref)), f"{what}: the KV pool differs from the clean launch's"
                continue
            bits = (lambda t: t.contiguous().view(torch.int32)) if b.dtype in (torch.float32, torch.int32) else bf16_bits
            assert torch.equal(bits(b[:T]), bits(ref)), f"{what}: {name} rows < T differ from the clean launch"
            assert torch.equal(bits(b[T:]), bits(_initial(b[T:]))), f"{what}: {name} changed past row T"
        if epi == "plain":
            assert _untouched(got["out"][:, N:]) and _untouched(want["out"][:, N:]), f"{what}: columns past N were written"


def _initial(t):
    """the sentinel a capacity buffer of t's kind starts with, in t's shape"""
    if t.dtype == torch.int32:
        return torch.full_like(t, -7)
    if t.dtype == torch.float32:
        return torch.full_like(t, -7.5)
    return _sentinel(*t.shape)
