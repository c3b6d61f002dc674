"""Numerics shared by the exact kernel tests: bf16 rounding and bit views, the reduction order and launch shape of the
row-norm kernels, and the checkers that hold RMSNorm, SiLU·up and RoPE to a float64 (or bit-exact) reference.

Each checker takes the kernel's output and the inputs as torch tensors on any device; the GPU tests run them on the
kernels' outputs, tests/test_elementwise_exact_cpu.py runs them on CPU emulations, faithful and subtly wrong, to show
they accept the first and reject the others."""
import numpy as np
import torch

from oracle import llama_oracle as O

# RMSNorm: the kernel's fp32 inv = rsqrtf(ss / H + eps) lies within RMS_DELTA * inv64 of the float64 value.  ss is a sum of
# positive terms through at most 8 * 4 + 10 roundings (each thread's 8 * VPT adds, then 5 butterfly levels in the warp and
# 5 more over the warp sums), each at most 2^-24 relative of the whole sum: 42 * 2^-24 in ss, 21 * 2^-24 in inv after the
# square root.  The IEEE division by H and the add of eps round once each (2^-24 relative, 2^-25 each in inv), and
# rsqrtf is within 2 ulps (4 * 2^-24 relative): 21 + 0.5 + 0.5 + 4 = 26.
RMS_DELTA = 26 * 2.0 ** -24

# SiLU: silu_bf16 is __fdividef(g, 1 + __expf(-g)).  __expf is ex2.approx(g * log2e) with log2e rounded to fp32: the
# rounded constant (0.22 * 2^-24 relative) and the rounded product (2^-24) move the exponent by 1.22 |g| 2^-24, which is
# 1.22 |g| 2^-24 relative in e^-g; ex2.approx adds at most 2 ulps (4 * 2^-24), 1 + e one rounding (2^-24) and __fdividef
# 2 ulps (4 * 2^-24).  e^-g enters s = g / (1 + e^-g) with a weight below 1, so s is within (9 + 1.22 |g|) 2^-24
# relative of float64; SILU_C0 and SILU_C1 round that up.
SILU_C0, SILU_C1 = 10.0, 1.25
# __fdividef returns 0 once the denominator passes 2^126, i.e. 1 + e^-g for bf16 g <= -87.5 (e^87.5 > 2^126 > e^87): there
# the kernel's silu is a signed zero where the true value is about g e^g (below 1e-36).  The fused GEMM epilogue shares
# silu_bf16, so this is pinned as a documented deviation rather than changed.
SILU_TAIL = -87.5


def bf16(x):
    """Round-to-nearest-even bf16 of fp32 values (float64 input is rounded to fp32 first), kept in float32."""
    return x.float().to(torch.bfloat16).float()


def bf16_bits(t):
    """int16 bit patterns of a bf16 tensor."""
    assert t.dtype == torch.bfloat16
    return t.contiguous().view(torch.int16)


def f32_bits(t):
    """int32 bit patterns of the fp32 values of t (bf16 values widen exactly): NaN-safe equality, and -0 != +0."""
    return t.float().contiguous().view(torch.int32)


def warp_sum(v):
    """__shfl_xor_sync butterfly over 32 fp32 lanes (offsets 16..1); every lane ends with the same value."""
    v = v.astype(np.float32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[np.arange(32) ^ o]).astype(np.float32)
    return v[0]


def norm_launch(rows, H):
    """(threads, vectors per thread) that rmsnorm() and the pooling / score kernels use for `rows` rows of H: one 8-element
    vector per thread below 512 rows or when H / 8 is not a multiple of 256, else 256 threads of H / 2048 vectors."""
    vecs = H // 8
    return (vecs, 1) if (rows < 512 or vecs % 256) else (256, vecs // 256)


def _ordered(bits):
    """int32 fp32 bit patterns -> int64 keys in value order (-0 sorts just below +0)."""
    b = np.asarray(bits, dtype=np.int64)
    return np.where(b >= 0, b, -(b & 0x7FFFFFFF) - 1)


def _unordered(keys):
    k = np.asarray(keys, dtype=np.int64)
    return np.where(k >= 0, k, (-k - 1) | 0x80000000).astype(np.uint32).view(np.int32)


def fp32_between(lo, hi, device="cpu"):
    """Every fp32 value in the closed interval [lo, hi] (lo, hi any real numbers), ascending, as a float32 tensor."""
    lo, hi = float(lo), float(hi)
    a, b = np.float32(lo), np.float32(hi)
    if float(a) < lo:
        a = np.nextafter(a, np.float32(np.inf))
    if float(b) > hi:
        b = np.nextafter(b, np.float32(-np.inf))
    ka, kb = _ordered(np.array(a).view(np.int32)), _ordered(np.array(b).view(np.int32))
    keys = np.arange(int(ka), int(kb) + 1, dtype=np.int64)
    return torch.from_numpy(_unordered(keys).view(np.float32).copy()).to(device)


def check_rmsnorm(v, w, out, eps):
    """RMSNorm rows against float64.  v: [rows, H] the normalised rows (bf16 values: the input, or bf16(x + res) in
    fused-add mode), w: [H] the bf16 weight, out: [rows, H] the kernel's output.  A row passes iff one fp32 r within
    RMS_DELTA * inv64 of inv64 = (mean(v^2) + eps)^-1/2 (float64) reproduces every element as bf16(bf16(fp32(v r)) w).
    Returns (passing rows [rows] bool, rows that needed a candidate other than the fp32 nearest inv64)."""
    v, w = v.float(), w.float()
    inv64 = (v.double().pow(2).mean(-1) + float(np.float32(eps))).rsqrt()
    got = f32_bits(out)

    def apply(vv, r):
        return f32_bits(bf16(bf16(vv * r) * w))
    ok = (apply(v, inv64.float()[:, None]) == got).all(-1)
    nonnearest = 0
    for i in (~ok).nonzero().flatten().tolist():
        r = fp32_between(inv64[i] * (1 - RMS_DELTA), inv64[i] * (1 + RMS_DELTA), v.device)
        if bool((apply(v[i][None, :], r[:, None]) == got[i][None, :]).all(-1).any()):
            ok[i] = True
            nonnearest += 1
    return ok, nonnearest


def check_silu(g, u, out):
    """SiLU(g) * u elementwise against float64.  g, u: the bf16 gate and up values, out: the kernel's output (same shape).
    With s64 = g / (1 + e^-g) in float64, the kernel's fp32 silu is within (SILU_C0 + SILU_C1 |g|) 2^-24 relative of s64,
    so s = bf16(silu) is bf16(s64), or, where that interval straddles a bf16 rounding boundary, either neighbour; then
    out = bf16(s u) exactly (the product of two bf16 values is exact in fp32).  For g <= SILU_TAIL: |out| <= 2^-100 |u|
    and no NaN.  Returns (passing elements bool, elements whose interval straddles a boundary)."""
    g, u = g.float(), u.float()
    tail = g <= SILU_TAIL
    g64 = g.double()
    s64 = g64 / (1 + torch.exp(-g64))
    b = (SILU_C0 + SILU_C1 * g64.abs()) * 2.0 ** -24 * s64.abs()
    s_lo, s_hi = bf16(s64 - b), bf16(s64 + b)
    got = f32_bits(out)
    ok = (f32_bits(bf16(s_lo * u)) == got) | (f32_bits(bf16(s_hi * u)) == got)
    out = out.float()
    ok_tail = ~torch.isnan(out) & (out.abs() <= 2.0 ** -100 * u.abs())
    straddle = (s_lo != s_hi) & ~tail
    return torch.where(tail, ok_tail, ok), int(straddle.sum())


def rope_expected(qkv, positions, cos_sin, Hq, Hkv, D):
    """The q and k heads of qkv [T, (Hq + 2 Hkv) D] rotated as the reference backend's bf16 neox RoPE does (every bf16 op
    rounds), at positions clamped to [0, max_pos), the kernels' contract: [T, Hq + Hkv, D] float32."""
    T = qkv.shape[0]
    pos = positions.long().clamp(0, cos_sin.shape[0] - 1)
    return O.rope_neox(qkv[:, :(Hq + Hkv) * D].float().reshape(T, Hq + Hkv, D), pos, cos_sin.float())
