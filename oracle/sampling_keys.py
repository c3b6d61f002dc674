"""The sampler's selection (kubeai_b200/csrc/sampling.cu, sample_kernel) restated as 16-bit key thresholds, in numpy: test
infrastructure, never imported by the package.

oracle/sampling.py and oracle/penalties.py state what is kept in float64 over values; this file states the same selection
the way the kernel finds it, over the order-preserving keys of the bf16 logits, and says which of the kernel's branches a
row takes.  tests/test_sampling_exact_cpu.py pins the two statements against each other, so a case built here is known to
reach the configuration it names, and its kept set is known to the bit.

For one row of bf16 bit patterns b[0..V) with temperature T, top_k k, top_p p and min_p (p and min_p as float32):
  - key(b) orders the values: -0 and +0 share one key; -NaN sits below -inf, +NaN above +inf;
  - z(key) = float32(value) / float32(T) in fp32, z_max = z(the row's largest key);
  - tm (min_p > 0): the smallest key t <= that largest key with float64(fp32(z(t) - z_max)) >= log(float64(min_p)), taken
    over every key (not by bisection), so a predicate that is not monotone in the key would show;
  - tk (0 < k < V): the k-th largest key of the row;
  - tp (0 < p < 1): with m_v = exp(fp32(z_v - z_max)) (float64 here, floor(expf(.) * 2^40) in the kernel) and Z the mass of
    the tokens with key >= max(tk, tm), the largest key t with mass(key >= max(t, tk, tm)) >= p * Z;
  - the race runs over the tokens with key >= max(tk, tm, tp);
  - bins and passes: bk = tk >> 8 (pass 3 builds its low-byte histogram), bm = tm >> 8 (pass 3b, when top-p and min_p are
    both on and bm is not the bin pass 3 already holds), bp = tp >> 8 (pass 4, unless the shared low-byte histogram already
    holds bin bp); z is recomputed from bm's histogram when tm > tk.

Top-p error bound.  The kernel's masses differ from these float64 m_v by, per token,
    2 ulp of expf (<= 2^-22 m_v)  +  the fp32 rounding of z_v - z_max (a relative error <= 2^-24 |d_v| in the exponent)
    +  the floor of m_v * 2^40 (< min(2^-40, m_v), and 0 when expf returns 0),
and the sums are exact integers (2^40 * 2^17 fits in 64 bits; their conversion to double adds 2^-52 relative).  The kernel
compares M_k >= p Z_k where M and Z are sums of such masses, so its decision equals the float64 one wherever
|M - p Z| > E_M + p E_Z; topp_error_bound returns 2 (E / Z) over the kept tokens, in units of probability, which bounds that
distance for every boundary.  Cases keep their top-p slack far above it, and one keeps it within ~10x.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

SAMPLING_EPS = np.float32(1e-5)
ALL_KEYS = np.arange(65536, dtype=np.uint32)


def key_of(bits):
    """Order-preserving 16-bit key of bf16 bit patterns (uint16 / int arrays): -0 folds onto +0."""
    b = np.asarray(bits, dtype=np.uint32) & np.uint32(0xFFFF)
    b = np.where(b == 0x8000, np.uint32(0), b)
    return np.where(b & 0x8000, ~b & np.uint32(0xFFFF), b | np.uint32(0x8000)).astype(np.uint32)


def bits_of_key(keys):
    """The bf16 bit pattern of a key (+0 for the key -0 and +0 share)."""
    k = np.asarray(keys, dtype=np.uint32)
    return np.where(k & 0x8000, k & np.uint32(0x7FFF), ~k & np.uint32(0xFFFF)).astype(np.uint32)


def f32_of_bits(bits):
    return (np.asarray(bits, dtype=np.uint32) << np.uint32(16)).view(np.float32)


def bf16_bits(values):
    """float32 values that are exact bf16 (checked) -> uint16 bit patterns; -0.0 keeps its sign."""
    v = np.asarray(values, dtype=np.float32)
    u = v.view(np.uint32)
    assert not (u & 0xFFFF).any(), "not a bf16 value"
    return (u >> np.uint32(16)).astype(np.uint16)


def z_of_bits(bits, T):
    """z = float32(l) / float32(T) in fp32 (numpy float32 division rounds to nearest, as __fdiv_rn)."""
    with np.errstate(invalid="ignore", over="ignore"):
        return (f32_of_bits(bits) / np.float32(T)).astype(np.float32)


def d_of_bits(bits, T, zmax):
    """fp32(z - z_max), the kernel's __fsub_rn."""
    with np.errstate(invalid="ignore"):
        return (z_of_bits(bits, T) - np.float32(zmax)).astype(np.float32)


@dataclass
class Selection:
    greedy: bool
    topk_on: bool
    topp_on: bool
    minp_on: bool
    kmax: int = 0
    tk: int = 0
    tm: int = 0
    tp: int = 0
    thr: int = 0
    bk: int = -1
    bm: int = -1
    bp: int = -1
    passes: tuple = ()          # of "3", "3b", "4": the low-byte histogram passes the kernel runs
    z_recomputed: bool = False  # tm > tk with top-p and min_p: Z comes from bm's histogram
    kept: np.ndarray = None     # bool [V]: the race's tokens (key >= thr), or the argmax alone when greedy
    masses: np.ndarray = None   # float64 [V]: exp(fp32(z - z_max)) (top-p rows)

    def describe(self):
        if self.greedy:
            return "greedy"
        on = "+".join(n for n, f in (("top_k", self.topk_on), ("top_p", self.topp_on), ("min_p", self.minp_on)) if f)
        return (f"{on or 'temperature'}: tk={self.tk:#06x} tm={self.tm:#06x} tp={self.tp:#06x} thr={self.thr:#06x} "
                f"bk={self.bk} bm={self.bm} bp={self.bp} passes={','.join(self.passes) or '-'}"
                f"{' z-recomputed' if self.z_recomputed else ''} kept={int(self.kept.sum())}")


def select(bits, temperature, top_k=0, top_p=1.0, min_p=0.0) -> Selection:
    """The kernel's thresholds, bins and passes for one row of bf16 bit patterns."""
    bits = np.asarray(bits).astype(np.uint32)
    V = bits.shape[0]
    T, p, mp = np.float32(temperature), np.float32(top_p), np.float32(min_p)
    keys = key_of(bits)
    if not T >= SAMPLING_EPS:
        f = f32_of_bits(bits)
        kept = np.zeros(V, dtype=bool)
        kept[int(np.argmax(np.where(np.isnan(f), -np.inf, f)))] = True
        return Selection(True, False, False, False, kept=kept)
    s = Selection(False, 0 < top_k < V, bool(0 < p < 1), bool(mp > 0))
    zmax = np.float32(0)
    if s.topp_on or s.minp_on:
        s.kmax = int(keys.max())
        zmax = z_of_bits(bits_of_key(s.kmax), T)
    if s.minp_on:
        lm = np.log(np.float64(mp))
        with np.errstate(invalid="ignore"):
            ok = d_of_bits(bits_of_key(ALL_KEYS), T, zmax).astype(np.float64) >= lm
        ok[s.kmax + 1:] = False
        s.tm = int(np.argmax(ok)) if ok.any() else s.kmax
    if s.topk_on:
        s.tk = int(np.sort(keys)[V - top_k])
        s.bk = s.tk >> 8
        s.passes += ("3",)
    lo_bin = s.bk if s.topk_on else -1
    if s.topp_on:
        with np.errstate(invalid="ignore", over="ignore"):
            m = np.exp(d_of_bits(bits, T, zmax).astype(np.float64))
        m = np.where(np.isnan(m), 0.0, m)
        s.masses = m
        base = max(s.tk, s.tm)
        inz = keys >= base
        Z = m[inz].sum()
        if s.minp_on:
            s.bm = s.tm >> 8
            if s.bm != lo_bin:
                s.passes += ("3b",)
            lo_bin = s.bm
            s.z_recomputed = s.tm > s.tk
        # mass(key >= t) over the kept tokens for every distinct row key t, high to low
        uk, inv = np.unique(keys[inz], return_inverse=True)                    # ascending distinct keys
        per = np.bincount(inv, weights=m[inz], minlength=len(uk))
        at_or_above = np.cumsum(per[::-1])[::-1]
        X = np.float64(p) * Z
        reach = np.flatnonzero(at_or_above >= X)
        s.tp = int(uk[reach[-1]]) if reach.size else base
        s.bp = s.tp >> 8
        if s.bp != lo_bin:
            s.passes += ("4",)
    s.thr = max(s.tk, s.tm, s.tp)
    s.kept = keys >= s.thr
    return s


def topp_error_bound(bits, temperature, kept):
    """Bound on how far (in probability) the kernel's top-p comparison can sit from the float64 one, over `kept`."""
    bits = np.asarray(bits).astype(np.uint32)
    keys = key_of(bits)
    zmax = z_of_bits(bits_of_key(int(keys.max())), temperature)
    d = d_of_bits(bits[kept], temperature, zmax).astype(np.float64)
    d = np.where(np.isfinite(d), d, -np.inf)
    with np.errstate(invalid="ignore"):
        m = np.exp(d)
        rel = np.where(m > 0, 2.0 ** -22 + np.expm1(2.0 ** -24 * np.abs(np.where(m > 0, d, 0.0))), 0.0)
    err = (m * rel + np.minimum(2.0 ** -40, m)).sum()
    Z = m.sum()
    return 2.0 * (err / Z + 2.0 ** -52)
