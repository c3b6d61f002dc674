"""Reference of the engine's sampler (kubeai_b200/csrc/sampling.cu) in numpy: test infrastructure, never imported by
the package.

Semantics (vLLM V1's vllm/v1/sample/sampler.py:223-297 and ops/topk_topp_sampler.py:328-416, made deterministic), for
one row of logits l[0..V):
  - temperature < 1e-5: argmax of l, lowest index on ties;
  - z_v = float32(l_v) / float32(temperature), in fp32;
  - top-k (0, -1 or >= V = off) keeps every token with z_v >= the k-th largest z;
  - top-p (>= 1 = off) keeps token v iff the softmax mass (over the top-k-kept tokens) of the kept tokens with z strictly
    greater than z_v is < p;
  - the token is the argmax over the kept tokens of z_v - log(E_v), E_v = -log(u_v), lowest index on ties, where
    u_v = ((x >> 9) + 0.5) * 2^-23 and x is word v & 3 of Philox4x32-10 with counter (v >> 2, n, 0, 0) and key
    (seed & 0xffffffff, seed >> 32).
The filter and the race run in float64 here; the kernel uses fp32 and fixed-point masses, so the two may part only where
the race's top-2 margin or the top-p boundary slack is tiny.  sample_ref returns both so that tests can exempt those
positions.
"""
from __future__ import annotations

import numpy as np

SAMPLING_EPS = np.float32(1e-5)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 arrays (or scalars) of uint32 counter words, broadcast together; key: (k0, k1).  Returns uint32 [4, ...]."""
    c = [np.asarray(x, dtype=np.uint64) for x in np.broadcast_arrays(*[np.asarray(x, dtype=np.uint64) for x in ctr])]
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    for r in range(10):
        if r:
            k0 = (k0 + _W0) & _MASK
            k1 = (k1 + _W1) & _MASK
        p0 = _M0 * c[0]            # 32 x 32 -> 64 bits: no overflow in uint64
        p1 = _M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return np.stack(c).astype(np.uint32)


def uniforms(seed: int, n, V: int):
    """u_v for v in [0, V) at generation index n (a scalar, or an array that broadcasts against [V])."""
    v = np.arange(V, dtype=np.uint64)
    n = np.asarray(n, dtype=np.uint64)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    words = philox4x32_10((v >> np.uint64(2), n[..., None] if n.ndim else n, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    x = np.choose((v & np.uint64(3)).astype(np.intp), list(words))
    return ((x >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23


def scaled(logits, temperature):
    """z = float32(l) / float32(T) in fp32, as float64."""
    return (np.asarray(logits, dtype=np.float32) / np.float32(temperature)).astype(np.float64)


def filter_mask(z, top_k=0, top_p=1.0):
    """(kept mask, top-p boundary slack) of one row of scaled logits z (float64).  The slack is the distance of p from
    the cumulative masses on either side of the kept / dropped boundary (inf when top-p is off)."""
    z = np.asarray(z, dtype=np.float64)
    V = z.shape[0]
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        kth = np.sort(z)[V - top_k]
        keep = z >= kth
    slack = np.inf
    if 0 < top_p < 1:
        zk = z[keep]
        p = np.exp(zk - zk.max())
        p /= p.sum()
        vals, inv = np.unique(zk, return_inverse=True)            # ascending distinct values
        per = np.bincount(inv, weights=p, minlength=len(vals))
        above = np.concatenate([np.cumsum(per[::-1])[::-1][1:], [0.0]])   # mass strictly above each value
        kept_vals = above < top_p                                  # the top value always (above = 0)
        i_lo = int(np.argmax(kept_vals))                           # the lowest kept value; i_lo - 1 the highest dropped
        slack = float(top_p - above[i_lo])
        if i_lo > 0:
            slack = min(slack, float(above[i_lo - 1] - top_p))
        kk = np.flatnonzero(keep)
        keep[kk[~kept_vals[inv]]] = False
    return keep, slack


def sample_ref(logits, temperature, top_k=0, top_p=1.0, seed=0, n=0):
    """(token, race margin, top-p slack) of one row.  The margin is the gap between the best and second-best race score
    among the kept tokens (inf when one token is kept, and for greedy rows the top-2 logit gap)."""
    l = np.asarray(logits, dtype=np.float32)
    V = l.shape[0]
    if not np.float32(temperature) >= SAMPLING_EPS:
        top2 = np.sort(l.astype(np.float64))[-2:]
        return int(np.argmax(l)), float(top2[1] - top2[0]) if V > 1 else np.inf, np.inf
    z = scaled(l, temperature)
    keep, slack = filter_mask(z, top_k, top_p)
    e = -np.log(uniforms(seed, n, V))
    score = np.where(keep, z - np.log(e), -np.inf)
    tok = int(np.argmax(score))
    kept = np.sort(score[keep])
    margin = float(kept[-1] - kept[-2]) if kept.size > 1 else np.inf
    return tok, margin, slack


def probs(logits, temperature, top_k=0, top_p=1.0):
    """The distribution the race draws from: softmax of z over the kept tokens (float64, zeros elsewhere)."""
    z = scaled(logits, temperature)
    keep, _ = filter_mask(z, top_k, top_p)
    p = np.where(keep, np.exp(z - z[keep].max()), 0.0)
    return p / p.sum()
