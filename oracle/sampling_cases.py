"""Constructed sampler rows (test infrastructure, never imported by the package): each case puts the kernel's thresholds
where it names, and states the configuration it must reach so the tests can check the coverage rather than claim it.

A row is built from tiers of (bf16 value, count) at seeded random positions over a floor of filler (-2^100: finite, a key
of its own, and zero mass and no chance in the race at any temperature used here).  Positive values share a high-byte bin
across two binades ([0.5, 2), [2, 8), [8, 32), ...); the low byte is the exponent's last bit and the 7 mantissa bits, so
2.0 is key 0xC000 (bin 192 = 0 mod 8, low byte 0) and the bf16 value just below it, 1.9921875, is key 0xBFFF (bin 191 =
7 mod 8, low byte 255).

Every case is sized so that, over the N generation indices it is drawn at, each kept token has an expected count of at
least MIN_COUNT, and so does each token of the nearest dropped key had it been kept: a threshold one key off changes the
set of drawn ids.  Cases where the nearest dropped key has no mass under any threshold (nothing dropped, or only filler
and -inf) say so with neighbour=False.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle.sampling_keys import (SAMPLING_EPS, bits_of_key, bf16_bits, d_of_bits, key_of, select, topp_error_bound,
                                  z_of_bits)

FILLER = np.float32(-2.0 ** 100)
NEG_INF = np.float32(-np.inf)
MIN_COUNT = 20.0
N_CHOICES = (4096, 8192, 16384, 32768, 65536)
V_SMALL = 203            # below one vector per thread, and not a multiple of 8: the scalar tail runs
V_SIZES = (V_SMALL, 1000, 128256)
TOPP_SLACK_MIN = 1e-3    # the ordinary cases' top-p slack; topp_near_bound sits at ~10x the error bound instead


def build_row(V, tiers, seed, filler=FILLER):
    """bf16 bit patterns [V]: tier values at seeded random positions, filler elsewhere."""
    vals = np.full(V, filler, dtype=np.float32)
    total = sum(c for _, c in tiers)
    assert total <= V, (total, V)
    pos = np.random.default_rng(seed).permutation(V)[:total]
    at = 0
    for v, c in tiers:
        vals[pos[at:at + c]] = np.float32(v)
        at += c
    return bf16_bits(vals)


def next_up(x):
    return np.nextafter(np.float32(x), np.float32(np.inf))


def minp_flip_pair(bits, T, value):
    """Adjacent float32 (lo, hi): min_p = lo keeps the tokens of `value`, min_p = hi drops them (the kernel's predicate)."""
    zmax = z_of_bits(bits_of_key(int(key_of(bits).max())), T)
    d = np.float64(d_of_bits(bf16_bits([value]), T, zmax)[0])
    mp = np.float32(np.exp(d))
    while np.log(np.float64(mp)) > d:
        mp = np.nextafter(mp, np.float32(0))
    while np.log(np.float64(next_up(mp))) <= d:
        mp = next_up(mp)
    assert np.log(np.float64(mp)) <= d < np.log(np.float64(next_up(mp)))
    return mp, next_up(mp)


def topp_near_bound(bits, T, value, times=10.0):
    """A float32 top_p that keeps the tie group of `value` with a slack of about `times` the kernel's error bound."""
    keys = key_of(bits)
    z = z_of_bits(bits, T).astype(np.float64)
    m = np.exp(z - z.max())
    kv = int(key_of(bf16_bits([value]))[0])
    above = m[keys > kv].sum() / m.sum()
    B = topp_error_bound(bits, T, keys >= kv)
    return np.float32(above + times * B)


@dataclass
class Case:
    name: str
    tiers: list
    T: float = 1.0
    top_k: object = 0          # int, or a function of V
    top_p: object = 1.0        # float, or a function of (bits, T)
    min_p: object = 0.0        # float, or a function of (bits, T)
    expect: object = None      # predicate over the Selection: the configuration the case exists for
    config: str = ""           # that configuration in words
    neighbour: bool = True
    filler: np.float32 = FILLER
    tags: tuple = field(default_factory=tuple)

    def row(self, V, seed=0):
        return build_row(V, self.tiers, seed + V, self.filler)

    def params(self, bits):
        """(T, top_k, top_p, min_p) for this row, as the kernel reads them."""
        V = bits.shape[0]
        k = self.top_k(V) if callable(self.top_k) else self.top_k
        p = self.top_p(bits, self.T) if callable(self.top_p) else self.top_p
        mp = self.min_p(bits, self.T) if callable(self.min_p) else self.min_p
        return np.float32(self.T), int(k), np.float32(p), np.float32(mp)


def probs_of(bits, T, kept):
    """The race's distribution over `kept` (float64): softmax of the fp32 z."""
    z = z_of_bits(bits, T).astype(np.float64)
    zk = np.where(kept, z, -np.inf)
    with np.errstate(invalid="ignore"):
        m = np.where(kept, np.exp(zk - zk.max()), 0.0)
    return m / m.sum(), z


def design(case, bits):
    """Check the case's sizing and configuration on one row; returns (Selection, params, N, report dict)."""
    T, k, p, mp = case.params(bits)
    sel = select(bits, T, k, p, mp)
    assert case.expect is None or case.expect(sel), f"{case.name}: not {case.config}: {sel.describe()}"
    keys = key_of(bits)
    if sel.greedy:
        q, live = np.zeros(bits.shape[0]), sel.kept
        q[live] = 1.0
    else:
        q, z = probs_of(bits, T, sel.kept)
        live = q > 0
    min_p_kept = float(q[live].min())
    below = keys < sel.thr
    nb = None
    if not sel.greedy and below.any():
        kd = int(keys[below].max())
        zd = np.float64(z_of_bits(bits_of_key(kd), T))
        zk = z[sel.kept].max()
        md = np.exp(zd - zk)
        cnt = int((keys == kd).sum())
        mass = np.exp(z[sel.kept] - zk).sum()
        nb = float(md / (mass + cnt * md))
    if case.neighbour:
        assert nb is not None and nb > 0, f"{case.name}: no dropped neighbour with mass"
    need = MIN_COUNT / min(min_p_kept, nb if case.neighbour else 1.0)
    N = next((n for n in N_CHOICES if n >= need), None)
    assert N is not None, f"{case.name}: needs {need:.0f} draws"
    slack = None
    if sel.topp_on:
        B = topp_error_bound(bits, T, sel.kept)
        m = sel.masses
        kept_mass = m[keys >= max(sel.tk, sel.tm)]
        Z = kept_mass.sum()
        above = m[keys > sel.tp].sum() / Z                       # < p: the boundary group is kept
        nxt = keys[(keys < sel.tp) & (keys >= max(sel.tk, sel.tm))]
        slack = float(p) - above if above > 0 else np.inf            # nothing above the top group: exact in the kernel
        if nxt.size:
            slack = min(slack, m[keys >= int(nxt.max())].sum() / Z - float(p))
        if "near_bound" in case.tags:
            assert 3 * B < slack < 30 * B, (case.name, slack, B)
        else:
            assert slack > TOPP_SLACK_MIN, (case.name, slack)
        slack = (slack, B)
    report = dict(N=N, kept=int(sel.kept.sum()), live=int(live.sum()), min_kept=N * min_p_kept,
                  min_neighbour=None if nb is None else N * nb, topp_slack=slack)
    return sel, (T, k, p, mp), N, report


def _v(*vals):
    return [np.float32(v) for v in vals]


CASES = [
    Case("temperature_only", [(1.0, 20), (0.5, 30), (0.0, 30)], T=0.8, neighbour=False, config="the race alone",
         expect=lambda s: not (s.topk_on or s.topp_on or s.minp_on) and s.thr == 0),
    Case("topk_kth_in_tie_group", [(3.0, 3), (2.5, 4), (2.0, 6), (1.75, 5)], top_k=10,
         config="top-k alone, the k-th value inside a tie group kept whole",
         expect=lambda s: s.passes == ("3",) and s.kept.sum() == 13),
    Case("topk_1_tie_at_max", [(4.0, 3), (3.875, 5)], top_k=1, config="k = 1 with the maximum tied three ways",
         expect=lambda s: s.kept.sum() == 3 and s.passes == ("3",)),
    Case("topk_V_minus_1", [(1.0, 10), (0.5, 10), (-2.0 ** 101, 1)], top_k=lambda V: V - 1, neighbour=False,
         config="k = V - 1: everything but the one lowest key",
         expect=lambda s: s.topk_on and s.kept.sum() == s.kept.shape[0] - 1),
    Case("topk_beyond_finite", [(1.0, 10), (0.0, 10)], top_k=50, filler=NEG_INF, neighbour=False,
         config="k above the number of finite logits (the rest -inf)",
         expect=lambda s: s.topk_on and s.tk == int(key_of(bf16_bits(_v(-np.inf)))[0])),
    Case("topp_boundary_in_max_bin", [(7.0, 2), (6.5, 3), (6.0, 4), (5.5, 10)], top_p=0.6,
         config="top-p alone, boundary in the maximum's bin",
         expect=lambda s: s.passes == ("4",) and s.bp == s.kmax >> 8),
    Case("topp_boundary_in_lower_bin", [(10.0, 2), (7.0, 6), (6.5, 8)], top_p=0.85,
         config="top-p alone, boundary in a bin below the maximum's",
         expect=lambda s: s.passes == ("4",) and s.bp < s.kmax >> 8),
    Case("topp_tie_group_kept_whole", [(3.0, 4), (2.0, 8), (1.0, 8)], top_p=0.6,
         config="top-p boundary at a tie group whose cumulative mass passes p: kept whole",
         expect=lambda s: s.kept.sum() == 12),
    Case("topp_tie_group_dropped_whole", [(3.0, 4), (2.0, 8), (1.0, 8)], top_p=0.45,
         config="top-p boundary at a tie group whose mass above is >= p: dropped whole",
         expect=lambda s: s.kept.sum() == 4),
    Case("topp_tiny", [(5.0, 3), (4.875, 4)], top_p=1e-6, config="p tiny: the top tie group alone",
         expect=lambda s: s.kept.sum() == 3 and s.tp == s.kmax),
    Case("topp_near_bound", [(3.0, 4), (2.0, 8), (1.0, 8)], top_p=lambda b, T: topp_near_bound(b, T, 2.0),
         config="top-p slack within ~10x of the kernel's error bound", tags=("near_bound",),
         expect=lambda s: s.kept.sum() == 12),
    Case("topk_topp_same_bin", [(6.0, 3), (5.0, 4), (4.0, 6), (3.5, 8), (3.0, 10)], top_k=13, top_p=0.7,
         config="top-k + top-p, bp == bk: pass 4 skipped",
         expect=lambda s: s.bp == s.bk and s.passes == ("3",) and s.thr == s.tp > s.tk),
    Case("topk_topp_higher_bin", [(10.0, 2), (9.0, 3), (7.0, 4), (6.0, 5)], top_k=9, top_p=0.8,
         config="top-k + top-p, bp > bk: pass 4 runs",
         expect=lambda s: s.bp > s.bk and s.passes == ("3", "4")),
    Case("minp_flip_keeps", [(2.0, 4), (1.0, 6), (0.0, 8)], min_p=lambda b, T: minp_flip_pair(b, T, 1.0)[0],
         config="min_p alone, the lower of two adjacent float32 min_p: the 1.0 tier kept",
         expect=lambda s: s.minp_on and s.thr == s.tm and s.kept.sum() == 10),
    Case("minp_flip_drops", [(2.0, 4), (1.0, 6), (0.0, 8)], min_p=lambda b, T: minp_flip_pair(b, T, 1.0)[1],
         config="min_p alone, the upper of the pair: the 1.0 tier dropped",
         expect=lambda s: s.minp_on and s.thr == s.tm and s.kept.sum() == 4),
    # fp32(z - z_max) equals log(float32 min_p) exactly only at min_p = 1 and d = 0.  A key below the row max has d = 0
    # when the division by T rounds both to one z: at T = 2^100, 2^-48 and 2^-48 * (1 + 2^-7) both become 2^-148.
    Case("minp_one_keeps_equal_z", [(2.0 ** -48 * 1.0078125, 6), (2.0 ** -48, 5), (2.0 ** -50, 8)], T=2.0 ** 100,
         min_p=1.0, config="min_p = 1 at a boundary of d = 0 exactly: a lower key with z equal to z_max is kept",
         expect=lambda s: s.tm <= int(key_of(bf16_bits(_v(2.0 ** -48)))[0]) < s.kmax and s.kept.sum() == 11),
    Case("minp_topk_tm_above_tk", [(3.0, 3), (2.5, 4), (2.0, 5), (1.0, 6)], top_k=12, min_p=0.5,
         config="min_p + top-k, tm > tk", expect=lambda s: s.tm > s.tk and s.thr == s.tm),
    Case("minp_topk_tm_below_tk", [(3.0, 3), (2.5, 4), (2.0, 5), (1.0, 6)], top_k=3, min_p=0.2,
         config="min_p + top-k, tm <= tk", expect=lambda s: s.tm <= s.tk and s.thr == s.tk),
    Case("minp_topp_same_bin", [(7.0, 2), (6.0, 4), (5.0, 6), (4.0, 8), (1.0, 10)], top_p=0.6, min_p=float(np.exp(-2.5)),
         config="min_p + top-p, bp == bm: pass 4 reuses pass 3b",
         expect=lambda s: s.bp == s.bm and s.passes == ("3b",) and s.z_recomputed and s.thr == s.tp > s.tm),
    Case("minp_topp_other_bin", [(10.0, 2), (9.0, 3), (7.0, 4), (6.0, 5), (3.0, 10)], top_p=0.8,
         min_p=float(np.exp(-3.5)), config="min_p + top-p, bp != bm: pass 4 runs",
         expect=lambda s: s.bp != s.bm and s.passes == ("3b", "4") and s.thr == s.tp),
    Case("all_three_pass4_reruns_bk", [(6.0, 3), (5.0, 4), (4.0, 6), (1.0, 8), (0.5, 10)], top_k=13, top_p=0.7,
         min_p=float(np.exp(-5.25)), config="top-k + top-p + min_p, tm <= tk, bm != bk, bp == bk: pass 4 re-runs bin bk",
         expect=lambda s: s.tm <= s.tk and s.bm != s.bk and s.bp == s.bk and s.passes == ("3", "3b", "4")),
    Case("all_three_tm_above_tk", [(7.0, 2), (6.0, 4), (5.0, 6), (4.0, 8), (1.0, 10)], top_k=30, top_p=0.6,
         min_p=float(np.exp(-2.5)), config="top-k + top-p + min_p, tm > tk, bp == bm",
         expect=lambda s: s.tm > s.tk and s.bp == s.bm != s.bk and s.z_recomputed and s.passes == ("3", "3b")),
    Case("edge_topk_bin0_low0", [(4.0, 3), (2.0, 5), (1.9921875, 6)], top_k=8,
         config="tk = 0xC000: bin 0 mod 8, low byte 0, the dropped key adjacent",
         expect=lambda s: s.tk == 0xC000),
    Case("edge_topk_bin7_low255", [(4.0, 3), (2.0, 5), (1.9921875, 6), (1.0, 6)], top_k=14,
         config="tk = 0xBFFF: bin 7 mod 8, low byte 255", expect=lambda s: s.tk == 0xBFFF),
    Case("edge_topp_bin0_low0", [(4.0, 3), (2.0, 5), (1.9921875, 6)], top_p=0.75,
         config="tp = 0xC000: bin 0 mod 8, low byte 0", expect=lambda s: s.tp == 0xC000),
    Case("edge_topp_bin7_low255", [(4.0, 3), (2.0, 5), (1.9921875, 6), (1.0, 8)], top_p=0.85,
         config="tp = 0xBFFF: bin 7 mod 8, low byte 255", expect=lambda s: s.tp == 0xBFFF),
    Case("edge_minp_bin7_low255", [(4.0, 3), (2.0, 5), (1.9921875, 6), (1.0, 8)],
         min_p=lambda b, T: minp_flip_pair(b, T, 1.9921875)[0], config="tm = 0xBFFF: bin 7 mod 8, low byte 255",
         expect=lambda s: s.tm == 0xBFFF and s.kept.sum() == 14),
    Case("signed_zero_tie", [(1.0, 3), (0.0, 4), (-0.0, 4), (-0.5, 5)], top_k=5,
         config="top-k boundary at a tie group of +0 and -0 (one key)", expect=lambda s: s.kept.sum() == 11),
    Case("temperature_eps", [(0.0, 3), (-2.0 ** -17, 4), (-2.0 ** -16, 5)], T=float(SAMPLING_EPS), neighbour=False,
         config="temperature exactly 1e-5: sampled", expect=lambda s: not s.greedy and s.kept.sum() == s.kept.shape[0]),
    Case("temperature_below_eps", [(0.0, 3), (-2.0 ** -17, 4), (-2.0 ** -16, 5)],
         T=float(np.nextafter(SAMPLING_EPS, np.float32(0))), neighbour=False,
         config="temperature one float32 below 1e-5: greedy", expect=lambda s: s.greedy),
    Case("temperature_flat", [(4.0, 10), (2.0, 10), (0.0, 10), (-3.0, 10)], T=100.0, neighbour=False,
         config="temperature 100: nearly flat", expect=lambda s: not s.greedy and s.thr == 0),
]

CASES_BY_NAME = {c.name: c for c in CASES}


def oracle_kept(bits, T, top_k=0, top_p=1.0, min_p=0.0):
    """(kept mask, top-p slack, min_p slack) of oracle/penalties.py + oracle/sampling.py on one row of bf16 bits."""
    from oracle.penalties import min_p_keep
    from oracle.sampling import filter_mask, scaled
    lf = z_of_bits(bits, 1.0)
    if not np.float32(T) >= SAMPLING_EPS:
        keep = np.zeros(lf.shape[0], dtype=bool)
        keep[int(np.argmax(lf))] = True
        return keep, np.inf, np.inf
    z = scaled(lf, T)
    mkeep, mslack = min_p_keep(z.astype(np.float32), float(min_p))
    keep, slack = filter_mask(np.where(mkeep, z, -np.inf), int(top_k), float(top_p))
    return keep & mkeep, slack, mslack


def race(bits, T, kept, seed, ns):
    """oracle/sampling.py's race restricted to the kept tokens that can win, vectorised over generation indices ns:
    (tokens [len(ns)], top-2 margins).  Kept tokens with zero softmax mass (filler, -inf) are left out after checking that
    no draw of E_v could lift them over a live token (an fp32 u_v keeps log(E_v) within [-16.7, 2.8])."""
    from oracle.sampling import philox4x32_10
    z = z_of_bits(bits, T).astype(np.float64)
    q, _ = probs_of(bits, T, kept)
    live = np.flatnonzero(q > 0)
    dead = kept & ~(q > 0)
    if dead.any():
        assert z[dead].max() < z[live].min() - 20.0
    ns = np.asarray(ns, dtype=np.uint64)
    ids = live.astype(np.uint64)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    words = philox4x32_10((ids[None, :] >> np.uint64(2), ns[:, None], 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    x = np.choose((ids & np.uint64(3)).astype(np.intp)[None, :], list(words))
    u = ((x >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    score = z[live][None, :] - np.log(-np.log(u))
    best = np.argmax(score, axis=1)
    if live.size > 1:
        top2 = np.partition(score, live.size - 2, axis=1)[:, -2:]
        margin = top2[:, 1] - top2[:, 0]
    else:
        margin = np.full(len(ns), np.inf)
    return live[best], margin
