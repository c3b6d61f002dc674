"""The sampler's key-threshold restatement (oracle/sampling_keys.py) against the float64 oracle (oracle/sampling.py,
oracle/penalties.py), and the constructed rows of oracle/sampling_cases.py: each case reaches the configuration it names,
its kept set equals the oracle's to the bit, and it is sized so that a threshold one key off would show on the GPU."""
import numpy as np
import pytest

from oracle.penalties import sample_ref
from oracle.sampling_cases import (CASES, MIN_COUNT, V_SIZES, build_row, design, minp_flip_pair, oracle_kept, race)
from oracle.sampling_keys import ALL_KEYS, bf16_bits, bits_of_key, f32_of_bits, key_of, select, topp_error_bound


def test_keys_order_every_bf16_value_and_fold_signed_zero():
    bits = ALL_KEYS
    f = f32_of_bits(bits)
    keys = key_of(bits)
    num = ~np.isnan(f)
    order = np.argsort(keys[num], kind="stable")
    assert (np.diff(f[num][order]) >= 0).all()                      # keys sort the values
    assert keys[0x8000] == keys[0x0000] == 0x8000                   # -0 and +0: one key
    assert len(np.unique(keys[num])) == num.sum() - 1               # every other value its own key
    back = bits_of_key(keys)
    assert (back[bits != 0x8000] == bits[bits != 0x8000]).all() and back[0x8000] == 0
    # +NaN above +inf, -NaN below -inf
    assert keys[0x7FC0] > keys[0x7F80] and keys[0xFFC0] < keys[0xFF80]
    assert key_of(bf16_bits([2.0]))[0] == 0xC000 and key_of(bf16_bits([1.9921875]))[0] == 0xBFFF


@pytest.mark.parametrize("V", V_SIZES)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_case_reaches_its_configuration_and_kept_set_equals_the_oracle(case, V):
    bits = case.row(V)
    sel, (T, k, p, mp), N, rep = design(case, bits)
    print(f"{case.name} V={V}: {sel.describe()} N={N} min expected count kept={rep['min_kept']:.0f} "
          f"nearest dropped={rep['min_neighbour'] and round(rep['min_neighbour'])} top-p (slack, bound)={rep['topp_slack']}")
    assert rep["min_kept"] >= MIN_COUNT
    want, slack, mslack = oracle_kept(bits, T, k, p, mp)
    assert np.array_equal(sel.kept, want), (np.flatnonzero(sel.kept != want), slack, mslack)


def test_every_configuration_is_reached():
    seen = {}
    for c in CASES:
        sel = design(c, c.row(1000))[0]
        seen.setdefault(sel.passes, []).append(c.name)
    print({"/".join(k) or "-": v for k, v in seen.items()})
    for passes in [(), ("3",), ("4",), ("3", "4"), ("3b",), ("3b", "4"), ("3", "3b"), ("3", "3b", "4")]:
        assert passes in seen, passes


def test_minp_flip_pair_moves_exactly_one_key():
    c = next(c for c in CASES if c.name == "minp_flip_keeps")
    for V in V_SIZES:
        bits = c.row(V)
        lo, hi = minp_flip_pair(bits, 1.0, 1.0)
        assert np.nextafter(lo, np.float32(1)) == hi
        a, b = select(bits, 1.0, min_p=lo), select(bits, 1.0, min_p=hi)
        flipped = np.unique(key_of(bits)[a.kept != b.kept])
        assert flipped.tolist() == [int(key_of(bf16_bits([1.0]))[0])] and (a.kept >= b.kept).all()
        for mp in (lo, hi):
            assert np.array_equal(select(bits, 1.0, min_p=mp).kept, oracle_kept(bits, 1.0, min_p=mp)[0])


def test_topp_error_bound_is_far_below_the_slacks():
    for c in CASES:
        bits = c.row(128256)
        sel, _, _, rep = design(c, bits)
        if sel.topp_on:
            slack, B = rep["topp_slack"]
            assert B < 1e-6 and slack > 3 * B, (c.name, slack, B)
            assert B == topp_error_bound(bits, c.T, sel.kept)


@pytest.mark.parametrize("seed", range(6))
def test_restatement_equals_the_oracle_on_random_rows(seed):
    """Random Gaussian rows and parameters: the kept sets agree wherever the top-p slack clears the float32 rounding of
    z - z_max (the restatement's masses) by far; min_p and top-k need no exemption (the same predicate and keys)."""
    rng = np.random.default_rng(seed)
    exempt = 0
    for _ in range(40):
        V = int(rng.choice([7, 203, 1000, 4096]))
        vals = (rng.standard_normal(V) * rng.choice([0.5, 3.0, 20.0])).astype(np.float32)
        vals[rng.random(V) < 0.05] = -np.inf
        vals[rng.integers(0, V, 3)] = vals[rng.integers(0, V)]               # ties
        bits = (vals.view(np.uint32) >> 16).astype(np.uint16)               # truncate to bf16
        T = np.float32(rng.choice([1e-5, 0.3, 1.0, 2.5]))
        k = int(rng.choice([0, 1, 2, 5, 50, V - 1, V]))
        p = np.float32(rng.choice([1.0, 0.99, 0.9, 0.5, 0.1, 1e-4]))
        mp = np.float32(rng.choice([0.0, 0.0, 1e-3, 0.05, 0.3, 0.9]))
        if not np.isfinite(f32_of_bits(bits)).any():
            continue
        sel = select(bits, T, k, p, mp)
        want, slack, _ = oracle_kept(bits, T, k, p, mp)
        if not np.array_equal(sel.kept, want):
            assert slack < 1e-6, (V, T, k, p, mp, slack)
            exempt += 1
    print(f"{exempt} of 40 rows exempt by top-p slack")
    assert exempt <= 2


def test_vectorised_race_equals_the_oracle_token_for_token():
    c = next(c for c in CASES if c.name == "all_three_pass4_reruns_bk")
    bits = c.row(1000)
    sel, (T, k, p, mp), _, _ = design(c, bits)
    lf = f32_of_bits(bits)
    ns = np.arange(0, 64 * 7, 7)
    toks, margins = race(bits, T, sel.kept, 0x1234_5678_9ABC, ns)
    for n, t, m in zip(ns, toks, margins):
        tok, margin, _, _ = sample_ref(lf, T, k, p, 0x1234_5678_9ABC, int(n), mp)
        assert tok == t and np.isclose(margin, m)


def test_builder_places_tiers_at_seeded_positions():
    a = build_row(1000, [(1.0, 5), (0.5, 7)], seed=3)
    assert np.array_equal(a, build_row(1000, [(1.0, 5), (0.5, 7)], seed=3))
    f = f32_of_bits(a)
    assert (f == 1.0).sum() == 5 and (f == 0.5).sum() == 7 and (f == -2.0 ** 100).sum() == 988
