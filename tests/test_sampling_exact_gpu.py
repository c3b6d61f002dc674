"""The sampler kernel (sample_kernel, kubeai_b200/csrc/sampling.cu) pinned to exact kept sets on constructed rows
(oracle/sampling_cases.py): at every case and vocabulary size the set of drawn ids equals the oracle's kept set, and every
draw is the oracle's race winner except where the race's top-2 margin is under 1e-4.  Then every greedy selector the
engine can run (argmax_rows, the sampler's greedy branch, the lm_head ARGMAX epilogue) against np.argmax on constructed
ties, greedy streams that must not depend on which of them ran, and the sampler on a row holding +NaN."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle.sampling_cases import CASES, V_SIZES, design, oracle_kept, probs_of, race
from oracle.sampling_keys import bf16_bits, f32_of_bits, key_of, select

pytestmark = pytest.mark.gpu
MARGIN = 1e-4                    # the race's fp32 scores may part from float64 only below this top-2 margin
SEED = 0x5EED_CA5E_0001
CHUNK = 4096
POISON = 0x7180                  # bf16 +2^100: past V in a row with ld > V; read, it would win every selection


def ld_of(V):
    return V if V % 8 == 0 else (V + 7) // 8 * 8 + 8


def sample_ld(logits, V, T, k, p, seed, n, mp):
    """b200_op_sample on bf16 logits [S, ld] read as [S, V]; each parameter a scalar or one per row."""
    from kubeai_b200._lib import check, lib
    S, ld = logits.shape
    rows = np.empty(S, dtype=[("temperature", "<f4"), ("top_k", "<i4"), ("top_p", "<f4"), ("seed_lo", "<u4"),
                              ("seed_hi", "<u4"), ("n", "<i4"), ("min_p", "<f4")])
    seed = np.broadcast_to(np.asarray(seed, dtype=object), (S,))
    rows["temperature"] = np.broadcast_to(np.asarray(T, dtype=np.float32), (S,))
    rows["top_k"] = np.broadcast_to(np.asarray(k, dtype=np.int32), (S,))
    rows["top_p"] = np.broadcast_to(np.asarray(p, dtype=np.float32), (S,))
    rows["seed_lo"] = [int(s) & 0xFFFFFFFF for s in seed]
    rows["seed_hi"] = [(int(s) >> 32) & 0xFFFFFFFF for s in seed]
    rows["n"] = np.broadcast_to(np.asarray(n, dtype=np.int32), (S,))
    rows["min_p"] = np.broadcast_to(np.asarray(mp, dtype=np.float32), (S,))
    rows_dev = torch.from_numpy(rows.view(np.int32).reshape(S, 7).copy()).cuda()
    out = torch.empty(S, dtype=torch.int32, device="cuda")
    check(lib().b200_op_sample(C.c_void_p(logits.data_ptr()), ld, C.c_void_p(rows_dev.data_ptr()), S, V,
                               C.c_void_p(out.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out.cpu().numpy()


def device_rows(bits, S, ld):
    """S copies of one row of bf16 bits, padded to ld with POISON."""
    V = bits.shape[0]
    buf = torch.full((S, ld), POISON, dtype=torch.int16, device="cuda")
    buf[:, :V] = torch.from_numpy(bits.view(np.int16)).cuda()
    return buf.view(torch.bfloat16)


def draw(bits, params, N, seed=SEED):
    """The row drawn at generation indices 0..N-1, CHUNK rows per launch."""
    V = bits.shape[0]
    T, k, p, mp = params
    buf = device_rows(bits, min(N, CHUNK), ld_of(V))
    return np.concatenate([sample_ld(buf[:min(CHUNK, N - c)], V, T, k, p, seed, np.arange(c, min(c + CHUNK, N)), mp)
                           for c in range(0, N, CHUNK)])


def live_kept(bits, params):
    """The oracle's kept tokens that can be drawn (nonzero mass), or the argmax of a greedy row."""
    keep = oracle_kept(bits, *params)[0]
    if not np.float32(params[0]) >= np.float32(1e-5):
        return keep
    return keep & (probs_of(bits, params[0], keep)[0] > 0)


@pytest.mark.parametrize("V", V_SIZES)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_kept_set_is_exact_and_every_draw_is_the_oracles(case, V):
    bits = case.row(V)
    sel, params, N, rep = design(case, bits)
    got = draw(bits, params, N)
    want = live_kept(bits, params)
    drawn = np.zeros(V, dtype=bool)
    drawn[got] = True
    assert np.array_equal(drawn, want), (f"{case.name} ({case.config}): drawn but not kept "
                                         f"{np.flatnonzero(drawn & ~want)[:8]}, kept but never drawn "
                                         f"{np.flatnonzero(want & ~drawn)[:8]}; {sel.describe()}")
    ns = np.arange(N)
    if sel.greedy:
        assert (got == int(np.flatnonzero(want)[0])).all()
        return
    toks = np.empty(N, dtype=np.int64)
    margins = np.empty(N)
    keep = oracle_kept(bits, *params)[0]
    for c in range(0, N, CHUNK):
        toks[c:c + CHUNK], margins[c:c + CHUNK] = race(bits, params[0], keep, SEED, ns[c:c + CHUNK])
    bad = got != toks
    print(f"{case.name} V={V}: {sel.describe()} N={N}, {int(bad.sum())} draws exempt (race margin < {MARGIN})")
    assert (margins[bad] < MARGIN).all(), (case.name, np.flatnonzero(bad & (margins >= MARGIN))[:8])
    assert bad.sum() <= max(2, N // 1000)


def test_tiny_vocabulary_below_one_vector_with_a_padded_stride():
    """V = 5 < 8 and ld = 8: only visit_row's scalar tail reads the row; the padding is never selected."""
    vals = np.array([1.0, 0.5, 1.0, -np.inf, 0.25], dtype=np.float32)
    bits = bf16_bits(vals)
    N = 4096
    for params in [(1.0, 0, 1.0, 0.0), (0.7, 2, 1.0, 0.0), (1.0, 0, 0.5, 0.0), (1.0, 0, 1.0, 0.5), (1.0, 3, 0.9, 0.3),
                   (0.0, 0, 1.0, 0.0), (2.0, 4, 0.99, 0.01)]:
        params = tuple(np.float32(x) if i != 1 else int(x) for i, x in enumerate(params))
        got = draw(bits, params, N)
        want = live_kept(bits, params)
        drawn = np.zeros(5, dtype=bool)
        drawn[got] = True
        assert np.array_equal(drawn, want), (params, got[:16])
        assert np.array_equal(select(bits, *params).kept & want, want)
        if params[0] >= 1e-5:
            toks, margins = race(bits, params[0], oracle_kept(bits, *params)[0], SEED, np.arange(N))
            assert (margins[got != toks] < MARGIN).all(), params


def test_batch_of_every_case_equals_each_case_alone():
    V, ns = 1000, np.array([0, 1, 77, 4095])
    rows, params, seeds = [], [], []
    for i, c in enumerate(CASES):
        bits = c.row(V)
        rows.append(bits)
        params.append(c.params(bits))
        seeds.append(SEED + i)
    S = len(CASES) * len(ns)
    buf = torch.from_numpy(np.repeat(np.stack(rows), len(ns), axis=0).view(np.int16)).cuda().view(torch.bfloat16)
    P = np.repeat(np.array([(float(T), k, float(p), float(mp)) for T, k, p, mp in params], dtype=object), len(ns), axis=0)
    batch = sample_ld(buf, V, P[:, 0].astype(np.float32), P[:, 1].astype(np.int32), P[:, 2].astype(np.float32),
                      np.repeat(seeds, len(ns)), np.tile(ns, len(CASES)), P[:, 3].astype(np.float32))
    assert batch.shape == (S,)
    for i, c in enumerate(CASES):
        T, k, p, mp = params[i]
        solo = sample_ld(device_rows(rows[i], len(ns), V), V, T, k, p, seeds[i], ns, mp)
        assert np.array_equal(batch[i * len(ns):(i + 1) * len(ns)], solo), c.name


# ------------------------------------------------------------------ greedy: every selector, constructed ties
def greedy_rows(V):
    """(name, float32 row, bf16-exact) with the maximum placed where the selectors' reductions meet."""
    rng = np.random.default_rng(V)
    base = -rng.integers(1, 200, V).astype(np.float32) / 64        # bf16-exact values in [-3.1, -0.015]
    out = []

    def at(name, pos, value=8.0, fill=None):
        r = base.copy() if fill is None else np.full(V, fill, dtype=np.float32)
        for q in pos:
            r[q] = value
        out.append((name, r))
    at("tie_across_slabs", [130, 300] if V > 300 else [5, 200])
    at("tie_within_lane", [256 + 4 * 5 + 1, 256 + 4 * 5 + 3] if V > 300 else [4 * 5 + 1, 4 * 5 + 3])
    if V >= 8 * 2049:   # thread 1000's first load, thread 0's second load and its next iteration
        at("tie_across_threads", [8 * 1000 + 2, 8 * 1024 + 1, 8 * 2048])
    else:
        at("tie_across_threads", [8 * (V // 8 - 1) - 6, 8 * 3 + 5])
    at("tie_at_ends", [0, V - 1])
    at("max_at_last", [V - 1])
    at("only_finite_at_last", [V - 1], value=-7.0, fill=-np.inf)
    r = np.full(V, -1.0, dtype=np.float32)
    r[3], r[7] = -0.0, 0.0
    out.append(("neg_zero_first", r))
    r = r.copy()
    r[3], r[7] = 0.0, -0.0
    out.append(("pos_zero_first", r))
    return out


@pytest.mark.parametrize("V", [203, 1000, 128256])
def test_greedy_selectors_agree_with_first_maximum(V):
    from kubeai_b200 import ops
    from kubeai_b200._lib import check, lib
    rows = greedy_rows(V)
    names = [n for n, _ in rows]
    want = np.array([int(np.argmax(r)) for _, r in rows])
    bits = np.stack([bf16_bits(r) for _, r in rows])
    ld = ld_of(V)
    pad = np.full((len(rows), ld), POISON, dtype=np.uint16)
    pad[:, :V] = bits
    buf = torch.from_numpy(pad.view(np.int16)).cuda().view(torch.bfloat16)
    am = torch.empty(len(rows), dtype=torch.int32, device="cuda")
    check(lib().b200_op_argmax(C.c_void_p(buf.data_ptr()), C.c_void_p(am.data_ptr()), len(rows), V, ld,
                               C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    got = {"argmax_rows": am.cpu().numpy(),
           "sample T=0": sample_ld(buf, V, 0.0, 0, 1.0, SEED, 0, 0.0),
           "sample T=0 with filters": sample_ld(buf, V, 0.0, 3, 0.5, SEED, 9, 0.2)}
    if ld == V:
        got["ops.sample"] = ops.sample(buf, 0.0).cpu().numpy()
        got["ops.argmax"] = ops.argmax(buf).cpu().numpy()
    for sel, g in got.items():
        assert np.array_equal(g, want), (sel, [(n, int(a), int(b)) for n, a, b in zip(names, g, want) if a != b])


@pytest.mark.parametrize("N,n_valid", [(1024, 0), (1024, 1000), (128256, 128000)])
def test_argmax_epilogue_on_constructed_ties(N, n_valid):
    """lm_head ARGMAX epilogue: exact ties from duplicated weight rows, placed across 128-column slabs, inside one lane's
    four columns and at both ends, with a larger maximum past n_valid that must be ignored."""
    from kubeai_b200 import ops
    T, K = 4, 256
    g = torch.Generator(device="cuda").manual_seed(N + n_valid)
    x = torch.randn(T, K, generator=g, device="cuda").abs().bfloat16()
    w0 = (torch.randn(N, K, generator=g, device="cuda") / 16).bfloat16()
    nv = n_valid or N
    big = torch.full((K,), 0.5, dtype=torch.bfloat16, device="cuda")
    tie_sets = {"across_slabs": [130, 300, 700], "within_lane": [512 + 4 * 9 + 1, 512 + 4 * 9 + 2, 512 + 4 * 9 + 3],
                "ends": [0, nv - 1], "last_only": [nv - 1]}
    for name, ties in tie_sets.items():
        w = w0.clone()
        w[ties] = big
        if n_valid:
            w[n_valid + 5] = 0.75                                # the largest logit, past n_valid
            w[N - 1] = 0.75
        plain, _ = ops.gemm3(x, w)
        ids, _ = ops.gemm3(x, w, epi=ops.EPI_ARGMAX, n_valid=n_valid)
        torch.cuda.synchronize()
        lg = plain.float().cpu().numpy()[:, :nv]
        assert (lg[:, ties] == lg[:, ties[:1]]).all(), f"{name}: the duplicated rows are not exact ties"
        want = np.argmax(lg, axis=1)
        assert (want == ties[0]).all(), name
        assert np.array_equal(ids.cpu().numpy(), want), (name, ids.cpu().numpy(), want)


# ------------------------------------------------------------------ engine: the greedy stream does not depend on the selector
NEIGHBOURS = {"epilogue (all greedy)": dict(temperature=0.0),
              "sample_kernel greedy branch": dict(temperature=0.9, top_p=0.9, seed=5),
              "argmax_rows (logprobs)": dict(temperature=0.0, logprobs=True, top_logprobs=3),
              "penalties then argmax_rows": dict(temperature=0.0, repetition_penalty=1.5)}


def test_greedy_streams_do_not_depend_on_the_selector():
    from kubeai_b200.engine import Engine, mini_config
    prompts = [list(np.random.default_rng(70 + i).integers(0, 512, 6 + 3 * i)) for i in range(5)]
    n_tok, nb = 16, 2
    streams = {}
    for mode, spec in NEIGHBOURS.items():
        with Engine(mini_config()) as e:
            rids = [e.submit(p, max_tokens=n_tok, **(spec if i == nb else {})) for i, p in enumerate(prompts)]
            for _ in range(n_tok):
                ran, info = e.step()
                assert ran and info.sampled == len(rids)       # the same batch shape at every step
            outs = [e.poll(r).tokens for r in rids]
        assert all(len(o) == n_tok for o in outs), mode
        streams[mode] = [o for i, o in enumerate(outs) if i != nb]
    first = next(iter(streams.values()))
    for mode, s in streams.items():
        assert s == first, mode


# ------------------------------------------------------------------ +NaN in a row
def test_positive_nan_row_pins_todays_selection():
    """A +NaN logit has the largest key (above +inf).  Greedy and temperature-only rows ignore it; top-k counts it as the
    largest key (so k - 1 real tokens stay); with top-p or min_p on, z_max is NaN and the row returns token 0."""
    V = 1000
    c = next(c for c in CASES if c.name == "topk_kth_in_tie_group")
    clean = c.row(V)
    nan_at = int(np.flatnonzero(f32_of_bits(clean) == np.float32(-2.0 ** 100))[5])     # a filler position, not token 0
    bits = clean.copy()
    bits[nan_at] = 0x7FC0
    assert np.isnan(f32_of_bits(bits)[nan_at]) and key_of(bits).max() == 0xFFC0
    N = 4096
    # greedy: the argmax of the other tokens
    g = draw(bits, (np.float32(0.0), 0, np.float32(1.0), np.float32(0.0)), 64)
    assert (g == int(np.argmax(f32_of_bits(clean)))).all()
    # temperature only, and top-k: the race never picks NaN; top-k 10 keeps the NaN key and the top 9 real tokens
    for k in (0, 10):
        params = (np.float32(1.0), k, np.float32(1.0), np.float32(0.0))
        got = draw(bits, params, N)
        assert nan_at not in got
        kept = select(bits, *params).kept.copy()
        kept[nan_at] = False
        toks, margins = race(clean, np.float32(1.0), kept, SEED, np.arange(N))
        assert (margins[got != toks] < MARGIN).all(), k
        if k:   # the NaN key takes one of the k places: the 2.0 tie group (ranks 9-14) is still reached and kept whole
            assert kept.sum() == 13 and set(np.unique(got)) == set(np.flatnonzero(kept))
    # top-p or min_p: token 0
    for params in [(1.0, 0, 0.9, 0.0), (1.0, 0, 1.0, 0.1), (1.0, 20, 0.9, 0.1)]:
        params = (np.float32(params[0]), params[1], np.float32(params[2]), np.float32(params[3]))
        assert (draw(bits, params, 64) == 0).all(), params
