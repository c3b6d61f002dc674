"""Sampling without a GPU: the oracle (oracle/sampling.py) against Philox4x32-10's known answers, vLLM's own top-k / top-p
mask and the distribution it draws from; the serving shell's validation of the sampling fields."""
import json

import numpy as np
import pytest
from scipy import stats

from kubeai_b200.server import PREFIX_HASH, Server
from oracle.sampling import filter_mask, philox4x32_10, probs, sample_ref, scaled, uniforms


def test_philox_known_answers():
    # Random123's known-answer vectors for philox4x32 with 10 rounds
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        assert tuple(int(x) for x in philox4x32_10(ctr, key)) == want
    u = uniforms(7, np.arange(3), 4096)
    assert u.shape == (3, 4096) and (u > 0).all() and (u < 1).all()
    assert np.array_equal(u[2], uniforms(7, 2, 4096))


def test_filter_matches_vllm_top_k_top_p_mask():
    ops = pytest.importorskip("vllm.v1.sample.ops.topk_topp_sampler")
    import torch
    rng = np.random.default_rng(3)
    V = 1000
    # distinct values (no ties), shuffled, spread over about +-8
    rows = np.stack([rng.permutation(np.cumsum(rng.uniform(0.002, 0.03, V)) - 8.0) for _ in range(200)]).astype(np.float32)
    assert all(len(np.unique(r)) == V for r in rows)
    checked = 0
    for T in (0.5, 1.0, 1.7):
        for k in (0, 1, 20, 500, V):
            for p in (1.0, 0.95, 0.6, 0.1):
                z = np.stack([scaled(r, T) for r in rows])
                got, slacks = zip(*[filter_mask(zr, k, p) for zr in z])
                zt = torch.from_numpy(z.astype(np.float32))
                masked = ops.apply_top_k_top_p_pytorch(zt.clone(), torch.full((200,), k if k > 0 else V, dtype=torch.long),
                                                       torch.full((200,), p, dtype=torch.float32) if p < 1 else None)
                want = torch.isfinite(masked).numpy()
                for g, w, s in zip(got, want, slacks):
                    if s < 1e-5:    # fp32 cumsum in vLLM vs float64 here: a coin flip at the boundary
                        continue
                    assert np.array_equal(g, w), (T, k, p)
                    checked += 1
    assert checked > 0.99 * 3 * 5 * 4 * 200


@pytest.mark.parametrize("T,k,p", [(1.0, 0, 1.0), (0.7, 5, 1.0), (1.3, 0, 0.8), (0.9, 6, 0.9)])
def test_race_frequencies_follow_the_filtered_softmax(T, k, p):
    rng = np.random.default_rng(11)
    l = (rng.standard_normal(12) * 1.5).astype(np.float32)
    want = probs(l, T, k, p)
    z = scaled(l, T)
    keep, _ = filter_mask(z, k, p)
    N = 40000
    e = -np.log(uniforms(0x1234_5678_9ABC, np.arange(N), l.size))          # [N, V]
    draws = np.argmax(np.where(keep, z - np.log(e), -np.inf), axis=1)
    assert keep[draws].all()
    counts = np.bincount(draws, minlength=l.size)[keep]
    res = stats.chisquare(counts, want[keep] * N)
    assert res.pvalue > 1e-3, (res, counts, want[keep] * N)
    # the one-row helper agrees with the vectorised race
    for n in (0, 1, 999):
        assert sample_ref(l, T, k, p, seed=0x1234_5678_9ABC, n=n)[0] == draws[n]


def test_greedy_rows_are_the_argmax_and_ignore_filters():
    l = np.array([0.5, 2.0, -1.0, 2.0, 1.0], dtype=np.float32)
    for T in (0.0, 9e-6):
        assert sample_ref(l, T, top_k=1, top_p=0.1, seed=5, n=3)[0] == 1     # lowest index among the tied maxima
    keep, _ = filter_mask(scaled(l, 1.0), top_k=1)
    assert keep.tolist() == [False, True, False, True, False]              # ties at the k-th value are kept
    keep, _ = filter_mask(scaled(l, 1.0), top_p=0.5)
    assert keep.tolist() == [False, True, False, True, False]              # a tie group is kept or dropped whole


@pytest.fixture()
def psrv():
    with Server([None], model="test-model", strategy=PREFIX_HASH) as s:
        yield s


def test_server_validates_sampling_fields(psrv):
    base = {"model": "test-model", "messages": [{"role": "user", "content": "hi"}]}
    ok = [{"temperature": 0.8}, {"temperature": 0}, {"temperature": 2, "top_p": 1}, {"top_p": 0.9, "top_k": 40},
          {"top_k": -1}, {"top_k": 0}, {"seed": 7}, {"seed": -3}, {"seed": 2 ** 53}, {"seed": 0, "temperature": 1.0},
          {"min_p": 0.1}, {"min_p": 0.1, "temperature": 0}, {"min_p": 0, "temperature": 0.7}, {"top_k": 5}]
    for extra in ok:
        st, out = psrv.parse_request("/openai/v1/chat/completions", json.dumps({**base, **extra}))
        assert st == 0, (extra, out)
    bad = [({"temperature": -0.1}, "temperature"), ({"top_p": 0}, "top_p"), ({"top_p": 1.5}, "top_p"),
           ({"top_p": -0.2}, "top_p"), ({"top_k": -2}, "top_k"), ({"top_k": 2.5}, "top_k"), ({"seed": 1.5}, "seed"),
           ({"seed": 2 ** 53 + 2}, "seed"), ({"seed": -(2 ** 54)}, "seed"), ({"temperature": 1e39}, "temperature"),
           ({"min_p": 0.1, "temperature": 0.7}, "min_p")]
    for extra, msg in bad:
        st, out = psrv.parse_request("/openai/v1/chat/completions", json.dumps({**base, **extra}))
        assert st == 400 and msg in out["error"], (extra, st, out)


def test_sampling_is_a_server_setting():
    """enable_sampling off (the default): a sampled request gets the greedy-only 400 after the field checks; on: it
    passes them (with no engine behind the replica it then fails at the engine, 502)."""
    body = {"model": "model1", "messages": [{"role": "user", "content": "hi"}], "max_tokens": 2}
    with Server([None], model="model1") as off, Server([None], model="model1", enable_sampling=True, max_retries=0) as on:
        r = off.handle("POST", "/openai/v1/chat/completions", json.dumps({**body, "temperature": 0.7}))
        assert r.status == 400 and "greedy" in r.json()["error"]
        for srv in (off, on):
            r = srv.handle("POST", "/openai/v1/chat/completions", json.dumps({**body, "temperature": -0.7}))
            assert r.status == 400 and "temperature" in r.json()["error"]
            r = srv.handle("POST", "/openai/v1/chat/completions", json.dumps({**body, "temperature": 0.7, "min_p": 0.1}))
            assert r.status == 400 and "min_p" in r.json()["error"]
        assert on.handle("POST", "/openai/v1/chat/completions", json.dumps({**body, "temperature": 0.7})).status == 502
