"""Logprobs, CPU-only parts: the oracle (oracle/logprobs.py) against vLLM's own Sampler.compute_logprobs /
gather_logprobs and its OpenAI response builders, and the serving shell's request-field matrix with enable_logprobs off
(today's 400s, word for word) and on."""
import json
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from kubeai_b200.server import Server
from oracle.logprobs import chat_logprobs, completion_logprobs, logprobs_ref, position_entries


TOL = 1e-6


def tie_free_rows(S, V, seed):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn(S, V, generator=g, dtype=torch.float64) * 3
    return rows.float()          # float32 values, distinct with probability 1


def test_oracle_equals_vllm_sampler():
    sampler = pytest.importorskip("vllm.v1.sample.sampler")
    S, V, N = 6, 3000, 20
    rows = tie_free_rows(S, V, 1)
    tokens = torch.tensor([0, 5, 17, 2999, 1234, 42], dtype=torch.int64)
    lp_v = sampler.Sampler.compute_logprobs(rows)
    for s in range(S):
        ref, ids = logprobs_ref(rows[s].numpy(), N)
        assert (np.abs(lp_v[s].double().numpy() - ref) <= TOL + 2.0 ** -22 * np.abs(ref)).all()   # fp32 output rounding
    try:
        got = sampler.Sampler.gather_logprobs(lp_v, N, tokens)
    except Exception as e:          # needs a custom op that may not run without a GPU
        pytest.skip(f"gather_logprobs does not run here: {e}")
    for s in range(S):
        ref, ids = logprobs_ref(rows[s].numpy(), N)
        assert got.logprob_token_ids[s, 0] == tokens[s]
        assert got.logprob_token_ids[s, 1:].tolist() == ids.tolist()
        assert abs(float(got.logprobs[s, 0]) - ref[tokens[s]]) <= TOL + 2.0 ** -22 * abs(ref[tokens[s]])
        assert (np.abs(got.logprobs[s, 1:].double().numpy() - ref[ids]) <= TOL + 2.0 ** -22 * np.abs(ref[ids])).all()


def records(seed, n_pos=4, N=5, V=300):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_pos):
        x = rng.standard_normal(V).astype(np.float32) * 3
        ref, ids = logprobs_ref(x, N)
        tok = int(ids[1]) if k % 2 else int(rng.integers(0, V))    # sampled token inside / outside the top N
        out.append((tok, np.float32(ref[tok]), ids, ref[ids].astype(np.float32)))
    return out


def token_str(t):
    return ["é", "a", "bb", " x", "\U0001f642"][t % 5] + str(t // 5)


def _vllm_builders():
    chat = pytest.importorskip("vllm.entrypoints.openai.chat_completion.serving")
    comp = pytest.importorskip("vllm.entrypoints.openai.completion.serving")
    lp_mod = pytest.importorskip("vllm.logprobs")
    return chat.OpenAIServingChat, comp.OpenAIServingCompletion, lp_mod.Logprob


def _vllm_dicts(recs, Logprob):
    out = []
    for tok, lp, ids, lps in recs:
        d = position_entries(tok, lp, ids, lps)
        out.append({t: Logprob(logprob=v, rank=None, decoded_token=token_str(t)) for t, v in d.items()})
    return out


@pytest.mark.parametrize("N", [0, 1, 5])
def test_response_builders_equal_vllm(N):
    Chat, Comp, Logprob = _vllm_builders()
    recs = [(t, lp, ids[:N], lps[:N]) for t, lp, ids, lps in records(N + 3)]
    tops = _vllm_dicts(recs, Logprob)
    ids = [r[0] for r in recs]
    fake = SimpleNamespace(return_tokens_as_token_ids=False)
    fake._get_decoded_token = Chat._get_decoded_token
    fake._get_top_logprobs = lambda *a: Chat._get_top_logprobs(fake, *a)
    want = Chat._create_chat_logprobs(fake, ids, tops, None, N).model_dump(mode="json")
    assert want == chat_logprobs(recs, N, token_str)
    want = Comp._create_completion_logprobs(fake, ids, tops, N, None, 7).model_dump(mode="json")
    assert want == completion_logprobs(recs, N, token_str, 7)


# ------------------------------------------------------------------ request fields
BASE_CHAT = {"model": "m", "messages": [{"role": "user", "content": "hi"}]}
BASE_COMP = {"model": "m", "prompt": "hi"}
CHAT_OK = [({"logprobs": True}, 0), ({"logprobs": True, "top_logprobs": 5}, 5), ({"logprobs": True, "top_logprobs": 20}, 20),
           ({"logprobs": False}, None), ({"logprobs": None, "top_logprobs": None}, None), ({"top_logprobs": 0}, None),
           ({"logprobs": True, "top_logprobs": 0}, 0), ({"logprobs": True, "top_logprobs": 3.0}, 3)]
CHAT_BAD = [{"logprobs": True, "top_logprobs": 21}, {"logprobs": True, "top_logprobs": -1},
            {"logprobs": True, "top_logprobs": 2.5}, {"logprobs": True, "top_logprobs": "5"}, {"top_logprobs": 5},
            {"logprobs": False, "top_logprobs": 1}, {"logprobs": 1}, {"logprobs": "yes"},
            {"logprobs": True, "prompt_logprobs": 1}, {"logprobs": True, "echo": True}]
COMP_OK = [({"logprobs": 0}, 0), ({"logprobs": 5}, 5), ({"logprobs": 20}, 20), ({"logprobs": None}, None), ({}, None)]
COMP_BAD = [{"logprobs": 21}, {"logprobs": -1}, {"logprobs": 1.5}, {"logprobs": True}, {"logprobs": "3"},
            {"logprobs": 2, "prompt_logprobs": 2}, {"logprobs": 2, "echo": True}, {"top_logprobs": 3}]


def _status(srv, path, body):
    st, out = srv.parse_request(path, json.dumps(body))
    return st, out.get("error", "")


def test_fields_keep_todays_400_when_off():
    with Server([None], model="m") as off:
        for extra, _ in CHAT_OK + [(b, None) for b in CHAT_BAD]:
            body = {**BASE_CHAT, **extra}
            want = 400 if any(isinstance(extra.get(k), (bool, int, float)) and extra.get(k) and extra.get(k) is not False
                              for k in ("logprobs", "top_logprobs", "prompt_logprobs", "echo")) else 0
            st, err = _status(off, "/v1/chat/completions", body)
            assert st == want, (extra, st, err)
            if st:
                assert err in ("bad request: logprobs is not supported by this engine",
                               "bad request: echo is not supported by this engine"), err
        for extra, _ in COMP_OK + [(b, None) for b in COMP_BAD]:
            st, err = _status(off, "/v1/completions", {**BASE_COMP, **extra})
            truthy = any(isinstance(extra.get(k), (bool, int, float)) and extra.get(k) and extra.get(k) > 0
                         for k in ("logprobs", "top_logprobs", "prompt_logprobs", "echo"))
            assert st == (400 if truthy else 0), (extra, st, err)


def test_fields_when_on():
    with Server([None], model="m", enable_logprobs=True) as on:
        for extra, _ in CHAT_OK:
            assert _status(on, "/v1/chat/completions", {**BASE_CHAT, **extra})[0] == 0, extra
        for extra in CHAT_BAD:
            st, err = _status(on, "/v1/chat/completions", {**BASE_CHAT, **extra})
            assert st == 400 and err.startswith("bad request: "), (extra, st, err)
        for extra, _ in COMP_OK:
            assert _status(on, "/v1/completions", {**BASE_COMP, **extra})[0] == 0, extra
        for extra in COMP_BAD:
            st, err = _status(on, "/v1/completions", {**BASE_COMP, **extra})
            assert st == 400 and err.startswith("bad request: "), (extra, st, err)
        assert "prompt_logprobs" in _status(on, "/v1/completions", {**BASE_COMP, "prompt_logprobs": 1})[1]
        assert "echo" in _status(on, "/v1/completions", {**BASE_COMP, "echo": True})[1]
        assert "needs" in _status(on, "/v1/chat/completions", {**BASE_CHAT, "top_logprobs": 2})[1]
