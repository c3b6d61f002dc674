"""Prompt logprobs and echo, CPU-only parts: the oracle (oracle/prompt_logprobs.py) against vLLM's own
Sampler.gather_logprobs ranks, its prompt-logprob dict builder and its OpenAI response builders, and the serving shell's
request-field matrix with enable_prompt_logprobs off (today's 400s, word for word) and on."""
import json
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from kubeai_b200.server import Server
from oracle.logprobs import logprobs_ref
from oracle.prompt_logprobs import echo_completion_logprobs, prompt_entry, prompt_logprobs_json, rank_ref


def _rows():
    g = torch.Generator().manual_seed(3)
    tie_free = (torch.randn(4, 2000, generator=g, dtype=torch.float64) * 3).float()
    # bf16 rows with ties at the target: all equal, 1000 equal to the target, target the max, target the min, -0 / +0
    tied = torch.randn(5, 2000, generator=g).bfloat16().float()
    tied[0] = 0.5
    tied[1, :1000] = tied[1, 7]
    tied[2, 11] = tied[2].max() + 1
    tied[3, 13] = tied[3].min() - 1
    tied[4, :500] = 0.0
    tied[4, 500:1000] = -0.0
    return torch.cat([tie_free, tied]), torch.tensor([5, 17, 1999, 0, 3, 7, 11, 13, 700])


def test_rank_equals_vllm_gather_logprobs():
    sampler = pytest.importorskip("vllm.v1.sample.sampler")
    rows, tokens = _rows()
    lp_v = sampler.Sampler.compute_logprobs(rows)
    with torch.compiler.set_stance("force_eager"):   # the compiled count needs a C++ toolchain, the eager one does not
        got = sampler.Sampler.gather_logprobs(lp_v, 20, tokens)
    for s in range(len(rows)):
        assert int(got.selected_token_ranks[s]) == rank_ref(rows[s].numpy(), tokens[s]), s
    assert [rank_ref(rows[s].numpy(), tokens[s]) for s in (4, 6, 7)] == [2000, 1, 2000]


@pytest.mark.parametrize("N", [0, 1, 5, 20])
def test_prompt_entry_equals_vllm(N):
    lp_mod = pytest.importorskip("vllm.logprobs")
    rows, tokens = _rows()
    for s in range(len(rows)):
        x = rows[s].numpy()
        lp, ids = logprobs_ref(x, N)
        t = int(tokens[s])
        rank = rank_ref(x, t)
        want = lp_mod.create_prompt_logprobs(False)
        lp_mod.append_logprobs_for_next_position(want, [t] + ids.tolist(), [float(lp[t])] + lp[ids].tolist(),
                                                 [str(i) for i in [t] + ids.tolist()], rank, N)
        got = prompt_entry(t, lp[t], rank, ids, lp[ids])
        assert list(want[1].keys()) == list(got.keys())
        assert {k: (v.logprob, v.rank) for k, v in want[1].items()} == got


def token_str(t):
    return ["é", "a", "bb", " x", "\U0001f642"][t % 5] + str(t // 5)


def _prompt_records(prompt, N, V=300, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(len(prompt) - 1):
        x = (rng.standard_normal(V) * 3).astype(np.float32)
        if k == 1:
            x[5] = -np.inf        # a -inf entry: clamped to -9999 by vLLM's clamp_prompt_logprobs
        lp, ids = logprobs_ref(x, N)
        t = int(prompt[k + 1])
        out.append((t, np.float32(lp[t]), rank_ref(x, t), ids, lp[ids].astype(np.float32)))
    return out


def _vllm_prompt_dicts(recs, Logprob):
    out = [None]
    for tok, lp, rank, ids, lps in recs:
        out.append({t: Logprob(logprob=v, rank=r, decoded_token=token_str(t))
                    for t, (v, r) in prompt_entry(tok, lp, rank, ids, lps).items()})
    return out


@pytest.mark.parametrize("N", [0, 1, 5])
def test_echo_and_prompt_logprobs_builders_equal_vllm(N):
    comp = pytest.importorskip("vllm.entrypoints.openai.completion.serving")
    proto = pytest.importorskip("vllm.entrypoints.openai.completion.protocol")
    engine_serving = pytest.importorskip("vllm.entrypoints.openai.engine.serving")
    lp_mod = pytest.importorskip("vllm.logprobs")
    prompt = [3, 5, 5, 250, 1, 7]
    recs = _prompt_records(prompt, N)
    rng = np.random.default_rng(9)
    outs = []
    for k in range(2):
        x = (rng.standard_normal(300) * 3).astype(np.float32)
        lp, ids = logprobs_ref(x, N)
        t = int(ids[0]) if k and N else 17 + k    # the second generated token is the top one when there is a top
        outs.append((t, np.float32(lp[t]), ids, lp[ids].astype(np.float32)))
    dicts = engine_serving.clamp_prompt_logprobs(_vllm_prompt_dicts(recs, lp_mod.Logprob))
    # prompt_logprobs as vLLM's pydantic response writes it
    choice = proto.CompletionResponseChoice(index=0, text="", prompt_logprobs=dicts).model_dump(mode="json")
    assert choice["prompt_logprobs"] == prompt_logprobs_json(recs, token_str)
    assert choice["prompt_logprobs"][2]["5"]["logprob"] == -9999.0 or 5 not in dict(prompt_entry(*recs[1]))
    # echo: _create_completion_logprobs over [None, prompt dicts..., output dicts...]
    fake = SimpleNamespace(return_tokens_as_token_ids=False)
    fake._get_decoded_token = comp.OpenAIServingCompletion._get_decoded_token
    tok = SimpleNamespace(decode=lambda t: token_str(t))
    out_dicts = [{t: lp_mod.Logprob(logprob=v, rank=None, decoded_token=token_str(t))
                  for t, v in {int(o[0]): float(o[1]), **{int(i): float(v) for i, v in zip(o[2], o[3])}}.items()}
                 for o in outs]
    for gen in (0, 2):   # max_tokens 0 (prompt only) and an echo followed by generated tokens
        want = comp.OpenAIServingCompletion._create_completion_logprobs(
            fake, prompt + [o[0] for o in outs[:gen]], dicts + out_dicts[:gen], N, tok).model_dump(mode="json")
        assert want == echo_completion_logprobs(prompt, recs, N, token_str, outs[:gen])


def test_echo_max_tokens_0_usage_is_vllms():
    """vLLM runs one token for an echo with max_tokens 0 and counts it: completion_tokens 1, the text is the prompt."""
    comp = pytest.importorskip("vllm.entrypoints.openai.completion.serving")
    proto = pytest.importorskip("vllm.entrypoints.openai.completion.protocol")
    req = proto.CompletionRequest(model="m", prompt=[1, 2, 3], echo=True, max_tokens=0)
    assert req.to_sampling_params(16, {}).max_tokens == 1
    out = SimpleNamespace(index=0, text="x", token_ids=[9], logprobs=None, finish_reason="length", stop_reason=None,
                          routed_experts=None)
    res = SimpleNamespace(prompt_token_ids=[1, 2, 3], prompt_logprobs=None, prompt="abc", outputs=[out],
                          num_cached_tokens=0, kv_transfer_params=None)
    fake = SimpleNamespace(enable_prompt_tokens_details=False, _raise_if_error=lambda *a: None, system_fingerprint=None)
    resp = comp.OpenAIServingCompletion.request_output_to_completion_response(
        fake, [res], req, "id", 0, "m", None, SimpleNamespace(final_usage_info=None))
    assert resp.choices[0].text == "abc" and resp.choices[0].finish_reason == "length"
    assert (resp.usage.prompt_tokens, resp.usage.completion_tokens, resp.usage.total_tokens) == (3, 1, 4)


# ------------------------------------------------------------------ request fields
BASE_CHAT = {"model": "m", "messages": [{"role": "user", "content": "hi"}]}
BASE_COMP = {"model": "m", "prompt": "hi"}
OK = [{"prompt_logprobs": 0}, {"prompt_logprobs": 1}, {"prompt_logprobs": 20}, {"prompt_logprobs": None},
      {"prompt_logprobs": 3.0}, {"prompt_logprobs": 0, "stream": True}, {"prompt_logprobs": 2, "logprobs": 1}]
COMP_OK = [{"echo": True}, {"echo": True, "logprobs": 1, "max_tokens": 1, "temperature": 0},
           {"echo": True, "max_tokens": 0}, {"echo": True, "logprobs": 5, "max_tokens": 0}, {"echo": False},
           {"echo": True, "stream": True, "logprobs": 2}]
BAD = [({"prompt_logprobs": -1}, "Requested prompt logprobs of 512, which is greater than max allowed: 20"),
       ({"prompt_logprobs": 21}, "Requested prompt logprobs of 21, which is greater than max allowed: 20"),
       ({"prompt_logprobs": -2}, "`prompt_logprobs` must be a positive value or -1."),
       ({"prompt_logprobs": 2.5}, "prompt_logprobs must be an integer"),
       ({"prompt_logprobs": "3"}, "prompt_logprobs must be an integer"),
       ({"prompt_logprobs": 1, "stream": True}, "`prompt_logprobs` are not available when `stream=True`."),
       ({"prompt_logprobs": -1, "stream": True}, "`prompt_logprobs` are not available when `stream=True`.")]


def _status(srv, path, body):
    st, out = srv.parse_request(path, json.dumps(body))
    return st, out.get("error", "")


def _old_refusal(extra, chat, logprobs_on):
    """The refusal the serving shell gave before prompt logprobs existed (its check order)."""
    def truthy(k):
        v = extra.get(k)
        return isinstance(v, (bool, int, float)) and v > 0
    if not logprobs_on and (truthy("logprobs") or truthy("top_logprobs") or truthy("prompt_logprobs")):
        return "bad request: logprobs is not supported by this engine"
    if truthy("prompt_logprobs"):
        return "bad request: prompt_logprobs is not supported by this engine"
    if truthy("echo"):
        return "bad request: echo is not supported by this engine"
    return ""


def test_fields_keep_todays_400_when_off():
    for kw in ({}, {"enable_logprobs": True}, {"enable_logprobs": True, "enable_sampling": True,
                                               "enable_logits_processors": True}):
        with Server([None], model="m", vocab=512, **kw) as off:
            for extra in OK + COMP_OK + [b for b, _ in BAD]:
                for path, base in (("/v1/chat/completions", BASE_CHAT), ("/v1/completions", BASE_COMP)):
                    chat = "chat" in path
                    body = {k: v for k, v in {**base, **extra}.items() if not (chat and k == "logprobs")}
                    want = _old_refusal(body, chat, bool(kw))
                    assert _status(off, path, body) == ((400, want) if want else (0, "")), (kw, path, body)


def test_fields_when_on():
    with Server([None], model="m", vocab=512, enable_logprobs=True, enable_prompt_logprobs=True) as on:
        for extra in OK:
            for path, base in (("/v1/chat/completions", BASE_CHAT), ("/v1/completions", BASE_COMP)):
                body = {**base, **extra}
                if "chat" in path and "logprobs" in extra:
                    body["logprobs"] = True
                assert _status(on, path, body) == (0, ""), (path, extra)
        for extra in COMP_OK:
            assert _status(on, "/v1/completions", {**BASE_COMP, **extra}) == (0, ""), extra
        for extra, msg in BAD:
            for path, base in (("/v1/chat/completions", BASE_CHAT), ("/v1/completions", BASE_COMP)):
                assert _status(on, path, {**base, **extra}) == (400, "bad request: " + msg), (path, extra)
        assert _status(on, "/v1/chat/completions", {**BASE_CHAT, "echo": True}) == \
            (400, "bad request: echo is not supported by this engine")
        # the other refusals keep their words
        assert _status(on, "/v1/completions", {**BASE_COMP, "top_logprobs": 3})[1] == \
            "bad request: top_logprobs on completions (use logprobs) is not supported by this engine"
