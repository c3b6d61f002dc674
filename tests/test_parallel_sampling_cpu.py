"""Parallel sampling (n), CPU-only parts: the oracle (oracle/parallel_sampling.py) against vLLM 0.22's child seeds, its
SamplingParams messages and its pydantic response models for n choices, and the serving shell's request-field matrix with
max_n off (today's 400, word for word) and on."""
import json
from types import SimpleNamespace

import pytest

from kubeai_b200.server import Server
from oracle.parallel_sampling import (chat_response, child_seeds, completion_response, n_error, stream_events, usage)


@pytest.mark.parametrize("seed", [None, 0, 7, 2 ** 40 + 3])
def test_child_seeds_equal_vllm(seed):
    ps = pytest.importorskip("vllm.v1.engine.parallel_sampling")
    from vllm import SamplingParams
    parent = SimpleNamespace(sampling_params=SamplingParams(n=4, seed=seed, temperature=0.8),
                             cached_child_sampling_params=None)
    for i in range(4):
        child = ps.ParentRequest._get_child_sampling_params(parent, i)
        assert child.n == 1 and child.seed == child_seeds(seed, 4)[i]
        assert child.temperature == 0.8


@pytest.mark.parametrize("n,temperature", [(0, 1.0), (-1, 1.0), (2, 0.0), (3, 0.5), (1, 0.0), (4, 0.7)])
def test_messages_equal_sampling_params(n, temperature):
    pytest.importorskip("vllm")
    from vllm import SamplingParams
    try:
        SamplingParams(n=n, temperature=temperature)
        want = None
    except ValueError as e:
        want = str(e)
    assert n_error(n, temperature, 8) == want
    assert n_error(9, 1.0, 8) == "n must be at most 8, got 9."
    assert n_error(1.5, 1.0, 8) == "n must be an integer"


def _project(full, ours):
    """vLLM's dump restricted to the keys the serving shell writes (recursively)."""
    if isinstance(ours, dict):
        return {k: _project(full[k], v) for k, v in ours.items()}
    if isinstance(ours, list) and isinstance(full, list):
        return [_project(f, o) for f, o in zip(full, ours)] + full[len(ours):]
    return full


@pytest.mark.parametrize("with_plp", [False, True])
def test_non_stream_builders_equal_vllm(with_plp):
    cp = pytest.importorskip("vllm.entrypoints.openai.chat_completion.protocol")
    pp = pytest.importorskip("vllm.entrypoints.openai.completion.protocol")
    ep = pytest.importorskip("vllm.entrypoints.openai.engine.protocol")
    plp = [None, {"5": {"logprob": -1.5, "rank": 2, "decoded_token": "x"}}] if with_plp else None
    texts = [("a b", None, "length"), ("", None, "stop"), ("zz", None, "length")]
    u = usage(11, 4, [3, 0, 2])
    assert u == dict(prompt_tokens=11, total_tokens=16, completion_tokens=5, prompt_tokens_details=dict(cached_tokens=4))
    vu = ep.UsageInfo(prompt_tokens=11, completion_tokens=5, total_tokens=16,
                      prompt_tokens_details=ep.PromptTokenUsageInfo(cached_tokens=4))
    chat = chat_response("chatcmpl-1", 5, "m", texts, u, plp)
    want = cp.ChatCompletionResponse(
        id="chatcmpl-1", created=5, model="m", usage=vu, prompt_logprobs=plp,
        choices=[cp.ChatCompletionResponseChoice(index=i, message=cp.ChatMessage(role="assistant", content=t), logprobs=lp,
                                                 finish_reason=fr) for i, (t, lp, fr) in enumerate(texts)]
    ).model_dump(mode="json")
    assert [c["index"] for c in want["choices"]] == [0, 1, 2]
    assert _project(want, chat) == chat
    comp = completion_response("cmpl-1", 5, "m", texts, u, plp)
    want = pp.CompletionResponse(
        id="cmpl-1", created=5, model="m", usage=vu,
        choices=[pp.CompletionResponseChoice(index=i, text=t, logprobs=lp, finish_reason=fr, prompt_logprobs=plp)
                 for i, (t, lp, fr) in enumerate(texts)]).model_dump(mode="json")
    assert _project(want, comp) == comp
    assert ("prompt_logprobs" in comp["choices"][1]) == with_plp and "prompt_logprobs" not in comp


def test_stream_event_order():
    steps = [[(1, False), (0, False)], [(0, True)], [(1, True)]]
    assert stream_events(True, 2, steps, True) == [("role", 0), ("role", 1), ("token", 0), ("token", 1), ("finish", 0),
                                                   ("finish", 1), ("usage", None), ("done", None)]
    assert stream_events(False, 2, steps, False)[:2] == [("token", 0), ("token", 1)]


# ------------------------------------------------------------------ request fields
BASE_CHAT = {"model": "m", "messages": [{"role": "user", "content": "hi"}]}
BASE_COMP = {"model": "m", "prompt": "hi"}
FIELDS = [{"n": 0}, {"n": -1}, {"n": 1}, {"n": 1.5}, {"n": 9}, {"n": 2}, {"n": 8}, {"n": None}, {"n": 2, "temperature": 0},
          {"n": 2, "temperature": 0.8}, {"n": 3.0, "temperature": 0.8}, {"n": "2", "temperature": 0.8},
          {"best_of": 2, "temperature": 0.8}, {"n": 2, "best_of": 2, "temperature": 0.8},
          {"n": 4, "temperature": 0.8, "logprobs": 2}, {"n": 4, "temperature": 0.8, "prompt_logprobs": 1},
          {"n": 4, "temperature": 0.8, "echo": True, "logprobs": 1}, {"n": 4, "temperature": 0.8, "stream": True}]


def _status(srv, path, body):
    st, out = srv.parse_request(path, json.dumps(body))
    return st, out.get("error", "")


def _want(body, chat, max_n):
    """The serving shell's answer: with max_n < 2 the refusal it gave before n existed; else vLLM's checks of n first."""
    n = body.get("n")
    if max_n >= 2 and n is not None:
        msg = n_error(n, body.get("temperature", 0.0), max_n) if not isinstance(n, str) else "n must be an integer"
        if msg:
            return 400, "bad request: " + msg
    elif isinstance(n, (int, float)) and n > 1:
        return 400, "bad request: n > 1 is not supported by this engine"
    if body.get("best_of", 1) > 1:
        return 400, "bad request: best_of > 1 is not supported by this engine"
    if chat and body.get("echo"):
        return 400, "bad request: echo is not supported by this engine"
    return 0, ""


@pytest.mark.parametrize("max_n", [0, 1, 8])
def test_request_field_matrix(max_n):
    with Server([None], model="m", vocab=512, enable_sampling=True, enable_logprobs=True, enable_prompt_logprobs=True,
                max_n=max_n) as srv:
        for extra in FIELDS:
            for path, base in (("/v1/chat/completions", BASE_CHAT), ("/v1/completions", BASE_COMP)):
                chat = "chat" in path
                body = {**base, **extra}
                if chat and "logprobs" in extra:
                    body["logprobs"] = True
                if body.get("stream") and "prompt_logprobs" in body:
                    continue
                assert _status(srv, path, body) == _want(body, chat, max_n), (max_n, path, body)


def test_zero_config_keeps_todays_refusal():
    with Server([None], model="m", vocab=512) as srv:
        assert _status(srv, "/v1/chat/completions", {**BASE_CHAT, "n": 2}) == \
            (400, "bad request: n > 1 is not supported by this engine")
