"""Oracle of vLLM 0.22's parallel sampling (the request field `n`) as the serving shell restates it: the child seeds
(vllm/v1/engine/parallel_sampling.py ParentRequest._get_child_sampling_params), the checks of n (SamplingParams._verify_args
and _verify_greedy_sampling, plus the server's max_n bound), the non-stream responses for n choices (chat_completion/serving.py
and completion/serving.py: one choice per index, usage summed over the choices, prompt_logprobs on every completions choice
and once at the top level of a chat response) and the stream's event order per choice."""
from __future__ import annotations


def child_seeds(seed, n):
    """The seed of each of n children: seed + i, or None (each child then draws its own) when the request has none."""
    return [None if seed is None else seed + i for i in range(n)]


def n_error(n, temperature, max_n):
    """The message of the server's 400 for a request's n (without the "bad request: " prefix), None when it is served."""
    if isinstance(n, bool) or not isinstance(n, (int, float)) or n != int(n):
        return "n must be an integer"
    n = int(n)
    if n < 1:
        return f"n must be at least 1, got {n}."
    if n > max_n:
        return f"n must be at most {max_n}, got {n}."
    if n > 1 and temperature < 1e-5:
        return f"n must be 1 when using greedy sampling, got {n}."
    return None


def usage(prompt_tokens, cached_tokens, completion_tokens_per_choice):
    """The prompt once, the completion tokens of every choice."""
    c = sum(completion_tokens_per_choice)
    return dict(prompt_tokens=prompt_tokens, total_tokens=prompt_tokens + c, completion_tokens=c,
                prompt_tokens_details=dict(cached_tokens=cached_tokens))


def chat_response(rid, created, model, choices, usage_dict, prompt_logprobs=None):
    """choices: [(text, logprobs or None, finish_reason)] in index order; prompt_logprobs: the list, or None when the request
    did not ask for it (the key is then absent)."""
    out = dict(id=rid, object="chat.completion", created=created, model=model,
               choices=[dict(index=i, message=dict(role="assistant", content=text), logprobs=lp, finish_reason=fr,
                             stop_reason=None) for i, (text, lp, fr) in enumerate(choices)],
               usage=usage_dict)
    if prompt_logprobs is not None:
        out["prompt_logprobs"] = prompt_logprobs
    return out


def completion_response(rid, created, model, choices, usage_dict, prompt_logprobs=None):
    """Same for completions: prompt_logprobs goes on every choice."""
    cs = []
    for i, (text, lp, fr) in enumerate(choices):
        c = dict(index=i, text=text, logprobs=lp, finish_reason=fr, stop_reason=None)
        if prompt_logprobs is not None:
            c["prompt_logprobs"] = prompt_logprobs
        cs.append(c)
    return dict(id=rid, object="text_completion", created=created, model=model, choices=cs, usage=usage_dict)


def stream_events(chat, n, steps, include_usage):
    """The (kind, index) sequence of a stream of n choices.  steps: per engine step, the choices that produced a token
    there, each as (index, finished); kind is "role" (chat, one per choice before anything else), "token", "finish" (the
    token chunk that carries the choice's finish_reason), "usage" and "done".  Within a step, chunks go out in ascending
    choice index."""
    ev = [("role", i) for i in range(n)] if chat and steps else []
    for step in steps:
        for i, fin in sorted(step):
            ev.append(("finish" if fin else "token", i))
    if include_usage:
        ev.append(("usage", None))
    ev.append(("done", None))
    return ev
