"""n-gram speculative decoding on the host: the engine's proposer (b200_ngram_propose) and the plain-Python oracle against
vLLM's _find_longest_matched_ngram_and_propose_tokens, and the speculative config rules of b200_engine_create."""
import ctypes as C

import numpy as np
import pytest

from oracle.spec_decode import accept, propose

vllm_ngram = pytest.importorskip("vllm.v1.spec_decode.ngram_proposer")
vllm_propose = vllm_ngram._find_longest_matched_ngram_and_propose_tokens


def engine_propose(toks, min_n, max_n, k, max_model_len):
    from kubeai_b200 import _lib
    arr = (C.c_int32 * max(len(toks), 1))(*[int(t) for t in toks])
    out = (C.c_int32 * max(k, 1))()
    n = _lib.lib().b200_ngram_propose(arr, len(toks), min_n, max_n, k, max_model_len, out)
    assert n >= 0, n
    return list(out[:n])


def want(toks, min_n, max_n, k, max_model_len):
    return vllm_propose(np.asarray(toks, dtype=np.int32), min_n, max_n, max_model_len, k).tolist()


def random_cases(seed, count):
    rng = np.random.default_rng(seed)
    for _ in range(count):
        n = int(rng.integers(0, 80))
        alphabet = int(rng.integers(2, 6))
        toks = rng.integers(0, alphabet, size=n).tolist()
        min_n = int(rng.integers(1, 6))
        max_n = int(rng.integers(min_n, 9))
        k = int(rng.integers(1, 6))
        max_model_len = n + int(rng.integers(0, 6))
        yield toks, min_n, max_n, k, max_model_len


EDGE_CASES = [
    ([1, 2], 3, 5, 3, 100),                       # context shorter than min_n
    ([7, 8, 9, 1, 7, 8], 2, 3, 3, 100),           # match at the very start
    ([1, 2, 5, 1, 2, 6, 1, 2, 7, 1, 2], 2, 2, 3, 100),   # several equal-length matches
    ([3] * 20, 1, 4, 3, 100),                     # matches longer than max_n
    ([1, 2, 3, 4, 5, 1, 2, 3, 4, 5, 1, 2, 3], 2, 5, 3, 100),
    ([1, 2, 3, 9, 9, 1, 2, 3], 3, 3, 3, 10),      # k clipped by max_model_len
    ([1, 2, 3, 9, 9, 1, 2, 3], 3, 3, 3, 8),       # no room at all
    ([4, 5, 4, 5], 2, 2, 3, 100),                 # k clipped by the end of the context
    ([4, 5, 6, 4, 5], 1, 1, 3, 100),
    ([], 1, 1, 3, 100),
    ([0], 1, 1, 3, 100),
]


@pytest.mark.parametrize("case", EDGE_CASES)
def test_proposer_edge_cases_match_vllm(case):
    assert engine_propose(*case) == want(*case)
    assert propose(*case) == want(*case)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_proposer_matches_vllm_on_random_contexts(seed):
    hits = 0
    for case in random_cases(seed, 2000):
        w = want(*case)
        assert engine_propose(*case) == w, case
        assert propose(*case) == w, case
        hits += bool(w)
    assert hits > 500   # small alphabets: most contexts have a match


def test_proposer_long_context_matches_vllm():
    rng = np.random.default_rng(5)
    block = rng.integers(0, 128256, size=97).tolist()
    toks = (block * 25)[:2000] + rng.integers(0, 50, size=30).tolist() + block[:7]
    for (mn, mx) in [(1, 1), (2, 5), (5, 5), (3, 12)]:
        assert engine_propose(toks, mn, mx, 3, 4096) == want(toks, mn, mx, 3, 4096)


def test_proposer_rejects_bad_arguments():
    from kubeai_b200 import _lib
    l = _lib.lib()
    arr = (C.c_int32 * 4)(1, 2, 1, 2)
    out = (C.c_int32 * 4)()
    assert l.b200_ngram_propose(arr, 4, 0, 2, 3, 100, out) == -1
    assert l.b200_ngram_propose(arr, 4, 3, 2, 3, 100, out) == -1
    assert l.b200_ngram_propose(arr, 4, 1, 2, -1, 100, out) == -1
    assert l.b200_ngram_propose(None, 4, 1, 2, 3, 100, out) == -1


def test_accept_rule():
    assert accept([5, 6, 7], [5, 6, 7, 8]) == [5, 6, 7, 8]
    assert accept([5, 6, 7], [5, 9, 7, 8]) == [5, 9]
    assert accept([5, 6, 7], [4, 6, 7, 8]) == [4]
    assert accept([5, 6, 7], [5, 6, 7, 8], finishes=lambda j, t: t == 6) == [5, 6]
    assert accept([], [3]) == [3]


def create_rc(**kw):
    from kubeai_b200 import _lib
    from kubeai_b200.engine import mini_config
    l = _lib.lib()
    e = C.c_void_p()
    rc = l.b200_engine_create(C.byref(mini_config(**kw)), C.byref(e))
    if rc == 0:
        l.b200_engine_destroy(e)
    return rc, l.b200_last_error().decode()


@pytest.mark.parametrize("kw", [
    dict(num_speculative_tokens=4),
    dict(num_speculative_tokens=-1),
    dict(num_speculative_tokens=3, prompt_lookup_min=4, prompt_lookup_max=3),
    dict(num_speculative_tokens=3, prompt_lookup_max=4, prompt_lookup_min=6),
    dict(num_speculative_tokens=3, prompt_lookup_min=6),          # max unset: 6 and 6, fine; min > max needs both
    dict(num_speculative_tokens=2, prompt_lookup_min=-1),
])
def test_speculative_config_rules(kw):
    rc, msg = create_rc(**kw)
    invalid = (kw.get("num_speculative_tokens", 0) not in range(0, 4) or kw.get("prompt_lookup_min", 0) < 0
               or (kw.get("prompt_lookup_min", 0) and kw.get("prompt_lookup_max", 0)
                   and kw["prompt_lookup_min"] > kw["prompt_lookup_max"]))
    if invalid:
        assert rc == -1, (rc, msg)
    else:
        assert rc in (0, -5), (rc, msg)   # -5: no device on this host


@pytest.mark.parametrize("mn, mx", [(0, 0), (0, 3), (7, 0), (2, 2), (1, 8)])
def test_speculative_lookup_defaults_are_accepted(mn, mx):
    rc, msg = create_rc(num_speculative_tokens=3, prompt_lookup_min=mn, prompt_lookup_max=mx)
    assert rc in (0, -5), (rc, msg)


def test_speculative_config_error_messages():
    rc, msg = create_rc(num_speculative_tokens=4)
    assert rc == -1 and "num_speculative_tokens must be in 0..3" in msg
    rc, msg = create_rc(num_speculative_tokens=1, prompt_lookup_min=4, prompt_lookup_max=3)
    assert rc == -1 and "prompt_lookup_min=4 must be <= prompt_lookup_max=3" in msg


def test_stats_and_step_info_carry_the_speculative_counters():
    from kubeai_b200 import _lib
    names = [f for f, _ in _lib.Stats._fields_]
    assert names[-4:] == ["spec_drafts", "spec_draft_tokens", "spec_accepted_tokens", "spec_accepted_per_pos"]
    assert _lib.Stats().spec_accepted_per_pos._length_ == 3
    assert [f for f, _ in _lib.StepInfo._fields_][-2:] == ["draft_tokens", "accepted_tokens"]


# ------------------------------------------------------------------------------------------------------------ serving
def parse(text):
    from kubeai_b200 import _lib
    from kubeai_b200.engine import default_config
    cfg = default_config()
    rc = _lib.lib().b200_speculative_config_parse(text.encode(), C.byref(cfg))
    return rc, _lib.lib().b200_last_error().decode(), (cfg.num_speculative_tokens, cfg.prompt_lookup_min, cfg.prompt_lookup_max)


@pytest.mark.parametrize("text, want", [
    ('{"method": "ngram", "num_speculative_tokens": 3}', (3, 0, 0)),
    ('{"method": "ngram", "num_speculative_tokens": 2, "prompt_lookup_max": 4}', (2, 0, 4)),
    ('{"num_speculative_tokens": 1, "method": "ngram", "prompt_lookup_min": 2, "prompt_lookup_max": 5}', (1, 2, 5)),
    ('{"method": "ngram", "num_speculative_tokens": 3, "prompt_lookup_min": null, "prompt_lookup_max": 3}', (3, 0, 3)),
])
def test_speculative_config_json_is_applied(text, want):
    rc, msg, got = parse(text)
    assert rc == 0, msg
    assert got == want


@pytest.mark.parametrize("text, words", [
    ('{"method": "eagle", "num_speculative_tokens": 3}', 'only "method": "ngram"'),
    ('{"method": "ngram", "model": "x", "num_speculative_tokens": 3}', 'unsupported key "model"'),
    ('{"num_speculative_tokens": 3}', '"method" is required'),
    ('{"method": "ngram", "num_speculative_tokens": 4}', "num_speculative_tokens must be in 1..3"),
    ('{"method": "ngram"}', "num_speculative_tokens must be in 1..3"),
    ('{"method": "ngram", "num_speculative_tokens": 0}', "num_speculative_tokens must be an integer >= 1"),
    ('{"method": "ngram", "num_speculative_tokens": 2.5}', "must be an integer"),
    ('{"method": "ngram", "num_speculative_tokens": 2, "prompt_lookup_min": 5, "prompt_lookup_max": 4}',
     "prompt_lookup_min=5 must be <= prompt_lookup_max=4"),
    ('{"method": "ngram", "num_speculative_tokens": 2, "prompt_lookup_min": 0}', "prompt_lookup_min must be an integer >= 1"),
    ('[1]', "expected a JSON object"),
    ('{"method": ', "speculative-config:"),
])
def test_speculative_config_json_refusals(text, words):
    rc, msg, got = parse(text)
    assert rc == -1 and words in msg, msg
    assert got == (0, 0, 0)   # the config is left as it was


def test_b200serve_speculative_config_option():
    import subprocess
    from pathlib import Path
    exe = Path(__file__).resolve().parent.parent / "kubeai_b200" / "bin" / "b200serve"
    assert exe.exists()
    r = subprocess.run([str(exe), "--speculative-config", '{"method": "eagle", "num_speculative_tokens": 2}'],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode == 2 and 'only "method": "ngram" is supported' in r.stderr
    r = subprocess.run([str(exe), "--speculative-config", '{"method": "ngram", "num_speculative_tokens": 4}'],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode == 2 and "num_speculative_tokens must be in 1..3" in r.stderr
