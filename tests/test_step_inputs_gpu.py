"""The step's input words on the engine (mini model, manual_step).

(a) The H2D bytes a step adds to the stats equal 4 x the words of its layout, computed here from the scripted schedule:
3T + S, padded to 4 words, then 4 per decode work item and 4 per prefill work item (64 query tokens each), a block table
of ceil(max_model_len / 16) words per sequence, 6 words per sampled row (7 when a row has min_p) only when a row samples,
8 per row with logits edits, 2 per logprobs row, 3 per prompt-logprob row and 2 per forked page.

(b) forward_logits stages its inputs outside the recorded steps: a replay after it recomputes the recorded step.
"""
import numpy as np
import pytest

from kubeai_b200.engine import Engine, mini_config
from oracle.spec_decode import propose

pytestmark = pytest.mark.gpu

MAX_MODEL_LEN = 256
BTAB = MAX_MODEL_LEN // 16
QB = 64   # kPrefillQueryBlock


def words(T, S, nd=0, np_=0, nseq=1, samp=0, n_pen=0, n_lp=0, n_plp=0, n_fork=0):
    w = 3 * T + S
    w = (w + 3) // 4 * 4
    return w + 4 * nd + 4 * np_ + nseq * BTAB + samp * S + 8 * n_pen + 2 * n_lp + 3 * n_plp + 2 * n_fork


def step_expect(e, T, S, dec=0, pre=0, **kw):
    """One step whose schedule is known: its shape and its H2D bytes."""
    before = e.stats().h2d_bytes
    ran, info = e.step()
    assert ran
    assert (info.tokens, info.sampled, info.decode_seqs, info.prefill_seqs) == (T, S, dec, pre)
    np_ = kw.pop("np_", -(-T // QB) if pre else 0)
    want = words(T, S, nd=dec, np_=np_, nseq=dec + pre, **kw)
    assert e.stats().h2d_bytes - before == 4 * want, kw
    return info


def prompt(rng, n):
    return rng.integers(0, 512, size=n).tolist()


def test_h2d_bytes_equal_the_layout_words():
    rng = np.random.default_rng(21)
    with Engine(mini_config(max_batched_tokens=64, max_model_len=MAX_MODEL_LEN)) as e:
        # greedy: a prefill chunk (no sampled row), the prompt's last chunk, then a decode
        e.submit(prompt(rng, 100), max_tokens=2)
        step_expect(e, 64, 0, pre=1)
        step_expect(e, 36, 1, pre=1)
        step_expect(e, 1, 1, dec=1)
        # sampled rows: 6 words each, 7 in a step with min_p
        e.submit(prompt(rng, 20), max_tokens=1, temperature=0.8, seed=1)
        step_expect(e, 20, 1, pre=1, samp=6)
        e.submit(prompt(rng, 20), max_tokens=1, temperature=0.8, seed=1, min_p=0.05)
        step_expect(e, 20, 1, pre=1, samp=7)
        # logits edits and logprobs of a greedy row
        e.submit(prompt(rng, 20), max_tokens=1, presence_penalty=0.5)
        step_expect(e, 20, 1, pre=1, n_pen=1)
        e.submit(prompt(rng, 20), max_tokens=1, logprobs=True, top_logprobs=3)
        step_expect(e, 20, 1, pre=1, n_lp=1)
        # prompt logprobs over two chunks: positions 0..63, then 64..98 (99 is the sampled row)
        e.submit(prompt(rng, 100), max_tokens=1, prompt_logprobs=2)
        step_expect(e, 64, 0, pre=1, n_plp=64)
        step_expect(e, 36, 1, pre=1, n_plp=35)
        # a fork of three members from a prompt that ends inside its third page: three sampled rows, two page copies
        e.submit_n(prompt(rng, 37), 3, max_tokens=1, temperature=0.8, seed=5)
        step_expect(e, 37, 3, pre=1, samp=6, n_fork=2)
        assert not e.step()[0], "every request above has finished"


def test_h2d_bytes_of_a_speculative_verify():
    block = [7, 100, 23, 311]
    toks = block * 8
    bias = {t: 12.0 for t in block}   # the generated tokens come from the block: the proposer finds a match
    with Engine(mini_config(max_model_len=MAX_MODEL_LEN, num_speculative_tokens=3, prompt_lookup_min=1,
                            prompt_lookup_max=3)) as e:
        rid = e.submit(toks, max_tokens=10, logit_bias=bias)
        step_expect(e, 32, 1, pre=1, n_pen=1)
        ctx = toks + e.poll(rid).tokens
        m = len(propose(ctx, 1, 3, 3, MAX_MODEL_LEN))
        assert m >= 1
        info = step_expect(e, 1 + m, 1 + m, dec=1, n_pen=1 + m)
        assert info.draft_tokens == m


def test_replay_after_forward_logits_recomputes_the_recorded_step():
    rng = np.random.default_rng(4)
    with Engine(mini_config(max_model_len=MAX_MODEL_LEN)) as e:
        rid = e.submit(prompt(rng, 20), max_tokens=3)
        e.step()
        assert len(e.poll(rid).tokens) == 1
        ran, info = e.step()   # a greedy decode: the one recorded step
        assert ran and info.decode_seqs == 1 and info.sampled == 1
        tok = e.poll(rid).tokens
        assert len(tok) == 1
        e.forward_logits(prompt(rng, 40))
        e.replay(1)
        assert e.tensor("step.sampled").view(np.int32)[:1].tolist() == tok
