"""Logits edits, CPU-only parts: the oracle (oracle/penalties.py) against vLLM's own apply_penalties (torch CPU path),
LogitBiasLogitsProcessor, MinTokensLogitsProcessor and MinPLogitsProcessor, and the serving shell's request fields with
enable_logits_processors off (today's 400s, word for word) and on (vLLM's ranges)."""
import json
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from kubeai_b200.server import PREFIX_HASH, Server
from oracle.penalties import bf16_round, edit, edit_f32, min_p_keep, named


def bf16_row(rng, V, scale=4.0):
    x = bf16_round((rng.standard_normal(V) * scale).astype(np.float32))
    x[rng.integers(0, V, 3)] = -np.inf          # masked entries stay masked
    x[rng.integers(0, V, 2)] = 0.0
    return x


def vllm_penalties(rows, prompts, outputs, pres, freq, rep):
    utils = pytest.importorskip("vllm.model_executor.layers.utils")
    S, V = rows.shape

    def pad(lists):
        n = max(1, max(len(x) for x in lists))
        return torch.tensor([list(x) + [V] * (n - len(x)) for x in lists], dtype=torch.int64)
    logits = torch.from_numpy(rows.copy())
    return utils.apply_penalties(logits, pad(prompts), pad(outputs), torch.tensor(pres, dtype=torch.float32),
                                 torch.tensor(freq, dtype=torch.float32), torch.tensor(rep, dtype=torch.float32)).numpy()


@pytest.mark.parametrize("V", [512, 3001])
def test_oracle_equals_vllm_apply_penalties(V):
    """Before the bf16 rounding the oracle is vLLM's arithmetic bit for bit (signed zeros aside), on histories in the
    prompt only, the output only and both, counts in the thousands, negative penalties and r on both sides of 1."""
    rng = np.random.default_rng(V)
    cases = [  # (prompt, output, presence, frequency, repetition)
        (rng.integers(0, V, 40), [], 0.0, 0.0, 1.3),
        ([], rng.integers(0, V, 60), 0.5, 0.5, 1.0),
        (rng.integers(0, V // 4, 300), rng.integers(0, V // 4, 300), -1.5, 2.0, 0.7),
        (rng.integers(0, V, 10), np.concatenate([np.full(3000, 7), rng.integers(0, V, 50)]), 2.0, -2.0, 1.1),
        (rng.integers(0, 4, 5), rng.integers(0, 4, 2000), -0.25, 0.125, 2.0),
        ([], [], 0.3, 0.3, 1.2),
    ]
    rows = np.stack([bf16_row(rng, V) for _ in cases])
    got = vllm_penalties(rows, [c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases],
                         [c[3] for c in cases], [c[4] for c in cases])
    for s, (p, o, pr, fr, rp) in enumerate(cases):
        want = edit_f32(rows[s], prompt=p, output=o, presence=pr, frequency=fr, repetition=rp)
        assert np.array_equal(want, got[s]), (s, np.flatnonzero(want != got[s])[:8])
        m = named(V, prompt=p, output=o, presence=pr, frequency=fr, repetition=rp)
        assert np.array_equal(want[~m], rows[s][~m])          # tokens no list names keep their value
        r = edit(rows[s], prompt=p, output=o, presence=pr, frequency=fr, repetition=rp)
        assert np.array_equal(r, bf16_round(want))
        fin = np.isfinite(want)
        ulp = np.abs(bf16_round(want[fin]).astype(np.float64) - want[fin])
        assert (ulp <= np.abs(want[fin]) * 2.0 ** -8 + 1e-45).all()    # rounding moves a value by at most half a bf16 ulp


def _processor(cls, params_list, V):
    iface = pytest.importorskip("vllm.v1.sample.logits_processor.interface")
    cfg = SimpleNamespace(scheduler_config=SimpleNamespace(max_num_seqs=8))
    proc = cls(cfg, torch.device("cpu"), False)
    added = [(i, p, list(prompt), output) for i, (p, prompt, output) in enumerate(params_list)]
    proc.update_state(iface.BatchUpdate(batch_size=len(params_list), removed=[], added=added, moved=[]))
    return proc


def test_oracle_equals_vllm_logit_bias_and_min_tokens():
    builtin = pytest.importorskip("vllm.v1.sample.logits_processor.builtin")
    from vllm import SamplingParams
    V, eos = 700, 2
    rng = np.random.default_rng(3)
    bias = {5: 250.0, 0: -3.5, V - 1: 0.75, 17: -1000.0}
    reqs = [dict(min_tokens=4, stop=[9, 11], out=[1, 2], ignore_eos=False),
            dict(min_tokens=4, stop=[9], out=[1, 2, 3, 4], ignore_eos=False),   # past min_tokens: no ban
            dict(min_tokens=3, stop=[], out=[], ignore_eos=True)]               # EOS is banned even with ignore_eos
    params = []
    for r in reqs:
        # from_optional is how vLLM's OpenAI server builds them: it clamps the biases to [-100, 100]
        sp = SamplingParams.from_optional(min_tokens=r["min_tokens"], stop_token_ids=r["stop"], max_tokens=20, ignore_eos=r["ignore_eos"],
                            logit_bias=bias)
        sp.update_from_generation_config({}, eos_token_id=eos)
        assert eos in sp.all_stop_token_ids
        params.append((sp, [3, 4], r["out"]))
    rows = np.stack([bf16_row(rng, V) for _ in reqs])
    logits = torch.from_numpy(rows.copy())
    logits = _processor(builtin.MinTokensLogitsProcessor, params, V).apply(logits)
    logits = _processor(builtin.LogitBiasLogitsProcessor, params, V).apply(logits)
    for s, r in enumerate(reqs):
        want = edit_f32(rows[s], output=r["out"], min_tokens=r["min_tokens"], stop_ids=r["stop"] + [eos], logit_bias=bias)
        assert np.array_equal(want, logits[s].numpy()), s


def test_oracle_min_p_equals_vllm_outside_the_boundary_slack():
    builtin = pytest.importorskip("vllm.v1.sample.logits_processor.builtin")
    from vllm import SamplingParams
    rng = np.random.default_rng(5)
    V, T = 4000, 0.8
    min_ps = [0.05, 0.3, 1.0, 1e-4]
    params = [(SamplingParams(temperature=T, min_p=m), [1], []) for m in min_ps]
    rows = np.stack([bf16_row(rng, V, 3.0) for _ in min_ps])
    z = torch.from_numpy((rows / np.float32(T)).astype(np.float32))
    got = _processor(builtin.MinPLogitsProcessor, params, V).apply(z.clone())
    for s, m in enumerate(min_ps):
        keep, slack = min_p_keep(z[s].numpy(), m)
        vkeep = np.isfinite(got[s].numpy()) & np.isfinite(z[s].numpy())
        if slack > 1e-5:          # vLLM compares fp32 probabilities: only a boundary closer than that may differ
            assert np.array_equal(keep & np.isfinite(z[s].numpy()), vkeep), (s, m)
        assert keep[np.argmax(z[s].numpy())]


@pytest.fixture()
def psrv_off():
    with Server([None], model="test-model", strategy=PREFIX_HASH) as s:
        yield s


@pytest.fixture()
def psrv_on():
    with Server([None], model="test-model", strategy=PREFIX_HASH, vocab=1000, enable_sampling=True,
                enable_logits_processors=True) as s:
        yield s


BASE = {"model": "test-model", "messages": [{"role": "user", "content": "hi"}]}
FIELDS = [{"presence_penalty": 0.5}, {"frequency_penalty": -2}, {"repetition_penalty": 1.1}, {"logit_bias": {"5": 1}},
          {"min_tokens": 4}, {"min_p": 0.1, "temperature": 0.7}]


def test_setting_off_keeps_every_400(psrv_off):
    for extra, msg in zip(FIELDS, ["penalties", "penalties", "penalties", "logit_bias", "min_tokens", "min_p"]):
        st, out = psrv_off.parse_request("/openai/v1/chat/completions", json.dumps({**BASE, **extra}))
        assert st == 400 and out["error"] == f"bad request: {'sampling penalties' if msg == 'penalties' else msg} " \
                                             f"is not supported by this engine", (extra, out)


def test_setting_on_accepts_and_refuses_what_vllm_does(psrv_on):
    ok = FIELDS + [{"presence_penalty": 2}, {"presence_penalty": -2.0}, {"repetition_penalty": 0.01},
                   {"repetition_penalty": 5}, {"min_p": 0}, {"min_p": 1}, {"min_tokens": 0}, {"logit_bias": {}},
                   {"logit_bias": None}, {"presence_penalty": None}, {"logit_bias": {"0": -100, "999": 100}},
                   {"logit_bias": {"5": 1e6, "6": -1e6}}, {"min_p": 0.5, "temperature": 0}, {"logit_bias": {"+7": 2}}]
    for extra in ok:
        for path in ("/openai/v1/chat/completions", "/openai/v1/completions"):
            body = {**BASE, **extra} if "chat" in path else {"model": "test-model", "prompt": "x", **extra}
            st, out = psrv_on.parse_request(path, json.dumps(body))
            assert st == 0, (extra, out)
    bad = [({"presence_penalty": 2.5}, "presence_penalty must be in [-2, 2]"),
           ({"frequency_penalty": -2.01}, "frequency_penalty must be in [-2, 2]"),
           ({"repetition_penalty": 0}, "repetition_penalty must be greater than zero"),
           ({"repetition_penalty": -1}, "repetition_penalty must be greater than zero"),
           ({"min_p": 1.5}, "min_p must be in [0, 1]"), ({"min_p": -0.1}, "min_p must be in [0, 1]"),
           ({"min_tokens": -1}, "min_tokens"), ({"min_tokens": 1.5}, "min_tokens"),
           ({"presence_penalty": "0.5"}, "presence_penalty must be a number"),
           ({"logit_bias": {"abc": 1}}, "logit_bias keys must be integer token ids"),
           ({"logit_bias": {"1.5": 1}}, "logit_bias keys must be integer token ids"),
           ({"logit_bias": {"1000": 1}}, "out-of-vocab token ids"), ({"logit_bias": {"-1": 1}}, "out-of-vocab"),
           ({"logit_bias": {"5": "x"}}, "logit_bias values must be numbers"), ({"logit_bias": [5]}, "logit_bias must be"),
           ({"logit_bias": {str(i): 1 for i in range(1025)}}, "at most 1024")]
    for extra, msg in bad:
        st, out = psrv_on.parse_request("/openai/v1/chat/completions", json.dumps({**BASE, **extra}))
        assert st == 400 and msg in out["error"], (extra, st, out)


def test_min_tokens_above_max_tokens_is_refused():
    body = {**BASE, "max_tokens": 3, "min_tokens": 4}
    with Server([None], model="test-model", enable_logits_processors=True, max_retries=0) as on:
        r = on.handle("POST", "/openai/v1/chat/completions", json.dumps(body))
        assert r.status == 400 and "min_tokens must be less than or equal to max_tokens=3" in r.json()["error"]
        assert on.handle("POST", "/openai/v1/chat/completions", json.dumps({**body, "min_tokens": 3})).status == 502


# ------------------------------------------------------------------ the token history (penalties.cu update_kernel)
THREADS = 256   # update_kernel's block size: the shift moves 256 records per chunk
MUTANTS = ["lowest_chunk_first", "guard_i_gt_pos", "insert_after", "count_on_miss", "clear_on_hit", "insert_when_full"]


def update_emulated(buf, lens, slot, t, cap, mutant=None):
    """update_kernel for one history row in numpy: buf int64 [slots * cap + 1, 4] holds the lists back to back (the row
    past the last list stands for whatever follows the buffer), lens [slots].  Thread 0 binary-searches the first record
    with id >= t and counts a hit; on a miss with n < cap the records [pos, n) move up by one in 256-record chunks,
    highest chunk first (each chunk is read by all threads, a barrier, then written), and {t, 1, 0, 0} goes to pos.
    `mutant` names one of MUTANTS, a wrong variant the checks must reject."""
    base, n = slot * cap, int(lens[slot])
    lst = buf[base:]
    lo, hi = 0, n
    while lo < hi:
        mid = (lo + hi) >> 1
        if lst[mid, 0] < t:
            lo = mid + 1
        else:
            hi = mid
    found = lo < n and lst[lo, 0] == t
    if found:
        lst[lo, 1] += 1
        if mutant == "clear_on_hit":
            lst[lo, 2:] = 0
        return
    if mutant == "count_on_miss" and lo < n:
        lst[lo, 1] += 1
    if n >= cap and mutant != "insert_when_full":
        return
    pos = lo + 1 if mutant == "insert_after" and lo < n else lo
    his = list(range(n, pos, -THREADS))
    if mutant == "lowest_chunk_first":
        his.reverse()
    tid = np.arange(THREADS)
    for hi in his:
        i = hi - THREADS + tid
        mine = ((i > pos) if mutant == "guard_i_gt_pos" else (i >= pos)) & (i < hi)
        e = lst[i[mine]].copy()           # every thread reads, __syncthreads, every thread writes
        lst[i[mine] + 1] = e
    lst[pos] = (t, 1, 0, 0)
    lens[slot] = n + 1


def history_cases(rng):
    """(prompt, output, stream, bias, stops, min_tokens, V, cap): lists from empty to several chunks, streams that mix
    repeats, fresh ids, prompt-only, bias-only and stop-only ids, and lists that reach their cap."""
    cases = []
    for V, n_p, n_o, n_s, cap in ((64, 0, 0, 40, 4096), (5000, 1500, 200, 300, 4096), (3000, 700, 0, 400, 4096),
                                  (1200, 1100, 50, 300, 800), (300, 250, 20, 200, 200)):
        prompt = rng.integers(0, V, n_p).tolist()
        output = rng.integers(0, V, n_o).tolist()
        bias = {int(t): float(rng.standard_normal() * 80) for t in rng.integers(0, V, 30)}
        stops = rng.integers(0, V, 8).tolist()
        seen = list(set(prompt) | set(output) | set(bias) | set(stops)) or [0]
        stream = np.where(rng.random(n_s) < 0.5, rng.choice(seen, n_s), rng.integers(0, V, n_s)).tolist()
        cases.append((prompt, output, stream, bias, stops, 10 ** 6, V, cap))
    return cases


def run_history(mutant):
    """Apply every case's stream token by token to two neighbouring lists (slot 1 with the case, slot 0 poisoned and
    never named): True iff every step gives records(prompt, output + stream so far) exactly, with the rest of the buffer,
    the other slot and the row past the buffer untouched."""
    from oracle.penalties import records
    rng = np.random.default_rng(17)
    for prompt, output, stream, bias, stops, min_tokens, V, cap in history_cases(rng):
        kw = dict(history=True, logit_bias=bias, stop_ids=stops, min_tokens=min_tokens)
        first = records(prompt, output, **kw)
        if len(first) > cap:
            continue
        buf = rng.integers(-2 ** 31, 2 ** 31, (2 * cap + 1, 4))
        buf[cap:cap + len(first)] = first
        lens = np.array([int(rng.integers(0, cap)), len(first)])
        poison = buf.copy()
        out, held = list(output), set(first[:, 0].tolist())
        for t in stream:
            update_emulated(buf, lens, 1, t, cap, mutant)
            if t in held or len(held) < cap:      # a full list drops a new id and keeps its length
                out.append(t)
                held.add(t)
            want = records(prompt, out, **kw)
            n = len(want)
            if lens[1] != n or not np.array_equal(buf[cap:cap + n], want):
                return False
            if not (np.array_equal(buf[:cap], poison[:cap]) and np.array_equal(buf[cap + n:], poison[cap + n:])):
                return False
    return True


def test_update_emulation_equals_records_step_by_step():
    """One update per sampled token keeps the list equal to the oracle's list of the longer output, across chunk
    boundaries, single- and multi-chunk shifts and full lists."""
    assert run_history(None)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_update_checks_reject_mutant(mutant):
    assert not run_history(mutant), f"{mutant} passed the history checks"


def test_records_build_rules():
    from oracle.penalties import PEN_BIAS, PEN_PROMPT, PEN_STOP, records
    r = records([5, 3, 5], [3, 9, 9, 9], history=True, logit_bias={7: 250.0, 3: -0.5, 9: -1e9}, stop_ids=[1, 7],
                min_tokens=5)
    assert r[:, 0].tolist() == [1, 3, 5, 7, 9]
    assert r[:, 1].tolist() == [0, 1, 0, 0, 3]
    assert r[:, 3].tolist() == [PEN_STOP, PEN_PROMPT | PEN_BIAS, PEN_PROMPT, PEN_BIAS | PEN_STOP, PEN_BIAS]
    assert r[:, 2].view(np.float32).tolist() == [0.0, -0.5, 0.0, 100.0, -100.0]
    # no history: only the bias and stop records; min_tokens reached: no stop records
    assert records([5], [3], history=False, logit_bias={2: 1.0}, stop_ids=[4], min_tokens=2)[:, 0].tolist() == [2, 4]
    assert records([5], [3], history=True, stop_ids=[4], min_tokens=1)[:, 0].tolist() == [3, 5]
    assert records().shape == (0, 4)
