"""n-gram speculative decoding on the GPU.

Attention: decode work items with q_count 1..4 (the last token and up to 3 drafts in one 16-row tile) through
b200_op_paged_attn (decode) and b200_op_paged_attn_decode_split, against an fp64 oracle on the bf16 inputs.  Pages the
block table does not name are NaN (a read shows up as a NaN output), rows past each item's last position are finite
poison, and the positions after q_pos0 + j carry keys aimed at row j's queries with large values, so a missing per-row
mask moves the output by O(1).

Engine: draft-rich workloads (prompts made of a repeated random block, logit_bias on a small token set) with
manual_step and kept logits: every emitted token is the oracle's on its kept raw row, every step emits the accepted
drafts plus one token, and the counters, limits and pages add up.
"""
import re

import numpy as np
import pytest
import torch

from kubeai_b200 import ops
from oracle import penalties
from oracle.spec_decode import accept, propose

pytestmark = pytest.mark.gpu

D = 128
RMS_C = 0.04
POISON_V = 512.0


def make_case(items, Hkv, seed):
    """items: (q_pos0, q_count).  Returns q [T, Hq*128], kv pool, block tables, work, and the fp64 oracle output."""
    g = torch.Generator().manual_seed(seed)
    Hq = 4 * Hkv
    lens = [p0 + qc for p0, qc in items]
    nbs = [(L + 15) // 16 for L in lens]
    used = sum(nbs)
    perm = torch.randperm(used + 4, generator=g)
    nan_block = int(perm[-1])
    kv = torch.full((used + 4, 2, Hkv, 16, D), float("nan"), dtype=torch.bfloat16)
    max_blocks = max(nbs) + 2
    btab = torch.full((len(items), max_blocks), nan_block, dtype=torch.int32)
    T = sum(qc for _, qc in items)
    q = torch.randn(T, Hq, D, generator=g).bfloat16()
    want = torch.zeros(T, Hq, D, dtype=torch.float64)
    work, pos, tok = [], 0, 0
    for s, ((p0, qc), L, nb) in enumerate(zip(items, lens, nbs)):
        blocks = perm[pos:pos + nb]
        pos += nb
        btab[s, :nb] = blocks.int()
        k = torch.randn(nb * 16, Hkv, D, generator=g)
        v = torch.randn(nb * 16, Hkv, D, generator=g)
        # each draft position's key aims at the queries of the rows that must not see it
        for i in range(1, qc):
            k[p0 + i] = 0.3 * q[tok:tok + i].float().reshape(i, Hkv, 4, D).sum((0, 2))
            v[p0 + i] = 32.0 * torch.sign(torch.randn(Hkv, D, generator=g))
        k[L:] *= 8.0
        v[L:] = POISON_V
        k, v = k.bfloat16(), v.bfloat16()
        kv[blocks, 0] = k.reshape(nb, 16, Hkv, D).permute(0, 2, 1, 3)
        kv[blocks, 1] = v.reshape(nb, 16, Hkv, D).permute(0, 2, 1, 3)
        for j in range(qc):
            ctx = p0 + j + 1
            kk = k[:ctx].double().repeat_interleave(4, dim=1)        # [ctx, Hq, D]
            vv = v[:ctx].double().repeat_interleave(4, dim=1)
            sc = torch.einsum("hd,thd->ht", q[tok + j].double(), kk) * D ** -0.5
            want[tok + j] = torch.einsum("ht,thd->hd", torch.softmax(sc, -1), vv)
        work.append((tok, qc, p0, s))
        tok += qc
    return (q.reshape(T, Hq * D).cuda(), kv.cuda(), btab.cuda(), torch.tensor(work, dtype=torch.int32).cuda(),
            want.reshape(T, Hq * D))


def run(q, kv, btab, work, Hkv, split):
    out = torch.full((q.shape[0], q.shape[1]), -7776.0, dtype=torch.bfloat16, device="cuda")
    ops.paged_attn(q, kv, btab, work, 4 * Hkv, Hkv, decode=True, out=out, split=split)
    torch.cuda.synchronize()
    return out


def check_close(got, want, what):
    got = got.double().cpu().reshape(got.shape[0], -1, D)
    want = want.reshape(want.shape[0], -1, D)
    assert torch.isfinite(got).all(), f"{what}: non-finite output (an unnamed page was read)"
    err = (got - want).abs().amax(-1)
    rms = want.pow(2).mean(-1).sqrt()
    worst = float((err / rms).max())
    assert worst <= RMS_C, f"{what}: max err/rms {worst:.4f}"


# drafts that start, straddle and end on a page (16) and on a 64-token tile boundary
POSITIONS = [0, 1, 12, 13, 14, 15, 16, 60, 61, 62, 63, 64, 65, 127, 1021, 2045, 4093]


@pytest.mark.parametrize("Hkv", [1, 8])
@pytest.mark.parametrize("split", [0, 1, 2, 5, 32])
def test_multi_position_decode_matches_oracle(Hkv, split):
    items = [(p0, qc) for p0 in POSITIONS for qc in (1, 2, 3, 4)]
    q, kv, btab, work, want = make_case(items, Hkv, seed=11 + Hkv + split)
    got = run(q, kv, btab, work, Hkv, split)
    check_close(got, want, f"Hkv={Hkv} split={split}")


@pytest.mark.parametrize("Hkv", [1, 8])
@pytest.mark.parametrize("split", [0, 3, 32])
def test_single_position_items_are_bit_identical_next_to_verify_items(Hkv, split):
    items = [(700, 1), (700, 4), (63, 1), (61, 4), (2000, 1), (15, 3), (1, 1)]
    q, kv, btab, work, want = make_case(items, Hkv, seed=5)
    mixed = run(q, kv, btab, work, Hkv, split)
    check_close(mixed, want, "mixed")
    ones = [i for i, (_, qc) in enumerate(items) if qc == 1]
    alone = run(q, kv, btab, work[ones].contiguous(), Hkv, split)
    for i in ones:
        t = int(work[i, 0])
        assert torch.equal(mixed[t].view(torch.int16), alone[t].view(torch.int16)), f"item {i}"
    # rows of the launch that no work item names keep the sentinel: nothing is written past q_count
    used = torch.zeros(q.shape[0], dtype=torch.bool)
    for i in ones:
        used[int(work[i, 0])] = True
    assert (alone[~used.cuda()].float() == -7776.0).all()


# ------------------------------------------------------------------------------------------------------------ engine
from kubeai_b200.engine import Engine, mini_config  # noqa: E402

V = 512


def block_prompt(seed, block=23, reps=6):
    rng = np.random.default_rng(seed)
    b = rng.integers(0, V, size=block).tolist()
    return (b * reps)[: block * reps - 3]


def drive(e, reqs, kcfg, max_steps=400):
    """Step the engine until every request finishes; for single-request steps check every emitted token against the oracle
    on the kept rows.  reqs: {rid: dict(prompt, params)}.  Returns {rid: tokens}, per-step (drafts, emitted) pairs."""
    out = {r: [] for r in reqs}
    done = {r: False for r in reqs}
    history = []
    for _ in range(max_steps):
        live = [r for r in reqs if not done[r]]
        ctx = {r: reqs[r]["prompt"] + out[r] for r in live}
        ran, info = e.step()
        assert ran
        rows = e.read_logits(info.sampled) if info.sampled else None
        got = {}
        for r in live:
            pr = e.poll(r)
            got[r] = pr.tokens
            out[r] += pr.tokens
            done[r] = pr.finished is not None
        if len(live) == 1 and rows is not None:
            r = live[0]
            p = reqs[r]["params"]
            n_gen = len(ctx[r]) - len(reqs[r]["prompt"])
            if n_gen > 0:
                # the drafts the engine proposed: the oracle's, with the engine's caps
                cap = min(kcfg["k"], p.get("max_tokens", 16) - n_gen - 1, 256 - len(ctx[r]) - 1)
                drafts = propose(ctx[r], kcfg["min"], kcfg["max"], cap, 256) if cap > 0 else []
                assert info.sampled == 1 + len(drafts), (info.sampled, drafts)
                assert info.draft_tokens == len(drafts)
                toks, tight = [], False
                for j in range(info.sampled):
                    edits = {}
                    if p.get("logit_bias") or p.get("min_tokens"):
                        edits = dict(logit_bias=p.get("logit_bias"), min_tokens=p.get("min_tokens", 0),
                                     output=[0] * (n_gen + j), stop_ids=p.get("stop_all", ()))
                    t, margin = _row_token(rows[j], p, n_gen + j, edits)
                    tight |= margin < 1e-4   # the float64 race cannot order the kernel's fp32 scores this close
                    toks.append(t)
                stops = set(p.get("stop_ids", ()))
                maxt = p.get("max_tokens", 16)
                want = accept(drafts, toks, finishes=lambda j, t: t in stops or n_gen + j + 1 >= maxt
                              or len(ctx[r]) + j + 1 >= 256)
                history.append((len(drafts), len(got[r])))
                if tight:
                    continue
                assert got[r] == want, (got[r], want, drafts)
                assert info.accepted_tokens == sum(1 for j, t in enumerate(want) if j < len(drafts) and t == drafts[j])
        if all(done.values()):
            return out, history
    raise AssertionError("requests did not finish")


def _row_token(row, p, n, edits):
    if edits:
        row = penalties.edit(row, **edits)
    t, margin, *_ = penalties.sample_ref(row, p.get("temperature", 0.0), p.get("top_k", 0), 1.0, p.get("seed", 0), n, 0.0)
    return t, margin


def bias_set(prompt, n=4):
    return {int(t): 12.0 for t in sorted(set(prompt))[:n]}


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("temperature", [0.0, 1.0])
def test_engine_verify_emits_the_oracle_tokens(k, temperature):
    kcfg = dict(k=k, min=1, max=3)
    with Engine(mini_config(num_speculative_tokens=k, prompt_lookup_min=1, prompt_lookup_max=3)) as e:
        e.set_keep_logits(True)
        free0 = e.stats().kv_blocks_free
        total_hist = []
        for seed in range(3):
            prompt = block_prompt(seed)
            params = dict(max_tokens=40, temperature=temperature, top_k=3 if temperature else 0, seed=100 + seed,
                          logit_bias=bias_set(prompt))
            rid = e.submit(prompt, max_tokens=40, temperature=temperature, top_k=params["top_k"], seed=params["seed"],
                           logit_bias=params["logit_bias"])
            out, hist = drive(e, {rid: dict(prompt=prompt, params=params)}, kcfg)
            assert len(out[rid]) == 40
            e.release(rid)
            total_hist += hist
        st = e.stats()
        assert st.spec_accepted_tokens > 0, total_hist
        assert st.spec_draft_tokens > st.spec_accepted_tokens, "no draft was ever rejected"
        assert st.spec_draft_tokens == sum(d for d, _ in total_hist)
        assert sum(st.spec_accepted_per_pos[j] for j in range(3)) == st.spec_accepted_tokens
        assert all(st.spec_accepted_per_pos[j] == 0 for j in range(k, 3))
        assert st.kv_blocks_free == free0


def test_engine_stops_and_limits_inside_a_verify():
    kcfg = dict(k=3, min=1, max=3)
    with Engine(mini_config(num_speculative_tokens=3, prompt_lookup_min=1, prompt_lookup_max=3, eos_token_id=-1)) as e:
        e.set_keep_logits(True)
        free0 = e.stats().kv_blocks_free
        prompt = block_prompt(7)
        bias = bias_set(prompt, 3)
        stop = sorted(bias)[1]
        # a stop id among the biased tokens ends the run inside an accepted run of drafts
        rid = e.submit(prompt, max_tokens=60, stop_ids=[stop], logit_bias=bias, min_tokens=9, ignore_eos=True)
        out, _ = drive(e, {rid: dict(prompt=prompt, params=dict(max_tokens=60, logit_bias=bias, min_tokens=9,
                                                               stop_ids=[stop], stop_all=[stop]))}, kcfg)
        toks = out[rid]
        assert stop not in toks[:9], "min_tokens must mask the stop id through every draft position"
        assert toks[-1] == stop or len(toks) == 60
        assert stop not in toks[:-1]
        e.release(rid)
        # max_tokens and max_model_len are never exceeded
        for mt in (1, 2, 5, 11):
            rid = e.submit(prompt, max_tokens=mt, logit_bias=bias)
            out, _ = drive(e, {rid: dict(prompt=prompt, params=dict(max_tokens=mt, logit_bias=bias))}, kcfg)
            assert len(out[rid]) == mt
            e.release(rid)
        long_prompt = (prompt * 3)[:240]
        rid = e.submit(long_prompt, max_tokens=100, logit_bias=bias)
        out, _ = drive(e, {rid: dict(prompt=long_prompt, params=dict(max_tokens=100, logit_bias=bias))}, kcfg)
        assert len(long_prompt) + len(out[rid]) == 256
        e.release(rid)
        assert e.stats().kv_blocks_free == free0


def test_engine_logprobs_of_verify_rows():
    with Engine(mini_config(num_speculative_tokens=3, prompt_lookup_min=1, prompt_lookup_max=3)) as e:
        e.set_keep_logits(True)
        prompt = block_prompt(3)
        bias = bias_set(prompt)
        rid = e.submit(prompt, max_tokens=30, logit_bias=bias, logprobs=True, top_logprobs=2)
        seen, recs = 0, []
        for _ in range(200):
            ran, info = e.step()
            rows = e.read_logits(info.sampled)
            pr = e.poll_logprobs(rid, 2)
            # the records are those of the rows of the emitted tokens, in order; rejected rows give none
            for j, t in enumerate(pr.tokens):
                ref = torch.log_softmax(torch.tensor(rows[j], dtype=torch.float32), -1)
                assert abs(float(ref[t]) - float(pr.lp[j])) < 1e-4
                order = np.lexsort((np.arange(V), -rows[j]))   # by logit, lowest id on ties
                assert list(pr.top_ids[j]) == [int(x) for x in order[:2]]
            seen += len(pr.tokens)
            if pr.finished:
                break
        assert seen == 30
        assert e.stats().spec_accepted_tokens > 0


def test_engine_mixed_batch_penalised_requests_decode_one_token():
    with Engine(mini_config(num_speculative_tokens=3, prompt_lookup_min=1, prompt_lookup_max=3)) as e:
        e.set_keep_logits(True)
        free0 = e.stats().kv_blocks_free
        prompt = block_prompt(4)
        bias = bias_set(prompt)
        b = e.submit(prompt[::-1], max_tokens=30, logit_bias=bias, presence_penalty=0.5, seed=1)
        a = e.submit(prompt, max_tokens=30, logit_bias=bias)
        outs = {a: [], b: []}
        for _ in range(200):
            ran, info = e.step()
            got = {r: e.poll(r).tokens for r in outs}
            if len(outs[b]) < 30 and outs[b]:
                # b (admitted first) has row 0 and never speculates: one token, equal to the oracle on its edited row
                assert len(got[b]) == 1
                row = e.read_logits(info.sampled)[0]
                want = penalties.edit(row, prompt=prompt[::-1], output=outs[b], presence=0.5, logit_bias=bias)
                assert got[b][0] == int(np.argmax(want))
            for r in outs:
                outs[r] += got[r]
            if len(outs[a]) == 30 and len(outs[b]) == 30:
                break
        assert len(outs[a]) == 30 and len(outs[b]) == 30
        assert e.stats().spec_accepted_tokens > 0
        e.release(a)
        e.release(b)
        assert e.stats().kv_blocks_free == free0


def test_engine_parallel_members_speculate_and_pages_return():
    with Engine(mini_config(num_speculative_tokens=3, prompt_lookup_min=1, prompt_lookup_max=3)) as e:
        free0 = e.stats().kv_blocks_free
        prompt = block_prompt(9)
        bias = bias_set(prompt)
        rids = e.submit_n(prompt, 4, max_tokens=60, temperature=1.0, top_k=2, seed=3, logit_bias=bias)
        multi = {r: 0 for r in rids}   # steps in which a member emitted more than one token: it accepted a draft
        member_drafts = 0
        for _ in range(300):
            ran, info = e.step()
            got = {r: e.poll(r) for r in rids}
            for r in rids:
                multi[r] += len(got[r].tokens) > 1
            member_drafts += info.draft_tokens   # only the members run in this engine
            if all(g.finished for g in got.values()) or not ran:
                break
        assert member_drafts > 0 and all(multi[r] > 0 for r in rids), multi
        for r in rids:
            e.release(r)
        assert e.stats().kv_blocks_free == free0


def test_engine_preemption_and_aborts_while_speculating():
    # a pool too small for all of them: sequences are preempted and recompute from their tokens
    with Engine(mini_config(num_speculative_tokens=3, prompt_lookup_min=1, prompt_lookup_max=3, num_kv_blocks=48)) as e:
        free0 = e.stats().kv_blocks_free
        prompts = [block_prompt(20 + i) for i in range(6)]
        rids = [e.submit(p, max_tokens=80, logit_bias=bias_set(p)) for p in prompts]
        outs = {r: [] for r in rids}
        fin = {}
        for step in range(2000):
            ran, _ = e.step()
            for r in rids:
                pr = e.poll(r)
                outs[r] += pr.tokens
                if pr.finished:
                    fin[r] = pr.finished
            if step == 30:
                e.abort(rids[-1])
            if len(fin) == len(rids) or not ran:
                break
        st = e.stats()
        assert st.preemptions > 0 and st.spec_accepted_tokens > 0
        assert fin[rids[-1]] == "aborted"
        assert all(len(outs[r]) == 80 and fin[r] == "length" for r in rids[:-1])
        for r in rids:
            e.release(r)
        assert e.stats().kv_blocks_free == free0
    # the streams equal those of an engine with room for all of them, up to rounding-level ties (checked on one)
    with Engine(mini_config(num_speculative_tokens=3, prompt_lookup_min=1, prompt_lookup_max=3)) as ref:
        r0 = ref.submit(prompts[0], max_tokens=80, logit_bias=bias_set(prompts[0]))
        want = []
        while len(want) < 80:
            ref.step()
            want += ref.poll(r0).tokens
    n = next((i for i, (x, y) in enumerate(zip(outs[rids[0]], want)) if x != y), 80)
    assert n >= 8, (outs[rids[0]], want)


def single_run_rows(e, prompt, bias, max_tokens):
    """Greedy run of one request with kept logits: its tokens and, per token, the bias-edited row it was chosen from."""
    rid = e.submit(prompt, max_tokens=max_tokens, logit_bias=bias)
    toks, rows = [], []
    while len(toks) < max_tokens:
        ran, info = e.step()
        got = e.poll(rid).tokens
        if got:
            kept = e.read_logits(info.sampled)
            for j, t in enumerate(got):
                rows.append(penalties.edit(kept[j], logit_bias=bias))
                toks.append(t)
    e.release(rid)
    return toks, rows


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_greedy_stream_with_and_without_speculation(seed):
    """The rule of test_vllm_parity_gpu.py: the streams agree up to the first position whose top-2 margin is below the
    logit difference measured between the two runs' kept rows (logits depend on the step's shape, DESIGN.md §8)."""
    prompt = block_prompt(40 + seed)
    bias = bias_set(prompt)
    with Engine(mini_config(num_speculative_tokens=3, prompt_lookup_min=1, prompt_lookup_max=3)) as e:
        e.set_keep_logits(True)
        on, rows_on = single_run_rows(e, prompt, bias, 48)
        assert e.stats().spec_accepted_tokens > 0
    with Engine(mini_config()) as e:
        e.set_keep_logits(True)
        off, rows_off = single_run_rows(e, prompt, bias, 48)
    diff = 0.0
    for i in range(48):
        d = np.abs(rows_on[i] - rows_off[i])
        diff = max(diff, float(np.max(d[np.isfinite(d)])))
        top2 = np.sort(rows_off[i])[-2:]
        if on[i] != off[i]:
            assert float(top2[1] - top2[0]) <= 2 * diff, (i, on, off, diff)
            break
    assert diff < 0.25, diff


def test_engine_prefix_cache_after_speculation():
    with Engine(mini_config(num_speculative_tokens=3, prompt_lookup_min=1, prompt_lookup_max=3)) as e:
        e.set_keep_logits(True)
        prompt = block_prompt(12)
        bias = bias_set(prompt)
        rid = e.submit(prompt, max_tokens=50, logit_bias=bias)
        toks = []
        for _ in range(200):
            e.step()
            pr = e.poll(rid)
            toks += pr.tokens
            if pr.finished:
                break
        assert e.stats().spec_accepted_tokens > 0
        e.release(rid)
        seq = prompt + toks
        # the hit reaches into the generated tokens: the pages the verify steps published
        p2 = seq[:-1]
        rid2 = e.submit(p2, max_tokens=1)
        ran, info = e.step()
        pr = e.poll(rid2)
        assert pr.finished and pr.usage[1] == (len(p2) - 1) // 16 * 16 > len(prompt), (pr.usage, len(prompt), len(p2))
        # the row computed over those cached pages equals a plain forward over the same tokens
        got = e.read_logits(1)[0]
        e.release(rid2)
    with Engine(mini_config()) as ref:
        want = ref.forward_logits(p2)[-1]
    err = np.abs(got - want)
    assert (err <= 0.15 + 1.6e-2 * np.abs(want)).all(), float(err.max())


# ------------------------------------------------------------------------------------------------------------ server
@pytest.fixture(params=[0, 3], ids=["off", "k3"])
def spec_stack(request):
    from kubeai_b200.server import LEAST_LOAD, Server
    engines = [Engine(mini_config(manual_step=0, max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512,
                                  num_speculative_tokens=request.param, prompt_lookup_min=1, prompt_lookup_max=3))]
    srv = Server(engines, model="mini", strategy=LEAST_LOAD, vocab=V, max_model_len=1024, enable_sampling=True,
                 enable_logits_processors=True)
    yield srv, request.param
    srv.close()
    engines[0].close()


def metric(text, name, **labels):
    lab = ",".join(f'{k}="{v}"' for k, v in dict(replica=0, **labels).items())
    m = re.search(re.escape(f"{name}{{{lab}}}") + r" (\d+)", text)
    assert m, name
    return int(m.group(1))


def test_server_over_a_speculating_engine(spec_stack):
    import json
    srv, k = spec_stack
    names = ["b200_engine_spec_decode_num_drafts_total", "b200_engine_spec_decode_num_draft_tokens_total",
             "b200_engine_spec_decode_num_accepted_tokens_total"]
    m0 = srv.metrics()
    assert all(metric(m0, n) == 0 for n in names)
    assert all(metric(m0, "b200_engine_spec_decode_num_accepted_tokens_per_pos_total", position=j) == 0 for j in range(3))
    prompt = block_prompt(50)
    bias = {str(t): v for t, v in bias_set(prompt).items()}
    for i in range(3):
        body = dict(model="mini", prompt=prompt, max_tokens=24, temperature=0, logit_bias=bias)
        r = srv.handle("POST", "/openai/v1/completions", json.dumps(body))
        j = r.json()
        assert r.status == 200 and j["object"] == "text_completion" and j["choices"][0]["finish_reason"] == "length"
        assert j["usage"]["completion_tokens"] == 24 and j["usage"]["prompt_tokens"] == len(prompt)
        rs = srv.handle("POST", "/openai/v1/completions", json.dumps(dict(body, stream=True,
                                                                          stream_options={"include_usage": True})))
        ev = rs.sse_events()
        assert ev[-1] == "[DONE]"
        chunks = [json.loads(x) for x in ev[:-1]]
        # one chunk per token, however many tokens a step emitted
        toks = [c for c in chunks if c["choices"]]
        assert len(toks) == 24 and [c["choices"][0]["finish_reason"] for c in toks] == [None] * 23 + ["length"]
        assert "".join(c["choices"][0]["text"] for c in toks) == j["choices"][0]["text"]
        assert chunks[-1]["usage"]["completion_tokens"] == 24
    m = srv.metrics()
    drafts, dtoks, acc = (metric(m, n) for n in names)
    per_pos = [metric(m, "b200_engine_spec_decode_num_accepted_tokens_per_pos_total", position=j) for j in range(3)]
    if k == 0:
        assert drafts == dtoks == acc == 0 and per_pos == [0, 0, 0]
    else:
        assert drafts > 0 and dtoks >= drafts and 0 < acc <= dtoks and sum(per_pos) == acc
