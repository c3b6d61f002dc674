"""Parallel sampling (n) on the GPU: the fork's page copy (b200_op_kv_copy_blocks) bit for bit against a torch index copy,
the engine's groups (b200_submit_n) on the 2-layer test model with kept logits (one prefill, n bit-identical fork rows,
every member's tokens against oracle/sampling.py with seed + i, KV exact through the copied tail page, pages returned), the
other request fields per member, preemption, aborts, prefix caching off, and the serving shell's n choices against the
oracle builders (oracle/parallel_sampling.py)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

from oracle.parallel_sampling import chat_response, completion_response, usage
from oracle.penalties import edit
from oracle.penalties import sample_ref as sample_edit_ref
from oracle.sampling import sample_ref

pytestmark = pytest.mark.gpu
V = 512
T_, TOP_P = 0.9, 0.95
MARGIN, SLACK = 1e-4, 1e-6   # oracle coin flips: race top-2 margin, top-p boundary slack


def _logit_close(got, want, what):
    err = np.abs(got - want)
    tol = 0.15 + 1.6e-2 * np.abs(want)   # the engine tests' logits tolerance
    assert (err <= tol).all(), f"{what}: max err {err.max():.4f}"


# ------------------------------------------------------------------ op
@pytest.mark.parametrize("layers,hkv,nblocks", [(2, 1, 24), (32, 8, 20)])   # mini and Llama-3-8B page shapes
def test_kv_copy_blocks_bit_exact(layers, hkv, nblocks):
    from kubeai_b200 import ops
    block_bytes = 2 * hkv * 16 * 128 * 2
    g = torch.Generator().manual_seed(layers)
    kv = torch.randint(-32768, 32767, (layers, nblocks, block_bytes // 2), generator=g, dtype=torch.int16)
    src, dst = [3, 3, 7, 1, 3], [10, 11, 2, 15, 19]   # pairs sharing a src; every other page is poison that must keep its bits
    want = kv.clone()
    want[:, dst] = kv[:, src]
    d = kv.cuda()
    ops.kv_copy_blocks(d, layers, nblocks * block_bytes, block_bytes, src, dst)
    torch.cuda.synchronize()
    assert torch.equal(d.cpu(), want)
    ops.kv_copy_blocks(d, layers, nblocks * block_bytes, block_bytes, [], [])   # no pairs: nothing
    torch.cuda.synchronize()
    assert torch.equal(d.cpu(), want)


# ------------------------------------------------------------------ engine
def _prompt(n, seed=0):
    return np.random.default_rng(seed).integers(0, V, size=n).tolist()


@pytest.fixture(scope="module")
def ref():
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(max_batched_tokens=256, num_kv_blocks=256)) as e:
        yield e


def run_group(prompt, n, max_tokens=6, seed=11, budget=256, sp=None, abort=None, **cfg):
    """One group to its end with kept logits.  Returns (tokens per member, kept rows per member [k, V], step infos, blocks
    free after the fork step, finish reasons, the engine's stats after release).  abort: {step: member} aborts before
    that step."""
    from kubeai_b200.engine import Engine, mini_config
    sp = dict(temperature=T_, top_p=TOP_P, **(sp or {}))
    with Engine(mini_config(max_batched_tokens=budget, **cfg)) as e:
        e.set_keep_logits(True)
        total = e.stats().kv_blocks_total
        rids = e.submit_n(prompt, n, max_tokens=max_tokens, seed=seed, **sp)
        assert e._l.b200_engine_unfinished(e._h) == n
        toks, rows, fin = [[] for _ in rids], [[] for _ in rids], [None] * n
        infos, free_fork = [], None
        for step in range(200):
            for i in (abort or {}).get(step, ()):
                e.abort(rids[i])
            ran, info = e.step()
            if not ran:
                break
            infos.append((info.tokens, info.sampled))
            kept = e.read_logits(info.sampled) if info.sampled else None
            polled = [e.poll(r) for r in rids]
            # rows in running order: the members in index order (a leader aborted before the fork still has its row there)
            j = info.sampled - sum(1 for pr in polled if pr.tokens) if free_fork is None else 0
            for i, pr in enumerate(polled):
                if pr.tokens:
                    rows[i].append(kept[j])
                    j += 1
                toks[i] += pr.tokens
                fin[i] = fin[i] or pr.finished
            if free_fork is None and info.sampled:
                free_fork = e.stats().kv_blocks_free
                assert j == info.sampled
        for i, r in enumerate(rids):   # a group aborted before its fork ends in a step that runs nothing
            fin[i] = fin[i] or e.poll(r).finished
            e.release(r)
        st = e.stats()
        assert st.kv_blocks_free == total and st.running == 0 and e._l.b200_engine_unfinished(e._h) == 0
        return toks, [np.array(r) for r in rows], infos, free_fork, fin, st, total


def check_tokens(toks, rows, seed, top_p=TOP_P):
    exempt = 0
    for i, (t, rs) in enumerate(zip(toks, rows)):
        for k, tok in enumerate(t):
            want, margin, slack = sample_ref(rs[k], T_, 0, top_p, seed + i, k)
            if margin < MARGIN or slack < SLACK:
                exempt += 1
                continue
            assert tok == want, (i, k, tok, want)
    assert exempt <= 2


@pytest.mark.parametrize("n_prompt,budget", [(1, 256), (15, 256), (16, 256), (17, 256), (33, 256), (200, 64)])
@pytest.mark.parametrize("n", [2, 4, 16])
def test_group_tokens_pages_and_kv(ref, n_prompt, budget, n):
    prompt = _prompt(n_prompt, n_prompt)
    max_tokens = 6
    toks, rows, infos, free_fork, fin, st, total = run_group(prompt, n, max_tokens=max_tokens, budget=budget)
    assert fin == ["length"] * n and all(len(t) == max_tokens for t in toks)
    # the n fork rows come from one lm_head launch over the same hidden row: bit-identical
    fork = np.stack([r[0] for r in rows])
    assert (fork.view(np.uint32) == fork[0].view(np.uint32)).all()
    check_tokens(toks, rows, 11)
    # the prompt is computed once: every step's tokens add up to it plus the members' decodes
    assert sum(t for t, _ in infos) == n_prompt + n * (max_tokens - 1)
    assert st.prompt_tokens == n_prompt and st.generated_tokens == n * max_tokens
    # pages after the fork: the prompt's, plus one copied tail per member 1..n-1 when the prompt ends inside a page
    pages = -(-n_prompt // 16) + ((n - 1) if n_prompt % 16 else 0)
    assert free_fork == total - pages
    # the members' KV (shared pages and copied tails) gives the logits of a plain forward over prompt + own tokens
    for i in range(n):
        want = ref.forward_logits(prompt + toks[i][:-1])[n_prompt - 1:]
        _logit_close(rows[i], want, f"member {i}")


def test_seedless_members_differ_and_reproduce():
    prompt = _prompt(20)
    a = run_group(prompt, 4, seed=5)[0]
    b = run_group(prompt, 4, seed=5)[0]
    assert a == b and len({tuple(t) for t in a}) > 1
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config()) as e:
        rids = e.submit_n(prompt, 4, max_tokens=6, temperature=T_)
        outs = [[] for _ in rids]
        while e.step()[0]:
            for i, r in enumerate(rids):
                outs[i] += e.poll(r).tokens
        assert all(len(o) == 6 for o in outs) and len({tuple(o) for o in outs}) > 1


def test_submit_n_refusals():
    from kubeai_b200 import B200Error
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(max_num_seqs=8)) as e:
        for n, kw in ((0, dict(temperature=1.0)), (-1, dict(temperature=1.0)), (9, dict(temperature=1.0)), (2, {})):
            with pytest.raises(B200Error) as ei:
                e.submit_n([1, 2, 3], n, **kw)
            assert ei.value.code == -1
        assert "greedy" in str(ei.value)
        assert len(e.submit_n([1, 2, 3], 1)) == 1 and len(e.submit_n([1, 2, 3], 8, temperature=1.0)) == 8


def test_members_edits_logprobs_and_prompt_records():
    """Penalties, min_tokens and logit_bias per member against oracle/penalties.py on the kept raw rows; each member's
    logprobs are its row's; the prompt records are the same for every member."""
    from kubeai_b200 import ops
    from kubeai_b200.engine import Engine, mini_config
    prompt = _prompt(21, 3)
    n, N, steps = 3, 3, 8
    sp = dict(temperature=T_, top_p=TOP_P, repetition_penalty=1.3, frequency_penalty=0.4, presence_penalty=0.2,
              logit_bias={7: 2.0, 300: -100.0}, min_tokens=4, logprobs=True, top_logprobs=N,
              prompt_logprobs=2)
    with Engine(mini_config(eos_token_id=4)) as e:
        e.set_keep_logits(True)
        rids = e.submit_n(prompt, n, max_tokens=steps, seed=21, **sp)
        outs = [[] for _ in rids]
        exempt = 0
        plp = []
        for k in range(steps):
            ran, info = e.step()
            assert ran and info.sampled == n
            rows = e.read_logits(n)
            recs = [e.poll_logprobs(r, N) for r in rids]
            toks = [rc.tokens[0] for rc in recs]
            lp, top_ids, _ = ops.logprobs(torch.from_numpy(rows).bfloat16().cuda(), toks, N)
            for i, rc in enumerate(recs):
                assert rc.lp[0] == lp[i].item() and rc.top_ids[0].tolist() == top_ids[i, :N].tolist()
                row = edit(rows[i], prompt=prompt, output=outs[i], presence=0.2, frequency=0.4, repetition=1.3,
                           min_tokens=4, stop_ids=[4], logit_bias=sp["logit_bias"])
                want, margin, slack, mslack = sample_edit_ref(row, T_, 0, TOP_P, 21 + i, k)
                if min(margin, slack, mslack) < 1e-4:
                    exempt += 1
                else:
                    assert toks[i] == want, (i, k, toks[i], want)
                outs[i].append(toks[i])
            if k == 0:
                plp = [e.poll_prompt_logprobs(r, len(prompt), 2) for r in rids]
        assert exempt <= 2
        assert all(300 not in o and 4 not in o[:4] for o in outs)
        assert plp[0] is not None
        for p in plp[1:]:   # bit for bit
            assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(plp[0], p))


def test_preemption_and_prefix_caching_off():
    """Under KV pressure members are preempted and recomputed, and still finish with every page returned; their fork
    tokens (sampled before any preemption) are the calm run's.  With the prefix cache off the fork still shares the
    prompt's pages by reference, and the run is the calm run token for token."""
    prompt = _prompt(40, 8)
    calm, rows, _, _, _, st, _ = run_group(prompt, 4, max_tokens=24, num_kv_blocks=128)
    assert st.preemptions == 0
    check_tokens(calm, rows, 11)
    pressed, _, _, _, fin, st, _ = run_group(prompt, 4, max_tokens=24, num_kv_blocks=8, max_model_len=64)
    assert st.preemptions > 0 and fin == ["length"] * 4 and all(len(t) == 24 for t in pressed)
    assert [t[0] for t in pressed] == [t[0] for t in calm]
    off, _, _, free_fork, fin, st, total = run_group(prompt, 4, max_tokens=24, num_kv_blocks=128, enable_prefix_caching=0)
    assert free_fork == total - 3 - 3 and st.cached_prompt_tokens == 0
    assert off == calm


@pytest.mark.parametrize("who,when", [((1,), 1), ((0,), 1), ((0, 1, 2), 1), ((2,), 5), ((0,), 5)])
def test_aborts(who, when):
    """Members aborted before the fork (prompt of 200 tokens, fork on the 4th step) or after it end "aborted"; the others
    finish; every page comes back (run_group checks)."""
    prompt = _prompt(200, 2)
    toks, rows, infos, _, fin, st, _ = run_group(prompt, 3, max_tokens=6, budget=64, abort={when: who})
    for i in range(3):
        if i in who:
            assert fin[i] == "aborted" and len(toks[i]) == (0 if when < 4 else when - 3)
        else:
            assert fin[i] == "length" and len(toks[i]) == 6
    if len(who) == 3:
        assert st.generated_tokens == 0
    check_tokens([t for t in toks], rows, 11)


# ------------------------------------------------------------------ server
def _detok(ids):
    from kubeai_b200._lib import lib
    buf = C.create_string_buffer(1 << 16)
    n = lib().b200_detokenize(V, (C.c_int32 * max(len(ids), 1))(*ids), len(ids), buf, 1 << 16)
    return buf.raw[:n].decode()


def _serve(body, route, max_n=8):
    from kubeai_b200.engine import Engine, mini_config
    from kubeai_b200.server import Server
    eng = Engine(mini_config(manual_step=0, max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512))
    srv = Server([eng], model="mini", vocab=V, max_model_len=1024, enable_sampling=True, enable_logprobs=True,
                 enable_prompt_logprobs=True, max_n=max_n)
    ids = srv.render_prompt("/v1/" + route, json.dumps(body)) if max_n >= 2 or body.get("n", 1) == 1 else None
    r = srv.handle("POST", "/openai/v1/" + route, json.dumps(body))
    st = eng.stats()
    srv.close()
    eng.close()
    return r, ids, st


def _engine_members(ids, n, max_tokens, seed):
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512)) as e:
        rids = e.submit_n(ids, n, max_tokens=max_tokens, ignore_eos=True, temperature=T_, seed=seed)
        outs = [[] for _ in rids]
        while e.step()[0]:
            for i, r in enumerate(rids):
                outs[i] += e.poll(r).tokens
        return outs


def _strip(d):
    return {k: v for k, v in d.items() if k not in ("id", "created")}


@pytest.mark.parametrize("route", ["chat/completions", "completions"])
def test_server_non_stream_equals_oracle_and_reproduces(route):
    n, mt = 4, 7
    body = dict(model="mini", max_tokens=mt, n=n, ignore_eos=True, temperature=T_, seed=17)
    body.update(messages=[{"role": "user", "content": "Tell me about the fox."}] if "chat" in route else dict(prompt="The fox"))
    r1, ids, st = _serve(body, route)
    r2, _, _ = _serve(body, route)
    assert r1.status == 200, r1.body
    assert st.prompt_tokens == len(ids) and st.kv_blocks_free == st.kv_blocks_total
    a, b = r1.json(), r2.json()
    assert _strip(a) == _strip(b)
    outs = _engine_members(ids, n, mt, 17)
    build = chat_response if "chat" in route else completion_response
    want = build(a["id"], a["created"], "mini", [(_detok(o), None, "length") for o in outs], usage(len(ids), 0, [mt] * n))
    assert a == want


@pytest.mark.parametrize("route", ["chat/completions", "completions"])
def test_server_stream_choices(route):
    n, mt = 3, 5
    body = dict(model="mini", max_tokens=mt, n=n, ignore_eos=True, temperature=T_, seed=4, stream=True,
                stream_options=dict(include_usage=True))
    body.update(messages=[{"role": "user", "content": "hi there"}] if "chat" in route else dict(prompt="hi there"))
    r, ids, _ = _serve(body, route)
    assert r.status == 200
    ev = r.sse_events()
    assert ev[-1] == "[DONE]"
    chunks = [json.loads(x) for x in ev[:-1]]
    assert chunks[-1]["choices"] == [] and chunks[-1]["usage"]["completion_tokens"] == n * mt
    assert chunks[-1]["usage"]["prompt_tokens"] == len(ids)
    body_chunks = chunks[:-1]
    if "chat" in route:   # one role chunk per choice first
        assert [c["choices"][0]["index"] for c in body_chunks[:n]] == list(range(n))
        assert all(c["choices"][0]["delta"].get("role") == "assistant" for c in body_chunks[:n])
        body_chunks = body_chunks[n:]
    texts, finishes = [""] * n, [0] * n
    for c in body_chunks:
        assert len(c["choices"]) == 1
        ch = c["choices"][0]
        i = ch["index"]
        assert finishes[i] == 0   # nothing after a choice's finish chunk
        texts[i] += ch["delta"]["content"] if "chat" in route else ch["text"]
        if ch["finish_reason"]:
            finishes[i] += 1
    assert finishes == [1] * n
    outs = _engine_members(ids, n, mt, 4)
    assert texts == [_detok(o) for o in outs]


def test_server_n1_bodies_and_off_refusal():
    body = dict(model="mini", max_tokens=6, ignore_eos=True, temperature=T_, seed=2, prompt="abc", logprobs=2)
    on, _, _ = _serve(body, "completions", max_n=8)
    off, _, _ = _serve(body, "completions", max_n=0)
    one, _, _ = _serve({**body, "n": 1}, "completions", max_n=8)
    assert _strip(on.json()) == _strip(off.json()) == _strip(one.json())
    r, _, _ = _serve({**body, "n": 2}, "completions", max_n=0)
    assert r.status == 400 and r.json()["error"] == "bad request: n > 1 is not supported by this engine"


def test_server_client_disconnect_frees_every_page():
    import time
    from kubeai_b200.engine import Engine, mini_config
    from kubeai_b200.server import Server
    eng = Engine(mini_config(manual_step=0, max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512))
    srv = Server([eng], model="mini", vocab=V, max_model_len=1024, enable_sampling=True, max_n=8)
    seen = []

    def on_chunk(c):
        seen.append(c)
        return len(seen) >= 6   # "client gone"

    body = dict(model="mini", messages=[{"role": "user", "content": "x" * 40}], max_tokens=200, n=4, temperature=T_,
                stream=True, ignore_eos=True)
    srv.handle("POST", "/openai/v1/chat/completions", json.dumps(body), on_chunk=on_chunk)
    for _ in range(100):
        if eng.stats().running == 0:
            break
        time.sleep(0.02)
    st = eng.stats()
    srv.close()
    eng.close()
    assert st.running == 0 and st.kv_blocks_free == st.kv_blocks_total and st.generated_tokens < 4 * 200
