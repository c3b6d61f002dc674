"""Prompt logprobs on the GPU: the ranked logprobs_rows kernel (b200_op_logprobs_rank) against the oracle
(oracle/prompt_logprobs.py), the engine's prompt records against the scratch logits they came from, the same prompt under
different schedules (chunk budgets, decoding neighbours, preemption, a cached prefix), the serving shell's prompt_logprobs
and echo JSON against the oracle builders, and the records against vLLM's prompt_logprobs on the 2-layer test model."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.logprobs import completion_logprobs, logprobs_ref
from oracle.prompt_logprobs import echo_completion_logprobs, prompt_logprobs_json, rank_ref

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24


def lp_bound(V):
    """fp32 error of lp = (l - m) - log(sum) against float64 (the bound of the generated-token records)."""
    return min((V / 1024 + 10 + 4) * EPS, 1.5e-5)


def ulp_bf16(x):
    return np.exp2(np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -20))) - 7)


# ------------------------------------------------------------------ op
def _hard_rows(V, g):
    rows, toks = [], []
    rows.append(torch.full((V,), 1.25)); toks.append(V // 2)                 # all equal
    r = torch.full((V,), -6.0)
    tie = torch.randperm(V, generator=g)[:min(1000, V // 2)]
    r[tie] = 2.0
    r[torch.randperm(V, generator=g)[:3]] = 4.0
    rows.append(r); toks.append(int(tie[5]) if float(r[int(tie[5])]) == 2.0 else int(tie[0]))   # ties at the target
    r = torch.randn(V, generator=g)
    r[V - 1] = 50.0
    rows.append(r); toks.append(V - 1)                                        # the target is the max
    r = torch.randn(V, generator=g)
    r[3] = -50.0
    rows.append(r); toks.append(3)                                            # the target is the min
    r = torch.randn(V, generator=g)
    r[: V // 4] = 0.0
    r[V // 4: V // 2] = -0.0
    rows.append(r); toks.append(V // 4 + 1)                                   # -0 and +0 are one logit
    return torch.stack(rows).bfloat16(), toks


@pytest.mark.parametrize("V", [512, 1000, 128256])
def test_op_rank_matches_oracle(V):
    from kubeai_b200 import ops
    g = torch.Generator().manual_seed(V)
    S = 64
    rand = (torch.randn(S, V, generator=g) * 3).bfloat16()
    hard, htoks = _hard_rows(V, g)
    logits = torch.cat([rand, hard])
    rng = np.random.default_rng(V)
    tokens = np.concatenate([rng.integers(0, V, S), htoks]).astype(np.int32)
    tokens[:S:3] = torch.argmax(rand.float(), 1).numpy()[::3]
    ns = rng.choice([0, 1, 5, 20], len(tokens)).astype(np.int32)
    ns[S:] = 20
    d = logits.cuda()
    lp, rank, ti, tl = (t.cpu().numpy() for t in ops.logprobs_rank(d, tokens, ns))
    lp0, ti0, tl0 = (t.cpu().numpy() for t in ops.logprobs(d, tokens, ns))
    assert lp.view(np.uint32).tolist() == lp0.view(np.uint32).tolist()         # the same bits as without ranks
    assert np.array_equal(ti, ti0) and np.array_equal(tl.view(np.uint32), tl0.view(np.uint32))
    lf = logits.float().numpy()
    for s in range(len(tokens)):
        assert rank[s] == rank_ref(lf[s], tokens[s]), (s, rank[s], rank_ref(lf[s], tokens[s]))
        ref, ids = logprobs_ref(lf[s], ns[s])
        assert np.array_equal(ti[s, :ns[s]], ids)
        assert abs(lp[s] - ref[tokens[s]]) <= lp_bound(V) + 2.0 ** -22 * abs(ref[tokens[s]])
    assert rank[S] == V and rank[S + 2] == 1 and rank[S + 3] == V


# ------------------------------------------------------------------ engine, exact against the scratch rows
def _scratch(e, V):
    return (e.tensor("step.prompt_logits").astype(np.uint32) << 16).view(np.float32).reshape(-1, V)


def _check_exact(rows, recs, toks, N):
    """rows: the fp32 logits the records came from; recs: (lp, rank, top_ids, top_lp) arrays."""
    lp, rank, ti, tl = recs
    V = rows.shape[1]
    for k in range(len(toks)):
        ref, ids = logprobs_ref(rows[k], N)
        assert np.array_equal(ti[k], ids), k
        assert rank[k] == rank_ref(rows[k], toks[k]), k
        want = np.concatenate([[ref[toks[k]]], ref[ids]])
        got = np.concatenate([[lp[k]], tl[k]]).astype(np.float64)
        assert (np.abs(got - want) <= lp_bound(V) + 2.0 ** -22 * np.abs(want)).all(), k


def test_engine_records_equal_oracle_on_their_rows():
    from kubeai_b200 import B200Error
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(1)
    V = 512
    with Engine(mini_config(max_batched_tokens=256, max_model_len=512)) as e:
        # one step, two whole prompts: rows 0..198 are A's positions, 199..237 B's
        A, B = rng.integers(0, V, 200).tolist(), rng.integers(0, V, 40).tolist()
        ra, rb = e.submit(A, max_tokens=2, prompt_logprobs=5), e.submit(B, max_tokens=2, prompt_logprobs=20)
        before = e.stats().d2h_bytes
        e.step()
        assert e.stats().d2h_bytes - before == 2 * 4 + 238 * 4 * 42
        rows = _scratch(e, V)
        got_a, got_b = e.poll_prompt_logprobs(ra, 200, 5), e.poll_prompt_logprobs(rb, 40, 20)
        _check_exact(rows[:199], got_a, A[1:], 5)
        _check_exact(rows[199:238], got_b, B[1:], 20)
        # a 300-token prompt in two chunks of 256 and 44 rows: nothing before the last chunk, then all 299 records
        while not (e.poll(ra).finished and e.poll(rb).finished):
            e.step()
        C = rng.integers(0, V, 300).tolist()
        rc = e.submit(C, max_tokens=1, prompt_logprobs=3)
        e.step()
        assert e.poll_prompt_logprobs(rc, 300, 3) is None
        first = _scratch(e, V)[:256].copy()
        e.step()
        second = _scratch(e, V)[:43].copy()
        got = e.poll_prompt_logprobs(rc, 300, 3)
        assert got is not None and len(got[0]) == 299
        _check_exact(np.concatenate([first, second]), got, C[1:], 3)
        assert len(e.poll(rc).tokens) == 1                            # the prompt records did not move the token cursor
        with pytest.raises(B200Error):
            e.poll_prompt_logprobs(e.submit([1, 2, 3]), 3, 0)
        for bad in (dict(prompt_logprobs=21), dict(prompt_logprobs=-1)):
            with pytest.raises(B200Error):
                e.submit([1, 2, 3], **bad)


# ------------------------------------------------------------------ engine, across schedules
PROMPT = np.random.default_rng(7).integers(0, 512, 150).tolist()
N_P = 5


def _run(cfg, plp, others=(), others_first=0, prefix_first=False):
    """The tokens, prompt records and usage of PROMPT (+ others submitted before it, stepped others_first times)."""
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(**cfg)) as e:
        if prefix_first:
            e.generate([PROMPT], max_tokens=2)
        rids = [e.submit(p, max_tokens=12) for p in others]
        for _ in range(others_first):
            e.step()
        r = e.submit(PROMPT, max_tokens=12, prompt_logprobs=plp)
        toks, recs, usage = [], None, None
        for _ in range(500):
            ran, _ = e.step()
            for o in rids:
                e.poll(o)
            pr = e.poll(r)
            toks += pr.tokens
            if toks and plp is not None and recs is None:
                recs = e.poll_prompt_logprobs(r, len(PROMPT), plp)
                assert recs is not None
            if pr.finished:
                usage = pr.usage
                break
        return toks, recs, usage, e.stats().preemptions


def _rows():
    """bf16 logits of PROMPT's positions from a plain forward of the same seeded model."""
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config()) as e:
        return e.forward_logits(PROMPT)[:-1]


def _check_close(recs, rows, what):
    lp, rank, ti, tl = recs
    assert len(lp) == len(PROMPT) - 1, what
    worst = 0.0
    for k in range(len(lp)):
        x = rows[k].astype(np.float64)
        margin = 4 * float(ulp_bf16(np.abs(x).max()))        # split-K and chunking differ between the runs
        ref, ids = logprobs_ref(x, N_P)
        t = PROMPT[k + 1]
        err = abs(lp[k] - ref[t])
        worst = max(worst, err / margin)
        assert err <= 2 * margin + lp_bound(512), (what, k, err, margin)
        if (np.abs(x - x[t]) <= 2 * margin).sum() == 1:       # no other logit near the token's: the rank is certain
            assert rank[k] == rank_ref(x, t), (what, k)
        srt = np.sort(x)[::-1]
        for j in range(N_P):
            if all(abs(srt[j] - srt[q]) > 2 * margin for q in (j - 1, j + 1) if 0 <= q < len(srt)):
                assert ti[k, j] == ids[j], (what, k, j)
    return worst


def test_records_across_schedules():
    rng = np.random.default_rng(11)
    others = [rng.integers(0, 512, n).tolist() for n in (20, 33, 47)]
    base = dict(max_batched_tokens=256)
    runs = {
        "alone": (base, {}),
        "chunks of 64": (dict(max_batched_tokens=64), {}),
        "chunks of 32 next to decodes": (dict(max_batched_tokens=32), dict(others=others, others_first=4)),
        "preempted": (dict(num_kv_blocks=16, max_model_len=224, enable_prefix_caching=0, max_batched_tokens=64),
                      dict(others=[rng.integers(0, 512, 60).tolist() for _ in range(4)], others_first=2)),
    }
    rows = _rows()
    for what, (cfg, kw) in runs.items():
        toks, recs, usage, pre = _run(cfg, N_P, **kw)
        toks0, _, _, pre0 = _run(cfg, None, **kw)
        assert toks == toks0 and pre == pre0, what           # asking for prompt logprobs changes no token
        if what == "preempted":
            assert pre > 0
        worst = _check_close(recs, rows, what)
        print(f"{what}: {len(recs[0])} records, worst |lp - oracle| = {worst:.2f} x 4 bf16 ulps of the row max")
    toks, recs, usage, _ = _run(base, N_P, prefix_first=True)
    assert usage[1] == 0                                      # cached_tokens: the cached prefix was not read
    _check_close(recs, rows, "after a cached prefix")
    toks1, _, usage1, _ = _run(base, None, prefix_first=True)
    assert usage1[1] == 144                                   # without the field the same prompt hits 9 blocks


# ------------------------------------------------------------------ serving shell
def f32(x):
    if isinstance(x, float):
        return float(np.float32(x))
    if isinstance(x, dict):
        return {k: f32(v) for k, v in x.items()}
    if isinstance(x, list):
        return [f32(v) for v in x]
    return x


def token_str(t):
    s = ""
    for _ in range(4):
        s = chr(ord("a") + t % 26) + s
        t //= 26
    return " " + s


CFG = dict(max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512)


def _engine_records(ids, n_prompt_lp, n_lp, max_tokens):
    """The same request on a fresh engine stepped alone: prompt records [(tok, lp, rank, ids, lps)], output records
    [(tok, lp, ids, lps)]."""
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(**CFG)) as e:
        r = e.submit(ids, max_tokens=max_tokens, prompt_logprobs=n_prompt_lp, logprobs=n_lp is not None,
                     top_logprobs=n_lp or 0)
        out = []
        while True:
            ran, _ = e.step()
            pr = e.poll_logprobs(r, n_lp) if n_lp is not None else e.poll(r)
            if n_lp is not None:
                out += list(zip(pr.tokens, pr.lp, pr.top_ids, pr.top_lp))
            if pr.finished or not ran:
                break
        lp, rank, ti, tl = e.poll_prompt_logprobs(r, len(ids), n_prompt_lp)
        return [(ids[k + 1], lp[k], rank[k], ti[k], tl[k]) for k in range(len(ids) - 1)], out


def test_server_json_equals_oracle_builders():
    from kubeai_b200.engine import Engine, mini_config
    from kubeai_b200.server import Server
    id_prompt = [5, 300, 17, 17, 400, 2, 99, 123]
    cases = []
    for prompt in ("The quick brown fox", id_prompt):
        for n in (0, 1, 5):
            for mt in (0, 1):
                cases.append(dict(prompt=prompt, echo=True, logprobs=n, max_tokens=mt))
        cases.append(dict(prompt=prompt, prompt_logprobs=3, max_tokens=4))
        cases.append(dict(prompt=prompt, echo=True, max_tokens=3))                                  # echo, no logprobs
        cases.append(dict(prompt=prompt, echo=True, logprobs=2, max_tokens=4, stream=True,
                          stream_options=dict(include_usage=True)))
        cases.append(dict(prompt=prompt, echo=True, logprobs=1, max_tokens=0, stream=True))
    cases.append(dict(prompt=id_prompt, echo=True, logprobs=1, max_tokens=1, temperature=0))          # lm-eval loglikelihood
    cases.append(dict(messages=[{"role": "user", "content": "Tell me about the fox."}], prompt_logprobs=4, max_tokens=3,
                      logprobs=True, top_logprobs=2))
    eng = Engine(mini_config(manual_step=0, **CFG))
    srv = Server([eng], model="mini", vocab=512, max_model_len=1024, enable_sampling=True, enable_logprobs=True,
                 enable_prompt_logprobs=True)
    try:
        for body in cases:
            chat = "messages" in body
            path = "/v1/chat/completions" if chat else "/v1/completions"
            body = dict(model="mini", ignore_eos=True, **body)
            ids = srv.render_prompt(path, json.dumps(body))
            r = srv.handle("POST", "/openai" + path, json.dumps(body))
            assert r.status == 200, (body, r.body)
            n_lp = body.get("top_logprobs", 0) if chat and body.get("logprobs") else (None if chat else body.get("logprobs"))
            n_p = body.get("prompt_logprobs", n_lp if body.get("echo") else None)
            mt = body["max_tokens"]
            precs, orecs = _engine_records(ids, n_p, n_lp, max(mt, 1)) if n_p is not None else ([], None)
            if n_p is None:
                orecs = None
            echo_text = body["prompt"] if isinstance(body.get("prompt"), str) else "".join(token_str(t) for t in ids)
            if body.get("stream"):
                chunks = [json.loads(x) for x in r.sse_events()[:-1]]
                first = chunks[0]["choices"][0]
                if mt == 0:
                    assert first["text"] == echo_text and len(chunks) == 1 + bool(body.get("stream_options"))
                    assert f32(first["logprobs"]) == f32(echo_completion_logprobs(ids, precs, n_lp, token_str))
                else:
                    assert first["text"] == echo_text + token_str(orecs[0][0])
                    assert f32(first["logprobs"]) == f32(echo_completion_logprobs(ids, precs, n_lp, token_str, orecs[:1]))
                    off = len(token_str(orecs[0][0]))
                    for k, c in enumerate(chunks[1:mt], start=1):
                        assert f32(c["choices"][0]["logprobs"]) == f32(completion_logprobs([orecs[k]], n_lp, token_str, off))
                        off += len(c["choices"][0]["text"])
                if body.get("stream_options"):
                    assert chunks[-1]["usage"]["completion_tokens"] == mt
                continue
            j = r.json()
            ch = j["choices"][0]
            if chat:
                assert f32(j["prompt_logprobs"]) == f32(prompt_logprobs_json(precs, token_str))
                assert "prompt_logprobs" not in ch
                continue
            if body.get("echo"):
                assert ch["text"].startswith(echo_text)
                assert (ch["text"] == echo_text) == (mt == 0)
            if n_lp is not None and body.get("echo"):
                want = echo_completion_logprobs(ids, precs, n_lp, token_str, orecs if mt else ())
                assert f32(ch["logprobs"]) == f32(want), body
                assert [token_str(t) for t in ids[1:]] == want["tokens"][1:len(ids)]
            if n_p is not None:
                assert f32(ch["prompt_logprobs"]) == f32(prompt_logprobs_json(precs, token_str)), body
            else:
                assert "prompt_logprobs" not in ch
            assert j["usage"]["prompt_tokens"] == len(ids) and j["usage"]["completion_tokens"] == max(mt, 1)
            if n_p is not None:
                assert j["usage"]["prompt_tokens_details"]["cached_tokens"] == 0
            try:
                from vllm.entrypoints.openai.completion.protocol import CompletionResponse
                CompletionResponse.model_validate(j)
            except ImportError:
                pass
    finally:
        srv.close()
        eng.close()


# ------------------------------------------------------------------ vLLM parity (2-layer test model)
def _vllm_ok():
    if os.environ.get("B200_SKIP_VLLM") == "1":
        return False
    try:
        import vllm  # noqa: F401
        return True
    except Exception:
        return False


LOGPROB_ULPS = 6.0


@pytest.mark.skipif(not _vllm_ok(), reason="vllm is not importable (or B200_SKIP_VLLM=1)")
def test_prompt_logprobs_match_vllm_on_the_test_model(tmp_path):
    os.environ.setdefault("HF_HUB_OFFLINE", "1")
    os.environ.setdefault("VLLM_NO_USAGE_STATS", "1")
    from safetensors.torch import save_file
    from vllm import LLM, SamplingParams

    from kubeai_b200.engine import Engine, config_from_hf
    from oracle.gen_golden import hf_model
    from oracle.weights import ModelCfg, make_weights
    cfg = ModelCfg()
    m = hf_model(cfg, make_weights(cfg), torch.bfloat16)
    m.config.save_pretrained(tmp_path)
    save_file({k: v.contiguous() for k, v in m.state_dict().items()}, str(tmp_path / "model.safetensors"))
    g = torch.Generator().manual_seed(29)
    prompts = [torch.randint(0, cfg.vocab, (int(n),), generator=g).tolist() for n in (5, 17, 40, 90, 150)]
    N = 5
    ecfg = config_from_hf(tmp_path, max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=256,
                          manual_step=1, seed=777)
    mine = []
    with Engine(ecfg) as e:
        e.load_safetensors(tmp_path)
        for p in prompts:
            r = e.submit(p, max_tokens=1, prompt_logprobs=N)
            while not e.poll(r).finished:
                e.step()
            mine.append((e.poll_prompt_logprobs(r, len(p), N), e.forward_logits(p)[:-1]))
    llm = LLM(model=str(tmp_path), skip_tokenizer_init=True, dtype="bfloat16", max_model_len=256, enforce_eager=True,
              gpu_memory_utilization=0.25, enable_prefix_caching=False, seed=0)
    outs = llm.generate([{"prompt_token_ids": p} for p in prompts],
                        SamplingParams(temperature=0.0, max_tokens=1, detokenize=False, prompt_logprobs=N))
    compared = ranks = 0
    for p, o, ((lp, rank, ti, tl), rows) in zip(prompts, outs, mine):
        ref = o.prompt_logprobs
        assert ref[0] is None and len(ref) == len(p)
        for k in range(len(p) - 1):
            d = ref[k + 1]
            t = p[k + 1]
            margin = LOGPROB_ULPS * float(ulp_bf16(np.abs(rows[k]).max()))
            assert abs(lp[k] - d[t].logprob) <= margin, (len(p), k, lp[k], d[t].logprob)
            x = rows[k].astype(np.float64)
            near = int((np.abs(x - x[t]) <= margin).sum()) - 1   # other logits within the margin of the token's
            assert abs(rank[k] - d[t].rank) <= near, (len(p), k, rank[k], d[t].rank, near)   # near == 0: equal
            ranks += near == 0
            compared += 1
    print(f"vLLM prompt_logprobs parity: {compared} positions, {ranks} with no other logit within the margin")
    assert compared == sum(len(p) - 1 for p in prompts)
