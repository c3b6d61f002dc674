"""Logprobs on the GPU: the logprobs_rows kernel (b200_op_logprobs) against the float64 oracle (oracle/logprobs.py), hard
rows, determinism, records of engine batches (mixed greedy / sampled / logprobs / preempted requests) and the serving
shell's JSON against vLLM's response builders, and the engine's records against vLLM on the 2-layer test model."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.logprobs import chat_logprobs, completion_logprobs, logprobs_ref

pytestmark = pytest.mark.gpu
EPS = 2.0 ** -24


def lp_bound(V):
    """fp32 error of lp = (l - m) - log(sum): the sum runs V/1024 sequential additions per thread and 10 tree levels,
    each rounding by <= 2^-24 relative, plus a few ulps from expf / logf; the two subtractions add 2^-22 |lp|."""
    return min((V / 1024 + 10 + 4) * EPS, 1.5e-5)


def bf16_rows(S, V, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(S, V, generator=g) * scale).bfloat16()


def check_rows(lf, tokens, ns, lp, top_ids, top_lp, V):
    """lf: float32 [S, V]; returns the largest error seen."""
    worst = 0.0
    tol_abs = lp_bound(V)
    for s in range(lf.shape[0]):
        ref, ids = logprobs_ref(lf[s], ns[s])
        n = len(ids)
        assert np.array_equal(top_ids[s, :n], ids), (s, top_ids[s, :n], ids)
        got = np.concatenate([[lp[s]], top_lp[s, :n]]).astype(np.float64)
        want = np.concatenate([[ref[tokens[s]]], ref[ids]])
        err = np.abs(got - want)
        assert (err <= tol_abs + 2.0 ** -22 * np.abs(want)).all(), (s, err.max())
        worst = max(worst, float(err.max()))
        assert (np.diff(top_lp[s, :n]) <= 0).all()
        hit = np.flatnonzero(top_ids[s, :n] == tokens[s])
        if len(hit):
            assert top_lp[s, hit[0]].view(np.uint32) == np.float32(lp[s]).view(np.uint32)
    return worst


def run_op(logits, tokens, ns):
    from kubeai_b200 import ops
    lp, ti, tl = ops.logprobs(logits, tokens, ns)
    return lp.cpu().numpy(), ti.cpu().numpy(), tl.cpu().numpy()


@pytest.mark.parametrize("V", [512, 1000, 128256])
@pytest.mark.parametrize("S", [1, 7, 128, 300])
def test_op_matches_oracle(V, S):
    logits = bf16_rows(S, V, seed=V * 3 + S)
    rng = np.random.default_rng(S + V)
    ns = rng.choice([0, 1, 5, 20], S).astype(np.int32)
    tokens = rng.integers(0, V, S).astype(np.int32)
    tokens[::3] = torch.argmax(logits.float(), 1).numpy()[::3]     # a third of the rows: the sampled token is the top one
    lp, ti, tl = run_op(logits.cuda(), tokens, ns)
    worst = check_rows(logits.float().numpy(), tokens, ns, lp, ti, tl, V)
    print(f"V={V} S={S}: max |lp - float64| = {worst:.3g} (bound {lp_bound(V):.3g} + 2^-22 |lp|)")


def test_hard_rows():
    V, N = 128256, 20
    rows = []
    rows.append(torch.full((V,), 1.25))                                    # all equal
    r = torch.full((V,), -6.0)
    g = torch.Generator().manual_seed(3)
    tie = torch.randperm(V, generator=g)[:1000]
    r[tie] = 2.0                                                           # 1000 ties across the 20th value
    above = torch.randperm(V, generator=g)[:3]
    r[above] = 4.0
    rows.append(r)
    r = torch.randn(V, generator=g)
    r[777] = 90.0                                                          # one far above the rest
    rows.append(r)
    r = torch.full((V,), -1.0)
    r[torch.arange(5, V, 9000)] = 0.0
    r[torch.arange(9, V, 7000)] = -0.0                                     # -0 and +0: one key
    rows.append(r)
    logits = torch.stack(rows).bfloat16()
    lf = logits.float().numpy()
    tokens = np.array([V - 1, int(tie.min()), 777, 9], dtype=np.int32)
    ns = np.full(4, N, dtype=np.int32)
    lp, ti, tl = run_op(logits.cuda(), tokens, ns)
    check_rows(lf, tokens, ns, lp, ti, tl, V)
    assert np.array_equal(ti[0], np.arange(N)) and np.allclose(tl[0], -np.log(V), atol=lp_bound(V), rtol=0)
    assert len(set(tl[0].view(np.uint32).tolist())) == 1 and tl[0, 0] == lp[0]
    assert sorted(ti[1, :3].tolist()) == sorted(above.tolist()) and ti[1, :3].tolist() == sorted(ti[1, :3].tolist())
    assert ti[1, 3:].tolist() == sorted(tie.tolist())[:17]
    assert ti[2, 0] == 777 and lp[2] == 0.0
    zeros = np.flatnonzero(lf[3] == 0)
    assert ti[3].tolist() == zeros[:N].tolist() and len(set(tl[3].view(np.uint32).tolist())) == 1
    # V = 1001 inside rows of ld = 1008
    from kubeai_b200._lib import check, lib
    from kubeai_b200.ops import _p, _stream
    S, V2, ld = 9, 1001, 1008
    full = bf16_rows(S, ld, seed=11).cuda()
    toks = np.arange(S, dtype=np.int32) * 111
    n2 = np.array([0, 1, 5, 20, 20, 5, 1, 0, 20], dtype=np.int32)
    t_d, n_d = torch.from_numpy(toks).cuda(), torch.from_numpy(n2).cuda()
    lp2 = torch.zeros(S, device="cuda")
    ti2 = torch.zeros(S, 20, dtype=torch.int32, device="cuda")
    tl2 = torch.zeros(S, 20, device="cuda")
    check(lib().b200_op_logprobs(_p(full), ld, S, V2, _p(t_d), _p(n_d), _p(lp2), _p(ti2), _p(tl2), _stream()))
    check_rows(full.float().cpu().numpy()[:, :V2], toks, n2, lp2.cpu().numpy(), ti2.cpu().numpy(), tl2.cpu().numpy(), V2)
    assert (ti2.cpu().numpy()[n2 == 0] == 0).all()          # entries past N are left as they were


def test_rows_are_independent_of_their_place():
    S, V = 128, 128256
    logits = bf16_rows(S, V, seed=21).cuda()
    rng = np.random.default_rng(4)
    ns = rng.choice([0, 1, 5, 20], S).astype(np.int32)
    tokens = rng.integers(0, V, S).astype(np.int32)
    a = run_op(logits, tokens, ns)
    perm = rng.permutation(S)
    b = run_op(logits[torch.from_numpy(perm).cuda()].contiguous(), tokens[perm], ns[perm])
    for x, y in zip(a, b):
        assert np.array_equal(x[perm].view(np.uint32), y.view(np.uint32))


# ------------------------------------------------------------------ engine (mini model)
PROMPTS = [list(np.random.default_rng(60 + i).integers(0, 512, 9 + 3 * i)) for i in range(8)]
SPECS = [dict(), dict(logprobs=True), dict(logprobs=True, top_logprobs=5), dict(temperature=0.8, seed=1),
         dict(temperature=0.9, top_p=0.9, seed=2, logprobs=True, top_logprobs=20),
         dict(temperature=1.0, top_k=5, seed=3, logprobs=True, top_logprobs=1), dict(logprobs=True, top_logprobs=20),
         dict(temperature=0.7, seed=4)]
N_TOK = 8


def no_lp(specs):
    return [{k: v for k, v in s.items() if k not in ("logprobs", "top_logprobs")} for s in specs]


def run_batch(specs, check):
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config()) as e:
        e.set_keep_logits(True)
        rids = [e.submit(p, max_tokens=N_TOK, **sp) for p, sp in zip(PROMPTS, specs)]
        outs = [[] for _ in rids]
        for step in range(N_TOK):
            before = e.stats().d2h_bytes
            ran, info = e.step()
            assert ran and info.sampled == len(rids)
            n_lp = sum(1 for s in specs if s.get("logprobs"))
            assert e.stats().d2h_bytes - before == 4 * len(rids) + n_lp * 4 * 41
            rows = e.read_logits(len(rids))
            for i, r in enumerate(rids):
                sp = specs[i]
                if not sp.get("logprobs"):
                    outs[i] += e.poll(r).tokens
                    continue
                n = sp.get("top_logprobs", 0)
                pr = e.poll_logprobs(r, n)
                assert len(pr.tokens) == 1 and pr.top_ids.shape == (1, n)
                outs[i] += pr.tokens
                if check:
                    check_rows(rows[i:i + 1], np.array(pr.tokens, np.int32), [n], pr.lp, pr.top_ids, pr.top_lp, 512)
        return outs


def test_engine_records_match_oracle_and_tokens_do_not_change():
    from kubeai_b200 import B200Error
    a = run_batch(SPECS, check=True)
    assert a == run_batch(no_lp(SPECS), check=False)
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config()) as e:
        r = e.submit([1, 2, 3])
        with pytest.raises(B200Error):
            e.poll_logprobs(r, 0)
        for bad in (dict(logprobs=True, top_logprobs=21), dict(logprobs=True, top_logprobs=-1), dict(top_logprobs=3)):
            with pytest.raises(B200Error):
                e.submit([1, 2, 3], **bad)


def test_engine_records_survive_preemption():
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, 512, size=40).tolist() for _ in range(6)]
    specs = [dict(logprobs=True, top_logprobs=(0, 3, 20)[i % 3]) if i % 2 == 0 else dict(temperature=0.8, seed=i)
             for i in range(6)]

    def run(sp_list):
        with Engine(mini_config(num_kv_blocks=14, max_model_len=224, enable_prefix_caching=0)) as e:
            rids = [e.submit(p, max_tokens=24, **s) for p, s in zip(prompts, sp_list)]
            outs, recs = [[] for _ in rids], [0] * len(rids)
            for _ in range(400):
                ran, _ = e.step()
                for i, r in enumerate(rids):
                    if sp_list[i].get("logprobs"):
                        pr = e.poll_logprobs(r, sp_list[i]["top_logprobs"])
                        recs[i] += len(pr.lp)
                        assert np.isfinite(pr.lp).all() and (pr.lp <= 0).all()
                    else:
                        pr = e.poll(r)
                    outs[i] += pr.tokens
                if not ran:
                    break
            assert e.stats().preemptions > 0
            return outs, recs

    outs, recs = run(specs)
    assert all(len(o) == 24 for o in outs)
    assert [recs[i] for i in range(0, 6, 2)] == [24, 24, 24]        # one record per generated token
    assert outs == run(no_lp(specs))[0]


def test_full_size_step():
    """128 rows at V = 128256, N = 20, as the lm_head of one decode step leaves them."""
    from kubeai_b200.engine import Engine, mini_config
    V = 128256
    with Engine(mini_config(vocab=V, max_num_seqs=128, max_batched_tokens=1024, num_kv_blocks=1024)) as e:
        e.set_keep_logits(True)
        rng = np.random.default_rng(8)
        rids = [e.submit(rng.integers(0, V, 4).tolist(), max_tokens=2, logprobs=True, top_logprobs=20) for _ in range(128)]
        e.step()
        for r in rids:
            e.poll_logprobs(r, 20)
        ran, info = e.step()
        assert ran and info.sampled == 128 and info.decode_seqs == 128
        rows = e.read_logits(128)
        got = [e.poll_logprobs(r, 20) for r in rids]
    tokens = np.array([g.tokens[0] for g in got], np.int32)
    worst = check_rows(rows, tokens, [20] * 128, np.concatenate([g.lp for g in got]),
                       np.concatenate([g.top_ids for g in got]), np.concatenate([g.top_lp for g in got]), V)
    assert (tokens == rows.argmax(1)).all()
    print(f"full-size step: max |lp - float64| = {worst:.3g}")


# ------------------------------------------------------------------ serving shell
def f32(x):
    """JSON floats compared as the fp32 values the engine computed."""
    if isinstance(x, float):
        return float(np.float32(x))
    if isinstance(x, dict):
        return {k: f32(v) for k, v in x.items()}
    if isinstance(x, list):
        return [f32(v) for v in x]
    return x


TOKENIZER_CORPUS = ["The quick brown fox jumps over the lazy dog. naïve café, 你好世界 \U0001f642 12345"] * 20


def _tokenizer(tmp_path):
    tokenizers = pytest.importorskip("tokenizers")
    from tokenizers import Regex, decoders, models, pre_tokenizers, trainers
    pattern = r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+"
    tok = tokenizers.Tokenizer(models.BPE(ignore_merges=True))
    tok.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(pattern), behavior="isolated", invert=False),
                                                 pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    specials = ["<|begin_of_text|>", "<|end_of_text|>", "<|start_header_id|>", "<|end_header_id|>", "<|eot_id|>"]
    tok.train_from_iterator(TOKENIZER_CORPUS, trainers.BpeTrainer(vocab_size=400, special_tokens=specials, show_progress=False,
                                                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet()))
    path = tmp_path / "tokenizer.json"
    tok.save(str(path))
    from kubeai_b200.tokenizer import Tokenizer
    return tok, Tokenizer(path)


CFG = dict(max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512)


def _records(ids, n, sampling):
    """poll_logprobs of the same request on a fresh engine, stepped alone: [(token, lp, top ids, top lp)]"""
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(**CFG)) as e:
        r = e.submit(ids, max_tokens=7, logprobs=True, top_logprobs=n, **sampling)
        recs = []
        while True:
            ran, _ = e.step()
            pr = e.poll_logprobs(r, n)
            recs += list(zip(pr.tokens, pr.lp, pr.top_ids, pr.top_lp))
            if pr.finished or not ran:
                return recs


@pytest.mark.parametrize("real_tok", [False, True])
def test_server_json_equals_oracle_builders(real_tok, tmp_path):
    from kubeai_b200.engine import Engine, mini_config
    from kubeai_b200.server import Server
    hf = mine = None
    if real_tok:
        hf, mine = _tokenizer(tmp_path)

        def token_str(t):
            return hf.decode([int(t)], skip_special_tokens=False)
    else:
        def token_str(t):
            s = ""
            for _ in range(4):
                s = chr(ord("a") + t % 26) + s
                t //= 26
            return " " + s
    cases = [(chat, stream, sampling, n) for chat in (True, False) for stream in (False, True)
             for sampling, n in ((dict(), 5), (dict(temperature=0.8, seed=7), 2))]
    for chat, stream, sampling, n in cases:
        eng = Engine(mini_config(manual_step=0, **CFG))
        srv = Server([eng], model="mini", vocab=512, max_model_len=1024, enable_sampling=True, enable_logprobs=True)
        if mine is not None:
            srv.set_tokenizer(mine)
        body = dict(model="mini", max_tokens=7, stream=stream, ignore_eos=True, **sampling)
        if chat:
            body.update(messages=[{"role": "user", "content": "Tell me about the fox."}], logprobs=True, top_logprobs=n)
            path = "/v1/chat/completions"
        else:
            body.update(prompt="The quick brown", logprobs=n)
            path = "/v1/completions"
        ids = srv.render_prompt(path, json.dumps(body))
        r = srv.handle("POST", "/openai" + path, json.dumps(body))
        srv.close()
        eng.close()
        assert r.status == 200, r.body
        recs = _records(ids, n, sampling)
        assert len(recs) == 7
        if stream:
            chunks = [json.loads(e) for e in r.sse_events()[:-1]]
            if chat:
                assert chunks[0]["choices"][0]["logprobs"] is None
                chunks = chunks[1:]
            assert len(chunks) == 7
            off = 0
            for k, c in enumerate(chunks):
                got = c["choices"][0]["logprobs"]
                if chat:
                    want = chat_logprobs([recs[k]], n, token_str)
                else:
                    want = completion_logprobs([recs[k]], n, token_str, off)
                    off += len(c["choices"][0]["text"])
                assert f32(got) == f32(want), (chat, k)
                _validate(c, chat, stream=True)
        else:
            j = r.json()
            got = j["choices"][0]["logprobs"]
            want = chat_logprobs(recs, n, token_str) if chat else completion_logprobs(recs, n, token_str)
            assert f32(got) == f32(want), chat
            _validate(j, chat, stream=False)
    if mine is not None:
        mine.close()


def _validate(obj, chat, stream):
    """vLLM's own pydantic response models accept the JSON, where they import."""
    try:
        if chat:
            from vllm.entrypoints.openai.chat_completion.protocol import (ChatCompletionResponse,
                                                                           ChatCompletionStreamResponse)
            (ChatCompletionStreamResponse if stream else ChatCompletionResponse).model_validate(obj)
        else:
            from vllm.entrypoints.openai.completion.protocol import CompletionResponse, CompletionStreamResponse
            (CompletionStreamResponse if stream else CompletionResponse).model_validate(obj)
    except ImportError:
        pass


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


def ulp_bf16(x):
    return np.exp2(np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -20))) - 7)


@pytest.mark.skipif(not _vllm_ok(), reason="vllm is not importable (or B200_SKIP_VLLM=1)")
def test_records_match_vllm_logprobs_on_the_test_model(tmp_path):
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
    g = torch.Generator().manual_seed(23)
    prompts = [torch.randint(0, cfg.vocab, (int(n),), generator=g).tolist() for n in (5, 17, 40, 90, 150)]
    N = 16
    ecfg = config_from_hf(tmp_path, max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=256,
                          manual_step=1, seed=777)
    mine = []
    with Engine(ecfg) as e:
        e.load_safetensors(tmp_path)
        for p in prompts:
            r = e.submit(p, max_tokens=N, logprobs=True, top_logprobs=5)
            recs = []
            while len(recs) < N:
                e.step()
                pr = e.poll_logprobs(r, 5)
                recs += list(zip(pr.tokens, pr.lp, pr.top_ids, pr.top_lp))
            rows = e.forward_logits(p + [t[0] for t in recs[:-1]])[len(p) - 1:]   # the row each token came from
            mine.append((recs, rows))
    llm = LLM(model=str(tmp_path), skip_tokenizer_init=True, dtype="bfloat16", max_model_len=256, enforce_eager=True,
              gpu_memory_utilization=0.25, enable_prefix_caching=False, seed=0)
    outs = llm.generate([{"prompt_token_ids": p} for p in prompts],
                        SamplingParams(temperature=0.0, max_tokens=N, ignore_eos=True, detokenize=False, logprobs=5))
    compared = 0
    for p, o, (recs, rows) in zip(prompts, outs, mine):
        ref = o.outputs[0]
        for k in range(N):
            if ref.token_ids[k] != recs[k][0]:
                break
            d = ref.logprobs[k]
            tok, lp, top_ids, top_lp = recs[k]
            scale = float(ulp_bf16(np.abs(rows[k]).max()))     # one bf16 ulp of the row's largest |logit|
            assert abs(lp - d[tok].logprob) <= LOGPROB_ULPS * scale, (len(p), k, lp, d[tok].logprob)
            vt = sorted(((v.rank, t, v.logprob) for t, v in d.items() if v.rank <= 5))
            vl = [x[2] for x in vt]
            for j in range(5):
                gap_ok = all(abs(vl[j] - vl[q]) > 2 * LOGPROB_ULPS * scale for q in (j - 1, j + 1) if 0 <= q < len(vl))
                if gap_ok and j < len(vt):
                    assert int(top_ids[j]) == vt[j][1], (len(p), k, j)
            compared += 1
    print(f"vLLM parity: {compared} positions compared")
    assert compared >= N
