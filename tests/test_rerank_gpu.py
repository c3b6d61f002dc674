"""Rerank on the GPU: the score_rows kernel against rmsnorm, a numpy emulation of its summation order and float64, a
score-head engine on sequence-classification checkpoints that HF transformers writes, score requests under every
scheduling path, the refusals, /v1/rerank through the serving shell and b200serve, and vLLM 0.22 parity.  The oracle is
tests/rerank_common.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from embeddings_common import hidden_rows
from kernel_numerics import norm_launch, warp_sum
from kubeai_b200 import B200Error, lib, ops
from kubeai_b200.engine import Engine, config_from_hf, mini_config
from kubeai_b200._lib import BEGIN_FN, WRITE_FN, ResponseWriter
from kubeai_b200.server import Server, tokenize
from oracle.weights import ModelCfg
from rerank_common import (activate, edit_config, llama3_tokenizer, logit_bound, rerank_body, resolve_activation,
                           score_weight, scores, write_seq_cls_checkpoint)

pytestmark = pytest.mark.gpu


def _kernel_logits(y, sw, rows):
    """score_rows_kernel's logits of one bf16 normed row y (fp32 values) in its fixed order: the block size and vectors per
    thread that rmsnorm() picks for `rows` rows; per label each thread's FMAs over its vectors i and elements j in visit
    order, the warp butterfly, then the warp sums added one after another in warp order."""
    H = y.size
    threads, vpt = norm_launch(rows, H)
    out = np.zeros(sw.shape[0], np.float32)
    for l in range(sw.shape[0]):
        acc = np.zeros(threads, np.float32)
        for i in range(vpt):
            for j in range(8):
                idx = (np.arange(threads) + i * threads) * 8 + j
                # fmaf: the product of two bf16 values is exact in fp64, so one rounding of the fp64 sum is the FMA
                acc = (acc.astype(np.float64) + y[idx].astype(np.float64) * sw[l, idx].astype(np.float64)).astype(np.float32)
        warps = [warp_sum(acc[k * 32:(k + 1) * 32]) for k in range(threads // 32)]
        t = np.float32(warps[0])
        for w in warps[1:]:
            t = np.float32(t + np.float32(w))
        out[l] = t
    return out


@pytest.mark.parametrize("H", [256, 2048, 4096, 8192])
@pytest.mark.parametrize("n", [7, 600])   # rmsnorm() and score_rows pick 256-thread CTAs of several vectors from 512 rows
def test_score_rows_matches_rmsnorm_order_emulation_and_float64(H, n):
    g = torch.Generator().manual_seed(H + n)
    hid = (torch.randn(64, H, generator=g) * 3).to(torch.bfloat16).cuda()
    hid[5] = 0
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).cuda()
    base = torch.tensor([3, 5, 0, 63, 17, 3, 40], dtype=torch.int32)
    rows = torch.cat([base, torch.randint(0, 64, (n - 7,), generator=g, dtype=torch.int32)]).cuda()
    y = ops.rmsnorm(hid, w, 1e-5, row_index=rows).float().cpu().numpy()
    for L in (1, 2, 3, 32):
        sw = (torch.randn(L, H, generator=g) / np.sqrt(H)).to(torch.bfloat16)
        swn = sw.float().numpy()
        off = torch.zeros(n, dtype=torch.int32).cuda()
        raw = ops.score_rows(hid, w, sw.cuda(), rows, off).cpu().numpy()
        # the normed rows are rmsnorm's: with L = H / 8 one-hot labels the logits would be the row itself; here, the
        # emulation of the kernel's order on rmsnorm's bf16 rows reproduces every bit
        k = min(n, 6)
        emu = np.stack([_kernel_logits(y[s], swn, n) for s in range(k)])
        assert np.array_equal(raw[:k].view(np.uint32), emu.view(np.uint32)), (L, raw[:k], emu)
        # fp32 bound from float64: H / (8 * vectors per thread) products per thread reduced through 8 * vpt + 5 + warps
        # roundings; each rounding is at most 2^-24 relative of a partial sum bounded by sum |y w|
        want = y.astype(np.float64) @ swn.astype(np.float64).T
        vpt = norm_launch(n, H)[1]
        warps = (H // 8 // vpt) // 32
        depth = 8 * vpt + 5 + warps
        bound = depth * 2.0 ** -24 * (np.abs(y).astype(np.float64) @ np.abs(swn).astype(np.float64).T) + 1e-30
        err = np.abs(raw - want)
        assert (err <= bound).all(), (L, (err / bound).max())
        print(f"score_rows H={H} rows={n} L={L}: max |logit - float64| / bound = {(err / bound).max():.3f}")
        # every activation against float64 of the kernel's own logits (IEEE expf is within 2 ulps)
        for act in (0, 1, 2, 3):
            on = torch.ones(n, dtype=torch.int32).cuda()
            got = ops.score_rows(hid, w, sw.cuda(), rows, on, activation=act).cpu().numpy()
            a = resolve_activation(L, act)
            ref = np.stack([activate(r, a) for r in raw.astype(np.float64)])
            if a == 3:
                assert np.array_equal(got.view(np.uint32), raw.view(np.uint32))
            else:
                assert np.isfinite(got).all()
                assert (np.abs(got - ref) <= 8 * np.spacing(np.abs(ref).astype(np.float32)) + 1e-37).all(), (L, act)
            # flags pick the rows that get the activation
            mixed = (torch.arange(n) % 2).to(torch.int32).cuda()
            gm = ops.score_rows(hid, w, sw.cuda(), rows, mixed, activation=act).cpu().numpy()
            assert np.array_equal(gm[0::2].view(np.uint32), raw[0::2].view(np.uint32))
            assert np.array_equal(gm[1::2].view(np.uint32), got[1::2].view(np.uint32))
    # row permutation changes no bit; zero rows launch nothing
    perm = torch.randperm(n, generator=g).cuda()
    on = torch.ones(n, dtype=torch.int32).cuda()
    a = ops.score_rows(hid, w, sw.cuda(), rows, on)
    b = ops.score_rows(hid, w, sw.cuda(), rows[perm].contiguous(), on)
    assert torch.equal(a[perm].view(torch.int32), b.view(torch.int32))
    z = ops.score_rows(hid, w, sw.cuda(), rows[:0], on[:0])
    assert z.shape == (0, 32)


def test_op_refuses_bad_shapes():
    l = lib()
    for H, L, act in [(100, 1, 0), (8448, 1, 0), (512, 0, 0), (512, 33, 0), (512, 1, 4), (512, 1, -1)]:
        assert l.b200_op_score_rows(None, None, None, None, None, 1, H, L, act, C.c_float(1e-5), None, None) == -1


# ------------------------------------------------------------------ engines on HF checkpoints
def _ec(d, **kw):
    base = dict(max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=128, manual_step=1)
    base.update(kw)
    return config_from_hf(str(d), **base)


def _check(got, cfg, ids, sw, activation=0, use_activation=True, hid=None):
    h = hid if hid is not None else hidden_rows(cfg, ids)
    x = scores(cfg, ids, sw, hid=h, use_activation=False)
    bound = logit_bound(cfg, ids, sw, hid=h)
    if not use_activation or resolve_activation(len(sw), activation) == 3:
        assert (np.abs(got - x) <= bound).all(), (got, x, bound)
        return
    a = resolve_activation(len(sw), activation)
    # sigmoid and softmax are 1/4- and 1/2-Lipschitz per logit (softmax: in the max norm, summed over the labels)
    want = activate(x, a)
    lim = (0.25 * bound) if a == 1 else 0.5 * bound.max() * len(sw) * np.ones_like(bound)
    assert (np.abs(got - want) <= lim + 1e-6).all(), (got, want, lim)


SHAPES = {"G4-D128": ModelCfg(), "G1-D128": ModelCfg(kv_heads=4), "G4-D64": ModelCfg(q_heads=8, kv_heads=2, head_dim=64)}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("tied", [False, True])
def test_engine_on_hf_seq_cls_checkpoint_matches_oracle(tmp_path, shape, tied):
    cfg = SHAPES[shape]
    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, cfg.vocab, size=n).tolist() for n in (1, 17, 200)]
    for L in (1, 3):
        d = tmp_path / f"L{L}"
        write_seq_cls_checkpoint(d, cfg, L, tie_word_embeddings=tied)
        ec = _ec(d)
        assert (ec.runner, ec.num_labels, ec.score_activation) == (1, L, 0)
        sw = score_weight(cfg, L)
        with Engine(ec) as e:
            e.load_safetensors(str(d))
            with pytest.raises(B200Error):
                e.tensor("lm_head")
            got_sw = (e.tensor("score").astype(np.uint32) << 16).view(np.float32).reshape(L, cfg.hidden)
            assert np.array_equal(got_sw, sw)
            on = e.score(prompts)
            off = e.score(prompts, use_activation=False)
        for p, a, b in zip(prompts, on, off):
            h = hidden_rows(cfg, p)
            _check(b, cfg, p, sw, use_activation=False, hid=h)
            _check(a, cfg, p, sw, hid=h)


def test_golden_is_reproduced(tmp_path):
    from pathlib import Path
    g = np.load(Path(__file__).parent / "golden" / "llama_mini_seqcls.npz")
    cfg = ModelCfg()
    ids = np.split(g["ids"], np.cumsum(g["lens"])[:-1])
    for L in (1, 3):
        write_seq_cls_checkpoint(tmp_path / f"L{L}", cfg, L)
        with Engine(_ec(tmp_path / f"L{L}")) as e:
            e.load_safetensors(str(tmp_path / f"L{L}"))
            got = e.score([p.tolist() for p in ids], use_activation=False)
        for p, x, want in zip(ids, got, g[f"logits_{L}"]):
            bound = logit_bound(cfg, p.tolist(), g[f"score_{L}"])
            assert (np.abs(x - want) <= bound + 0.05).all(), (L, x, want)


def _score_cfg(L=1, **kw):
    base = dict(runner=1, num_labels=L, max_model_len=256, max_batched_tokens=256)
    base.update(kw)
    return mini_config(**base)


LENS = [1, 15, 16, 17, 200, 256]


def test_scheduling_variations_stay_within_the_oracle_bound_and_free_pages():
    cfg = ModelCfg()
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, cfg.vocab, size=n).tolist() for n in LENS]
    hid = [hidden_rows(cfg, p) for p in prompts]
    for L in (1, 3):
        with Engine(_score_cfg(L)) as e:
            sw = (e.tensor("score").astype(np.uint32) << 16).view(np.float32).reshape(L, cfg.hidden)
            alone = np.stack([e.score([p], use_activation=False)[0] for p in prompts])
            for x, p, h in zip(alone, prompts, hid):
                _check(x, cfg, p, sw, use_activation=False, hid=h)
            assert e.stats().kv_blocks_free == e.stats().kv_blocks_total
        for budget in (256, 16, 48):   # batched, and chunked under a small budget
            with Engine(_score_cfg(L, max_batched_tokens=budget)) as e:
                xs = e.score(prompts, use_activation=False)
                for x, p, h in zip(xs, prompts, hid):
                    _check(x, cfg, p, sw, use_activation=False, hid=h)
                assert e.stats().kv_blocks_free == e.stats().kv_blocks_total
    # page pressure: 20 pages hold one 256-token prompt but not all of them at once
    with Engine(_score_cfg(1, num_kv_blocks=20, max_batched_tokens=64)) as e:
        sw = (e.tensor("score").astype(np.uint32) << 16).view(np.float32).reshape(1, cfg.hidden)
        xs = e.score(prompts, use_activation=False)
        for x, p, h in zip(xs, prompts, hid):
            _check(x, cfg, p, sw, use_activation=False, hid=h)
        assert e.stats().kv_blocks_free == e.stats().kv_blocks_total


def test_a_long_query_shared_by_many_documents_hits_the_prefix_cache():
    cfg = ModelCfg()
    rng = np.random.default_rng(8)
    query = rng.integers(0, cfg.vocab, size=130).tolist()
    docs = [rng.integers(0, cfg.vocab, size=int(n)).tolist() for n in rng.integers(1, 100, size=24)]
    pairs = [query + d for d in docs]
    with Engine(_score_cfg(1, max_num_seqs=32, num_kv_blocks=512)) as e:
        sw = (e.tensor("score").astype(np.uint32) << 16).view(np.float32).reshape(1, cfg.hidden)
        first = e.score(pairs[:1])
        before = e.stats().cached_prompt_tokens
        rest = e.score(pairs[1:])
        # every later pair reads the query's 8 full pages from the cache
        assert e.stats().cached_prompt_tokens - before == 128 * (len(pairs) - 1)
    for x, p in zip(np.concatenate([first, rest]), pairs):
        _check(x, cfg, p, sw)
    # and the same scores with the prefix cache off, within the same bound
    with Engine(_score_cfg(1, max_num_seqs=32, num_kv_blocks=512, enable_prefix_caching=0)) as e:
        cold = e.score(pairs)
        assert e.stats().cached_prompt_tokens == 0
    for x, p in zip(cold, pairs):
        _check(x, cfg, p, sw)


def test_fixed_admission_is_bit_reproducible_and_abort_frees_pages():
    rng = np.random.default_rng(9)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (30, 100, 7, 64)]
    outs = []
    for _ in range(2):
        with Engine(_score_cfg(3, max_batched_tokens=64)) as e:
            e._l.b200_engine_set_fixed_admission(e._h, 1)
            outs.append(e.score(prompts))
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))
    with Engine(_score_cfg(1, max_batched_tokens=32)) as e:
        rid = e.submit_score(prompts[1])
        e.step()
        e.abort(rid)
        e.step()
        v, fin, _ = e.poll_score(rid)
        assert v is None and fin == "aborted"
        assert e.stats().kv_blocks_free == e.stats().kv_blocks_total


def test_refusals(tmp_path):
    with Engine(_score_cfg(2)) as e:
        with pytest.raises(B200Error, match="has a score head \\(num_labels = 2\\): submit score requests with b200_submit_score"):
            e.submit_embed([1, 2, 3])
        with pytest.raises(B200Error, match="b200_submit_embed"):
            e.submit([1, 2, 3])
        with pytest.raises(B200Error, match="exceeds max_model_len"):
            e.submit_score([1] * 257)
        rid = e.submit_score([1, 2])
        vec = np.zeros(512, np.float32)
        assert e._l.b200_poll_embedding(e._h, rid, vec.ctypes.data_as(C.c_void_p), 512, C.byref(C.c_int32()), None) == -1
        assert b"is not an embedding request" in lib().b200_last_error()
        out = np.zeros(3, np.float32)
        assert e._l.b200_poll_score(e._h, rid, out.ctypes.data_as(C.c_void_p), 3, C.byref(C.c_int32()), None) == -1
        assert b"num_labels 2" in lib().b200_last_error()
        e.release(rid)
    with Engine(_score_cfg(0)) as e:
        with pytest.raises(B200Error, match="has no score head"):
            e.submit_score([1, 2, 3])
    with Engine(mini_config()) as e:
        with pytest.raises(B200Error, match="generate runner: score requests need"):
            e.submit_score([1, 2, 3])
        with pytest.raises(B200Error, match="generate runner: embedding requests need"):
            e.submit_embed([1, 2, 3])
    with pytest.raises(B200Error, match="mix heads"):
        with Engine(_score_cfg(1)) as a, Engine(_score_cfg(0)) as b:
            Server([a, b], model="m")
    with pytest.raises(B200Error, match="mix heads"):
        with Engine(_score_cfg(1)) as a, Engine(_score_cfg(2)) as b:
            Server([a, b], model="m")
    # the loader: a missing or misshapen score.weight, and a seq-cls checkpoint in a generate or embedding engine
    cfg = ModelCfg()
    write_seq_cls_checkpoint(tmp_path / "s3", cfg, 3)
    ec = _ec(tmp_path / "s3")
    ec.num_labels = 2
    with Engine(ec) as e:
        with pytest.raises(B200Error, match=r"score.weight: shape \[3,512\] != expected \[2,512\]"):
            e.load_safetensors(str(tmp_path / "s3"))
    from embeddings_common import write_base_checkpoint
    write_base_checkpoint(tmp_path / "base", cfg, "LlamaModel")
    with Engine(_score_cfg(1)) as e:
        with pytest.raises(B200Error, match=r"missing tensor score.weight: the engine has a score head of \[1, 512\]"):
            e.load_safetensors(str(tmp_path / "base"))
    for kw, what in [(dict(), "a generator"), (dict(runner=1), "an embedding model")]:
        with Engine(mini_config(**kw)) as e:
            with pytest.raises(B200Error, match=f"served by a pooling engine with num_labels > 0, not loaded as {what}"):
                e.load_safetensors(str(tmp_path / "s3"))
    with pytest.raises(B200Error, match="needs the pooling runner"):
        Engine(mini_config(num_labels=3))


def test_embedding_engine_pool_rows_outputs_are_unchanged():
    """An embedding engine's vectors are the pool_rows kernel's on the engine's own final-normed rows: the same bits as
    b200_op_pool_rows on rmsnorm of the oracle-free hidden rows is checked in test_embeddings_gpu; here the engine's step
    gives the same bits with and without a score-head engine alive beside it."""
    rng = np.random.default_rng(4)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (3, 77, 256)]
    with Engine(mini_config(runner=1)) as e:
        a = e.embed(prompts)
    with Engine(mini_config(runner=1)) as e, Engine(_score_cfg(1)) as s:
        s.score(prompts)
        b = e.embed(prompts)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ------------------------------------------------------------------ the serving shell
_LEN = ("This model's maximum context length is 256 tokens. However, you requested 0 output tokens and your prompt "
        "contains {q}{n} input tokens, for a total of {q}{n} tokens. Please reduce the length of the input prompt or the "
        "number of requested output tokens.")
_DEC = "reading model from body: decoding: json: cannot unmarshal JSON {t} into Go {g} within \"{w}\""
REFUSED = [
    ({"max_tokens_per_query": 8}, "max_tokens_per_query (per-document truncation) is not supported by this engine"),
    ({"max_tokens_per_doc": 8}, "max_tokens_per_doc (per-document truncation) is not supported by this engine"),
    ({"truncate_prompt_tokens": 8}, "truncate_prompt_tokens is not supported by this engine"),
    ({"instruction": "be nice"}, "instruction is not supported by this engine"),
    ({"chat_template_kwargs": {"a": 1}}, "chat_template_kwargs is not supported by this engine"),
    ({"priority": 1}, "priority is not supported by this engine"),
    ({"use_activation": "yes"}, "use_activation must be a boolean or null"),
    ({"add_special_tokens": 1}, "add_special_tokens must be a boolean"),
    ({"documents": []}, "documents must not be empty"),
    ({"documents": None}, "documents must not be empty"),
    ({"query": "", "documents": [""]}, "the query and document must not both be empty"),
    ({"query": "x" * 300, "documents": ["d"]}, _LEN.format(q="", n=301)),
    ({"query": "x" * 256, "documents": ["d"]}, _LEN.format(q="at least ", n=257)),
    ({"query": 1}, _DEC.format(t="number", g="string", w="/query")),
    ({"documents": "d"}, _DEC.format(t="string", g="[]string", w="/documents")),
    ({"documents": ["a", 2]}, _DEC.format(t="number", g="string", w="/documents/1")),
    ({"top_n": 1.5}, _DEC.format(t="number", g="int", w="/top_n")),
    ({"top_n": "2"}, _DEC.format(t="string", g="int", w="/top_n")),
]


def _serve(e, **kw):
    return Server([e], model="m", vocab=512, max_model_len=256, **kw)


def _body(s, body):
    r = s.handle("POST", "/openai/v1/rerank", json.dumps(dict(model="m", **body)))
    return r


def test_server_rerank_bodies_equal_the_oracle_builder():
    cfg = ModelCfg()
    docs = ["Paris is the capital of France.", "berlin", "x", "Paris is the capital of France.", "ok then " * 5]
    q = "What is the capital of France?"
    with Engine(_score_cfg(1, manual_step=0)) as e, _serve(e) as s:
        # the engine's scores of the same ids, submitted directly
        ids = [tokenize(q, vocab=512) + tokenize(d, vocab=512) for d in docs]
        rids = [e.submit_score(p) for p in ids]
        direct = []
        for r in rids:
            while True:
                e.wait(r, 1.0)
                v, fin, _ = e.poll_score(r)
                if fin is not None:
                    break
            direct.append(v[0])
            e.release(r)
        direct = np.array(direct, np.float32)
        ntok = sum(map(len, ids))
        for top_n in (None, 0, -3, 1, 2, 4, 5, 9):
            body = {"query": q, "documents": docs} if top_n is None else {"query": q, "documents": docs, "top_n": top_n}
            r = _body(s, body)
            assert r.status == 200, r.body
            j = r.json()
            assert j.pop("id").startswith("score-")
            assert j == rerank_body("m", docs, direct, ntok, top_n or 0), top_n
            # the printed score reads back as the engine's fp32 to the bit
            got = np.array([x["relevance_score"] for x in j["results"]], np.float32)
            assert np.array_equal(got.view(np.uint32), direct[[x["index"] for x in j["results"]]].view(np.uint32))
        # the same body twice gives the same bytes but the id
        a, b = _body(s, {"query": q, "documents": docs}).json(), _body(s, {"query": q, "documents": docs}).json()
        a.pop("id"), b.pop("id")
        assert a == b
        # ties: docs 0 and 3 are one text, so one score; the earlier document comes first
        res = _body(s, {"query": q, "documents": docs}).json()["results"]
        order = [x["index"] for x in res]
        assert order.index(0) + 1 == order.index(3) or direct[0] != direct[3]
        # use_activation false gives the raw logits
        raw = _body(s, {"query": q, "documents": docs, "use_activation": False}).json()
        rv = {x["index"]: x["relevance_score"] for x in raw["results"]}
        for i, v in rv.items():
            assert abs(1 / (1 + np.exp(-v)) - direct[i]) < 1e-6
        for body in ({"use_activation": None}, {"add_special_tokens": True}, {"add_special_tokens": False},
                     {"max_tokens_per_doc": 0, "max_tokens_per_query": 0, "priority": None, "instruction": None}):
            r = _body(s, dict(query=q, documents=docs, **body)).json()
            r.pop("id")
            assert r == rerank_body("m", docs, direct, ntok), body
        # routes of a score-head server
        m = s.handle("GET", "/openai/v1/models").json()
        assert m["data"][0]["features"] == ["Reranking"]
        for path, body in [("/v1/completions", '{"model":"m","prompt":"x"}'), ("/v1/chat/completions", '{"model":"m"}'),
                           ("/v1/embeddings", '{"model":"m","input":"x"}')]:
            c = s.handle("POST", "/openai" + path, body)
            assert (c.status, c.json()) == (404, {"error": "model not found: this engine serves Reranking only"})
        # ParseRequest accepts the path here: the model / adapter split, no prefix
        st, pr = s.parse_request("/v1/rerank", '{"model":"m","query":"abc","documents":["d"]}', prefix_chars=2)
        assert st == 0 and (pr["model"], pr["adapter"], pr["prefix"]) == ("m", "", "")
        st, pr = s.parse_request("/v1/rerank", '{"model":"other","query":"abc","documents":["d"]}')
        assert (st, pr["error"]) == (404, 'model not found: "other"')
        for body, msg in REFUSED:
            full = {"query": q, "documents": docs}
            full.update(body)
            b = _body(s, full)
            assert (b.status, b.body) == (400, json.dumps({"error": "bad request: " + msg}, separators=(",", ":"),
                                                          ensure_ascii=False).encode() + b"\n"), body
        # a replica failure before anything was sent retries the whole request
        s._l.b200_server_inject_fault(s._h, 0, 1)
        rr = _body(s, {"query": q, "documents": docs})
        assert rr.status == 200 and "b200_request_retries_total 1" in s.metrics()
        # a client that went away is noticed at the response write: 499, and its requests are released
        body = json.dumps({"model": "m", "query": q, "documents": docs}).encode()
        w = ResponseWriter(None, BEGIN_FN(lambda _u, st, ct: 0), WRITE_FN(lambda _u, d, n: 1))
        assert s._l.b200_server_handle(s._h, b"POST", b"/openai/v1/rerank", b"application/json", body, len(body),
                                       C.byref(w)) == 499
        assert e._l.b200_engine_unfinished(e._h) == 0
        st = e.stats()
        assert st.running == 0 and st.kv_blocks_free == st.kv_blocks_total
    # an embedding server keeps its 404 on /v1/rerank and ParseRequest's 400; several labels get vLLM's scalar message
    with Engine(mini_config(runner=1, manual_step=0)) as e, _serve(e) as s:
        r = _body(s, {"query": q, "documents": docs})
        assert (r.status, r.body) == (404, b'{"error":"model not found: this engine serves TextEmbedding only"}\n')
        st, pr = s.parse_request("/v1/rerank", '{"model":"m","query":"q","documents":["d"]}')
        assert (st, pr["error"]) == (400, 'bad request: reading model from body: unknown path: "/v1/rerank"')
    with Engine(_score_cfg(3, manual_step=0)) as e, _serve(e) as s:
        r = _body(s, {"query": q, "documents": docs})
        assert r.status == 400 and "pooled_data should be a scalar score" in r.json()["error"]


def test_server_tokenizes_pairs_with_the_checkpoint_template(tmp_path):
    from kubeai_b200.tokenizer import Tokenizer
    hf = llama3_tokenizer(tmp_path / "tokenizer.json", "llama3", vocab_size=500)
    q, docs = "What is the capital of France?", ["Paris is the capital.", "The quick brown fox"]
    with Tokenizer(tmp_path / "tokenizer.json") as tok:
        for join in (0, 1):
            with Engine(_score_cfg(1, manual_step=0, score_join_pair=join)) as e, _serve(e) as s:
                s.set_tokenizer(tok)
                ids = [hf.encode(q + d).ids if join else hf.encode(q, d).ids for d in docs]
                want = [None] * len(ids)
                rids = [e.submit_score(p) for p in ids]
                for i, r in enumerate(rids):
                    while True:
                        e.wait(r, 1.0)
                        v, fin, _ = e.poll_score(r)
                        if fin is not None:
                            break
                    want[i] = v[0]
                    e.release(r)
                j = _body(s, {"query": q, "documents": docs}).json()
                j.pop("id")
                assert j == rerank_body("m", docs, np.array(want, np.float32), sum(map(len, ids))), join


def test_b200serve_model_dir_on_a_seq_cls_checkpoint(tmp_path):
    import socket
    import subprocess
    import time
    import urllib.request
    from pathlib import Path
    cfg = ModelCfg()
    write_seq_cls_checkpoint(tmp_path, cfg, 1)
    binp = Path(__file__).resolve().parent.parent / "kubeai_b200" / "bin" / "b200serve"
    for extra in ([], ["--runner", "pooling"]):
        with socket.socket() as so:
            so.bind(("127.0.0.1", 0))
            port = so.getsockname()[1]
        proc = subprocess.Popen([str(binp), "--gpus", "1", "--model", "m", "--model-dir", str(tmp_path), "--port", str(port),
                                 "--host", "127.0.0.1", "--max-model-len", "256", "--max-num-seqs", "16",
                                 "--max-num-batched-tokens", "256", *extra], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        try:
            base = f"http://127.0.0.1:{port}/openai/v1"
            for _ in range(300):
                try:
                    models = json.loads(urllib.request.urlopen(base + "/models", timeout=2).read())
                    break
                except Exception:
                    assert proc.poll() is None, proc.stdout.read().decode()
                    time.sleep(0.2)
            assert models["data"][0]["features"] == ["Reranking"]
            req = urllib.request.Request(base + "/rerank", data=json.dumps(
                {"model": "m", "query": "abc", "documents": ["d e f", "g"]}).encode(), headers={"Content-Type": "application/json"})
            j = json.loads(urllib.request.urlopen(req, timeout=60).read())
            assert sorted(r["index"] for r in j["results"]) == [0, 1]
            sw = score_weight(cfg, 1)
            for r in j["results"]:
                d = ["d e f", "g"][r["index"]]
                ids = tokenize("abc", vocab=512) + tokenize(d, vocab=512)
                _check(np.array([r["relevance_score"]]), cfg, ids, sw)
        finally:
            proc.terminate()
            proc.wait(timeout=30)
    # the generate runner is refused for a score head, never loaded as a generator
    r = subprocess.run([str(binp), "--gpus", "1", "--model", "m", "--model-dir", str(tmp_path), "--runner", "generate",
                        "--max-model-len", "256"], capture_output=True, text=True, timeout=120)
    assert r.returncode != 0 and "needs the pooling runner" in r.stderr


# ------------------------------------------------------------------ vLLM parity (2-layer test model)
def _vllm_ok():
    if os.environ.get("B200_SKIP_VLLM") == "1":
        return False
    try:
        import vllm  # noqa: F401
        return True
    except Exception:
        return False


@pytest.mark.skipif(not _vllm_ok(), reason="vllm is not importable (or B200_SKIP_VLLM=1)")
def test_rerank_matches_vllm_pooling_runner_on_the_test_model(tmp_path):
    """vLLM 0.22 with runner="pooling" in bf16 reranks the same (query, document) pairs on the same
    LlamaForSequenceClassification checkpoint and tokenizer.json: every relevance_score within 0.01 of the engine's, and
    the same order wherever vLLM's neighbouring scores differ by more than 0.01."""
    os.environ.setdefault("HF_HUB_OFFLINE", "1")
    os.environ.setdefault("VLLM_NO_USAGE_STATS", "1")
    from transformers import PreTrainedTokenizerFast
    from vllm import LLM
    from kubeai_b200.tokenizer import Tokenizer
    cfg = ModelCfg()
    write_seq_cls_checkpoint(tmp_path, cfg, 1)
    hf = llama3_tokenizer(tmp_path / "tokenizer.json", "llama3", vocab_size=cfg.vocab)
    PreTrainedTokenizerFast(tokenizer_object=hf, bos_token="<|begin_of_text|>", eos_token="<|end_of_text|>",
                            pad_token="<|end_of_text|>").save_pretrained(str(tmp_path))
    edit_config(tmp_path, pad_token_id=hf.token_to_id("<|end_of_text|>"))
    q = "What is the capital of France?"
    docs = ["Paris is the capital and largest city of France.", "The quick brown fox jumps over the lazy dog.",
            "naïve café déjà vu", "Reranking scores a query against each document.", "12345 67 890", "France", "?"]
    ec = _ec(tmp_path, manual_step=0)
    with Engine(ec) as e, _serve(e) as s, Tokenizer(tmp_path / "tokenizer.json") as tok:
        e.load_safetensors(str(tmp_path))
        s.set_tokenizer(tok)
        mine = s.handle("POST", "/openai/v1/rerank", json.dumps({"model": "m", "query": q, "documents": docs})).json()
    llm = LLM(model=str(tmp_path), runner="pooling", dtype="bfloat16", max_model_len=256, enforce_eager=True,
              gpu_memory_utilization=0.25, enable_prefix_caching=False, seed=0)
    outs = llm.score(q, docs, use_tqdm=False)
    theirs = np.array([o.outputs.score for o in outs], np.float64)
    got = np.zeros(len(docs))
    for r in mine["results"]:
        got[r["index"]] = r["relevance_score"]
    delta = np.abs(got - theirs)
    print(f"vLLM rerank parity: {len(docs)} documents, max |delta relevance_score| {delta.max():.6f}")
    assert delta.max() <= 0.01, (got, theirs)
    vo = np.argsort(-theirs, kind="stable")
    mo = [r["index"] for r in mine["results"]]
    for a, b in zip(vo, vo[1:]):
        if theirs[a] - theirs[b] > 0.01:
            assert mo.index(a) < mo.index(b), (mo, list(vo))
