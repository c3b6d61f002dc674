"""Embeddings on the GPU: the pool_rows kernel against rmsnorm and a float64 normalisation, a pooling engine on base-model
checkpoints that HF transformers writes, embedding requests under every scheduling path, the refusals, and /v1/embeddings
through the serving shell.  The oracle is tests/embeddings_common.py."""
import base64
import ctypes as C
import json

import numpy as np
import pytest
import torch

from embeddings_common import hidden_rows, pool, write_base_checkpoint, write_word_tokenizer
from kernel_numerics import norm_launch, warp_sum
from kubeai_b200 import B200Error, lib
from kubeai_b200.engine import Engine, config_from_hf, mini_config
from kubeai_b200._lib import BEGIN_FN, WRITE_FN, ResponseWriter
from kubeai_b200.server import Server, tokenize
from oracle.weights import ModelCfg

pytestmark = pytest.mark.gpu

# DESIGN §2: bf16 kernels against the bf16-rounding oracle
ATOL, RTOL = 0.15, 1.6e-2


def _p(t):
    return C.c_void_p(t.data_ptr())


def _ulp(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def _kernel_normalize(y, rows):
    """pool_rows_kernel's normalisation of one bf16 row y (fp32 values) in its fixed order: the block size and vectors per
    thread that rmsnorm() picks for `rows` rows, each thread's squares summed in visit order (a bf16 square is exact in
    fp32, so the kernel's FMA is one rounded add), the warp butterflies, then the warp sums in warp order; IEEE sqrt and
    division."""
    H = y.size
    threads, vpt = norm_launch(rows, H)
    acc = np.zeros(threads, np.float32)
    for i in range(vpt):
        for j in range(8):
            idx = (np.arange(threads) + i * threads) * 8 + j
            acc = (acc + (y[idx] * y[idx]).astype(np.float32)).astype(np.float32)
    warps = np.array([warp_sum(acc[k * 32:(k + 1) * 32]) for k in range(threads // 32)], np.float32)
    ss = warp_sum(np.concatenate([warps, np.zeros(32 - warps.size, np.float32)]))
    return (y / np.maximum(np.sqrt(np.float32(ss)), np.float32(1e-12))).astype(np.float32)


@pytest.mark.parametrize("H", [256, 2048, 4096, 8192])
@pytest.mark.parametrize("n", [7, 600])   # rmsnorm() and pool_rows pick 256-thread CTAs of several vectors from 512 rows
def test_pool_rows_matches_rmsnorm_and_float64_normalize(H, n):
    l = lib()
    g = torch.Generator().manual_seed(H)
    hid = (torch.randn(64, H, generator=g) * 3).to(torch.bfloat16).cuda()
    hid[5] = 0   # a zero row normalises to 0, not NaN
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).cuda()
    base = torch.tensor([3, 5, 0, 63, 17, 3, 40], dtype=torch.int32)
    rows = torch.cat([base, torch.randint(0, 64, (n - 7,), generator=g, dtype=torch.int32)]).cuda()
    ref = torch.empty(n, H, dtype=torch.bfloat16).cuda()
    assert l.b200_op_rmsnorm(_p(hid), None, _p(w), _p(ref), _p(rows), n, H, C.c_float(1e-5), None) == 0
    for flag in (0, 1):
        flags = torch.full((n,), flag, dtype=torch.int32).cuda()
        out = torch.empty(n, H, dtype=torch.float32).cuda()
        assert l.b200_op_pool_rows(_p(hid), _p(w), _p(rows), _p(flags), n, H, C.c_float(1e-5), _p(out), None) == 0
        torch.cuda.synchronize()
        o = out.cpu().numpy()
        y = ref.float().cpu().numpy()
        if not flag:
            assert np.array_equal(o.view(np.uint32), y.view(np.uint32))   # the fp32 of the bf16 normed rows, bit for bit
            continue
        assert np.isfinite(o).all() and (o[1] == 0).all()
        # bit for bit the kernel's fixed order, emulated in numpy fp32 (a multiply by a reciprocal, rsqrtf, another
        # reduction order or squares of unrounded values would each move bits here) ...
        emu = np.stack([_kernel_normalize(y[s], n) for s in range(min(n, 12))])
        assert np.array_equal(o[:len(emu)].view(np.uint32), emu.view(np.uint32))
        # ... and within the bound of that order from float64: a sum of squares through d = 8 * vectors per thread + 10
        # roundings (the thread's adds, then 5 butterfly levels twice) is off by at most d * 2^-24 relative, the square
        # root halves that, and sqrt and the division add half an ulp each
        yd = y.astype(np.float64)
        want = yd / np.maximum(np.linalg.norm(yd, axis=1, keepdims=True), 1e-12)
        vpt = norm_launch(n, H)[1]
        u = _ulp(want.astype(np.float32))
        bound = 0.5 * (8 * vpt + 10) * 2.0 ** -24 * np.abs(want) + u
        assert (np.abs(o - want) <= bound).all()
        ulps = np.abs(o - want) / np.maximum(u, 2.0 ** -149)
        print(f"pool_rows H={H} rows={n}: at most {ulps.max():.2f} fp32 ulps from float64 (bound "
              f"{(bound / np.maximum(u, 2.0 ** -149)).max():.2f})")
    # row order: a permutation of the rows permutes the outputs and changes no bit
    perm = torch.randperm(n, generator=g).cuda()
    flags = torch.ones(n, dtype=torch.int32).cuda()
    a = torch.empty(n, H, dtype=torch.float32).cuda()
    b = torch.empty(n, H, dtype=torch.float32).cuda()
    l.b200_op_pool_rows(_p(hid), _p(w), _p(rows), _p(flags), n, H, C.c_float(1e-5), _p(a), None)
    rp = rows[perm].contiguous()
    l.b200_op_pool_rows(_p(hid), _p(w), _p(rp), _p(flags), n, H, C.c_float(1e-5), _p(b), None)
    torch.cuda.synchronize()
    assert torch.equal(a[perm].view(torch.int32), b.view(torch.int32))


def _pool_cfg(**kw):
    base = dict(runner=1, max_model_len=256, max_batched_tokens=256)
    base.update(kw)
    return mini_config(**base)


def _check(v, ids, cfg, normalize=True, hid=None):
    h = hid if hid is not None else hidden_rows(cfg, ids)
    want = pool(h[-1], normalize)
    if normalize:
        assert abs(np.linalg.norm(v.astype(np.float64)) - 1) <= 1e-6
        cos = float(v.astype(np.float64) @ want / np.linalg.norm(v.astype(np.float64)))
        assert cos >= 0.9999, cos
    else:
        err = np.abs(v - want)
        assert (err <= ATOL + RTOL * np.abs(want)).all(), err.max()


@pytest.mark.parametrize("arch", ["MistralModel", "LlamaModel"])
@pytest.mark.parametrize("dtype,shards", [(torch.bfloat16, 1), (torch.float32, 3)])
def test_engine_on_hf_base_checkpoint_matches_oracle(tmp_path, arch, dtype, shards):
    cfg = ModelCfg()
    write_base_checkpoint(tmp_path, cfg, arch, dtype, shards)
    ec = config_from_hf(str(tmp_path), max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=128,
                        manual_step=1)
    assert ec.runner == 1 and ec.sliding_window == (256 if arch == "MistralModel" else 0)
    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, cfg.vocab, size=n).tolist() for n in (1, 17, 200)]
    with Engine(ec) as e:
        e.load_safetensors(str(tmp_path))
        with pytest.raises(B200Error):
            e.tensor("lm_head")
        vn = e.embed(prompts, normalize=True)
        vr = e.embed(prompts, normalize=False)
    for p, a, b in zip(prompts, vn, vr):
        h = hidden_rows(cfg, p)
        _check(a, p, cfg, True, h)
        _check(b, p, cfg, False, h)


def test_golden_is_reproduced(tmp_path):
    from pathlib import Path
    g = np.load(Path(__file__).parent / "golden" / "mistral_mini_embed.npz")
    cfg = ModelCfg()
    write_base_checkpoint(tmp_path, cfg, "MistralModel", torch.bfloat16, 1)
    ec = config_from_hf(str(tmp_path), max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=128,
                        manual_step=1)
    with Engine(ec) as e:
        e.load_safetensors(str(tmp_path))
        v = e.embed([g["ids"].tolist()])[0]
    want = g["embed_fp32"].astype(np.float64)
    assert float(v.astype(np.float64) @ want) >= 0.9999


LENS = [1, 15, 16, 17, 200, 256]


def test_scheduling_variations_stay_within_tolerance_and_free_pages():
    cfg = ModelCfg()
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, cfg.vocab, size=n).tolist() for n in LENS]
    hid = [hidden_rows(cfg, p) for p in prompts]
    # alone
    with Engine(_pool_cfg()) as e:
        for p, h in zip(prompts, hid):
            _check(e.embed([p])[0], p, cfg, True, h)
        assert e.stats().kv_blocks_free == e.stats().kv_blocks_total
        # prefix-cache hit: the same prompts again read their cached pages (a hit covers at most len - 1 tokens)
        before = e.stats().cached_prompt_tokens
        for p, h in zip(prompts, hid):
            _check(e.embed([p])[0], p, cfg, True, h)
        assert e.stats().cached_prompt_tokens > before
    # batched, and chunked under a small budget
    for budget in (256, 16, 48):
        with Engine(_pool_cfg(max_batched_tokens=budget)) as e:
            vs = e.embed(prompts)
            for v, p, h in zip(vs, prompts, hid):
                _check(v, p, cfg, True, h)
            assert e.stats().kv_blocks_free == e.stats().kv_blocks_total
    # a pool of 20 pages holds one 256-token prompt (16 pages) but not all of them at once: admission waits for pages.
    # (Only the oldest running prompt takes a whole-budget chunk, so embedding requests alone never preempt each other.)
    with Engine(_pool_cfg(num_kv_blocks=20, max_batched_tokens=64)) as e:
        vs = e.embed(prompts)
        for v, p, h in zip(vs, prompts, hid):
            _check(v, p, cfg, True, h)
        assert e.stats().kv_blocks_free == e.stats().kv_blocks_total


def test_fixed_admission_schedule_is_bit_reproducible_and_abort_frees_pages():
    rng = np.random.default_rng(9)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (30, 100, 7, 64)]
    outs = []
    for _ in range(2):
        with Engine(_pool_cfg(max_batched_tokens=64)) as e:
            e._l.b200_engine_set_fixed_admission(e._h, 1)
            outs.append(e.embed(prompts))
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))
    with Engine(_pool_cfg(max_batched_tokens=32)) as e:
        rid = e.submit_embed(prompts[1])
        e.step()
        e.abort(rid)
        e.step()
        v, fin, _ = e.poll_embedding(rid)
        assert v is None and fin == "aborted"
        assert e.stats().kv_blocks_free == e.stats().kv_blocks_total


def test_refusals():
    with Engine(_pool_cfg()) as e:
        with pytest.raises(B200Error, match="b200_submit_embed"):
            e.submit([1, 2, 3])
        with pytest.raises(B200Error):
            e.submit_embed([1] * 257)
        rid = e.submit_embed([1] * 256)
        e.embed([[2, 3]])
        e.release(rid)
    with Engine(mini_config()) as e:
        with pytest.raises(B200Error, match="runner = pooling"):
            e.submit_embed([1, 2, 3])
    with pytest.raises(B200Error, match="max_model_len 256 exceeds sliding_window 128"):
        Engine(_pool_cfg(sliding_window=128))
    with pytest.raises(B200Error, match="speculative"):
        Engine(_pool_cfg(num_speculative_tokens=1))
    with pytest.raises(B200Error, match="mix"):
        with Engine(_pool_cfg()) as a, Engine(mini_config()) as b:
            Server([a, b], model="m")


_LEN = ("This model's maximum context length is 256 tokens. However, you requested 0 output tokens and your prompt "
        "contains {q}{n} input tokens, for a total of {q}{n} tokens. Please reduce the length of the input prompt or the "
        "number of requested output tokens.")
_SHAPE = "input must be a string, a list of strings, a list of token ids or a list of token id lists"
# every refused field of /v1/embeddings with its exact message (after "bad request: ")
REFUSED = [
    ({"input": [1], "dimensions": 8}, 'Model "m" does not support matryoshka representation, changing output dimensions '
                                      'will lead to poor results.'),
    ({"input": [1], "embed_dtype": "float16"}, "embed_dtype other than float32 is not supported by this engine"),
    ({"input": [1], "embed_dtype": "bfloat16"}, "embed_dtype other than float32 is not supported by this engine"),
    ({"input": [1], "endianness": "big"}, "endianness other than native or little is not supported by this engine"),
    ({"input": [1], "truncate_prompt_tokens": 8}, "truncate_prompt_tokens is not supported by this engine"),
    ({"input": [1], "truncate_prompt_tokens": -1}, "truncate_prompt_tokens is not supported by this engine"),
    ({"messages": [{"role": "user", "content": "hi"}]}, "chat-form embeddings (messages) are not supported by this engine"),
    ({"input": [1], "encoding_format": "bytes"}, 'encoding_format must be "float" or "base64"'),
    ({"input": [1], "encoding_format": 1}, 'encoding_format must be "float" or "base64"'),
    ({"input": [1], "use_activation": "yes"}, "use_activation must be a boolean or null"),
    ({"input": [1], "use_activation": 1}, "use_activation must be a boolean or null"),
    ({"input": "x", "add_special_tokens": "no"}, "add_special_tokens must be a boolean"),
    ({}, "input is required"),
    ({"input": None}, "input is required"),
    ({"input": 7}, _SHAPE),
    ({"input": {"a": 1}}, _SHAPE),
    ({"input": ["a", 1]}, _SHAPE),
    ({"input": [1, "a"]}, _SHAPE),
    ({"input": [[1], 2]}, _SHAPE),
    ({"input": [True]}, _SHAPE),
    ({"input": []}, "input must not be empty"),
    ({"input": ""}, "input must not be empty"),
    ({"input": [[1], []]}, "input must not be empty"),
    ({"input": [512]}, "token ids must be integers in [0, 512)"),
    ({"input": [-1]}, "token ids must be integers in [0, 512)"),
    ({"input": [1.5]}, "token ids must be integers in [0, 512)"),
    ({"input": [[1], [2, 600]]}, "token ids must be integers in [0, 512)"),
    ({"input": [1] * 257}, _LEN.format(q="at least ", n=257)),
    ({"input": [1] * 300}, _LEN.format(q="", n=300)),
    ({"input": [[1], [2] * 258]}, _LEN.format(q="", n=258)),
]


def _serve(e, **kw):
    return Server([e], model="m", vocab=512, max_model_len=256, **kw)


def test_server_embeddings_float_base64_order_usage_and_retry():
    cfg = ModelCfg()
    rng = np.random.default_rng(2)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (5, 40, 1)]
    with Engine(_pool_cfg(manual_step=0)) as e, _serve(e) as s:
        r = s.handle("POST", "/openai/v1/embeddings", json.dumps({"model": "m", "input": prompts}))
        assert r.status == 200, r.body
        j = r.json()
        assert j["object"] == "list" and j["id"].startswith("embd-") and j["model"] == "m"
        assert j["usage"] == {"prompt_tokens": 46, "total_tokens": 46, "completion_tokens": 0, "prompt_tokens_details": None}
        assert [d["index"] for d in j["data"]] == [0, 1, 2] and all(d["object"] == "embedding" for d in j["data"])
        vj = np.array([d["embedding"] for d in j["data"]], dtype=np.float64).astype(np.float32)
        for v, p in zip(vj, prompts):
            _check(v, p, cfg)
        # the JSON floats are the exact fp32 values; base64 carries the same bits
        r64 = s.handle("POST", "/openai/v1/embeddings", json.dumps({"model": "m", "input": prompts, "encoding_format": "base64"}))
        vb = np.stack([np.frombuffer(base64.b64decode(d["embedding"]), "<f4") for d in r64.json()["data"]])
        assert np.array_equal(vb.view(np.uint32), vj.view(np.uint32))
        one = s.handle("POST", "/openai/v1/embeddings", json.dumps({"model": "m", "input": prompts[1], "use_activation": False}))
        _check(np.array(one.json()["data"][0]["embedding"], dtype=np.float32), prompts[1], cfg, normalize=False)
        # a replica failure before anything was sent retries the whole request
        s._l.b200_server_inject_fault(s._h, 0, 1)
        rr = s.handle("POST", "/openai/v1/embeddings", json.dumps({"model": "m", "input": prompts}))
        assert rr.status == 200 and "b200_request_retries_total 1" in s.metrics()
        vr = np.array([d["embedding"] for d in rr.json()["data"]], dtype=np.float32)
        assert np.array_equal(vr.view(np.uint32), vj.view(np.uint32))
        # routes and refusals of a pooling server
        m = s.handle("GET", "/openai/v1/models").json()
        assert m["data"][0]["features"] == ["TextEmbedding"]
        c = s.handle("POST", "/openai/v1/completions", '{"model":"m","prompt":"x"}')
        assert (c.status, c.json()) == (404, {"error": "model not found: this engine serves TextEmbedding only"})
        for body, msg in REFUSED:
            b = s.handle("POST", "/openai/v1/embeddings", json.dumps(dict(model="m", **body)))
            assert (b.status, b.body) == (400, json.dumps({"error": "bad request: " + msg}, separators=(",", ":"),
                                                          ensure_ascii=False).encode() + b"\n"), body
        # text inputs go through the (synthetic) tokenizer: the vectors are those of the same ids given as ids
        texts = ["hello world", " abcd efgh!", "x"]
        ids = [tokenize(x, vocab=512) for x in texts]
        want = np.array([d["embedding"] for d in s.handle("POST", "/openai/v1/embeddings", json.dumps(
            {"model": "m", "input": ids})).json()["data"]], dtype=np.float32)
        for body in ({"input": texts}, {"input": texts, "add_special_tokens": False}, {"input": texts, "use_activation": None},
                     {"input": texts, "encoding_format": "float", "embed_dtype": "float32", "endianness": "little"}):
            got = s.handle("POST", "/openai/v1/embeddings", json.dumps(dict(model="m", **body)))
            assert got.status == 200, got.body
            gv = np.array([d["embedding"] for d in got.json()["data"]], dtype=np.float32)
            assert np.array_equal(gv.view(np.uint32), want.view(np.uint32)), body
            assert got.json()["usage"]["prompt_tokens"] == sum(map(len, ids))
        one = s.handle("POST", "/openai/v1/embeddings", json.dumps({"model": "m", "input": texts[0]})).json()
        assert len(one["data"]) == 1 and np.array_equal(np.array(one["data"][0]["embedding"], np.float32).view(np.uint32),
                                                        want[0].view(np.uint32))
        # a client that went away is noticed when the response is written (one write at the end): 499, and its
        # requests are released
        body = json.dumps({"model": "m", "input": prompts}).encode()
        w = ResponseWriter(None, BEGIN_FN(lambda _u, st, ct: 0), WRITE_FN(lambda _u, d, n: 1))   # every write fails
        assert s._l.b200_server_handle(s._h, b"POST", b"/openai/v1/embeddings", b"application/json", body, len(body),
                                       C.byref(w)) == 499
        assert e._l.b200_engine_unfinished(e._h) == 0
        st = e.stats()
        assert st.running == 0 and st.kv_blocks_free == st.kv_blocks_total


def test_b200serve_model_dir_on_mistral_model(tmp_path):
    import os
    import socket
    import subprocess
    import time
    import urllib.request
    from pathlib import Path
    cfg = ModelCfg()
    write_base_checkpoint(tmp_path, cfg, "MistralModel", torch.bfloat16, 1)
    binp = Path(__file__).resolve().parent.parent / "kubeai_b200" / "bin" / "b200serve"
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    proc = subprocess.Popen([str(binp), "--gpus", "1", "--model", "m", "--model-dir", str(tmp_path), "--port", str(port),
                             "--host", "127.0.0.1", "--max-model-len", "256", "--max-num-seqs", "16",
                             "--max-num-batched-tokens", "256"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    try:
        base = f"http://127.0.0.1:{port}/openai/v1"
        for _ in range(300):
            try:
                models = json.loads(urllib.request.urlopen(base + "/models", timeout=2).read())
                break
            except Exception:
                assert proc.poll() is None, proc.stdout.read().decode()
                time.sleep(0.2)
        assert models["data"][0]["features"] == ["TextEmbedding"]
        req = urllib.request.Request(base + "/embeddings", data=json.dumps({"model": "m", "input": [[1, 2, 3, 4]]}).encode(),
                                     headers={"Content-Type": "application/json"})
        j = json.loads(urllib.request.urlopen(req, timeout=60).read())
        _check(np.array(j["data"][0]["embedding"], dtype=np.float32), [1, 2, 3, 4], cfg)
    finally:
        proc.terminate()
        proc.wait(timeout=30)


def test_mistral_for_causal_lm_gives_the_llama_logits(tmp_path):
    from oracle.gen_golden import hf_model
    from oracle.weights import make_weights
    cfg = ModelCfg()
    m = hf_model(cfg, make_weights(cfg), torch.bfloat16)
    m.save_pretrained(str(tmp_path / "llama"))
    mc = json.loads((tmp_path / "llama" / "config.json").read_text())
    (tmp_path / "mistral").mkdir()
    for f in (tmp_path / "llama").iterdir():
        if f.name != "config.json":
            (tmp_path / "mistral" / f.name).symlink_to(f)
    mc.update(architectures=["MistralForCausalLM"], model_type="mistral", sliding_window=None)
    (tmp_path / "mistral" / "config.json").write_text(json.dumps(mc))
    ids = list(range(1, 60))
    outs = []
    for d in ("llama", "mistral"):
        ec = config_from_hf(str(tmp_path / d), max_model_len=256, max_num_seqs=16, max_batched_tokens=256,
                            num_kv_blocks=128, manual_step=1)
        assert ec.runner == 0
        with Engine(ec) as e:
            e.load_safetensors(str(tmp_path / d))
            outs.append(e.forward_logits(ids))
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))


# ------------------------------------------------------------------ vLLM parity (2-layer test model)
def _vllm_ok():
    import os
    if os.environ.get("B200_SKIP_VLLM") == "1":
        return False
    try:
        import vllm  # noqa: F401
        return True
    except Exception:
        return False


@pytest.mark.skipif(not _vllm_ok(), reason="vllm is not importable (or B200_SKIP_VLLM=1)")
def test_embeddings_match_vllm_pooling_runner_on_the_test_model(tmp_path):
    """vLLM 0.22 with runner="pooling" in bf16 embeds the same token-id prompts on the same MistralModel checkpoint (last
    token, normalised): the cosine of every vector to the engine's is at least 0.999."""
    import os
    os.environ.setdefault("HF_HUB_OFFLINE", "1")
    os.environ.setdefault("VLLM_NO_USAGE_STATS", "1")
    from vllm import LLM
    from vllm.config import PoolerConfig
    cfg = ModelCfg()
    write_base_checkpoint(tmp_path, cfg, "MistralModel", torch.bfloat16, 1)
    write_word_tokenizer(tmp_path, cfg.vocab)   # vLLM's pooling entry point builds its IO processors from a tokenizer
    g = torch.Generator().manual_seed(31)
    prompts = [torch.randint(0, cfg.vocab, (int(n),), generator=g).tolist() for n in (1, 5, 17, 40, 90, 150, 256)]
    ec = config_from_hf(str(tmp_path), max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=128,
                        manual_step=1)
    with Engine(ec) as e:
        e.load_safetensors(str(tmp_path))
        mine = e.embed(prompts)
    llm = LLM(model=str(tmp_path), runner="pooling", dtype="bfloat16", max_model_len=256,
              enforce_eager=True, gpu_memory_utilization=0.25, enable_prefix_caching=False, seed=0,
              pooler_config=PoolerConfig(seq_pooling_type="LAST", use_activation=True))
    outs = llm.embed([{"prompt_token_ids": p} for p in prompts], use_tqdm=False)
    cos = []
    for p, o, v in zip(prompts, outs, mine):
        r = np.asarray(o.outputs.embedding, dtype=np.float64)
        assert r.shape == (cfg.hidden,) and abs(np.linalg.norm(r) - 1) < 1e-3
        cos.append(float(r @ v.astype(np.float64) / (np.linalg.norm(r) * np.linalg.norm(v.astype(np.float64)))))
    print(f"vLLM pooling-runner parity: {len(cos)} prompts, minimum cosine {min(cos):.6f}")
    assert min(cos) >= 0.999, cos
