"""Logits edits on the GPU: b200_op_penalize bit for bit against the oracle (oracle/penalties.py), min_p in
b200_op_sample token for token, engine batches that mix edited and plain requests, histories across chunked prefill,
prefix-cache hits and preemption, forcing and banning tokens, logprobs of edited requests, the serving shell, and greedy
streams against vLLM on the 2-layer test model."""
import json
import os

import numpy as np
import pytest
import torch

from oracle.penalties import edit, named, sample_ref

pytestmark = pytest.mark.gpu


def bits(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def f32(b):
    return (np.asarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def bf16_rows(S, V, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(S, V, generator=g) * scale).bfloat16()
    x[:, 3] = float("-inf")
    return x


def spec_rows(rng, S, V, max_len):
    out = []
    for s in range(S):
        n_p = int(rng.integers(1, max_len // 2))
        n_o = int(rng.integers(0, max_len - n_p))
        hot = rng.integers(0, V, 8)
        r = dict(prompt=rng.integers(0, V, n_p).tolist(),
                 output=np.where(rng.random(n_o) < 0.5, rng.choice(hot, n_o), rng.integers(0, V, n_o)).tolist())
        k = s % 5
        if k == 0:
            r.update(repetition_penalty=1.3)
        elif k == 1:
            r.update(presence_penalty=0.5, frequency_penalty=0.5, logit_bias={0: 100.0, V - 1: -100.0, 7: 2.5})
        elif k == 2:
            r.update(repetition_penalty=0.8, presence_penalty=-1.0, frequency_penalty=-0.25, min_tokens=n_o + 1,
                     stop_ids=[1, V - 2])
        elif k == 3:
            r.update(logit_bias={int(t): float(rng.standard_normal() * 50) for t in rng.integers(0, V, 20)}, min_tokens=0,
                     stop_ids=[5])
        else:
            r.update(frequency_penalty=2.0, repetition_penalty=2.0, logit_bias={V // 2: 150.0})
        out.append(r)
    return out


def oracle_kw(r):
    return dict(prompt=r.get("prompt", ()), output=r.get("output", ()), presence=r.get("presence_penalty", 0.0),
                frequency=r.get("frequency_penalty", 0.0), repetition=r.get("repetition_penalty", 1.0),
                min_tokens=r.get("min_tokens", 0), stop_ids=r.get("stop_ids", ()), logit_bias=r.get("logit_bias"))


@pytest.mark.parametrize("V", [512, 1000, 128256])
def test_op_equals_oracle_bit_for_bit(V):
    from kubeai_b200 import ops
    rng = np.random.default_rng(V)
    S = 10
    specs = spec_rows(rng, S, V, 2048)
    raw = bf16_rows(S, V, V).cuda()
    raw_bits = bits(raw)
    logits = raw.clone()
    edited = ops.penalize(logits, specs)
    torch.cuda.synchronize()
    assert np.array_equal(bits(logits), raw_bits)                     # the restore returns the raw rows exactly
    got = bits(edited)
    for s, r in enumerate(specs):
        want = edit(f32(raw_bits[s]), **oracle_kw(r))
        m = named(V, **oracle_kw(r))
        assert np.array_equal(got[s][~m], raw_bits[s][~m]), s         # entries outside the list keep their bits
        gw = f32(got[s][m])
        ww = want[m]
        assert np.array_equal(gw.view(np.uint32), ww.view(np.uint32)), (s, np.flatnonzero(gw != ww)[:5])
    # rows are edited independently of their place: a permutation permutes the result
    perm = rng.permutation(S)
    edited2 = ops.penalize(raw[perm].contiguous(), [specs[i] for i in perm])
    assert np.array_equal(bits(edited2), got[perm])
    # restore=False leaves the edits in place
    inplace = ops.penalize(raw.clone(), specs, restore=False)
    assert np.array_equal(bits(inplace), got)


def test_min_p_sample_equals_oracle():
    from kubeai_b200 import ops
    compared = exempt = 0
    for V, S in ((512, 64), (128256, 16)):
        raw = bf16_rows(S, V, 11 + V, scale=2.0).cuda()
        lf = f32(bits(raw))
        for T, k, p, mp in ((0.8, 0, 1.0, 0.05), (1.0, 50, 0.95, 0.1), (0.7, 0, 0.9, 0.2), (1.5, 5, 1.0, 0.5),
                            (0.9, 0, 0.95, 0.0), (0.0, 0, 1.0, 0.3)):
            seeds = [1000 + s for s in range(S)]
            got = ops.sample(raw, T, k, p, seeds, n=3, min_p=mp).cpu().numpy()
            base = ops.sample(raw, T, k, p, seeds, n=3).cpu().numpy()
            if mp == 0.0:
                assert np.array_equal(got, base)                         # min_p 0 is today's kernel
            for s in range(S):
                tok, margin, slack, mslack = sample_ref(lf[s], T, k, p, seeds[s], 3, mp)
                if min(margin, slack, mslack) < 1e-4:
                    exempt += 1
                    continue
                assert got[s] == tok, (V, T, k, p, mp, s)
                compared += 1
    assert compared > 10 * exempt


PROMPTS = [list(range(7, 7 + n)) for n in (5, 9, 3, 12, 6, 8)]
N_TOK = 10


def engine_specs(V):
    return [dict(),
            dict(repetition_penalty=1.3),
            dict(temperature=0.8, top_p=0.95, seed=5, presence_penalty=0.5, frequency_penalty=0.5),
            dict(logit_bias={11: 3.0, 40: -100.0, V - 1: 1.0}),
            dict(min_tokens=6, stop_ids=[17], ignore_eos=True),
            dict(temperature=0.9, seed=9, min_p=0.05, repetition_penalty=1.2, logit_bias={2: 1.5})]


def run_batch(specs, prompts=PROMPTS, check=False, **cfg):
    from kubeai_b200.engine import Engine, mini_config
    kw = dict(eos_token_id=4)
    kw.update(cfg)
    with Engine(mini_config(**kw)) as e:
        e.set_keep_logits(True)
        rids = [e.submit(p, max_tokens=N_TOK, **sp) for p, sp in zip(prompts, specs)]
        outs = [[] for _ in rids]
        exempt = 0
        for step in range(N_TOK):
            ran, info = e.step()
            assert ran and info.sampled == len(rids)
            rows = e.read_logits(len(rids))
            for i, r in enumerate(rids):
                t = e.poll(r).tokens
                assert len(t) == 1
                if check:
                    sp = specs[i]
                    stops = list(sp.get("stop_ids", ())) + [4]
                    row = edit(rows[i], prompt=prompts[i], output=outs[i], presence=sp.get("presence_penalty", 0.0),
                               frequency=sp.get("frequency_penalty", 0.0), repetition=sp.get("repetition_penalty", 1.0),
                               min_tokens=sp.get("min_tokens", 0), stop_ids=stops, logit_bias=sp.get("logit_bias"))
                    tok, margin, slack, mslack = sample_ref(row, sp.get("temperature", 0.0), sp.get("top_k", 0),
                                                            sp.get("top_p", 1.0), sp.get("seed", 0), step,
                                                            sp.get("min_p", 0.0))
                    if min(margin, slack, mslack) < 1e-4 and sp.get("temperature", 0.0) > 0:
                        exempt += 1
                    else:
                        assert t[0] == tok, (i, step, t[0], tok)
                outs[i] += t
        assert exempt <= 2
        return outs


def test_engine_batch_tokens_equal_oracle():
    specs = engine_specs(512)
    mixed = run_batch(specs, check=True)
    # the plain request's stream does not depend on its edited neighbours
    alone = run_batch([specs[0]], prompts=PROMPTS[:1])
    assert mixed[0] == alone[0]
    assert 40 not in mixed[3]
    assert 17 not in mixed[4][:6] and 4 not in mixed[4][:6]


def run_to_end(specs, prompts, max_tokens, stagger=False, **cfg):
    """Every request to its end; stagger: request i is submitted after step i (a later one can hit the prefix cache)."""
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(eos_token_id=4, **cfg)) as e:
        rids = []
        if not stagger:
            rids = [e.submit(p, max_tokens=max_tokens, **s) for p, s in zip(prompts, specs)]
        outs = [[] for _ in prompts]
        for k in range(2000):
            if stagger and k < len(prompts):
                rids.append(e.submit(prompts[k], max_tokens=max_tokens, **specs[k]))
            ran, _ = e.step()
            for i, r in enumerate(rids):
                outs[i] += e.poll(r).tokens
            if not ran:
                break
        return outs, e.stats()


def test_histories_survive_chunked_prefill_prefix_hits_and_preemption():
    """The same requests through chunked prefill, a prefix-cache hit (whose cached prompt tokens still count for the
    repetition penalty) and forced preemption give the streams of an unpressured run.  Different step shapes round the
    logits differently, so streams are compared up to the first position whose edited top-2 margin is a rounding
    coin-flip (< 0.25, the engine tests' rule)."""
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(7)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (40, 150, 60, 33, 90, 45)]
    prompts[3] = prompts[0][:32] + [9]                       # shares two full blocks with prompt 0: a prefix-cache hit
    specs = [dict(repetition_penalty=1.5, frequency_penalty=0.3), dict(presence_penalty=1.0, repetition_penalty=1.2),
             dict(frequency_penalty=1.0, logit_bias={5: 2.0}), dict(repetition_penalty=2.0),
             dict(min_tokens=10, stop_ids=[1, 2, 3], ignore_eos=True, repetition_penalty=1.1), dict()]
    calm, st = run_to_end(specs, prompts, 24, num_kv_blocks=256, max_model_len=256)
    assert st.preemptions == 0
    margins = []
    with Engine(mini_config(eos_token_id=4, num_kv_blocks=256, max_model_len=256)) as e:
        for p, sp, out in zip(prompts, specs, calm):
            rows = e.forward_logits(p + out[:-1])[len(p) - 1:]
            m = []
            for k in range(len(out)):
                ed = np.sort(edit(rows[k], prompt=p, output=out[:k], presence=sp.get("presence_penalty", 0.0),
                                  frequency=sp.get("frequency_penalty", 0.0),
                                  repetition=sp.get("repetition_penalty", 1.0), min_tokens=sp.get("min_tokens", 0),
                                  stop_ids=list(sp.get("stop_ids", ())) + [4],
                                  logit_bias=sp.get("logit_bias")).astype(np.float64))
                m.append(ed[-1] - ed[-2])
            margins.append(m)

    def same(got, which):
        compared = 0
        for i, w in zip(which, got):
            for k, (a, b) in enumerate(zip(calm[i], w)):
                if margins[i][k] < 0.25:
                    break
                assert a == b, (i, k)
                compared += 1
        return compared
    chunked, st = run_to_end(specs, prompts, 24, num_kv_blocks=256, max_model_len=256, max_batched_tokens=32)
    n = same(chunked, range(6))
    cached, st = run_to_end([specs[0], specs[3]], [prompts[0], prompts[3]], 24, stagger=True, num_kv_blocks=256,
                            max_model_len=256)
    assert st.cached_prompt_tokens > 0
    n += same(cached, [0, 3])
    pressed, st = run_to_end(specs, prompts, 24, num_kv_blocks=22, max_model_len=224, enable_prefix_caching=0)
    assert st.preemptions > 0
    n += same(pressed, range(6))
    assert n >= 50, n


def test_logit_bias_forces_and_bans_and_min_tokens_holds_eos():
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(eos_token_id=4)) as e:
        free = e.generate([[1, 2, 3]], max_tokens=8)[0]
        r = e.submit([1, 2, 3], max_tokens=8, logit_bias={77: 100.0})
        forced = []
        while len(forced) < 8:
            e.step()
            forced += e.poll(r).tokens
        assert forced == [77] * 8
        banned_tok = free[0]
        r = e.submit([1, 2, 3], max_tokens=8, logit_bias={banned_tok: -100.0})
        out = []
        while len(out) < 8:
            e.step()
            out += e.poll(r).tokens
        assert banned_tok not in out
        # +100 on EOS and a stop id: neither appears before min_tokens, then EOS ends the request
        r = e.submit([1, 2, 3], max_tokens=12, ignore_eos=False, stop_ids=[9], min_tokens=5, logit_bias={4: 100.0, 9: 100.0})
        out, fin = [], None
        for _ in range(20):
            e.step()
            pr = e.poll(r)
            out += pr.tokens
            fin = pr.finished
            if fin:
                break
        assert len(out) == 6 and out[-1] in (4, 9) and not set(out[:5]) & {4, 9} and fin == "stop"
        from kubeai_b200 import B200Error
        for bad in (dict(presence_penalty=2.5), dict(frequency_penalty=-3), dict(repetition_penalty=-1.0),
                    dict(min_p=1.5), dict(min_tokens=9), dict(min_tokens=-1), dict(logit_bias={512: 1.0}),
                    dict(logit_bias={-1: 1.0}), dict(logit_bias={5: float("nan")}),
                    dict(logit_bias={i: 1.0 for i in range(1025)})):
            with pytest.raises(B200Error):
                e.submit([1, 2, 3], max_tokens=8, **bad)


def test_logprobs_of_edited_requests_are_raw():
    from kubeai_b200 import ops
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config()) as e:
        e.set_keep_logits(True)
        specs = [dict(repetition_penalty=1.4, logit_bias={9: 5.0}), dict(temperature=0.8, seed=1, frequency_penalty=1.0)]
        rids = [e.submit(p, max_tokens=5, logprobs=True, top_logprobs=4, **s) for p, s in zip(PROMPTS, specs)]
        for _ in range(5):
            e.step()
            rows = torch.from_numpy(e.read_logits(2)).bfloat16().cuda()
            recs = [e.poll_logprobs(r, 4) for r in rids]
            toks = [rc.tokens[0] for rc in recs]
            lp, top_ids, top_lp = ops.logprobs(rows, toks, 4)
            for i, rc in enumerate(recs):
                assert rc.lp[0] == lp[i].item() and rc.top_ids[0].tolist() == top_ids[i, :4].tolist()
                assert np.array_equal(rc.top_lp[0], top_lp[i, :4].cpu().numpy())


def test_server_streams_the_engine_tokens():
    from kubeai_b200.engine import Engine, mini_config
    from kubeai_b200.server import Server
    fields = dict(presence_penalty=0.4, frequency_penalty=0.6, repetition_penalty=1.2, min_tokens=3,
                  logit_bias={"21": 4.0, "300": -100})
    body = dict(model="mini", max_tokens=7, stream=True, ignore_eos=True, temperature=0.7, seed=3, min_p=0.05,
                messages=[{"role": "user", "content": "Tell me about the fox."}], **fields)
    eng = Engine(mini_config(manual_step=0, max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512))
    srv = Server([eng], model="mini", vocab=512, max_model_len=1024, enable_sampling=True, enable_logits_processors=True)
    ids = srv.render_prompt("/v1/chat/completions", json.dumps(body))
    r = srv.handle("POST", "/openai/v1/chat/completions", json.dumps(body))
    srv.close()
    eng.close()
    assert r.status == 200, r.body
    from kubeai_b200.engine import Engine as E2
    with E2(mini_config(max_model_len=1024, max_batched_tokens=512, num_kv_blocks=512)) as e:
        rid = e.submit(ids, max_tokens=7, ignore_eos=True, temperature=0.7, seed=3, min_p=0.05, presence_penalty=0.4,
                       frequency_penalty=0.6, repetition_penalty=1.2, min_tokens=3, logit_bias={21: 4.0, 300: -100.0})
        want = []
        while len(want) < 7:
            e.step()
            want += e.poll(rid).tokens
    from kubeai_b200._lib import lib
    import ctypes as C
    buf = C.create_string_buffer(4096)
    n = lib().b200_detokenize(512, (C.c_int32 * 7)(*want), 7, buf, 4096)
    text = "".join(json.loads(ev)["choices"][0]["delta"].get("content", "") or "" for ev in r.sse_events()[:-1])
    assert text == buf.raw[:n].decode()


def _vllm_ok():
    if os.environ.get("B200_SKIP_VLLM") == "1":
        return False
    try:
        import vllm  # noqa: F401
        return True
    except Exception:
        return False


# The raw logits of the two engines differ by up to ~6 bf16 ulps of a row's largest logit (the logprobs parity test's
# bound), so a top-2 margin after the penalties smaller than that may flip between them.
MARGIN_ULPS = 8.0


@pytest.mark.skipif(not _vllm_ok(), reason="vllm is not importable (or B200_SKIP_VLLM=1)")
def test_greedy_penalized_streams_match_vllm(tmp_path):
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
    prompts = [torch.randint(0, cfg.vocab, (int(n),), generator=g).tolist() for n in (5, 17, 40, 90, 9, 33, 64, 120)]
    N = 24
    pen = dict(repetition_penalty=1.3, frequency_penalty=0.5)
    ecfg = config_from_hf(tmp_path, max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=256,
                          manual_step=1, seed=777)
    mine = []
    with Engine(ecfg) as e:
        e.load_safetensors(tmp_path)
        for p in prompts:
            r = e.submit(p, max_tokens=N, **pen)
            out = []
            while len(out) < N:
                e.step()
                out += e.poll(r).tokens
            mine.append(out)
    llm = LLM(model=str(tmp_path), skip_tokenizer_init=True, dtype="bfloat16", max_model_len=256, enforce_eager=True,
              gpu_memory_utilization=0.25, enable_prefix_caching=False, seed=0, logprobs_mode="processed_logits")
    outs = llm.generate([{"prompt_token_ids": p} for p in prompts],
                        SamplingParams(temperature=0.0, max_tokens=N, ignore_eos=True, detokenize=False, logprobs=2, **pen))
    compared = 0
    for o, out in zip(outs, mine):
        ref = list(o.outputs[0].token_ids)
        for k in range(N):
            top = sorted((v.logprob for v in o.outputs[0].logprobs[k].values()), reverse=True)[:2]   # after penalties
            ulp = np.exp2(np.floor(np.log2(max(abs(top[0]), 2.0 ** -20))) - 7)
            if (top[0] - top[1]) < MARGIN_ULPS * ulp:
                break
            assert ref[k] == out[k], (k, (top[0] - top[1]) / ulp, ref, out)
            compared += 1
    assert compared >= len(prompts), compared
    print(f"vLLM parity with penalties: {compared} positions compared")
