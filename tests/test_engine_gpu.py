"""GPU parity of the whole engine (scheduler + paged KV + prefix cache + forward + greedy) through
the C ABI against the CPU oracle and the HF golden fixture."""
import threading
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle.llama_oracle import LlamaOracle
from oracle.weights import ModelCfg, cos_sin_cache, f32_to_bf16_bits, make_weights, tensor_specs

pytestmark = pytest.mark.gpu
GOLD = np.load(Path(__file__).parent / "golden" / "llama_mini.npz")


@pytest.fixture(scope="module")
def oracle():
    cfg = ModelCfg()
    return LlamaOracle(cfg, make_weights(cfg))


@pytest.fixture()
def eng():
    from kubeai_b200.engine import Engine, mini_config
    e = Engine(mini_config())
    yield e
    e.close()


def test_weights_bit_exact_with_numpy_replica(eng):
    cfg = ModelCfg()
    w = make_weights(cfg)
    for name, shape, _, _ in tensor_specs(cfg):
        got = eng.tensor(name)
        assert np.array_equal(got, w[name].reshape(-1)), name
    cs = eng.tensor("cos_sin").reshape(cfg.max_model_len, 128)
    want = f32_to_bf16_bits(cos_sin_cache(cfg))
    # host libm cosf/sinf/powf vs numpy differ in the last fp32 bits at large angles: a few entries
    # land on the other side of a bf16 rounding boundary
    diff = np.abs(cs.astype(np.int32) - want.astype(np.int32))
    assert diff.max() <= 2 and (diff > 0).mean() < 0.002, (diff.max(), (diff > 0).mean())


def _logit_close(got, want, what):
    err = np.abs(got - want)
    tol = 0.15 + 1.6e-2 * np.abs(want)   # logits std ~4: two bf16 ulps at |x|~8-16 plus vLLM's rtol
    assert (err <= tol).all(), f"{what}: max err {err.max():.4f}, {int((err > tol).sum())} outside tolerance"


def test_forward_logits_match_oracle_and_hf_golden(eng, oracle):
    ids = GOLD["ids"]
    got = eng.forward_logits(ids)
    want, _ = oracle.forward(ids)
    _logit_close(got, want.numpy(), "engine vs oracle")
    _logit_close(got, GOLD["logits_fp32"], "engine vs HF fp32 golden")
    # greedy token agreement wherever the oracle's top-1/top-2 margin is not a rounding coin-flip
    top2 = np.sort(want.numpy(), axis=-1)[:, -2:]
    solid = (top2[:, 1] - top2[:, 0]) > 0.25
    assert (got.argmax(-1)[solid] == want.numpy().argmax(-1)[solid]).all()
    # single-token forward (decode-kernel path for position 0)
    g1 = eng.forward_logits(ids[:1])
    _logit_close(g1, want.numpy()[:1], "single token")


def test_greedy_generation_token_for_token(eng, oracle):
    ids = GOLD["ids"].tolist()
    out = eng.generate([ids], max_tokens=12)[0]
    want, rows = oracle.generate(ids, 12)
    margins = [float(torch.sort(r)[0][-1] - torch.sort(r)[0][-2]) for r in rows]
    # tokens must match up to the first position where the oracle itself is within rounding of a tie
    for i, (a, b) in enumerate(zip(out, want)):
        if margins[i] < 0.25:
            break
        assert a == b, f"token {i}: engine {a} oracle {b} (margin {margins[i]:.3f})"
    assert out == GOLD["greedy"].tolist() or min(margins) < 0.25


def test_continuous_batching_prefix_cache_and_chunked_prefill(oracle):
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(3)
    base = rng.integers(0, 512, size=70).tolist()
    prompts = [base[:70], base[:48] + rng.integers(0, 512, size=9).tolist(), base[:5],
               rng.integers(0, 512, size=33).tolist(), base[:70] + [1, 2, 3]]
    want = [oracle.generate(p, 8) for p in prompts]
    for budget, caching in [(256, 1), (32, 1), (16, 0)]:   # 32/16: prompts are prefilled in chunks
        with Engine(mini_config(max_batched_tokens=budget, enable_prefix_caching=caching)) as e:
            outs = e.generate(prompts[:3], max_tokens=8)
            outs += e.generate(prompts[3:], max_tokens=8)     # second wave hits the prefix cache
            st = e.stats()
            if caching:
                assert st.cached_prompt_tokens >= 64, st.cached_prompt_tokens   # base[:70] -> 4 full blocks
            else:
                assert st.cached_prompt_tokens == 0
            for i, (o, (w, rows)) in enumerate(zip(outs, want)):
                for j, (a, b) in enumerate(zip(o, w)):
                    m = torch.sort(rows[j])[0]
                    if float(m[-1] - m[-2]) < 0.25:
                        break
                    assert a == b, f"budget {budget} prompt {i} token {j}: {a} != {b}"
            assert st.kv_blocks_free == st.kv_blocks_total, "all KV pages must return to the pool"


def test_large_prefill_steps_use_multi_tile_gemm(oracle):
    """A 600-token prompt in one step (two 512-token GEMM tiles, prefill attention over 38 query tiles)."""
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(11)
    prompts = [rng.integers(0, 512, size=600).tolist(), rng.integers(0, 512, size=333).tolist()]
    with Engine(mini_config(max_model_len=1024, max_batched_tokens=1024, num_kv_blocks=256)) as e:
        outs = e.generate(prompts, max_tokens=6)
    ocfg = ModelCfg(max_model_len=1024)
    big = LlamaOracle(ocfg, make_weights(ocfg))
    for p, o in zip(prompts, outs):
        w, rows = big.generate(p, 6)
        for j, (a, b) in enumerate(zip(o, w)):
            m = torch.sort(rows[j])[0]
            if float(m[-1] - m[-2]) < 0.25:
                break
            assert a == b, f"token {j}: {a} != {b}"


def test_preemption_under_kv_pressure_keeps_outputs(oracle):
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(5)
    prompts = [rng.integers(0, 512, size=40).tolist() for _ in range(6)]
    want = [oracle.generate(p, 24) for p in prompts]
    # 6 seqs x 64 tokens = 24 pages needed; give 14 so the scheduler must preempt and recompute (the pool must still hold
    # one max_model_len sequence: 14 pages = 224 tokens)
    with Engine(mini_config(num_kv_blocks=14, max_model_len=224, enable_prefix_caching=0)) as e:
        outs = e.generate(prompts, max_tokens=24)
        assert e.stats().preemptions > 0
    for i, (o, (w, rows)) in enumerate(zip(outs, want)):
        assert len(o) == 24
        for j, (a, b) in enumerate(zip(o, w)):
            m = torch.sort(rows[j])[0]
            if float(m[-1] - m[-2]) < 0.25:
                break
            assert a == b, f"prompt {i} token {j}"


def test_background_thread_submit_wait_poll_abort():
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config(manual_step=0)) as e:
        rng = np.random.default_rng(9)
        results = {}

        def client(i):
            rid = e.submit(rng.integers(0, 512, size=20 + i).tolist(), max_tokens=10)
            toks = []
            while True:
                assert e.wait(rid, 30.0)
                pr = e.poll(rid)
                toks += pr.tokens
                if pr.finished:
                    results[i] = (toks, pr.finished, pr.usage)
                    break
            e.release(rid)

        th = [threading.Thread(target=client, args=(i,)) for i in range(8)]
        [t.start() for t in th]
        [t.join(60) for t in th]
        assert len(results) == 8
        for i, (toks, fin, usage) in results.items():
            assert len(toks) == 10 and fin == "length" and usage[0] == 20 + i and usage[2] == 10
        rid = e.submit(list(range(30)), max_tokens=200)
        e.abort(rid)
        for _ in range(200):
            e.wait(rid, 0.05)
            pr = e.poll(rid)
            if pr.finished:
                break
        assert pr.finished == "aborted"


def test_stop_token_and_eos():
    from kubeai_b200.engine import Engine, mini_config
    with Engine(mini_config()) as e:
        ids = GOLD["ids"].tolist()
        full = e.generate([ids], max_tokens=6)[0]
        rid = e.submit(ids, max_tokens=6, stop_ids=[full[2]])
        toks, fin = [], None
        for _ in range(20):
            e.step()
            pr = e.poll(rid)
            toks += pr.tokens
            if pr.finished:
                fin = pr.finished
                break
        assert toks == full[:3] and fin == "stop"


def test_pipelined_run_matches_single_steps_and_delivers_to_waiting_threads():
    """b200_engine_run (tokens of step N published after step N+1 is enqueued) yields the same tokens as one
    synchronous b200_engine_step at a time, streams them to threads blocked in b200_wait, and honours aborts."""
    from kubeai_b200.engine import Engine, mini_config
    g = torch.Generator().manual_seed(5)
    prompts = [torch.randint(0, 512, (n,), generator=g).tolist() for n in (5, 33, 70, 16, 121)]
    with Engine(mini_config()) as e:
        want = e.generate(prompts, max_tokens=20)
    with Engine(mini_config()) as e:
        rids = [e.submit(p, max_tokens=20) for p in prompts]
        victim = e.submit(prompts[0], max_tokens=200)
        got = [[] for _ in rids]

        def client(i):
            while True:
                e.wait(rids[i], 5.0)
                pr = e.poll(rids[i])
                got[i] += pr.tokens
                if pr.finished is not None:
                    return

        ths = [threading.Thread(target=client, args=(i,)) for i in range(len(rids))]
        for t in ths:
            t.start()
        infos = e.run(3)
        assert len(infos) == 3 and infos[0].tokens > 0
        e.abort(victim)
        total = 3
        while any(t.is_alive() for t in ths) and total < 400:
            total += len(e.run(8, 2000))
        for t in ths:
            t.join(timeout=10)
        assert got == want
        pr = e.poll(victim)
        while pr.finished is None:
            e.run(1, 1000)
            pr = e.poll(victim)
        assert pr.finished == "aborted"
        st = e.stats()
        assert st.running == 0 and st.waiting == 0


def test_full_size_llama3_8b_run_is_deterministic_and_accounts_prefix_reuse():
    """BASELINE config 2 shape (Llama-3-8B, 128 sequences, <=2k context) — too big for the CPU oracle, so checked through
    size-independent properties: two independent engines produce identical token streams for the same multi-turn
    workload (fixed schedules, no atomics in any reduction), every id is a vocabulary id, each request yields exactly
    max_tokens ids, and the second turn's cached prefix is what the block-hash chain must give."""
    from kubeai_b200.engine import Engine, default_config
    g = torch.Generator().manual_seed(11)
    first = [torch.randint(0, 128000, (int(n),), generator=g).tolist() for n in torch.randint(40, 300, (128,), generator=g)]
    follow = [torch.randint(0, 128000, (int(n),), generator=g).tolist() for n in torch.randint(20, 90, (128,), generator=g)]

    def run():
        cfg = default_config(manual_step=1, max_num_seqs=128, max_batched_tokens=2048, max_model_len=2048, kv_fraction=0.2)
        with Engine(cfg) as e:
            t1 = e.generate(first, max_tokens=12)
            turn2 = [p + o + f for p, o, f in zip(first, t1, follow)]
            rids = [e.submit(p, max_tokens=8) for p in turn2]
            t2, usage = [[] for _ in rids], [None] * len(rids)
            pending = set(range(len(rids)))
            while pending:
                ran = e.run(16, 1000)
                for i in list(pending):
                    pr = e.poll(rids[i])
                    t2[i] += pr.tokens
                    if pr.finished is not None:
                        usage[i] = pr.usage
                        pending.discard(i)
                assert ran or not pending
            return t1, t2, usage

    a1, a2, ua = run()
    b1, b2, ub = run()
    assert a1 == b1 and a2 == b2 and ua == ub
    assert all(len(o) == 12 for o in a1) and all(len(o) == 8 for o in a2)
    assert all(0 <= t < 128256 for o in a1 + a2 for t in o)
    for p, o, (prompt_tokens, cached, completion) in zip(first, a1, ua):
        # turn 1 computed len(p) + 11 tokens of KV (the 12th id was sampled, never fed back): every FULL 16-token block of
        # it is in the prefix cache, and turn 2 starts with exactly those tokens
        assert cached == ((len(p) + 11) // 16) * 16 and completion == 8 and prompt_tokens > cached


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_engines_on_two_devices_in_one_process_agree():
    """One process, one engine per GPU (how b200serve --gpus N runs the replicas): per-device kernel attributes, tensor
    maps and workspaces must not leak between devices."""
    from kubeai_b200.engine import Engine, mini_config
    g = torch.Generator().manual_seed(9)
    prompts = [torch.randint(0, 512, (n,), generator=g).tolist() for n in (7, 40, 130)]
    outs = []
    for dev_id in (0, 1, 0):
        with Engine(mini_config(device=dev_id)) as e:
            outs.append(e.generate(prompts, max_tokens=10))
    assert outs[0] == outs[1] == outs[2]
    with Engine(mini_config(device=0)) as e0, Engine(mini_config(device=1)) as e1:   # both alive at once
        r0 = [e0.submit(p, max_tokens=10) for p in prompts]
        r1 = [e1.submit(p, max_tokens=10) for p in prompts]
        for _ in range(200):
            e0.step(); e1.step()
        assert [e0.poll(r).tokens for r in r0] == outs[0]
        assert [e1.poll(r).tokens for r in r1] == outs[0]


def test_llama3_rope_scaling_matches_hf_golden():
    """Llama-3.1 style RoPE frequency scaling (ADVICE r1): cos/sin table vs the numpy replica, logits vs HF."""
    from kubeai_b200.engine import Engine, mini_config
    from oracle.gen_golden import ROPE3
    gold = np.load(Path(__file__).parent / "golden" / "llama_mini_rope3.npz")
    cfg = ModelCfg(**ROPE3)
    with Engine(mini_config(**ROPE3)) as e:
        cs = e.tensor("cos_sin").reshape(cfg.max_model_len, 128)
        want = f32_to_bf16_bits(cos_sin_cache(cfg))
        diff = np.abs(cs.astype(np.int32) - want.astype(np.int32))
        assert diff.max() <= 2 and (diff > 0).mean() < 0.002, (diff.max(), (diff > 0).mean())
        plain = f32_to_bf16_bits(cos_sin_cache(ModelCfg()))
        assert (cs != plain).mean() > 0.3                              # the scaling is not a no-op
        got = e.forward_logits(gold["ids"])
        _logit_close(got, gold["logits_fp32"], "engine (llama3 rope) vs HF fp32 golden")
        out = e.generate([gold["ids"].tolist()], max_tokens=12)[0]
    o = LlamaOracle(cfg, make_weights(cfg))
    want_t, rows = o.generate(gold["ids"].tolist(), 12)
    for i, (a, b) in enumerate(zip(out, want_t)):
        if float(torch.sort(rows[i])[0][-1] - torch.sort(rows[i])[0][-2]) < 0.25:
            break
        assert a == b, f"token {i}"


def test_create_time_validation_of_pool_and_shapes():
    """ADVICE r1: a pool that cannot hold one max_model_len sequence, and shapes the kernels reject, fail at create."""
    from kubeai_b200 import B200Error
    from kubeai_b200.engine import Engine, mini_config
    with pytest.raises(B200Error, match="KV pool too small"):
        Engine(mini_config(max_model_len=256, num_kv_blocks=8))        # needs 16 pages
    with pytest.raises(B200Error, match="unsupported model/config"):
        Engine(mini_config(hidden=576))                                # not a multiple of 256
    with pytest.raises(B200Error, match="unsupported model/config"):
        Engine(mini_config(vocab=509))
    with pytest.raises(B200Error, match="rope scaling"):
        Engine(mini_config(rope_scaling_type=2, rope_factor=0.0))
    with Engine(mini_config(max_model_len=256, num_kv_blocks=16)) as e:   # exactly one sequence fits
        rng = np.random.default_rng(3)
        outs = e.generate([rng.integers(0, 512, size=200).tolist(), rng.integers(0, 512, size=120).tolist()], max_tokens=50)
        assert [len(o) for o in outs] == [50, 50]                      # served one after the other through preemption
        assert e.stats().preemptions >= 0


def test_decode_paths_agree_token_for_token(oracle, monkeypatch):
    """The two decode paths — unfused kernels (B200_FUSED_DECODE=0) and one fused launch per projection (default) — keep
    the same rounding points and split-K orders: same greedy streams, and both the oracle's wherever its margin is not a
    rounding coin-flip."""
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(11)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (5, 17, 40, 64, 90, 121, 33, 8)]
    outs = {}
    for name, env in (("unfused", {"B200_FUSED_DECODE": "0"}), ("per_gemm", {})):
        for k in ("B200_FUSED_DECODE",):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        with Engine(mini_config(max_num_seqs=8, max_batched_tokens=128)) as e:
            outs[name] = e.generate(prompts, max_tokens=20)
            st = e.stats()
            outs[name + "_launches"] = st.kernel_launches
    assert outs["per_gemm"] == outs["unfused"]
    assert outs["per_gemm_launches"] < outs["unfused_launches"]
    for p, o in zip(prompts, outs["per_gemm"]):
        w, rows = oracle.generate(p, 20)
        for j, (a, b) in enumerate(zip(o, w)):
            srt = torch.sort(rows[j])[0]
            if float(srt[-1] - srt[-2]) < 0.25:
                break
            assert a == b, f"token {j}"


def test_large_step_paths_agree_token_for_token(monkeypatch):
    """Steps of more than 128 tokens: the pair kernel with fused epilogues (default) against fp32 segments + elementwise
    kernels (B200_FUSED_PREFILL=0).  Same segment order, same rounding points: the same greedy streams, fewer launches."""
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(12)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (150, 170, 200, 40, 129, 190, 64, 131)]
    outs = {}
    for name, env in (("segments", {"B200_FUSED_PREFILL": "0"}), ("fused", {})):
        monkeypatch.delenv("B200_FUSED_PREFILL", raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        with Engine(mini_config(max_num_seqs=8, max_batched_tokens=512, max_model_len=256)) as e:
            outs[name] = e.generate(prompts, max_tokens=12)
            outs[name + "_launches"] = e.stats().kernel_launches
    assert outs["fused"] == outs["segments"]
    # the test model's projections have fewer tiles than the device has CTA pairs, so most of its launches keep the segment
    # form either way; tests/test_fullsize_gpu.py::test_full_size_prefill_burst_step_matches_oracle covers the full shapes
    assert outs["fused_launches"] <= outs["segments_launches"]


def test_few_long_sequences_decode_through_split_kv_attention(oracle, monkeypatch):
    """Two sequences with long contexts: the engine splits each context over several attention CTAs (attn_decode_split);
    same tokens as with the split disabled, and the oracle's wherever its margin is not a rounding coin-flip."""
    from kubeai_b200.engine import Engine, mini_config
    rng = np.random.default_rng(21)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (230, 150)]
    outs = {}
    for name, env in (("split", None), ("one_cta", "1")):
        monkeypatch.delenv("B200_ATTN_SPLIT", raising=False)
        if env:
            monkeypatch.setenv("B200_ATTN_SPLIT", env)
        with Engine(mini_config(max_num_seqs=4, max_batched_tokens=256, max_model_len=256)) as e:
            outs[name] = e.generate(prompts, max_tokens=16)
            outs[name + "_launches"] = e.stats().kernel_launches
    assert outs["split_launches"] > outs["one_cta_launches"], "the split path (with its merge kernel) did not run"
    for p, a, b in zip(prompts, outs["split"], outs["one_cta"]):
        w, rows = oracle.generate(p, 16)
        for j, (x, y, z) in enumerate(zip(a, b, w)):
            srt = torch.sort(rows[j])[0]
            if float(srt[-1] - srt[-2]) < 0.25:
                break
            assert x == z and y == z, f"token {j}"
