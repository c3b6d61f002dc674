"""Group sizes G = q_heads / kv_heads from 1 to 16 on the GPU.

Attention: decode and verify items (G * q_count <= 16 rows of the mma tile) through b200_op_paged_attn and
b200_op_paged_attn_decode_split, and chunked-prefill items through b200_op_paged_attn_prefill_tc, against an fp64 oracle
on the bf16 inputs.  Pages the block table does not name are NaN, rows past each item's last position are finite poison,
and the positions after q_pos0 + j carry keys aimed at row j's queries, so a wrong row map or a missing per-row mask
moves the output by O(1).

Engine: mini models at G = 1, 3 and 8 against the CPU oracle (logits, greedy tokens, chunked prefill, the prefix cache,
preemption, n > 1 forks, speculative decoding at k_max(G)); the G = 3 tied golden loaded from an HF checkpoint; one
Llama-3.2-3B-shaped layer at full size; vLLM parity; b200serve with a tokenizer on a G = 3 checkpoint.
"""
import json
import re
import subprocess
import time
import urllib.request
from pathlib import Path

import numpy as np
import pytest
import torch

from kubeai_b200 import B200Error, ops

pytestmark = pytest.mark.gpu

D = 128
RMS_C = 0.04
POISON_V = 512.0
GROUPS = [1, 2, 3, 5, 6, 7, 8, 16]


def k_max(G):
    return min(3, 16 // G - 1)


# ------------------------------------------------------------------------------------------------------------ attention
def make_case(items, Hkv, G, seed, prefill=False):
    """items: (q_pos0, q_count).  Returns q [T, Hq*128], kv pool, block tables, work, and the fp64 oracle output."""
    g = torch.Generator().manual_seed(seed)
    Hq = G * Hkv
    lens = [p0 + qc for p0, qc in items]
    nbs = [(L + 15) // 16 for L in lens]
    used = sum(nbs)
    perm = torch.randperm(used + 4, generator=g)
    nan_block = int(perm[-1])
    kv = torch.full((used + 4, 2, Hkv, 16, D), float("nan"), dtype=torch.bfloat16)
    btab = torch.full((len(items), max(nbs) + 2), nan_block, dtype=torch.int32)
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
        # each later position's key aims at the queries of the rows that must not see it
        for i in range(1, min(qc, 16)):
            k[p0 + i] = 0.3 * q[tok:tok + i].float().reshape(i, Hkv, G, D).sum((0, 2))
            v[p0 + i] = 32.0 * torch.sign(torch.randn(Hkv, D, generator=g))
        k[L:] *= 8.0
        v[L:] = float("nan") if prefill else POISON_V    # the prefill kernel reads no token past the context
        k, v = k.bfloat16(), v.bfloat16()
        kv[blocks, 0] = k.reshape(nb, 16, Hkv, D).permute(0, 2, 1, 3)
        kv[blocks, 1] = v.reshape(nb, 16, Hkv, D).permute(0, 2, 1, 3)
        kk = k[:L].double().repeat_interleave(G, dim=1)           # [L, Hq, D]: q head h reads KV head h // G
        vv = v[:L].double().repeat_interleave(G, dim=1)
        sc = torch.einsum("jhd,thd->hjt", q[tok:tok + qc].double(), kk) * D ** -0.5
        sc = sc.masked_fill(torch.arange(L)[None, None, :] > (p0 + torch.arange(qc))[None, :, None], float("-inf"))
        want[tok:tok + qc] = torch.einsum("hjt,thd->jhd", torch.softmax(sc, -1), vv)
        work.append((tok, qc, p0, s))
        tok += qc
    return (q.reshape(T, Hq * D).cuda(), kv.cuda(), btab.cuda(), torch.tensor(work, dtype=torch.int32).cuda(),
            want.reshape(T, Hq * D))


def run(q, kv, btab, work, Hq, Hkv, split):
    out = torch.full((q.shape[0], q.shape[1]), -7776.0, dtype=torch.bfloat16, device="cuda")
    ops.paged_attn(q, kv, btab, work, Hq, Hkv, decode=True, out=out, split=split)
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


# positions that start, straddle and end on a page (16) and on a 64-token tile boundary
POSITIONS = [0, 1, 13, 15, 16, 49, 60, 63, 64, 127, 1021, 2045, 4093]


@pytest.mark.parametrize("G", GROUPS)
@pytest.mark.parametrize("split", [0, 1, 2, 5, 32])
def test_decode_and_verify_attention_matches_oracle(G, split):
    Hkv = 2
    items = [(p0, qc) for p0 in POSITIONS for qc in range(1, 16 // G + 1)]
    q, kv, btab, work, want = make_case(items, Hkv, G, seed=101 * G + split)
    check_close(run(q, kv, btab, work, G * Hkv, Hkv, split), want, f"G={G} split={split}")


@pytest.mark.parametrize("G", [1, 3, 8])
def test_decode_attention_with_eight_kv_heads(G):
    items = [(p0, qc) for p0 in (0, 62, 1000, 2047) for qc in range(1, 16 // G + 1)]
    q, kv, btab, work, want = make_case(items, 8, G, seed=7 + G)
    for split in (0, 3):
        check_close(run(q, kv, btab, work, 8 * G, 8, split), want, f"G={G} Hkv=8 split={split}")


@pytest.mark.parametrize("G", GROUPS + [4])
@pytest.mark.parametrize("split", [0, 3, 32])
def test_single_position_items_are_bit_identical_next_to_verify_items(G, split):
    Hkv = 2
    qm = 16 // G
    items = [(700, 1), (700, qm), (63, 1), (64 - qm // 2, qm), (2000, 1), (15, max(1, qm - 1)), (1, 1)]
    q, kv, btab, work, want = make_case(items, Hkv, G, seed=5 + G)
    mixed = run(q, kv, btab, work, G * Hkv, Hkv, split)
    check_close(mixed, want, "mixed")
    ones = [i for i, (_, qc) in enumerate(items) if qc == 1]
    alone = run(q, kv, btab, work[ones].contiguous(), G * Hkv, Hkv, split)
    used = torch.zeros(q.shape[0], dtype=torch.bool)
    for i in ones:
        t = int(work[i, 0])
        used[t] = True
        assert torch.equal(mixed[t].view(torch.int16), alone[t].view(torch.int16)), f"item {i}"
    assert (alone[~used.cuda()].float() == -7776.0).all()      # nothing is written past an item's rows


@pytest.mark.parametrize("G", GROUPS + [4])
def test_chunked_prefill_attention_matches_oracle(G):
    """Ragged work items of 1..64 query tokens after cached prefixes of 0..1900 tokens, one CTA per query head."""
    Hkv = 2
    items = [(0, 64), (0, 1), (0, 37), (16, 64), (63, 5), (64, 64), (100, 17), (500, 64), (1000, 48), (1900, 64), (7, 63)]
    q, kv, btab, work, want = make_case(items, Hkv, G, seed=300 + G, prefill=True)
    Hq = G * Hkv
    out = torch.full((q.shape[0], Hq * D), -7776.0, dtype=torch.bfloat16, device="cuda")
    ops.paged_attn_prefill_tc(q, kv, btab, work, Hq, Hkv, out=out)
    torch.cuda.synchronize()
    check_close(out, want, f"prefill G={G}")


@pytest.mark.parametrize("hq, hkv", [(2, 2), (6, 2), (8, 1), (16, 1)])
def test_op_level_paged_attn_refuses_decode_0_and_uneven_groups(hq, hkv):
    q, kv, btab, work, _ = make_case([(0, 16)], hkv, hq // hkv, seed=1)
    for head_dim in (None, 64, 128):
        with pytest.raises(B200Error, match=r"decode = 0 is not served; chunked prefill is b200_op_paged_attn_prefill_tc"):
            ops.paged_attn(q, kv, btab, work, hq, hkv, decode=False, head_dim=head_dim)
    with pytest.raises(B200Error, match="kv_heads must divide q_heads"):
        ops.paged_attn(q, kv, btab, work, 2 * hkv + 1 if hkv > 1 else 17, hkv, decode=True)


# ------------------------------------------------------------------------------------------------------------ engine
from kubeai_b200.engine import Engine, config_from_hf, default_config, mini_config  # noqa: E402
from oracle.llama_oracle import LlamaOracle  # noqa: E402
from oracle.weights import ModelCfg, make_weights  # noqa: E402

SHAPES = {1: dict(hidden=256, q_heads=2, kv_heads=2), 3: dict(hidden=768, q_heads=6, kv_heads=2),
          8: dict(hidden=1024, q_heads=8, kv_heads=1)}
_ORACLES = {}


def oracle(G):
    if G not in _ORACLES:
        cfg = ModelCfg(**SHAPES[G])
        _ORACLES[G] = LlamaOracle(cfg, make_weights(cfg))
    return _ORACLES[G]


def prompts(seed, lens):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 512, size=n).tolist() for n in lens]


def greedy_matches_oracle(o, prompt, got, n):
    want, rows = o.generate(prompt, n)
    for j, (a, b) in enumerate(zip(got, want)):
        m = torch.sort(rows[j])[0]
        if float(m[-1] - m[-2]) < 0.25:      # the oracle itself is within rounding of a tie: stop comparing
            return j
        assert a == b, f"greedy token {j}: engine {a} vs oracle {b}"
    return n


@pytest.mark.parametrize("G", [1, 3, 8])
def test_engine_logits_and_greedy_tokens_match_oracle(G):
    o = oracle(G)
    ps = prompts(G, [37, 1, 16, 120, 200])
    with Engine(mini_config(**SHAPES[G])) as e:
        for p in ps[:2] + ps[3:4]:
            got = e.forward_logits(p)
            want = o.forward(p)[0].numpy()
            err = np.abs(got - want)
            assert (err <= 0.15 + 1.6e-2 * np.abs(want)).all() and err.mean() < 0.04, (G, len(p), err.max())
        outs = e.generate(ps, max_tokens=12)
    compared = sum(greedy_matches_oracle(o, p, out, 12) for p, out in zip(ps, outs))
    assert compared >= len(ps), compared        # near-ties end the comparison early on these small models


@pytest.mark.parametrize("G", [1, 3, 8])
def test_engine_chunked_prefill_prefix_cache_and_preemption_follow_the_oracle(G):
    """48-token prefill chunks, a second pass through the prefix cache and a pool that holds one sequence (the rest wait
    or are preempted and recomputed): every stream is the oracle's up to its first near-tie.  Logits depend on the step's
    shape (DESIGN §8), so streams of different schedules are compared through the oracle, not with each other."""
    ps = prompts(10 + G, [230, 150, 90, 200, 17, 64])
    o = oracle(G)
    runs = []
    with Engine(mini_config(max_batched_tokens=48, **SHAPES[G])) as e:
        runs.append(e.generate(ps, max_tokens=20))
        runs.append(e.generate(ps, max_tokens=20))
    with Engine(mini_config(num_kv_blocks=17, **SHAPES[G])) as e:
        runs.append(e.generate(ps, max_tokens=20))
    for p, *outs in zip(ps, *runs):
        want, rows = o.generate(p, 20)
        for out in outs:
            assert len(out) == 20
            for j, (a, b) in enumerate(zip(out, want)):
                m = torch.sort(rows[j])[0]
                if float(m[-1] - m[-2]) < 0.25:
                    break
                assert a == b, (len(p), j)


@pytest.mark.parametrize("G", [1, 3, 8])
def test_engine_parallel_samples_fork_at_any_group_size(G):
    """n = 4 members of one prefill sample exactly what four separate requests with seeds s + i sample."""
    p = prompts(20 + G, [75])[0]
    with Engine(mini_config(**SHAPES[G])) as e:
        rids = e.submit_n(p, 4, max_tokens=16, temperature=0.9, top_p=0.95, seed=123)
        got = {r: [] for r in rids}
        while e.step()[0]:
            for r in rids:
                got[r] += e.poll(r).tokens
        members = [got[r] + e.poll(r).tokens for r in rids]
        for r in rids:
            e.release(r)
        singles = []
        for i in range(4):
            rid = e.submit(p, max_tokens=16, temperature=0.9, top_p=0.95, seed=123 + i)
            toks = []
            while e.step()[0]:
                toks += e.poll(rid).tokens
            singles.append(toks + e.poll(rid).tokens)
            e.release(rid)
    assert members == singles
    assert len({tuple(m) for m in members}) > 1


@pytest.mark.parametrize("G", [1, 3, 8])
def test_engine_speculative_decoding_at_k_max(G):
    """Prompts of a repeated random block and 1..3-token lookups give the n-gram proposer drafts; every emitted greedy
    token equals the oracle's on rows the oracle does not call a tie."""
    k = k_max(G)
    rng = np.random.default_rng(30 + G)
    ps = []
    for n in (23, 31, 40):
        b = rng.integers(0, 512, size=n).tolist()
        ps.append((b * 5)[: 5 * n - 3])
    with Engine(mini_config(num_speculative_tokens=k, prompt_lookup_min=1, prompt_lookup_max=3, **SHAPES[G])) as e:
        spec = e.generate(ps, max_tokens=24)
        st = e.stats()
    assert st.spec_draft_tokens > 0, st.spec_draft_tokens      # verify items of 1 + k positions ran
    assert st.spec_draft_tokens <= k * st.spec_drafts
    o = oracle(G)
    assert sum(greedy_matches_oracle(o, p, s, 24) for p, s in zip(ps, spec)) >= len(ps)


@pytest.mark.parametrize("G", [5, 8, 9, 16])
def test_create_refuses_drafts_past_k_max(G):
    with pytest.raises(B200Error, match=rf"num_speculative_tokens={k_max(G) + 1} exceeds {k_max(G)}, .* with {G} query heads"):
        Engine(mini_config(hidden=1024, q_heads=G, kv_heads=1, num_speculative_tokens=k_max(G) + 1))
    if k_max(G) > 0:
        with Engine(mini_config(hidden=1024, q_heads=G, kv_heads=1, num_speculative_tokens=k_max(G))) as e:
            assert len(e.generate([[1, 2, 3] * 20], max_tokens=4)[0]) == 4


def test_engine_loaded_from_tied_group_size_3_checkpoint_matches_golden(tmp_path):
    from scripts.gen_golden_gqa import GQA3, tied_weights, write_checkpoint
    gold = np.load(Path(__file__).parent / "golden" / "llama_mini_gqa3.npz")
    write_checkpoint(tmp_path)
    assert json.loads((tmp_path / "config.json").read_text())["tie_word_embeddings"] is True
    cfg = config_from_hf(tmp_path, max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=128,
                         manual_step=1, seed=999)
    assert (cfg.q_heads, cfg.kv_heads, cfg.rope_scaling_type, cfg.rope_factor) == (6, 2, 2, 32.0)
    w = tied_weights(ModelCfg(**GQA3))
    with Engine(cfg) as e:
        e.load_safetensors(tmp_path)
        for name in ("embed", "lm_head", "layers.0.wqkv", "layers.1.wo", "final_norm"):
            assert np.array_equal(e.tensor(name), w[name].reshape(-1)), name
        got = e.forward_logits(gold["ids"])
        toks = e.generate([gold["ids"].tolist()], max_tokens=12)[0]
    ref = gold["logits_fp32"]
    err, hf_err = np.abs(got - ref), np.abs(gold["logits_bf16"] - ref)
    assert (err <= 0.25 + 1.6e-2 * np.abs(ref)).all(), err.max()
    assert err.mean() <= 1.2 * hf_err.mean(), (err.mean(), hf_err.mean())
    o = LlamaOracle(ModelCfg(**GQA3), w)
    assert greedy_matches_oracle(o, gold["ids"].tolist(), toks, 12) >= 1


# ------------------------------------------------------------------------------------------------- full size (3B shape)
import test_fullsize_gpu as F  # noqa: E402   the 8B layer tests, run here on the 3B geometry

SHAPE_3B = dict(num_layers=1, hidden=3072, q_heads=24, kv_heads=8, intermediate=8192, vocab=128256, max_model_len=2048,
                rope_scaling_type=2, rope_factor=32.0, rope_low_freq_factor=1.0, rope_high_freq_factor=4.0,
                rope_original_max_pos=8192)


@pytest.fixture(scope="module")
def layer_3b():
    from oracle import llama_oracle as O
    from oracle.weights import bf16_bits_to_f32, cos_sin_cache
    e = Engine(default_config(manual_step=1, max_num_seqs=128, max_batched_tokens=1536, num_kv_blocks=128 * 129 + 64, **SHAPE_3B))
    cfg = ModelCfg(**SHAPE_3B)
    H, I, V = cfg.hidden, cfg.intermediate, cfg.vocab
    shapes = {"embed": (V, H), "lm_head": (V, H), "final_norm": (H,), "layers.0.wqkv": (cfg.qkv_rows, H),
              "layers.0.wo": (H, cfg.q_heads * D), "layers.0.wgu": (2 * I, H), "layers.0.wdown": (H, I),
              "layers.0.norm1": (H,), "layers.0.norm2": (H,)}
    w = {n: torch.from_numpy(bf16_bits_to_f32(e.tensor(n)).copy()).reshape(s) for n, s in shapes.items()}
    cs = O.r(torch.from_numpy(cos_sin_cache(cfg)))
    yield e, cfg, w, cs
    e.close()


@pytest.mark.parametrize("T", [128, 1536])
def test_llama32_3b_shape_prefill_logits_match_oracle(layer_3b, T):
    F.test_full_size_layer_prefill_logits_match_oracle(layer_3b, T)


def test_llama32_3b_shape_decode_step_of_128_sequences_matches_oracle(layer_3b):
    F.test_full_size_decode_step_of_128_sequences_matches_oracle(layer_3b)


# ------------------------------------------------------------------------------------------------- vLLM parity
import test_vllm_parity_gpu as VP  # noqa: E402


@pytest.mark.skipif(not VP._vllm_ok(), reason="vllm is not importable (or B200_SKIP_VLLM=1)")
@pytest.mark.parametrize("G", [1, 3, 8])
def test_logits_and_greedy_tokens_match_vllm(tmp_path, G):
    from safetensors.torch import save_file
    from oracle.gen_golden import hf_model
    from scripts.gen_golden_gqa import write_checkpoint
    if G == 3:
        write_checkpoint(tmp_path)           # tied embeddings, llama3 rope scaling
    else:
        cfg = ModelCfg(**SHAPES[G])
        m = hf_model(cfg, make_weights(cfg), torch.bfloat16)
        m.config.save_pretrained(tmp_path)
        save_file({k: v.contiguous() for k, v in m.state_dict().items()}, str(tmp_path / "model.safetensors"))
    g = torch.Generator().manual_seed(17 + G)
    lens = [5, 16, 33, 70, 121, 200] + torch.randint(2, 220, (10,), generator=g).tolist()
    ps = [torch.randint(0, 512, (int(n),), generator=g).tolist() for n in lens]
    N = 24
    ecfg = config_from_hf(tmp_path, max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=256,
                          manual_step=1, seed=777)
    with Engine(ecfg) as e:
        e.load_safetensors(tmp_path)
        mine = e.generate(ps, max_tokens=N)
        logits = {tuple(p): e.forward_logits(p) for p in ps}
    llm = VP._llm(tmp_path, 256, 0.15)
    try:
        res = VP._compare(f"2-layer test model, G = {G}", llm, lambda p: logits[tuple(p)], mine, ps, N, topk=20)
    finally:
        del llm
        import gc
        gc.collect()
        torch.cuda.empty_cache()
    assert sum(r["identical_prefix"] == N for r in res["greedy"]) >= len(ps) // 2


# ------------------------------------------------------------------------------------------------- b200serve
def test_b200serve_answers_a_chat_request_on_a_group_size_3_checkpoint(tmp_path):
    pytest.importorskip("tokenizers")
    from tokenizers import Regex, Tokenizer as HFTokenizer, decoders, models, pre_tokenizers, trainers
    from kubeai_b200._lib import LIB_PATH
    from scripts.gen_golden_gqa import write_checkpoint
    write_checkpoint(tmp_path)
    pat = r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+"
    hf = HFTokenizer(models.BPE(ignore_merges=True))
    hf.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(pat), behavior="isolated"),
                                                pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    hf.decoder = decoders.ByteLevel()
    specials = ["<|begin_of_text|>", "<|end_of_text|>", "<|start_header_id|>", "<|end_header_id|>", "<|eot_id|>"]
    hf.train_from_iterator(["hello world, how are you today? I'm fine thanks; it's 12345 o'clock"] * 50,
                           trainers.BpeTrainer(vocab_size=504, special_tokens=specials,
                                               initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False))
    hf.save(str(tmp_path / "tokenizer.json"))
    bindir = LIB_PATH.parent.parent / "bin"
    srv = subprocess.Popen([str(bindir / "b200serve"), "--gpus", "1", "--model", "mini3", "--model-dir", str(tmp_path),
                            "--port", "0", "--host", "127.0.0.1", "--max-model-len", "256", "--max-num-batched-tokens", "256",
                            "--max-num-seqs", "8", "--gpu-memory-utilization", "0.05"], stderr=subprocess.PIPE, text=True)
    try:
        port = None
        t0 = time.time()
        while time.time() - t0 < 120:
            line = srv.stderr.readline()
            m = re.search(r"on http://127.0.0.1:(\d+)/", line or "")
            if m:
                port = int(m.group(1))
                break
            assert srv.poll() is None, line
        assert port, "b200serve did not come up"
        body = dict(model="mini3", messages=[{"role": "user", "content": "hello world, how are you?"}], max_tokens=12,
                    temperature=0)
        req = urllib.request.Request(f"http://127.0.0.1:{port}/openai/v1/chat/completions", data=json.dumps(body).encode(),
                                     headers={"Content-Type": "application/json"})
        r = json.loads(urllib.request.urlopen(req, timeout=60).read())
        ch = r["choices"][0]
        assert ch["message"]["role"] == "assistant" and isinstance(ch["message"]["content"], str)
        assert ch["finish_reason"] in ("stop", "length")
        assert r["usage"]["prompt_tokens"] > 5 and 1 <= r["usage"]["completion_tokens"] <= 12
    finally:
        srv.terminate()
        srv.wait(20)
