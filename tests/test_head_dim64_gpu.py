"""64-dimensional heads (head_dim 64) on the GPU, through the C ABI.

Attention: decode and verify items through b200_op_paged_attn_hd / b200_op_paged_attn_decode_split_hd and chunked-prefill
items through b200_op_paged_attn_prefill_tc_hd against an fp64 oracle on the bf16 inputs, with NaN pages the block tables do
not name, finite poison past each item and keys aimed at masked rows (the cases of test_gqa_gpu.py at D = 64).  The _hd
entry points at 128 give the bits of the functions without _hd.

qkv epilogue: GEMM3_EPI_ROPE_KV at D = 64 against b200_op_rope_kvwrite_hd and the oracle's rope_neox on the GEMM's own
product, bit for bit, including slabs that hold the last k head and the first v head (odd kv_heads).

Engine: mini models at D = 64 (G = 4, G = 2 with 3 KV heads, G = 8) against the CPU oracle; the head_dim 64 tied golden
loaded from an HF checkpoint; one Llama-3.2-1B-shaped layer at full size; vLLM parity; b200serve on a head_dim 64 checkpoint.
"""
import json
import math
import re
import subprocess
import time
import urllib.request
from pathlib import Path

import numpy as np
import pytest
import torch

from kubeai_b200 import B200Error, ops
from oracle import llama_oracle as O

pytestmark = pytest.mark.gpu

D = 64
RMS_C = 0.04
POISON_V = 512.0
GROUPS = [1, 2, 3, 4, 8, 16]


def k_max(G):
    return min(3, 16 // G - 1)


# ------------------------------------------------------------------------------------------------------------ attention
def make_case(items, Hkv, G, seed, prefill=False, d=D):
    """items: (q_pos0, q_count).  Returns q [T, Hq*d], kv pool [blocks][2][Hkv][16][d], block tables, work, fp64 oracle."""
    g = torch.Generator().manual_seed(seed)
    Hq = G * Hkv
    lens = [p0 + qc for p0, qc in items]
    nbs = [(L + 15) // 16 for L in lens]
    used = sum(nbs)
    perm = torch.randperm(used + 4, generator=g)
    nan_block = int(perm[-1])
    kv = torch.full((used + 4, 2, Hkv, 16, d), float("nan"), dtype=torch.bfloat16)
    btab = torch.full((len(items), max(nbs) + 2), nan_block, dtype=torch.int32)
    T = sum(qc for _, qc in items)
    q = torch.randn(T, Hq, d, generator=g).bfloat16()
    want = torch.zeros(T, Hq, d, dtype=torch.float64)
    work, pos, tok = [], 0, 0
    for s, ((p0, qc), L, nb) in enumerate(zip(items, lens, nbs)):
        blocks = perm[pos:pos + nb]
        pos += nb
        btab[s, :nb] = blocks.int()
        k = torch.randn(nb * 16, Hkv, d, generator=g)
        v = torch.randn(nb * 16, Hkv, d, generator=g)
        for i in range(1, min(qc, 16)):
            k[p0 + i] = 0.3 * q[tok:tok + i].float().reshape(i, Hkv, G, d).sum((0, 2))
            v[p0 + i] = 32.0 * torch.sign(torch.randn(Hkv, d, generator=g))
        k[L:] *= 8.0
        v[L:] = float("nan") if prefill else POISON_V
        k, v = k.bfloat16(), v.bfloat16()
        kv[blocks, 0] = k.reshape(nb, 16, Hkv, d).permute(0, 2, 1, 3)
        kv[blocks, 1] = v.reshape(nb, 16, Hkv, d).permute(0, 2, 1, 3)
        kk = k[:L].double().repeat_interleave(G, dim=1)
        vv = v[:L].double().repeat_interleave(G, dim=1)
        sc = torch.einsum("jhd,thd->hjt", q[tok:tok + qc].double(), kk) * d ** -0.5
        sc = sc.masked_fill(torch.arange(L)[None, None, :] > (p0 + torch.arange(qc))[None, :, None], float("-inf"))
        want[tok:tok + qc] = torch.einsum("hjt,thd->jhd", torch.softmax(sc, -1), vv)
        work.append((tok, qc, p0, s))
        tok += qc
    return (q.reshape(T, Hq * d).cuda(), kv.cuda(), btab.cuda(), torch.tensor(work, dtype=torch.int32).cuda(),
            want.reshape(T, Hq * d))


def run(q, kv, btab, work, Hq, Hkv, split, head_dim=D):
    out = torch.full((q.shape[0], q.shape[1]), -7776.0, dtype=torch.bfloat16, device="cuda")
    ops.paged_attn(q, kv, btab, work, Hq, Hkv, decode=True, out=out, split=split, head_dim=head_dim)
    torch.cuda.synchronize()
    return out


def check_close(got, want, what, d=D):
    got = got.double().cpu().reshape(got.shape[0], -1, d)
    want = want.reshape(want.shape[0], -1, d)
    assert torch.isfinite(got).all(), f"{what}: non-finite output (an unnamed page was read)"
    err = (got - want).abs().amax(-1)
    rms = want.pow(2).mean(-1).sqrt()
    worst = float((err / rms).max())
    assert worst <= RMS_C, f"{what}: max err/rms {worst:.4f}"


POSITIONS = [0, 1, 13, 15, 16, 49, 60, 63, 64, 127, 1021, 2045, 4093]


@pytest.mark.parametrize("G", GROUPS)
@pytest.mark.parametrize("split", [0, 1, 2, 5, 32])
def test_decode_and_verify_attention_matches_oracle(G, split):
    Hkv = 2
    items = [(p0, qc) for p0 in POSITIONS for qc in range(1, 16 // G + 1)]
    q, kv, btab, work, want = make_case(items, Hkv, G, seed=103 * G + split)
    check_close(run(q, kv, btab, work, G * Hkv, Hkv, split), want, f"D=64 G={G} split={split}")


@pytest.mark.parametrize("G", [1, 4, 8])
def test_decode_attention_with_eight_kv_heads(G):
    items = [(p0, qc) for p0 in (0, 62, 1000, 2047) for qc in range(1, 16 // G + 1)]
    q, kv, btab, work, want = make_case(items, 8, G, seed=9 + G)
    for split in (0, 3):
        check_close(run(q, kv, btab, work, 8 * G, 8, split), want, f"D=64 G={G} Hkv=8 split={split}")


@pytest.mark.parametrize("G", [2, 4, 16])
def test_single_position_items_are_bit_identical_next_to_verify_items(G):
    Hkv = 2
    qm = 16 // G
    items = [(700, 1), (700, qm), (63, 1), (64 - qm // 2, qm), (2000, 1), (15, max(1, qm - 1)), (1, 1)]
    q, kv, btab, work, want = make_case(items, Hkv, G, seed=15 + G)
    for split in (0, 3):
        mixed = run(q, kv, btab, work, G * Hkv, Hkv, split)
        check_close(mixed, want, "mixed")
        ones = [i for i, (_, qc) in enumerate(items) if qc == 1]
        alone = run(q, kv, btab, work[ones].contiguous(), G * Hkv, Hkv, split)
        used = torch.zeros(q.shape[0], dtype=torch.bool)
        for i in ones:
            t = int(work[i, 0])
            used[t] = True
            assert torch.equal(mixed[t].view(torch.int16), alone[t].view(torch.int16)), f"item {i}"
        assert (alone[~used.cuda()].float() == -7776.0).all()


@pytest.mark.parametrize("G", GROUPS)
def test_chunked_prefill_attention_matches_oracle(G):
    """Ragged work items of 1..64 query tokens after cached prefixes of 0..1900 tokens, items crossing pages."""
    Hkv = 2
    items = [(0, 64), (0, 1), (0, 37), (16, 64), (63, 5), (64, 64), (100, 17), (500, 64), (1000, 48), (1900, 64), (7, 63)]
    q, kv, btab, work, want = make_case(items, Hkv, G, seed=310 + G, prefill=True)
    Hq = G * Hkv
    out = torch.full((q.shape[0], Hq * D), -7776.0, dtype=torch.bfloat16, device="cuda")
    ops.paged_attn_prefill_tc(q, kv, btab, work, Hq, Hkv, out=out, head_dim=D)
    torch.cuda.synchronize()
    check_close(out, want, f"prefill D=64 G={G}")


def test_hd_entry_points_at_128_give_the_bits_of_the_old_ones():
    G, Hkv = 4, 2
    items = [(p0, qc) for p0 in (0, 15, 64, 700, 2045) for qc in (1, 2, 4)]
    q, kv, btab, work, _ = make_case(items, Hkv, G, seed=77, d=128)
    for split in (0, 1, 4):
        a = run(q, kv, btab, work, G * Hkv, Hkv, split, head_dim=None)
        b = run(q, kv, btab, work, G * Hkv, Hkv, split, head_dim=128)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), split
    pitems = [(0, 64), (16, 40), (500, 64)]
    q, kv, btab, work, _ = make_case(pitems, Hkv, G, seed=78, prefill=True, d=128)
    a = ops.paged_attn_prefill_tc(q, kv, btab, work, G * Hkv, Hkv)
    b = ops.paged_attn_prefill_tc(q, kv, btab, work, G * Hkv, Hkv, head_dim=128)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_op_level_paged_attn_refuses_head_dim_96():
    q, kv, btab, work, _ = make_case([(0, 16)], 2, 4, seed=1)
    with pytest.raises(B200Error, match="head_dim=96; 64 and 128 are served"):
        ops.paged_attn(q, kv, btab, work, 8, 2, decode=True, head_dim=96)


# ------------------------------------------------------------------------------------------------ qkv epilogue, KV pages
def dev(x):
    return x.to(torch.bfloat16).cuda().contiguous()


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).bfloat16()


@pytest.mark.parametrize("T,Hq,Hkv,K,force", [(128, 32, 8, 2048, 0), (128, 8, 2, 512, 0), (50, 6, 3, 512, 2), (1, 2, 1, 512, 1),
                                              (77, 8, 1, 512, 0), (300, 32, 8, 2048, 0), (200, 10, 5, 512, 0)])
def test_rope_kv_epilogue_at_head_dim_64_is_bit_exact(T, Hq, Hkv, K, force):
    """The fused epilogue on the GEMM's own plain product equals rope_kvwrite_hd on that product and the oracle's rope_neox,
    bit for bit; slot -1 and unnamed slots are not written.  Odd kv_heads put the last k head and the first v head in one
    128-row slab."""
    from oracle.weights import ModelCfg, cos_sin_cache
    N = (Hq + 2 * Hkv) * D
    x, w = rnd(T, K, seed=24), rnd(N, K, scale=1 / math.sqrt(K), seed=25)
    max_pos = 2048
    cs = O.r(torch.from_numpy(cos_sin_cache(ModelCfg(max_model_len=max_pos, head_dim=D, rope_scaling_type=2, rope_factor=32.0,
                                                     rope_original_max_pos=64)))).cuda()
    assert cs.shape == (max_pos, D)
    g = torch.Generator().manual_seed(26)
    pos = torch.randint(0, max_pos, (T,), generator=g, dtype=torch.int32)
    nblocks = T + 8
    slots = torch.randperm(nblocks * 16, generator=g)[:T].to(torch.int32)
    if T > 3:
        slots[3] = -1
    kv = torch.zeros(nblocks, 2, Hkv, 16, D, dtype=torch.bfloat16, device="cuda")
    qkv = torch.zeros(T, N, dtype=torch.bfloat16, device="cuda")
    plain, sch = ops.gemm3(x, w, force=force)
    ops.gemm3(x, w, epi=ops.EPI_ROPE_KV, out=qkv, positions=pos.cuda(), slots=slots.cuda(), cos_sin=dev(cs), kv_layer=kv,
              q_heads=Hq, kv_heads=Hkv, force=force, head_dim=D)
    # the separate kernel on the same product
    qkv2 = plain.clone()
    kv2 = torch.zeros_like(kv)
    ops.rope_kvwrite(qkv2, pos.cuda(), slots.cuda(), dev(cs), kv2, Hq, Hkv, head_dim=D)
    torch.cuda.synchronize()
    assert torch.equal(qkv[:, :Hq * D].view(torch.int16), qkv2[:, :Hq * D].view(torch.int16)), "q rows: fused vs separate"
    assert torch.equal(kv.view(torch.int16), kv2.view(torch.int16)), "KV pages: fused vs separate"
    p = plain.float()
    q = O.rope_neox(p[:, :Hq * D].reshape(T, Hq, D), pos.long().cuda(), cs)
    k = O.rope_neox(p[:, Hq * D:(Hq + Hkv) * D].reshape(T, Hkv, D), pos.long().cuda(), cs)
    v = p[:, (Hq + Hkv) * D:].reshape(T, Hkv, D)
    assert torch.equal(qkv[:, :Hq * D].float().reshape(T, Hq, D), q), "rotated q rows"
    kvc = kv.float()
    for t in range(T):
        s = int(slots[t])
        if s < 0:
            continue
        assert torch.equal(kvc[s // 16, 0, :, s % 16], k[t]), f"K page row of token {t}"
        assert torch.equal(kvc[s // 16, 1, :, s % 16], v[t]), f"V page row of token {t}"
    used = torch.zeros(nblocks * 16, dtype=torch.bool)
    used[slots[slots >= 0].long()] = True
    untouched = kvc.permute(0, 3, 1, 2, 4).reshape(nblocks * 16, 2, Hkv, D)[~used.cuda()]
    assert not bool(untouched.any()), "only the named slots are written"


def test_kv_copy_blocks_at_the_head_dim_64_page_shape():
    Hkv, L, nb = 2, 3, 40
    block_bytes = 2 * Hkv * 16 * D * 2
    kv = rnd(L, nb, 2, Hkv, 16, D, seed=31).contiguous()
    before = kv.clone()
    src, dst = [3, 5, 3, 17], [20, 21, 22, 39]
    ops.kv_copy_blocks(kv, L, nb * block_bytes, block_bytes, src, dst)
    torch.cuda.synchronize()
    want = before.clone()
    for s, d in zip(src, dst):
        want[:, d] = before[:, s]
    assert torch.equal(kv.view(torch.int16), want.view(torch.int16))


# ------------------------------------------------------------------------------------------------------------ engine
from kubeai_b200.engine import Engine, config_from_hf, default_config, mini_config  # noqa: E402
from oracle.llama_oracle import LlamaOracle  # noqa: E402
from oracle.weights import ModelCfg, make_weights  # noqa: E402

SHAPES = {4: dict(hidden=512, q_heads=8, kv_heads=2, head_dim=64), 2: dict(hidden=512, q_heads=6, kv_heads=3, head_dim=64),
          8: dict(hidden=1024, q_heads=16, kv_heads=2, head_dim=64)}
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
        if float(m[-1] - m[-2]) < 0.25:
            return j
        assert a == b, f"greedy token {j}: engine {a} vs oracle {b}"
    return n


@pytest.mark.parametrize("G", [4, 2, 8])
def test_engine_logits_and_greedy_tokens_match_oracle(G):
    o = oracle(G)
    ps = prompts(40 + G, [37, 1, 16, 120, 200])
    with Engine(mini_config(**SHAPES[G])) as e:
        for p in ps[:2] + ps[3:4]:
            got = e.forward_logits(p)
            want = o.forward(p)[0].numpy()
            err = np.abs(got - want)
            assert (err <= 0.15 + 1.6e-2 * np.abs(want)).all() and err.mean() < 0.04, (G, len(p), err.max())
        outs = e.generate(ps, max_tokens=12)
    compared = sum(greedy_matches_oracle(o, p, out, 12) for p, out in zip(ps, outs))
    assert compared >= len(ps), compared


@pytest.mark.parametrize("G", [4, 2])
def test_engine_chunked_prefill_prefix_cache_and_preemption_follow_the_oracle(G):
    ps = prompts(50 + G, [230, 150, 90, 200, 17, 64])
    o = oracle(G)
    runs = []
    with Engine(mini_config(max_batched_tokens=48, **SHAPES[G])) as e:
        runs.append(e.generate(ps, max_tokens=20))
        runs.append(e.generate(ps, max_tokens=20))
        assert e.stats().cached_prompt_tokens > 0
    with Engine(mini_config(max_batched_tokens=96, **SHAPES[G])) as e:
        runs.append(e.generate(ps, max_tokens=20))
    with Engine(mini_config(num_kv_blocks=17, **SHAPES[G])) as e:
        runs.append(e.generate(ps, max_tokens=20))
        assert e.stats().preemptions > 0
    for p, *outs in zip(ps, *runs):
        want, rows = o.generate(p, 20)
        for out in outs:
            assert len(out) == 20
            for j, (a, b) in enumerate(zip(out, want)):
                m = torch.sort(rows[j])[0]
                if float(m[-1] - m[-2]) < 0.25:
                    break
                assert a == b, (len(p), j)


@pytest.mark.parametrize("G", [4, 2])
def test_engine_parallel_samples_fork_at_head_dim_64(G):
    """n = 4 members of one prefill (a 75-token prompt ends inside a page) sample what four separate requests sample."""
    p = prompts(60 + G, [75])[0]
    with Engine(mini_config(**SHAPES[G])) as e:
        rids = e.submit_n(p, 4, max_tokens=16, temperature=0.9, top_p=0.95, seed=321)
        got = {r: [] for r in rids}
        while e.step()[0]:
            for r in rids:
                got[r] += e.poll(r).tokens
        members = [got[r] + e.poll(r).tokens for r in rids]
        for r in rids:
            e.release(r)
        singles = []
        for i in range(4):
            rid = e.submit(p, max_tokens=16, temperature=0.9, top_p=0.95, seed=321 + i)
            toks = []
            while e.step()[0]:
                toks += e.poll(rid).tokens
            singles.append(toks + e.poll(rid).tokens)
            e.release(rid)
    assert members == singles
    assert len({tuple(m) for m in members}) > 1


@pytest.mark.parametrize("G", [4, 2, 8])
def test_engine_speculative_decoding_at_k_max(G):
    k = k_max(G)
    rng = np.random.default_rng(70 + G)
    ps = []
    for n in (23, 31, 40):
        b = rng.integers(0, 512, size=n).tolist()
        ps.append((b * 5)[: 5 * n - 3])
    with Engine(mini_config(num_speculative_tokens=k, prompt_lookup_min=1, prompt_lookup_max=3, **SHAPES[G])) as e:
        spec = e.generate(ps, max_tokens=24)
        st = e.stats()
    assert st.spec_draft_tokens > 0, st.spec_draft_tokens
    assert st.spec_draft_tokens <= k * st.spec_drafts
    o = oracle(G)
    assert sum(greedy_matches_oracle(o, p, s, 24) for p, s in zip(ps, spec)) >= len(ps)


@pytest.mark.parametrize("var", ["B200_FUSED_DECODE", "B200_FUSED_PREFILL"])
def test_unfused_forms_give_the_fused_bits(monkeypatch, var):
    """The separate RoPE / KV-write kernel and the fused qkv epilogue round alike at D = 64: same logits bits, same streams."""
    ps = prompts(80, [150, 170, 40, 129, 9])
    outs = {}
    for name in ("unfused", "fused"):
        monkeypatch.delenv(var, raising=False)
        if name == "unfused":
            monkeypatch.setenv(var, "0")
        with Engine(mini_config(max_num_seqs=8, max_batched_tokens=512, **SHAPES[4])) as e:
            outs[name] = e.generate(ps, max_tokens=12)
            outs[name + "_logits"] = e.forward_logits(ps[0]) if var == "B200_FUSED_PREFILL" else e.forward_logits(ps[2][:1])
    assert outs["fused"] == outs["unfused"]
    assert np.array_equal(outs["fused_logits"].view(np.uint32), outs["unfused_logits"].view(np.uint32))


def test_engine_loaded_from_tied_head_dim_64_checkpoint_matches_golden(tmp_path):
    from scripts.gen_golden_gqa import tied_weights
    from scripts.gen_golden_hd64 import HD64, write_checkpoint
    gold = np.load(Path(__file__).parent / "golden" / "llama_mini_hd64.npz")
    write_checkpoint(tmp_path)
    hc = json.loads((tmp_path / "config.json").read_text())
    assert hc["tie_word_embeddings"] is True and hc["head_dim"] == 64
    cfg = config_from_hf(tmp_path, max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=128,
                         manual_step=1, seed=999)
    assert (cfg.q_heads, cfg.kv_heads, cfg.head_dim, cfg.rope_scaling_type, cfg.rope_factor) == (8, 2, 64, 2, 32.0)
    w = tied_weights(ModelCfg(**HD64))
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
    o = LlamaOracle(ModelCfg(**HD64), w)
    assert greedy_matches_oracle(o, gold["ids"].tolist(), toks, 12) >= 1


# ------------------------------------------------------------------------------------------------- full size (1B shape)
import test_fullsize_gpu as F  # noqa: E402   the 8B layer tests, run here on the Llama-3.2-1B geometry

SHAPE_1B = dict(num_layers=1, hidden=2048, q_heads=32, kv_heads=8, head_dim=64, intermediate=8192, vocab=128256,
                max_model_len=2048, rope_scaling_type=2, rope_factor=32.0, rope_low_freq_factor=1.0, rope_high_freq_factor=4.0,
                rope_original_max_pos=8192)


@pytest.fixture(scope="module")
def layer_1b():
    from oracle.weights import bf16_bits_to_f32, cos_sin_cache
    e = Engine(default_config(manual_step=1, max_num_seqs=128, max_batched_tokens=1536, num_kv_blocks=128 * 129 + 64, **SHAPE_1B))
    cfg = ModelCfg(**SHAPE_1B)
    H, I, V = cfg.hidden, cfg.intermediate, cfg.vocab
    shapes = {"embed": (V, H), "lm_head": (V, H), "final_norm": (H,), "layers.0.wqkv": (cfg.qkv_rows, H),
              "layers.0.wo": (H, cfg.q_heads * D), "layers.0.wgu": (2 * I, H), "layers.0.wdown": (H, I),
              "layers.0.norm1": (H,), "layers.0.norm2": (H,)}
    w = {n: torch.from_numpy(bf16_bits_to_f32(e.tensor(n)).copy()).reshape(s) for n, s in shapes.items()}
    cs = O.r(torch.from_numpy(cos_sin_cache(cfg)))
    yield e, cfg, w, cs
    e.close()


# Share of the logits past F.LOGIT_ULPS_BULK ulps.  test_fullsize_gpu.py's 1e-5 was set at hidden 4096; at the 1B shape's
# hidden 2048 / intermediate 8192 a prefill of 128 tokens puts 5.5e-5 of them there at D = 64 and 7.1e-5 at D = 128 (a 16:4
# layer of the same shape), measured on an H100: the split-K orders of those GEMMs, not the head size, set it.
BULK_1B = 1e-4


@pytest.mark.parametrize("T", [128, 1536])
def test_llama32_1b_shape_prefill_logits_match_oracle(layer_1b, T):
    e, cfg, w, cs = layer_1b
    rng = np.random.default_rng(T)
    ids = rng.integers(0, cfg.vocab, size=T).tolist()
    got = e.forward_logits(ids)
    rows = sorted(set(range(0, T, max(1, T // 96))) | {T - 1, T - 2, 15, 16, 17})
    want = F.oracle_layer(cfg, w, cs, ids, rows)
    g = got[rows]
    err = np.abs(g - want)
    scale = F.ulp_bf16(np.maximum(np.abs(want), np.sqrt((want ** 2).mean(-1, keepdims=True))))
    assert (err <= F.LOGIT_ULPS * scale + 1e-3).all(), float((err / scale).max())
    assert float((err > F.LOGIT_ULPS_BULK * scale + 1e-3).mean()) < BULK_1B
    assert err.mean() < 0.5 * float(scale.mean())
    margin = np.sort(want, axis=-1)[:, -2:]
    solid = (margin[:, 1] - margin[:, 0]) > 4 * F.ulp_bf16(margin[:, 1])
    assert (g.argmax(-1)[solid] == want.argmax(-1)[solid]).all()


def test_llama32_1b_shape_decode_step_of_128_sequences_matches_oracle(layer_1b):
    F.test_full_size_decode_step_of_128_sequences_matches_oracle(layer_1b)


# ------------------------------------------------------------------------------------------------- vLLM parity
import test_vllm_parity_gpu as VP  # noqa: E402


@pytest.mark.skipif(not VP._vllm_ok(), reason="vllm is not importable (or B200_SKIP_VLLM=1)")
def test_logits_and_greedy_tokens_match_vllm_at_head_dim_64(tmp_path):
    from scripts.gen_golden_hd64 import write_checkpoint
    write_checkpoint(tmp_path)
    g = torch.Generator().manual_seed(91)
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
        res = VP._compare("2-layer test model, head_dim 64", llm, lambda p: logits[tuple(p)], mine, ps, N, topk=20)
    finally:
        del llm
        import gc
        gc.collect()
        torch.cuda.empty_cache()
    assert sum(r["identical_prefix"] == N for r in res["greedy"]) >= len(ps) // 2


# ------------------------------------------------------------------------------------------------- b200serve
def test_b200serve_answers_a_chat_request_on_a_head_dim_64_checkpoint(tmp_path):
    pytest.importorskip("tokenizers")
    from tokenizers import Regex, Tokenizer as HFTokenizer, decoders, models, pre_tokenizers, trainers
    from kubeai_b200._lib import LIB_PATH
    from scripts.gen_golden_hd64 import write_checkpoint
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
    srv = subprocess.Popen([str(bindir / "b200serve"), "--gpus", "1", "--model", "mini64", "--model-dir", str(tmp_path),
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
        body = dict(model="mini64", messages=[{"role": "user", "content": "hello world, how are you?"}], max_tokens=12,
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
