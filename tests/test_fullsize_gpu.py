"""Parity at BASELINE config 2's model size (Llama-3-8B shapes: hidden 4096, 32 query / 8 KV heads of 128, intermediate 14336,
vocab 128256), default-on in the GPU suite (VERDICT r1 item 1):

  * one full-size decoder layer + lm_head through the engine against the oracle's ops on the same weights, for a
    T=128 prefill, a T=1536 prefill and a 128-sequence decode step over contexts 16..2047 (the production decode batch);
  * paged attention at Hq/Hkv = 32/8 with 128 sequences, contexts {16, 1023, 2048} and ragged ones, shuffled block
    tables, for decode and for chunked prefill on top of a cached prefix.

Tolerances.  Ops: vLLM's bf16 kernel tolerance (vllm/ir/tolerances.py:13-24: atol 1e-3, rtol 1.6e-2).  Logits: stated in
bf16 ulps — |got - want| <= LOGIT_ULPS * ulp_bf16(max(|want|, rms of the row)) + 1e-3, ulp_bf16(x) = 2^(floor(log2 x) - 7)
— a logit is one bf16 rounding of a 4096-term fp32 dot product of values that themselves carry up to one ulp of upstream
difference, so 2 ulps is the floor for two correct bf16 pipelines; the measured maxima are printed.  Asserted: every
logit within 6 ulps, all but 1e-5 of them within 3, mean under half an ulp.
"""
import math

import numpy as np
import pytest
import torch

from oracle import llama_oracle as O
from oracle.weights import ModelCfg, bf16_bits_to_f32, cos_sin_cache

pytestmark = pytest.mark.gpu
LOGIT_ULPS = 6.0          # hard bound; all but 1e-5 of the logits must be within LOGIT_ULPS_BULK
LOGIT_ULPS_BULK = 3.0
SHAPE = dict(num_layers=1, hidden=4096, q_heads=32, kv_heads=8, intermediate=14336, vocab=128256, max_model_len=2048)


def ulp_bf16(x: np.ndarray) -> np.ndarray:
    a = np.maximum(np.abs(x), 2.0 ** -20)
    return np.exp2(np.floor(np.log2(a)) - 7)


def logits_close(got, want, what):
    """|got - want| in bf16 ulps of max(|logit|, the row's RMS logit): a small logit is the cancellation of terms of the
    row's typical size, so its error scale is the row's, not its own."""
    err = np.abs(got - want)
    scale = ulp_bf16(np.maximum(np.abs(want), np.sqrt((want ** 2).mean(-1, keepdims=True))))
    tol = LOGIT_ULPS * scale + 1e-3
    worst = float((err / scale).max())
    print(f"{what}: max |dlogit| {err.max():.4f}, max error {worst:.2f} bf16 ulps of the logit, mean |dlogit| {err.mean():.5f}")
    assert (err <= tol).all(), f"{what}: {int((err > tol).sum())} of {err.size} logits outside {LOGIT_ULPS} ulps (worst {worst:.2f})"
    assert float((err > LOGIT_ULPS_BULK * scale + 1e-3).mean()) < 1e-5, "all but 1e-5 of the logits within 3 ulps"
    assert err.mean() < 0.5 * float(scale.mean()), "mean error under half an ulp"
    return worst


@pytest.fixture(scope="module")
def layer():
    """A one-layer engine at the full shapes and its weights as oracle tensors (read back through the C ABI; the seeded
    init itself is pinned bit-exactly on the numpy replica by test_engine_gpu.py)."""
    from kubeai_b200.engine import Engine, default_config
    e = Engine(default_config(manual_step=1, max_num_seqs=128, max_batched_tokens=1536, num_kv_blocks=128 * 129 + 64, **SHAPE))
    cfg = ModelCfg(**SHAPE)
    names = ["embed", "final_norm", "lm_head"] + ["layers.0." + n for n in ("wqkv", "wo", "wgu", "wdown", "norm1", "norm2")]
    w = {}
    for n in names:
        w[n] = torch.from_numpy(bf16_bits_to_f32(e.tensor(n)).copy())
    H, I, V = cfg.hidden, cfg.intermediate, cfg.vocab
    for n, shp in (("embed", (V, H)), ("lm_head", (V, H)), ("layers.0.wqkv", (cfg.qkv_rows, H)), ("layers.0.wo", (H, H)),
                   ("layers.0.wgu", (2 * I, H)), ("layers.0.wdown", (H, I))):
        w[n] = w[n].reshape(shp)
    cs = O.r(torch.from_numpy(cos_sin_cache(cfg)))
    yield e, cfg, w, cs
    e.close()


def oracle_layer(cfg, w, cs, ids, rows):
    """Logits of the positions `rows` of one sequence `ids` through the one-layer model (oracle ops, full prefill)."""
    D, Hq, Hkv = cfg.head_dim, cfg.q_heads, cfg.kv_heads
    n = len(ids)
    pos = torch.arange(n)
    hidden = w["embed"][torch.as_tensor(ids, dtype=torch.long)]
    h = O.rms_norm(hidden, w["layers.0.norm1"], cfg.rms_eps)
    qkv = O.gemm(h, w["layers.0.wqkv"])
    q = O.rope_neox(qkv[:, :Hq * D].reshape(n, Hq, D), pos, cs)
    k = O.rope_neox(qkv[:, Hq * D:(Hq + Hkv) * D].reshape(n, Hkv, D), pos, cs)
    v = qkv[:, (Hq + Hkv) * D:].reshape(n, Hkv, D)
    rows = torch.as_tensor(rows, dtype=torch.long)
    a = O.attention(q[rows], k, v, pos[rows], 1.0 / math.sqrt(D)).reshape(len(rows), Hq * D)
    o = O.gemm(a, w["layers.0.wo"])
    h2, res = O.fused_add_rms_norm(o, hidden[rows], w["layers.0.norm2"], cfg.rms_eps)
    down = O.gemm(O.silu_and_mul(O.gemm(h2, w["layers.0.wgu"])), w["layers.0.wdown"])
    hf, _ = O.fused_add_rms_norm(down, res, w["final_norm"], cfg.rms_eps)
    return O.gemm(hf, w["lm_head"]).numpy()


@pytest.mark.parametrize("T", [128, 1536])
def test_full_size_layer_prefill_logits_match_oracle(layer, T):
    e, cfg, w, cs = layer
    rng = np.random.default_rng(T)
    ids = rng.integers(0, cfg.vocab, size=T).tolist()
    got = e.forward_logits(ids)
    rows = sorted(set(range(0, T, max(1, T // 96))) | {T - 1, T - 2, 15, 16, 17})
    want = oracle_layer(cfg, w, cs, ids, rows)
    logits_close(got[rows], want, f"prefill T={T} ({len(rows)} rows x {cfg.vocab})")
    margin = np.sort(want, axis=-1)[:, -2:]
    solid = (margin[:, 1] - margin[:, 0]) > 4 * ulp_bf16(margin[:, 1])
    assert (got[rows].argmax(-1)[solid] == want.argmax(-1)[solid]).all()


def test_full_size_decode_step_of_128_sequences_matches_oracle(layer):
    """The production decode batch: 128 sequences with contexts from 17 to 2047 tokens (ragged last pages), prefilled in
    chunks by the scheduler while the earlier ones already decode; the first step in which ALL 128 decode (T = 128, the
    shape of ~80% of the bench's steps) is compared row by row with the oracle's last-position logits."""
    e, cfg, w, cs = layer
    rng = np.random.default_rng(5)
    # the longest prompt is submitted (hence prefilled) last: it decodes exactly once before it reaches max_model_len, and
    # that one step is the step in which all 128 sequences decode together
    lens = [16, 17, 31, 1023, 1024, 1025, 500, 33] + rng.integers(16, 1900, size=117).tolist() + [1990, 2020, 2046]
    prompts = [rng.integers(0, cfg.vocab, size=n).tolist() for n in lens]
    e.set_keep_logits(True)
    rids = [e.submit(p, max_tokens=400) for p in prompts]
    gen = [[] for _ in rids]
    lg = None
    try:
        hist = []
        for _ in range(600):
            ran, info = e.step()
            st = e.stats()
            assert ran, f"engine idle after {len(hist)} steps: running {st.running} waiting {st.waiting} kv_free {st.kv_blocks_free} " \
                        f"preemptions {st.preemptions}; last steps (T, decode, prefill): {hist[-12:]}; finished: " \
                        f"{[(i, len(g), e.poll(r).finished) for i, (g, r) in enumerate(zip(gen, rids)) if e.poll(r).finished][:8]}"
            hist.append((info.tokens, info.decode_seqs, info.prefill_seqs))
            for i, r in enumerate(rids):
                gen[i] += e.poll(r).tokens
            if info.prefill_seqs == 0 and info.decode_seqs == len(rids):
                assert info.tokens == len(rids) and info.sampled == len(rids)
                lg = e.read_logits(len(rids))       # rows in scheduling order = submission order
                break
    finally:
        for r in rids:
            e.release(r)
        e.set_keep_logits(False)
        while e.step()[0]:                            # released while running: the engine drops them at its next step
            pass
    assert lg is not None, "no step with all 128 sequences decoding"
    ctx = [lens[i] + len(gen[i]) - 1 for i in range(len(rids))]      # tokens each row attended over (incl. itself)
    assert max(ctx) == 2047 and min(ctx) < 150
    assert all(int(lg[i].argmax()) == gen[i][-1] for i in range(len(rids))), "the sampled id is the argmax of the kept logits"
    sel = sorted(range(len(rids)), key=lambda i: ctx[i])
    sel = sel[:4] + sel[-4:] + sel[4:-4:6]            # the extremes and every 6th in between (CPU time of the oracle)
    G = lg[sel]
    Wn = np.stack([oracle_layer(cfg, w, cs, prompts[i] + gen[i][:-1], [ctx[i] - 1])[0] for i in sel])
    logits_close(G, Wn, f"decode step T=128, {len(sel)} of 128 sequences (contexts {min(ctx)}..{max(ctx)})")
    m = np.sort(Wn, axis=-1)[:, -2:]
    solid = (m[:, 1] - m[:, 0]) > 4 * ulp_bf16(m[:, 1])
    assert (G.argmax(-1)[solid] == Wn.argmax(-1)[solid]).all()


@pytest.mark.parametrize("mode", ["fused_epilogues", "fp32_segments"])
def test_full_size_prefill_burst_step_matches_oracle(layer, mode, monkeypatch):
    """A prefill burst as the scheduler runs it (T = 1500 new tokens of four prompts in ONE step, the sampled rows only):
    the GEMMs with RoPE / SiLU*up / residual add in their epilogues (default) and with plain outputs plus the separate
    elementwise kernels (B200_FUSED_PREFILL=0), each against the oracle."""
    from kubeai_b200.engine import Engine, default_config
    _, cfg, w, cs = layer
    monkeypatch.setenv("B200_FUSED_PREFILL", "0" if mode == "fp32_segments" else "1")
    rng = np.random.default_rng(77)
    lens = [700, 450, 300, 50]
    prompts = [rng.integers(0, cfg.vocab, size=n).tolist() for n in lens]
    with Engine(default_config(manual_step=1, max_num_seqs=8, max_batched_tokens=1536, num_kv_blocks=256, **SHAPE)) as e:
        e.set_keep_logits(True)
        rids = [e.submit(p, max_tokens=2) for p in prompts]
        ran, info = e.step()
        assert ran and info.tokens == sum(lens) and info.prefill_seqs == len(lens) and info.sampled == len(lens)
        got = e.read_logits(len(lens))
        launches = e.stats().kernel_launches
        for r in rids:
            e.release(r)
    want = np.stack([oracle_layer(cfg, w, cs, p, [len(p) - 1])[0] for p in prompts])
    logits_close(got, want, f"prefill burst T={sum(lens)} ({mode})")
    _BURST[mode] = (got, launches)
    if len(_BURST) == 2:   # both forms round at the same points: same bits, fewer launches with the fused epilogues
        assert np.array_equal(_BURST["fused_epilogues"][0], _BURST["fp32_segments"][0]), "the two forms differ"
        assert _BURST["fused_epilogues"][1] < _BURST["fp32_segments"][1]


_BURST = {}


# --------------------------------------------------------------------------------------------- attention, production shape
def _pool(seq_lens, Hkv, seed, extra=7):
    """Random bf16 K/V for every sequence scattered into a shuffled page pool [blocks][K|V][head][16][128]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    nb_total = sum((l + 15) // 16 for l in seq_lens) + extra
    perm = torch.randperm(nb_total, generator=torch.Generator().manual_seed(seed)).tolist()
    kv = torch.zeros(nb_total, 2, Hkv, 16, 128, dtype=torch.bfloat16, device="cuda")
    max_blocks = (max(seq_lens) + 15) // 16
    btab = torch.zeros(len(seq_lens), max_blocks, dtype=torch.int32)
    ks, vs = [], []
    for s, L in enumerate(seq_lens):
        nb = (L + 15) // 16
        blocks = torch.tensor([perm.pop() for _ in range(nb)])
        btab[s, :nb] = blocks.int()
        k = torch.randn(nb * 16, Hkv, 128, generator=g, device="cuda").bfloat16()
        v = torch.randn(nb * 16, Hkv, 128, generator=g, device="cuda").bfloat16()
        kv[blocks.cuda(), 0] = k.reshape(nb, 16, Hkv, 128).permute(0, 2, 1, 3)
        kv[blocks.cuda(), 1] = v.reshape(nb, 16, Hkv, 128).permute(0, 2, 1, 3)
        ks.append(k[:L].float())
        vs.append(v[:L].float())     # rows past L stay in the page as (finite) garbage the kernel must mask
    return kv, btab.cuda(), ks, vs


def _attn_close(got, want, what):
    err = (got - want).abs()
    tol = 4e-3 + 1.6e-2 * want.abs()          # vLLM bf16 tolerance (rtol 1.6e-2) + bf16 rounding of P and of the output
    assert bool((err <= tol).all()), f"{what}: max err {float(err.max()):.4g}, {int((err > tol).sum())} outside tolerance"


def test_decode_attention_at_production_shape():
    """Hq/Hkv = 32/8, 128 sequences, contexts {16, 1023, 2048} plus ragged lengths, shuffled block tables."""
    from kubeai_b200 import ops
    Hq, Hkv = 32, 8
    rng = np.random.default_rng(9)
    lens = [16, 1023, 2048, 1, 15, 17, 2047, 1024] + rng.integers(1, 2049, size=120).tolist()
    kv, btab, ks, vs = _pool(lens, Hkv, seed=21)
    g = torch.Generator(device="cuda").manual_seed(3)
    q = torch.randn(len(lens), (Hq + 2 * Hkv) * 128, generator=g, device="cuda").bfloat16()
    # work items in a shuffled order (the engine sorts them longest-first; any order must work)
    order = rng.permutation(len(lens)).tolist()
    work = torch.tensor([[i, 1, lens[i] - 1, i] for i in order], dtype=torch.int32).cuda()
    got = ops.paged_attn(q, kv, btab, work, Hq, Hkv, decode=True).float()
    torch.cuda.synchronize()
    for i, L in enumerate(lens):
        qi = q[i, :Hq * 128].float().reshape(1, Hq, 128)
        want = O.attention(qi, ks[i], vs[i], torch.tensor([L - 1], device="cuda"), 128 ** -0.5).reshape(1, Hq * 128)
        _attn_close(got[i:i + 1], want, f"decode seq {i} ctx {L}")


@pytest.mark.parametrize("split", [2, 5, 16, 32])
def test_split_kv_decode_attention_matches_oracle_and_the_unsplit_kernel(split):
    """Few decoding sequences: each context is cut into `split` slices streamed by different CTAs, partial softmax states
    merged by a second kernel.  Slices may be empty (a 1-token context split 32 ways)."""
    from kubeai_b200 import ops
    Hq, Hkv = 32, 8
    lens = [2048, 1023, 17, 300, 1, 64, 65, 1999]
    kv, btab, ks, vs = _pool(lens, Hkv, seed=23)
    g = torch.Generator(device="cuda").manual_seed(5)
    q = torch.randn(len(lens), (Hq + 2 * Hkv) * 128, generator=g, device="cuda").bfloat16()
    work = torch.tensor([[i, 1, L - 1, i] for i, L in enumerate(lens)], dtype=torch.int32).cuda()
    base = ops.paged_attn(q, kv, btab, work, Hq, Hkv, decode=True).float()
    for rep in range(2):
        got = ops.paged_attn(q, kv, btab, work, Hq, Hkv, decode=True, split=split).float()
        torch.cuda.synchronize()
        for i, L in enumerate(lens):
            qi = q[i, :Hq * 128].float().reshape(1, Hq, 128)
            want = O.attention(qi, ks[i], vs[i], torch.tensor([L - 1], device="cuda"), 128 ** -0.5).reshape(1, Hq * 128)
            _attn_close(got[i:i + 1], want, f"split {split} seq {i} ctx {L}")
        # against the one-CTA form: only the order of the fp32 merge differs
        assert float((got - base).abs().max()) <= 2 ** -7 * float(base.abs().max()) + 1e-3
    assert torch.equal(ops.paged_attn(q, kv, btab, work, Hq, Hkv, decode=True, split=1).float(), base)


@pytest.mark.parametrize("kernel", ["tensor_core", "mma_sync"])
def test_chunked_prefill_attention_at_production_shape_with_cached_prefix(kernel):
    from kubeai_b200 import ops
    Hq, Hkv = 32, 8
    qb = 64 if kernel == "tensor_core" else 16
    case = [(2048, 512), (1023, 1023), (16, 16), (1500, 37), (2047, 1), (777, 300), (64, 64), (1025, 1000)]   # (context, new tokens)
    lens = [c[0] for c in case]
    kv, btab, ks, vs = _pool(lens, Hkv, seed=22)
    T = sum(n for _, n in case)
    g = torch.Generator(device="cuda").manual_seed(4)
    q = torch.randn(T, (Hq + 2 * Hkv) * 128, generator=g, device="cuda").bfloat16()
    work, spans, tok = [], [], 0
    for i, (L, n) in enumerate(case):
        for j in range(0, n, qb):
            work.append([tok + j, min(qb, n - j), L - n + j, i])
        spans.append(tok)
        tok += n
    wt = torch.tensor(work, dtype=torch.int32).cuda()
    got = (ops.paged_attn_prefill_tc(q, kv, btab, wt, Hq, Hkv) if kernel == "tensor_core"
           else ops.paged_attn(q, kv, btab, wt, Hq, Hkv, decode=False)).float()
    torch.cuda.synchronize()
    for i, (L, n) in enumerate(case):
        t0 = spans[i]
        qi = q[t0:t0 + n, :Hq * 128].float().reshape(n, Hq, 128)
        want = O.attention(qi, ks[i], vs[i], torch.arange(L - n, L, device="cuda"), 128 ** -0.5).reshape(n, Hq * 128)
        _attn_close(got[t0:t0 + n], want, f"prefill seq {i} ctx {L} new {n}")
