"""Parity of the engine against the vLLM wheel of this image — the closest runnable stand-in for the reference's backend
pod (the repo pins vllm/vllm-openai:v0.10.2, charts/kubeai/values.yaml:45; the image has 0.22) — both loading the SAME HF
checkpoint.  Default-on whenever `import vllm` works (VERDICT r1 item 1c); B200_SKIP_VLLM=1 skips it (vLLM needs a few
minutes to start).  Two things are compared on >= 32 prompts:

  * LOGITS, through vLLM's prompt logprobs: for every prompt position the log-probabilities vLLM reports (the prompt's own
    next token and its top-k) against log_softmax of the engine's bf16 logits at that position.  Stated tolerance:
    |d logprob| <= LOGPROB_ULPS bf16 ulps of the position's largest |logit| (ulp_bf16(x) = 2^(floor(log2|x|) - 7): 0.0625 at
    |x| in 8..16, 0.125 at 16..32) — two correct bf16 pipelines differ by the rounding of the final 4096-term dot product
    (1 ulp) plus what the layers' bf16 intermediates feed into it.  The measured maxima of every run go to the JSON
    report (REPORT).
  * greedy TOKENS: streams may part only where vLLM's own top-2 candidates are within MARGIN_ULPS bf16 ulps of the top
    logit of each other.  MARGIN_ULPS = 4 is the measured bound on how far ONE logit of the 32-layer model moves between the
    two pipelines (max |d logprob| 3.7-4 ulps over three runs): a margin below it can flip.  Observed first-difference
    margins over three runs of 64 prompts: 0 (exact ties) .. 0.375 = 3 ulps at |logit| 16..32; the seeded random weights
    give near-flat distributions, which is what makes ties this common.
"""
import json
import os
from pathlib import Path

import numpy as np
import pytest
import torch


def _vllm_ok():
    if os.environ.get("B200_SKIP_VLLM") == "1":
        return False
    try:
        import vllm  # noqa: F401
        return True
    except Exception:
        return False


pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not _vllm_ok(), reason="vllm is not importable (or B200_SKIP_VLLM=1)")]
LOGPROB_ULPS = 6.0
MARGIN_ULPS = 4.0
REPORT = Path(__file__).resolve().parent.parent / "gpurun_out" / "vllm_parity.json"


def ulp_bf16(x):
    return np.exp2(np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** -20))) - 7)


def _compare(name, llm, engine_logits, engine_greedy, prompts, N, topk):
    """engine_logits(p) -> fp32 [len(p), V]; engine_greedy: list of token lists."""
    from vllm import SamplingParams
    sp = SamplingParams(temperature=0.0, max_tokens=N, ignore_eos=True, detokenize=False, logprobs=2, prompt_logprobs=topk)
    outs = llm.generate([{"prompt_token_ids": p} for p in prompts], sp)
    worst_ulps, worst_abs, n_cmp, sum_abs = 0.0, 0.0, 0, 0.0
    top1_agree = top1_total = 0
    for p, o in zip(prompts, outs):
        lg = engine_logits(p)                                    # [len, V]
        lse = np.log(np.exp((lg - lg.max(-1, keepdims=True)).astype(np.float64)).sum(-1)) + lg.max(-1).astype(np.float64)
        for j in range(1, len(p)):
            d = o.prompt_logprobs[j]
            if not d:
                continue
            toks = np.fromiter(d.keys(), dtype=np.int64)
            ref = np.array([d[int(t)].logprob for t in toks], dtype=np.float64)
            keep = np.isfinite(ref)
            toks, ref = toks[keep], ref[keep]
            mine = lg[j - 1, toks].astype(np.float64) - lse[j - 1]
            err = np.abs(mine - ref)
            scale = ulp_bf16(np.abs(lg[j - 1]).max())
            worst_ulps = max(worst_ulps, float((err / scale).max()))
            worst_abs = max(worst_abs, float(err.max()))
            sum_abs += float(err.sum())
            n_cmp += len(err)
            ranks = {int(t): d[int(t)].rank for t in toks}
            r1 = [t for t, r in ranks.items() if r == 1]
            if r1:
                top1_total += 1
                top1_agree += int(int(lg[j - 1].argmax()) == r1[0])
    report = []
    for p, o, got in zip(prompts, outs, engine_greedy):
        ref = list(o.outputs[0].token_ids)
        k = next((j for j in range(N) if ref[j] != got[j]), N)
        margin = None
        if k < N:
            lp = sorted((v.logprob for v in o.outputs[0].logprobs[k].values()), reverse=True)
            margin = lp[0] - lp[1] if len(lp) > 1 else float("inf")
        report.append((len(p), k, margin))
    top_ulp = float(ulp_bf16(np.array([max(float(np.abs(engine_logits(p)[-1]).max()) for p in prompts)])).max())
    res = dict(model=name, prompts=len(prompts), logprobs_compared=n_cmp, max_abs_dlogprob=round(worst_abs, 4),
               max_dlogprob_in_bf16_ulps_of_the_logit=round(worst_ulps, 2), mean_abs_dlogprob=round(sum_abs / max(1, n_cmp), 5),
               prompt_top1_agreement=[top1_agree, top1_total],
               greedy=[dict(prompt_len=a, identical_prefix=b, of=N, vllm_top2_margin_at_first_difference=c) for a, b, c in report])
    print(json.dumps(res))
    try:
        if REPORT.parent.is_dir():
            prev = json.loads(REPORT.read_text()) if REPORT.exists() else []
            REPORT.write_text(json.dumps(prev + [res], indent=1))
    except OSError:
        pass
    assert n_cmp > 0
    assert worst_ulps <= LOGPROB_ULPS, f"{name}: logprob differs by {worst_ulps:.2f} bf16 ulps of the logit (> {LOGPROB_ULPS})"
    # a top-2 margin can flip when it is under the sum of the two candidates' deviations: MARGIN_ULPS, or twice the worst
    # one-logit deviation this very run measured (itself bounded by LOGPROB_ULPS above), whichever is larger
    allowed = max(MARGIN_ULPS, 2.0 * worst_ulps) * top_ulp + 1e-3
    for plen, k, margin in report:
        assert k == N or margin <= allowed, (plen, k, margin, top_ulp, worst_ulps)
    return res


def _llm(path, max_len, util):
    os.environ.setdefault("HF_HUB_OFFLINE", "1")
    os.environ.setdefault("VLLM_NO_USAGE_STATS", "1")
    from vllm import LLM
    return LLM(model=str(path), skip_tokenizer_init=True, dtype="bfloat16", max_model_len=max_len, enforce_eager=True,
               gpu_memory_utilization=util, enable_prefix_caching=False, seed=0)


def test_logits_and_greedy_tokens_match_vllm_on_the_test_model(tmp_path):
    from safetensors.torch import save_file
    from kubeai_b200.engine import Engine, config_from_hf
    from oracle.gen_golden import hf_model
    from oracle.weights import ModelCfg, make_weights
    cfg = ModelCfg()
    m = hf_model(cfg, make_weights(cfg), torch.bfloat16)
    m.config.save_pretrained(tmp_path)
    save_file({k: v.contiguous() for k, v in m.state_dict().items()}, str(tmp_path / "model.safetensors"))
    g = torch.Generator().manual_seed(17)
    lens = [5, 16, 33, 70, 121, 200] + torch.randint(2, 220, (26,), generator=g).tolist()
    prompts = [torch.randint(0, cfg.vocab, (int(n),), generator=g).tolist() for n in lens]
    N = 24
    ecfg = config_from_hf(tmp_path, max_model_len=256, max_num_seqs=16, max_batched_tokens=256, num_kv_blocks=256,
                          manual_step=1, seed=777)
    with Engine(ecfg) as e:
        e.load_safetensors(tmp_path)
        mine = e.generate(prompts, max_tokens=N)
        logits = {tuple(p): e.forward_logits(p) for p in prompts}
    llm = _llm(tmp_path, 256, 0.25)
    res = _compare("2-layer test model (hidden 512, vocab 512)", llm, lambda p: logits[tuple(p)], mine, prompts, N, topk=20)
    assert sum(g["identical_prefix"] == N for g in res["greedy"]) >= len(prompts) // 2


@pytest.mark.skipif(os.environ.get("B200_SKIP_VLLM_8B") == "1", reason="B200_SKIP_VLLM_8B=1 (writes a 16 GB checkpoint)")
def test_full_size_llama3_8b_logits_and_greedy_tokens_match_vllm(tmp_path):
    """BASELINE config 2's model: the engine's seeded Llama-3-8B weights are exported as an HF checkpoint, vLLM loads it,
    and both sides' logits (prompt logprobs) and greedy streams are compared on 32 prompts of 5..700 tokens."""
    from safetensors.torch import save_file
    from transformers import LlamaConfig
    from kubeai_b200.engine import Engine, default_config
    L, H, I, V, Hq, Hkv, D = 32, 4096, 14336, 128256, 32, 8, 128
    g = torch.Generator().manual_seed(23)
    lens = [5, 17, 64, 150, 333, 700] + torch.randint(8, 400, (26,), generator=g).tolist()
    prompts = [torch.randint(0, 128000, (int(n),), generator=g).tolist() for n in lens]
    N = 16

    def bf16(bits: np.ndarray, rows: int, cols: int) -> torch.Tensor:
        return torch.from_numpy(bits.view(np.int16).reshape(rows, cols)).view(torch.bfloat16)

    logits_dir = tmp_path / "engine_logits"
    logits_dir.mkdir()
    with Engine(default_config(manual_step=1, max_num_seqs=32, max_batched_tokens=2048, max_model_len=2048, kv_fraction=0.05)) as e:
        mine = e.generate(prompts, max_tokens=N)
        for i, p in enumerate(prompts):
            np.save(logits_dir / f"{i}.npy", e.forward_logits(p).astype(np.float32))
        weight_map = {}

        def dump(fn, tensors):
            save_file({k: v.contiguous() for k, v in tensors.items()}, str(tmp_path / fn))
            weight_map.update({k: fn for k in tensors})

        dump("model-head.safetensors", {
            "model.embed_tokens.weight": bf16(e.tensor("embed"), V, H), "lm_head.weight": bf16(e.tensor("lm_head"), V, H),
            "model.norm.weight": bf16(e.tensor("final_norm"), 1, H).reshape(H)})
        for l in range(L):
            p, q = f"layers.{l}.", f"model.layers.{l}."
            wqkv = bf16(e.tensor(p + "wqkv"), (Hq + 2 * Hkv) * D, H)
            wgu = bf16(e.tensor(p + "wgu"), 2 * I, H)
            dump(f"model-layer-{l:02d}.safetensors", {
                q + "self_attn.q_proj.weight": wqkv[:Hq * D], q + "self_attn.k_proj.weight": wqkv[Hq * D:(Hq + Hkv) * D],
                q + "self_attn.v_proj.weight": wqkv[(Hq + Hkv) * D:], q + "self_attn.o_proj.weight": bf16(e.tensor(p + "wo"), H, Hq * D),
                q + "mlp.gate_proj.weight": wgu[:I], q + "mlp.up_proj.weight": wgu[I:],
                q + "mlp.down_proj.weight": bf16(e.tensor(p + "wdown"), H, I),
                q + "input_layernorm.weight": bf16(e.tensor(p + "norm1"), 1, H).reshape(H),
                q + "post_attention_layernorm.weight": bf16(e.tensor(p + "norm2"), 1, H).reshape(H)})
    (tmp_path / "model.safetensors.index.json").write_text(json.dumps({"metadata": {}, "weight_map": weight_map}))
    LlamaConfig(vocab_size=V, hidden_size=H, intermediate_size=I, num_hidden_layers=L, num_attention_heads=Hq,
                num_key_value_heads=Hkv, max_position_embeddings=2048, rms_norm_eps=1e-5, rope_theta=500000.0,
                tie_word_embeddings=False, torch_dtype="bfloat16", bos_token_id=1, eos_token_id=2).save_pretrained(tmp_path)
    llm = _llm(tmp_path, 2048, 0.45)
    index = {tuple(p): i for i, p in enumerate(prompts)}
    res = _compare("Llama-3-8B shape, seeded random weights", llm, lambda p: np.load(logits_dir / f"{index[tuple(p)]}.npy"),
                   mine, prompts, N, topk=5)
    assert any(g["identical_prefix"] == N for g in res["greedy"])
