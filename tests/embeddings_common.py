"""TEST INFRASTRUCTURE — the last-token pooling oracle and HF base-model checkpoints for the embedding tests.

The oracle restates vLLM 0.22's embed pooling (model_executor/layers/pooler/: LastPool, then PoolerNormalize, i.e.
F.normalize of the pooled row): the final-normed bf16 hidden row of the last prompt position, converted to fp32 and
normalised in float64 as x / max(||x||, 1e-12).  The hidden rows come from oracle/llama_oracle.py with its lm_head replaced
by the identity, so the "logits" it returns are the final-normed rows themselves (a bf16 row times the identity is exact).
"""
from __future__ import annotations

from pathlib import Path

import numpy as np
import torch

from oracle.llama_oracle import LlamaOracle
from oracle.weights import ModelCfg, make_weights


def hidden_rows(cfg: ModelCfg, ids, weights=None) -> np.ndarray:
    """fp32 [n, H] of the bf16 final-normed hidden rows of one sequence."""
    o = LlamaOracle(cfg, weights if weights is not None else make_weights(cfg))
    o.w["lm_head"] = torch.eye(cfg.hidden, dtype=torch.float32)
    h, _ = o.forward(list(ids))
    return h.numpy().astype(np.float32)


def pool(h_last: np.ndarray, normalize: bool = True) -> np.ndarray:
    """float64 [H]: the last position's row, L2-normalised when normalize."""
    x = np.asarray(h_last, dtype=np.float32).astype(np.float64)
    return x / max(float(np.linalg.norm(x)), 1e-12) if normalize else x


def hf_base_model(cfg: ModelCfg, arch: str, dtype, sliding_window=None):
    """transformers' MistralModel or LlamaModel (arch) with the seeded oracle weights."""
    from oracle.gen_golden import hf_model
    full = hf_model(cfg, make_weights(cfg), torch.float32)
    sd = {k[len("model."):]: v for k, v in full.state_dict().items() if k.startswith("model.")}
    if arch == "MistralModel":
        from transformers import MistralConfig, MistralModel
        hc = MistralConfig(vocab_size=cfg.vocab, hidden_size=cfg.hidden, intermediate_size=cfg.intermediate,
                           num_hidden_layers=cfg.num_layers, num_attention_heads=cfg.q_heads,
                           num_key_value_heads=cfg.kv_heads, head_dim=cfg.head_dim,
                           max_position_embeddings=cfg.max_model_len, rms_norm_eps=cfg.rms_eps,
                           rope_parameters=dict(rope_type="default", rope_theta=cfg.rope_theta),
                           sliding_window=sliding_window if sliding_window is not None else cfg.max_model_len,
                           tie_word_embeddings=False, hidden_act="silu")
        hc._attn_implementation = "eager"
        m = MistralModel(hc)
    else:
        from transformers import LlamaModel
        hc = full.config
        m = LlamaModel(hc)
    m.load_state_dict({k: v for k, v in sd.items() if "rotary" not in k}, strict=False)
    m.config.architectures = [arch]
    return m.to(dtype).eval()


def write_base_checkpoint(d: Path, cfg: ModelCfg, arch: str = "MistralModel", dtype=torch.bfloat16, shards: int = 1,
                          sliding_window=None):
    """An HF checkpoint of a base model as transformers writes it: tensors without the "model." prefix, no lm_head."""
    m = hf_base_model(cfg, arch, dtype, sliding_window)
    m.save_pretrained(str(d), max_shard_size=("1GB" if shards == 1 else "200KB"), safe_serialization=True)
    return m


def write_word_tokenizer(d: Path, vocab: int):
    """A word-level HF tokenizer over ids 0..vocab-1 ("t<id>"), for tools that need a tokenizer beside a checkpoint whose
    prompts are given as token ids."""
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    tok = Tokenizer(models.WordLevel({f"t{i}": i for i in range(vocab)}, unk_token="t0"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="t0", bos_token="t1", eos_token="t2").save_pretrained(str(d))
