"""TEST INFRASTRUCTURE — generate tests/golden/llama_mini_hd64.npz with HF transformers (run in the build container; the
GPU box only reads the committed fixture).

    python -m scripts.gen_golden_hd64

The Llama-3.2-1B geometry at test size: 64-dimensional heads with 4 query heads per KV head (8:2, so hidden 512 is
q_heads * head_dim), tied embeddings and llama3 rope scaling with factor 32.  Weights come from oracle/weights.py with the
embedding tied to the lm_head matrix, and the logits from transformers' LlamaForCausalLM built with tie_word_embeddings=True,
as scripts/gen_golden_gqa.py does at G = 3.  `write_checkpoint` writes the same model as an HF checkpoint without an
lm_head tensor, as Llama-3.2-1B ships.
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

from oracle.weights import ModelCfg
from scripts.gen_golden_gqa import tied_hf_model

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "llama_mini_hd64.npz"
HD64 = dict(hidden=512, q_heads=8, kv_heads=2, head_dim=64, rope_scaling_type=2, rope_factor=32.0, rope_low_freq_factor=1.0,
            rope_high_freq_factor=4.0, rope_original_max_pos=64)


def write_checkpoint(d: Path, dtype=torch.bfloat16) -> ModelCfg:
    from safetensors.torch import save_file
    cfg = ModelCfg(**HD64)
    m = tied_hf_model(cfg, dtype)
    sd = {k: v.contiguous() for k, v in m.state_dict().items() if k != "lm_head.weight"}
    m.config.save_pretrained(d)
    save_file(sd, str(Path(d) / "model.safetensors"))
    return cfg


def main():
    cfg = ModelCfg(**HD64)
    rng = np.random.default_rng(11)
    ids = rng.integers(0, cfg.vocab, size=40).astype(np.int64)
    x = torch.from_numpy(ids)[None]
    with torch.no_grad():
        m32 = tied_hf_model(cfg, torch.float32)
        assert m32.config.head_dim == 64 and m32.lm_head.weight.data_ptr() == m32.model.embed_tokens.weight.data_ptr()
        l32 = m32(x).logits[0].float().numpy()
        l16 = tied_hf_model(cfg, torch.bfloat16)(x).logits[0].float().numpy()
        gen = m32.generate(x, max_new_tokens=12, do_sample=False)[0, len(ids):].numpy()
        # transformers' rotary table for this config (llama3 scaling), for the cos_sin_cache check
        rot = m32.model.rotary_emb
        pos = torch.arange(cfg.max_model_len)[None]
        cos, sin = rot(torch.zeros(1, dtype=torch.float32), pos)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, ids=ids, logits_fp32=l32.astype(np.float32), logits_bf16=l16.astype(np.float32),
                        greedy=gen.astype(np.int64), hf_cos=cos[0].numpy().astype(np.float32),
                        hf_sin=sin[0].numpy().astype(np.float32),
                        cfg=np.array([cfg.num_layers, cfg.hidden, cfg.q_heads, cfg.kv_heads, cfg.head_dim, cfg.intermediate,
                                      cfg.vocab, cfg.max_model_len, cfg.seed]))
    top2 = np.sort(l32, axis=-1)[:, -2:]
    print("wrote", OUT, l32.shape, "greedy", gen.tolist())
    print("logit std %.3f  mean top1-top2 margin %.3f  min margin %.4f" %
          (l32.std(), (top2[:, 1] - top2[:, 0]).mean(), (top2[:, 1] - top2[:, 0]).min()))


if __name__ == "__main__":
    sys.exit(main())
