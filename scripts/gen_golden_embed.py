"""TEST INFRASTRUCTURE — generate tests/golden/mistral_mini_embed.npz with HF transformers (run in the build container; the
GPU box only reads the committed fixture).

    python -m scripts.gen_golden_embed

A tiny MistralModel (the e5-mistral-7b-instruct architecture at test size: no lm_head, tensors without the "model." prefix)
with the seeded weights of oracle/weights.py and sliding_window = max_position_embeddings, so sliding-window attention is
full attention.  It stores the prompt ids, transformers' last_hidden_state in fp32 and in bf16, and the last-token
embedding L2-normalised in float64 from the fp32 row (vLLM's LastPool + normalize).
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
from embeddings_common import hf_base_model  # noqa: E402
from oracle.weights import ModelCfg  # noqa: E402

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "mistral_mini_embed.npz"


def main():
    cfg = ModelCfg()
    rng = np.random.default_rng(13)
    ids = rng.integers(0, cfg.vocab, size=48).astype(np.int64)
    x = torch.from_numpy(ids)[None]
    with torch.no_grad():
        h32 = hf_base_model(cfg, "MistralModel", torch.float32)(x).last_hidden_state[0].float().numpy()
        h16 = hf_base_model(cfg, "MistralModel", torch.bfloat16)(x).last_hidden_state[0].float().numpy()
    last = h32[-1].astype(np.float64)
    emb = last / max(np.linalg.norm(last), 1e-12)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, ids=ids, hidden_fp32=h32.astype(np.float32), hidden_bf16=h16.astype(np.float32),
                        embed_fp32=emb.astype(np.float32),
                        cfg=np.array([cfg.num_layers, cfg.hidden, cfg.q_heads, cfg.kv_heads, cfg.head_dim, cfg.intermediate,
                                      cfg.vocab, cfg.max_model_len, cfg.seed]))
    print("wrote", OUT, h32.shape)


if __name__ == "__main__":
    sys.exit(main())
