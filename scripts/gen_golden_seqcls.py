"""TEST INFRASTRUCTURE — generate tests/golden/llama_mini_seqcls.npz with HF transformers (run in the build container; the
GPU box only reads the committed fixture).

    python -m scripts.gen_golden_seqcls

A tiny LlamaForSequenceClassification with the seeded weights of oracle/weights.py and the score weights of
tests/rerank_common.py, at num_labels 1 and 3, run on the CPU in fp32 with one prompt per batch (so the pooled position is
the last one, whatever pad_token_id says).  It stores the prompt ids, their lengths, the score weights and transformers'
logits for each label count.
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
from rerank_common import hf_seq_cls_model, score_weight  # noqa: E402
from oracle.weights import ModelCfg  # noqa: E402

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden" / "llama_mini_seqcls.npz"
LENS = (1, 9, 48, 130)


def main():
    cfg = ModelCfg()
    rng = np.random.default_rng(17)
    prompts = [rng.integers(0, cfg.vocab, size=n).astype(np.int64) for n in LENS]
    out = dict(ids=np.concatenate(prompts), lens=np.array(LENS),
               cfg=np.array([cfg.num_layers, cfg.hidden, cfg.q_heads, cfg.kv_heads, cfg.head_dim, cfg.intermediate,
                             cfg.vocab, cfg.max_model_len, cfg.seed]))
    for L in (1, 3):
        m = hf_seq_cls_model(cfg, L, torch.float32)
        with torch.no_grad():
            out[f"logits_{L}"] = np.stack([m(torch.from_numpy(p)[None]).logits[0].float().numpy() for p in prompts])
        out[f"score_{L}"] = score_weight(cfg, L)
    OUT.parent.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    sys.exit(main())
