"""TEST INFRASTRUCTURE — the score-head oracle, HF sequence-classification checkpoints and a Llama-3-pipeline tokenizer for
the rerank tests.

The oracle restates what vLLM 0.22 runs for a *ForSequenceClassification checkpoint on its pooling runner
(model_executor/models/adapters.py as_seq_cls_model, layers/pooler/): LastPool takes the final-normed hidden row of the
last prompt position, the `score` linear runs in fp32 (head_dtype defaults to fp32 for pooling models) on that bf16 row,
and PoolerClassify applies get_act_fn's activation when use_activation: sigmoid for one label, softmax for more, or what
problem_type asks for.  Here the logits are taken in float64 from the bf16 row and the bf16 score weight.  The hidden rows
come from tests/embeddings_common.py (oracle/llama_oracle.py with an identity lm_head).
"""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

from embeddings_common import hidden_rows
from oracle.weights import ModelCfg, make_weights

SIGMOID, SOFTMAX, NONE = 1, 2, 3   # b200_config.score_activation (0 = by label count)


def resolve_activation(num_labels: int, activation: int = 0) -> int:
    return activation or (SIGMOID if num_labels == 1 else SOFTMAX)


def activate(logits, activation: int):
    """float64 [L]: get_act_fn's activation of one row of logits."""
    x = np.asarray(logits, dtype=np.float64)
    if activation == SIGMOID:
        return 1.0 / (1.0 + np.exp(-x))
    if activation == SOFTMAX:
        e = np.exp(x - x.max())
        return e / e.sum()
    return x


def score_weight(cfg: ModelCfg, num_labels: int, seed: int = 7) -> np.ndarray:
    """fp32 [L, H] of bf16-representable score weights (HF's normal init scale, seeded)."""
    g = torch.Generator().manual_seed(seed * 1000 + num_labels)
    w = torch.randn(num_labels, cfg.hidden, generator=g) * (2.0 / np.sqrt(cfg.hidden))
    return w.to(torch.bfloat16).float().numpy()


def logits(cfg: ModelCfg, ids, sw: np.ndarray, weights=None, hid=None) -> np.ndarray:
    """float64 [L]: the score logits of the last position of one prompt."""
    h = hid if hid is not None else hidden_rows(cfg, ids, weights)
    return h[-1].astype(np.float64) @ np.asarray(sw, dtype=np.float64).T


def scores(cfg: ModelCfg, ids, sw, activation: int = 0, use_activation: bool = True, weights=None, hid=None):
    x = logits(cfg, ids, sw, weights, hid)
    return activate(x, resolve_activation(len(sw), activation)) if use_activation else x


def logit_bound(cfg: ModelCfg, ids, sw, hid=None, atol=0.15, rtol=1.6e-2) -> np.ndarray:
    """float64 [L]: how far the engine's logits may lie from the oracle's when each bf16 hidden element lies within
    atol + rtol * |h| of the oracle's (DESIGN §2): sum_h |w[l, h]| * (atol + rtol * |y_h|)."""
    h = hid if hid is not None else hidden_rows(cfg, ids)
    y = np.abs(h[-1].astype(np.float64))
    return np.abs(np.asarray(sw, dtype=np.float64)) @ (atol + rtol * y)


def hf_seq_cls_model(cfg: ModelCfg, num_labels: int, dtype, arch: str = "LlamaForSequenceClassification",
                     tie_word_embeddings: bool = False, problem_type=None, sw=None):
    """transformers' LlamaForSequenceClassification (or Mistral's) with the seeded oracle weights and score_weight()."""
    from oracle.gen_golden import hf_model
    full = hf_model(cfg, make_weights(cfg), torch.float32)
    hc = full.config
    hc.num_labels = num_labels
    hc.problem_type = problem_type
    hc.pad_token_id = 0
    hc.tie_word_embeddings = tie_word_embeddings
    if arch.startswith("Mistral"):
        from transformers import MistralConfig, MistralForSequenceClassification
        mc = MistralConfig(**{k: v for k, v in hc.to_dict().items() if k not in ("model_type", "architectures")})
        mc.sliding_window = None
        mc._attn_implementation = "eager"
        m = MistralForSequenceClassification(mc)
    else:
        from transformers import LlamaForSequenceClassification
        m = LlamaForSequenceClassification(hc)
    sd = {k: v for k, v in full.state_dict().items() if k.startswith("model.") and "rotary" not in k}
    sd["score.weight"] = torch.from_numpy(score_weight(cfg, num_labels) if sw is None else sw)
    missing, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected and all("rotary" in k for k in missing), (missing, unexpected)
    m.config.architectures = [arch]
    return m.to(dtype).eval()


def write_seq_cls_checkpoint(d: Path, cfg: ModelCfg, num_labels: int, dtype=torch.bfloat16, **kw):
    m = hf_seq_cls_model(cfg, num_labels, dtype, **kw)
    m.save_pretrained(str(d), safe_serialization=True)
    return m


def edit_config(d: Path, **kw):
    p = Path(d) / "config.json"
    c = json.loads(p.read_text())
    for k, v in kw.items():
        if v is None:
            c.pop(k, None)
        else:
            c[k] = v
    p.write_text(json.dumps(c))


# ------------------------------------------------------------------ a tokenizer.json of the Llama-3 pipeline
PATTERN = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+")
SPECIALS = ["<|begin_of_text|>", "<|end_of_text|>", "<|start_header_id|>", "<|end_header_id|>", "<|eot_id|>"]
CORPUS = [
    "What is the capital of France? Paris is the capital and largest city of France.",
    "The quick brown fox jumps over the lazy dog. Reranking scores a query against each document.",
    "naïve café déjà vu, straße — ¿qué tal? Привет, мир! 你好，世界！ 12345 67 890",
] * 20


def llama3_tokenizer(path: Path, post_processor: str = "llama3", vocab_size: int = 500):
    """Write a tokenizer.json of the Llama-3 pipeline (trained on a small corpus, ids < vocab_size).  post_processor:
    "llama3" = Sequence[ByteLevel, TemplateProcessing] as Llama-3 ships it (single "<|begin_of_text|> $A", pair
    "<|begin_of_text|> $A <|begin_of_text|> $B:1"), "template" = a bare TemplateProcessing with another pair layout, "none"
    = no post-processor.  Returns the HF tokenizers object."""
    from tokenizers import Regex, Tokenizer, decoders, models, pre_tokenizers, processors, trainers
    tok = Tokenizer(models.BPE(ignore_merges=True))
    tok.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(PATTERN), behavior="isolated", invert=False),
                                                 pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    tr = trainers.BpeTrainer(vocab_size=vocab_size, special_tokens=SPECIALS,
                             initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False)
    tok.train_from_iterator(CORPUS, tr)
    bos, eot = tok.token_to_id("<|begin_of_text|>"), tok.token_to_id("<|eot_id|>")
    if post_processor == "llama3":
        tok.post_processor = processors.Sequence([
            processors.ByteLevel(trim_offsets=False),
            processors.TemplateProcessing(single="<|begin_of_text|> $A", pair="<|begin_of_text|> $A <|begin_of_text|> $B:1",
                                          special_tokens=[("<|begin_of_text|>", bos)])])
    elif post_processor == "template":
        tok.post_processor = processors.TemplateProcessing(
            single="<|begin_of_text|> $A <|eot_id|>", pair="<|begin_of_text|> $A <|eot_id|> $B:1 <|eot_id|>:1",
            special_tokens=[("<|begin_of_text|>", bos), ("<|eot_id|>", eot)])
    tok.save(str(path))
    return tok


# ------------------------------------------------------------------ vLLM's RerankResponse
def rerank_body(model: str, documents, scores_, prompt_tokens: int, top_n: int = 0) -> dict:
    """vLLM 0.22's ServingScores._request_output_to_rerank_response as a dict (the id left out): results in document
    order, sorted by relevance_score with Python's stable sort(reverse=True), cut to top_n when 0 < top_n <
    len(documents)."""
    results = [{"index": i, "document": {"text": d, "multi_modal": None}, "relevance_score": float(s)}
               for i, (d, s) in enumerate(zip(documents, scores_))]
    results.sort(key=lambda r: r["relevance_score"], reverse=True)
    n = top_n if top_n > 0 else len(documents)
    if n < len(documents):
        results = results[:n]
    return {"model": model, "usage": {"prompt_tokens": prompt_tokens, "total_tokens": prompt_tokens}, "results": results}
