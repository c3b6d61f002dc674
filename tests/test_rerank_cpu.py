"""Rerank, CPU parts: the score-head config read from a *ForSequenceClassification checkpoint and its refusals, the
create-time rules, the score oracle against HF transformers' LlamaForSequenceClassification
(tests/golden/llama_mini_seqcls.npz, made by scripts/gen_golden_seqcls.py), pair tokenization against the HF `tokenizers`
wheel, ParseRequest on /v1/rerank of a server without a score head, and the oracle's response builder against vLLM's
pydantic RerankResponse."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from kubeai_b200 import B200Error
from kubeai_b200.engine import Engine, config_from_hf, mini_config
from kubeai_b200.server import Server
from oracle.weights import ModelCfg
from rerank_common import activate, hf_seq_cls_model, llama3_tokenizer, logits, rerank_body, score_weight

GOLDEN = Path(__file__).parent / "golden" / "llama_mini_seqcls.npz"


def _cfg_dir(tmp_path, **kw):
    c = dict(num_hidden_layers=2, hidden_size=512, num_attention_heads=4, num_key_value_heads=1, intermediate_size=1024,
             vocab_size=512, rms_norm_eps=1e-5, rope_theta=10000.0, model_type="llama",
             architectures=["LlamaForSequenceClassification"])
    for k, v in kw.items():
        if v is None:
            c.pop(k, None)
        else:
            c[k] = v
    (tmp_path / "config.json").write_text(json.dumps(c))
    return str(tmp_path)


@pytest.mark.parametrize("arch,model_type", [("LlamaForSequenceClassification", "llama"),
                                             ("MistralForSequenceClassification", "mistral")])
def test_config_from_hf_reads_the_score_head(tmp_path, arch, model_type):
    def cfg(**kw):
        return config_from_hf(_cfg_dir(tmp_path, architectures=[arch], model_type=model_type, **kw))
    c = cfg()   # HF's default: 2 labels, no problem_type, use_sep_token true
    assert (c.runner, c.num_labels, c.score_activation, c.score_join_pair) == (1, 2, 0, 0)
    assert cfg(id2label={"0": "LABEL_0"}).num_labels == 1
    assert cfg(id2label={str(i): f"L{i}" for i in range(5)}).num_labels == 5
    assert cfg(num_labels=7, id2label={"0": "a"}).num_labels == 7   # num_labels wins over id2label
    assert cfg(num_labels=32).num_labels == 32
    # vLLM's get_act_fn
    for pt, n, act in [("regression", 1, 3), ("regression", 4, 3), ("single_label_classification", 1, 1),
                       ("single_label_classification", 3, 2), ("multi_label_classification", 1, 1),
                       ("multi_label_classification", 3, 1), (None, 1, 0), (None, 3, 0)]:
        assert cfg(num_labels=n, problem_type=pt).score_activation == act, (pt, n)
    assert cfg(use_sep_token=True).score_join_pair == 0
    assert cfg(use_sep_token=False).score_join_pair == 1
    # a causal LM or base model keeps no head
    for a in ("LlamaForCausalLM", "LlamaModel"):
        c = config_from_hf(_cfg_dir(tmp_path, architectures=[a], num_labels=3), num_labels=2)
        assert c.num_labels == 0 and c.runner == (0 if a.endswith("CausalLM") else 1)


def test_config_from_hf_refusals(tmp_path):
    with pytest.raises(B200Error, match="33 labels is not supported: a score head has 1 to 32 labels"):
        config_from_hf(_cfg_dir(tmp_path, num_labels=33))
    with pytest.raises(B200Error, match="0 labels is not supported"):
        config_from_hf(_cfg_dir(tmp_path, num_labels=0))
    with pytest.raises(B200Error, match="architecture BertForSequenceClassification is not supported"):
        config_from_hf(_cfg_dir(tmp_path, architectures=["BertForSequenceClassification"], model_type="bert"))
    with pytest.raises(B200Error, match="architecture LlamaForTokenClassification is not supported"):
        config_from_hf(_cfg_dir(tmp_path, architectures=["LlamaForTokenClassification"]))
    with pytest.raises(B200Error, match='problem_type "ordinal" is not supported'):
        config_from_hf(_cfg_dir(tmp_path, problem_type="ordinal"))
    # the sentence-transformers pooling check of the embedding path applies to a score head too
    d = _cfg_dir(tmp_path)
    (tmp_path / "modules.json").write_text(json.dumps([
        {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"}]))
    (tmp_path / "1_Pooling").mkdir()
    (tmp_path / "1_Pooling" / "config.json").write_text(json.dumps({"pooling_mode_mean_tokens": True}))
    with pytest.raises(B200Error, match='pooling mode "mean_tokens"'):
        config_from_hf(d)


def test_create_time_rules_are_checked_before_the_device():
    for kw, msg in [(dict(num_labels=1), "a score head \\(num_labels = 1\\) needs the pooling runner"),
                    (dict(runner=1, num_labels=33), "num_labels 33 is not supported"),
                    (dict(runner=1, num_labels=-1), "num_labels -1 is not supported"),
                    (dict(runner=1, num_labels=1, score_activation=4), "score_activation must be 0"),
                    (dict(runner=1, num_labels=1, score_activation=-1), "score_activation must be 0")]:
        with pytest.raises(B200Error, match=msg) as ei:
            Engine(mini_config(**kw))
        assert ei.value.code == -1


def test_oracle_matches_hf_sequence_classification_on_the_golden():
    g = np.load(GOLDEN)
    cfg = ModelCfg()
    ids = np.split(g["ids"], np.cumsum(g["lens"])[:-1])
    for L in (1, 3):
        assert np.array_equal(g[f"score_{L}"], score_weight(cfg, L))
        for p, want in zip(ids, g[f"logits_{L}"]):
            got = logits(cfg, p.tolist(), g[f"score_{L}"])
            # the oracle's bf16 rows against transformers' fp32 forward
            assert np.allclose(got, want, atol=0.05, rtol=0.02), (L, got, want)


def test_activations_are_vllm_get_act_fn():
    x = np.array([-3.0, 0.5, 2.0])
    t = torch.from_numpy(x)
    assert np.allclose(activate(x, 1), torch.sigmoid(t).numpy())
    assert np.allclose(activate(x, 2), torch.softmax(t, -1).numpy())
    assert np.array_equal(activate(x, 3), x)
    # HF's LlamaForSequenceClassification score head is the same linear
    cfg = ModelCfg()
    m = hf_seq_cls_model(cfg, 3, torch.float32)
    assert np.array_equal(m.score.weight.detach().numpy(), score_weight(cfg, 3))


@pytest.fixture(scope="module")
def toks(tmp_path_factory):
    from kubeai_b200.tokenizer import Tokenizer
    out = {}
    for pp in ("llama3", "template", "none"):
        path = tmp_path_factory.mktemp("tok") / "tokenizer.json"
        hf = llama3_tokenizer(path, pp)
        out[pp] = (hf, Tokenizer(path))
    yield out
    for _, mine in out.values():
        mine.close()


PAIRS = [("What is the capital of France?", "Paris is the capital and largest city of France."),
         ("q", ""), ("", "d"), ("naïve café", " 你好，世界！ 12345"), ("a<|eot_id|>b", "c <|begin_of_text|> d"),
         ("  spaces  ", "\n\nnewlines\r\n"), ("The quick brown fox", "jumps over the lazy dog.")]


@pytest.mark.parametrize("pp", ["llama3", "template", "none"])
def test_pair_ids_equal_hf_tokenizers(toks, pp):
    hf, mine = toks[pp]
    for q, d in PAIRS:
        assert mine.encode_pair(q, d) == hf.encode(q, d).ids, (pp, q, d)                       # use_sep_token true
        assert mine.encode_pair(q, d, join=True) == hf.encode(q + d).ids, (pp, q, d)           # use_sep_token false
        assert mine.encode_pair(q, d, add_special_tokens=False) == hf.encode(q, d, add_special_tokens=False).ids
        assert mine.encode_pair(q, d, join=True, add_special_tokens=False) == hf.encode(q + d, add_special_tokens=False).ids
    if pp == "llama3":   # Llama-3's pair layout: <|begin_of_text|> A <|begin_of_text|> B
        bos = hf.token_to_id("<|begin_of_text|>")
        ids = mine.encode_pair("q", "d")
        assert ids[0] == bos and ids.count(bos) == 2


def test_rerank_parse_request_without_a_score_head_is_unchanged():
    """A generate server (and, on the GPU, an embedding server) keeps ParseRequest's 400 on /v1/rerank and its 404 route."""
    with Server([None], model="test-model") as s:
        st, r = s.parse_request("/v1/rerank", '{"model": "test-model", "query": "q", "documents": ["d"]}')
        assert (st, r["error"]) == (400, 'bad request: reading model from body: unknown path: "/v1/rerank"')
        st, r = s.parse_request("/v1/rerank", '{"model": "test-model", "query": 1}')
        assert (st, r["error"]) == (400, 'bad request: reading model from body: unknown path: "/v1/rerank"')
        h = s.handle("POST", "/openai/v1/rerank", '{"model":"test-model","query":"q","documents":["d"]}')
        assert (h.status, h.body) == (404, b'{"error":"model not found: this engine serves TextGeneration only"}\n')


@pytest.mark.parametrize("top_n", [0, -1, 1, 2, 4, 5, 9])
def test_response_builder_is_vllm_rerank_response(top_n):
    proto = pytest.importorskip("vllm.entrypoints.pooling.scoring.protocol")
    docs = ["a", "b", "c", "d", "e"]
    sc = np.array([0.25, 0.75, 0.25, 0.9, 0.75], dtype=np.float32)   # ties keep document order
    results = [proto.RerankResult(index=i, document=proto.RerankDocument(text=d), relevance_score=float(s))
               for i, (d, s) in enumerate(zip(docs, sc))]
    results.sort(key=lambda x: x.relevance_score, reverse=True)    # vLLM's _request_output_to_rerank_response
    n = top_n if top_n > 0 else len(results)
    if n < len(docs):
        results = results[:n]
    want = proto.RerankResponse(id="score-x", model="m", results=results,
                                usage=proto.RerankUsage(prompt_tokens=40, total_tokens=40)).model_dump()
    want.pop("id")
    assert rerank_body("m", docs, sc, 40, top_n) == want
    assert [r["index"] for r in want["results"]][:3] == [3, 1, 4][:min(3, n)]
