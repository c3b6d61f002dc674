"""Embeddings, CPU parts: the last-token pooling oracle against vLLM's normalize activation and HF transformers'
MistralModel / LlamaModel last_hidden_state (tests/golden/mistral_mini_embed.npz, made by scripts/gen_golden_embed.py), the
runner, sliding window and pooling config read from a checkpoint directory, ParseRequest on /v1/embeddings, and the bytes
a generate server keeps on the embeddings and models routes."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from embeddings_common import hf_base_model, hidden_rows, pool
from kubeai_b200 import B200Error
from kubeai_b200.engine import config_from_hf
from kubeai_b200.server import Server
from oracle.weights import ModelCfg

GOLDEN = Path(__file__).parent / "golden" / "mistral_mini_embed.npz"
ATOL, RTOL = 0.15, 1.6e-2   # DESIGN §2: bf16 rounding paths against each other


def test_oracle_matches_hf_last_hidden_state_on_the_golden():
    g = np.load(GOLDEN)
    cfg = ModelCfg()
    h = hidden_rows(cfg, g["ids"].tolist())
    for ref in (g["hidden_bf16"], g["hidden_fp32"]):
        assert (np.abs(h - ref) <= ATOL + RTOL * np.abs(ref)).all(), np.abs(h - ref).max()
    e = pool(h[-1])
    assert float(e @ g["embed_fp32"].astype(np.float64)) >= 0.9999


@pytest.mark.parametrize("arch", ["MistralModel", "LlamaModel"])
def test_oracle_matches_hf_base_models(arch):
    cfg = ModelCfg()
    ids = np.random.default_rng(1).integers(0, cfg.vocab, size=33).tolist()
    with torch.no_grad():
        ref = hf_base_model(cfg, arch, torch.float32)(torch.tensor([ids])).last_hidden_state[0].numpy()
    h = hidden_rows(cfg, ids)
    assert (np.abs(h - ref) <= ATOL + RTOL * np.abs(ref)).all()


def test_pool_is_vllm_last_pool_and_normalize():
    act = pytest.importorskip("vllm.model_executor.layers.pooler.activations")
    cfg = ModelCfg()
    h = hidden_rows(cfg, [5, 6, 7, 300, 2])
    last = torch.from_numpy(h)[-1:]   # LastPool: the last position of the sequence
    got = act.PoolerNormalize().forward_chunk(last)[0].numpy()
    want = pool(h[-1])
    assert np.abs(got - want).max() <= 4 * np.spacing(np.float32(1.0))
    assert np.array_equal(pool(h[-1], normalize=False), h[-1].astype(np.float64))
    assert (pool(np.zeros(8, np.float32)) == 0).all()


def _cfg_dir(tmp_path, **kw):
    c = dict(num_hidden_layers=2, hidden_size=512, num_attention_heads=4, num_key_value_heads=1, intermediate_size=1024,
             vocab_size=32000, rms_norm_eps=1e-5, rope_theta=10000.0, model_type="llama", architectures=["LlamaForCausalLM"])
    c.update(kw)
    (tmp_path / "config.json").write_text(json.dumps(c))
    return str(tmp_path)


@pytest.mark.parametrize("arch,model_type,sw,runner", [
    ("LlamaForCausalLM", "llama", None, 0), ("MistralForCausalLM", "mistral", 4096, 0), ("LlamaModel", "llama", None, 1),
    ("MistralModel", "mistral", 4096, 1), ("MistralModel", "mistral", None, 1)])
def test_config_from_hf_runner_and_sliding_window(tmp_path, arch, model_type, sw, runner):
    d = _cfg_dir(tmp_path, architectures=[arch], model_type=model_type, sliding_window=sw)
    c = config_from_hf(d)
    assert (c.runner, c.sliding_window) == (runner, sw or 0)
    c = config_from_hf(d, runner=1)          # vLLM's --runner pooling on any checkpoint: ForCausalLM resets it to 0
    assert c.runner == (0 if arch.endswith("ForCausalLM") else 1)


def test_config_from_hf_refuses_unknown_model_type_and_non_last_pooling(tmp_path):
    with pytest.raises(B200Error, match='model_type "qwen2" is not supported'):
        config_from_hf(_cfg_dir(tmp_path, model_type="qwen2"))
    d = _cfg_dir(tmp_path, architectures=["MistralModel"], model_type="mistral")
    (tmp_path / "modules.json").write_text(json.dumps([
        {"idx": 0, "name": "0", "path": "", "type": "sentence_transformers.models.Transformer"},
        {"idx": 1, "name": "1", "path": "1_Pooling", "type": "sentence_transformers.models.Pooling"},
        {"idx": 2, "name": "2", "path": "2_Normalize", "type": "sentence_transformers.models.Normalize"}]))
    (tmp_path / "1_Pooling").mkdir()
    modes = ["cls_token", "mean_tokens", "max_tokens", "mean_sqrt_len_tokens", "weightedmean_tokens", "lasttoken"]
    for mode in modes:
        (tmp_path / "1_Pooling" / "config.json").write_text(json.dumps(
            {"word_embedding_dimension": 512, **{f"pooling_mode_{m}": m == mode for m in modes}}))
        if mode == "lasttoken":
            assert config_from_hf(d).runner == 1
        else:
            with pytest.raises(B200Error, match=f'pooling mode "{mode}"'):
                config_from_hf(d)
    # last token beside another mode is refused too, naming the other one
    (tmp_path / "1_Pooling" / "config.json").write_text(json.dumps(
        {"pooling_mode_lasttoken": True, "pooling_mode_mean_tokens": True}))
    with pytest.raises(B200Error, match='pooling mode "mean_tokens"'):
        config_from_hf(d)
    # a generation checkpoint is not pooled: its sentence-transformers files are not read
    d = _cfg_dir(tmp_path, architectures=["MistralForCausalLM"], model_type="mistral")
    assert config_from_hf(d).runner == 0


@pytest.fixture()
def srv():
    with Server([None], model="model1", adapters=["adapter3"]) as s:
        yield s


def test_parse_request_on_embeddings(srv):
    st, r = srv.parse_request("/v1/embeddings", '{"model":"model1_adapter3","input":"some long text here"}', prefix_chars=4)
    assert st == 0 and (r["model"], r["adapter"], r["requested_model"], r["prefix"]) == ("model1", "adapter3", "model1_adapter3", "")
    st, r = srv.parse_request("/v1/embeddings", '{"model":"other","input":[1,2]}')
    assert (st, r["error"]) == (404, 'model not found: "other"')
    st, r = srv.parse_request("/v1/embeddings", '{"input":[1,2]}')
    assert (st, r["error"]) == (400, "bad request: reading model from body: missing 'model' field")


def test_generate_server_keeps_its_embeddings_and_models_bytes(srv):
    r = srv.handle("POST", "/openai/v1/embeddings", '{"model":"model1","input":"x"}')
    assert (r.status, r.body) == (404, b'{"error":"model not found: this engine serves TextGeneration only"}\n')
    r = srv.handle("GET", "/openai/v1/models")
    assert r.body == (b'{"object":"list","data":[{"id":"model1","object":"model","created":0,"owned_by":"kubeai-b200",'
                      b'"features":["TextGeneration"]},{"id":"model1_adapter3","object":"model","created":0,'
                      b'"owned_by":"kubeai-b200","features":["TextGeneration"]}]}')
