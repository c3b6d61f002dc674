"""Group sizes other than 4 query heads per KV head, on the CPU: the config rules of b200_config_from_hf and of
b200_engine_create (the speculative draft cap k_max(G) = min(3, 16 / G - 1)), and the CPU oracle at G = 3 with tied
embeddings and llama3 rope scaling pinned against HF transformers (tests/golden/llama_mini_gqa3.npz, made by
scripts/gen_golden_gqa.py)."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

from kubeai_b200 import B200Error
from kubeai_b200.engine import config_from_hf

GOLD = np.load(Path(__file__).parent / "golden" / "llama_mini_gqa3.npz")
BASE = dict(model_type="llama", hidden_size=1024, intermediate_size=1024, num_hidden_layers=2, vocab_size=512,
            head_dim=128, rms_norm_eps=1e-5, rope_theta=500000.0, hidden_act="silu")


def k_max(G):
    return min(3, 16 // G - 1)


def _cfg(tmp_path, hq, hkv):
    (tmp_path / "config.json").write_text(json.dumps(dict(BASE, num_attention_heads=hq, num_key_value_heads=hkv)))
    return config_from_hf(tmp_path)


@pytest.mark.parametrize("hq, hkv", [(8, 8), (24, 8), (8, 1), (16, 1), (32, 8)])
def test_config_from_hf_accepts_group_sizes_1_to_16(tmp_path, hq, hkv):
    c = _cfg(tmp_path, hq, hkv)
    assert (c.q_heads, c.kv_heads) == (hq, hkv)


@pytest.mark.parametrize("hq, hkv", [(5, 2), (32, 1), (8, 3)])
def test_config_from_hf_refuses_other_ratios(tmp_path, hq, hkv):
    with pytest.raises(B200Error, match=rf"GQA ratio {hq}:{hkv} is not supported \(kv_heads must divide q_heads, "
                                        r"with 1 to 16 query heads per KV head\)"):
        _cfg(tmp_path, hq, hkv)


def test_k_max_table():
    assert [k_max(G) for G in range(1, 17)] == [3, 3, 3, 3, 2, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0]


def create_rc(**kw):
    from kubeai_b200 import _lib
    from kubeai_b200.engine import mini_config
    l = _lib.lib()
    e = C.c_void_p()
    rc = l.b200_engine_create(C.byref(mini_config(**kw)), C.byref(e))
    if rc == 0:
        l.b200_engine_destroy(e)
    return rc, l.b200_last_error().decode()


@pytest.mark.parametrize("hq, hkv", [(2, 2), (6, 2), (4, 1), (5, 1), (6, 1), (8, 1), (9, 1), (16, 1)])
def test_create_refuses_drafts_past_k_max(hq, hkv):
    """num_speculative_tokens above k_max(G) is refused before any device work, with a message naming G and the cap;
    k_max(G) itself is accepted (-5: no device on this host)."""
    G = hq // hkv
    for k in range(0, 4):
        rc, msg = create_rc(hidden=1024, q_heads=hq, kv_heads=hkv, num_speculative_tokens=k)
        if k <= k_max(G):
            assert rc in (0, -5), (G, k, rc, msg)
        else:
            assert rc == -1, (G, k, rc, msg)
            assert msg == (f"num_speculative_tokens={k} exceeds {k_max(G)}, the most drafts a verify step holds with "
                           f"{G} query heads per KV head"), msg


def test_oracle_at_group_size_3_with_tied_embeddings_matches_hf():
    from oracle import llama_oracle as O
    from oracle.weights import ModelCfg
    from scripts.gen_golden_gqa import GQA3, tied_weights
    cfg = ModelCfg(**GQA3)
    assert cfg.q_heads // cfg.kv_heads == 3
    assert GOLD["cfg"].tolist() == [cfg.num_layers, cfg.hidden, cfg.q_heads, cfg.kv_heads, cfg.intermediate, cfg.vocab,
                                    cfg.max_model_len, cfg.seed]
    o = O.LlamaOracle(cfg, tied_weights(cfg))
    l = o.forward(GOLD["ids"])[0].numpy()
    # the tied logits reach |23|: the bf16 oracle must be no farther from HF's fp32 model than HF's own bf16 model is
    ref = GOLD["logits_fp32"]
    err, hf_err = np.abs(l - ref), np.abs(GOLD["logits_bf16"] - ref)
    assert err.max() <= hf_err.max() and err.mean() <= hf_err.mean(), (err.max(), hf_err.max(), err.mean(), hf_err.mean())
    err = np.abs(l - GOLD["logits_bf16"])
    assert (err <= 0.25 + 1.6e-2 * np.abs(GOLD["logits_bf16"])).all() and err.mean() < 0.04, err.max()
    toks, rows = o.generate(GOLD["ids"].tolist(), 12)
    for j, (a, b) in enumerate(zip(toks, GOLD["greedy"].tolist())):
        m = np.sort(rows[j].numpy())
        if m[-1] - m[-2] < 0.25:
            break
        assert a == b, j
