"""64-dimensional heads on the CPU: the head_dim rules of b200_config_from_hf and of b200_engine_create, the rotary table at
D = 64 against transformers', and the CPU oracle at D = 64 (Llama-3.2-1B geometry at test size: 8:2 heads, tied
embeddings, llama3 rope scaling) pinned against HF transformers (tests/golden/llama_mini_hd64.npz, made by
scripts/gen_golden_hd64.py)."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from kubeai_b200 import B200Error
from kubeai_b200.engine import config_from_hf, safetensors_list

GOLD = np.load(Path(__file__).parent / "golden" / "llama_mini_hd64.npz")
BASE = dict(model_type="llama", intermediate_size=1024, num_hidden_layers=2, vocab_size=512, rms_norm_eps=1e-5,
            rope_theta=500000.0, hidden_act="silu")
# Llama-3.2-1B's config.json (architecture fields)
LLAMA32_1B = dict(model_type="llama", hidden_size=2048, num_attention_heads=32, num_key_value_heads=8, head_dim=64,
                  intermediate_size=8192, num_hidden_layers=16, vocab_size=128256, rms_norm_eps=1e-5, rope_theta=500000.0,
                  hidden_act="silu", tie_word_embeddings=True, max_position_embeddings=131072, bos_token_id=128000,
                  eos_token_id=128001, rope_scaling=dict(factor=32.0, high_freq_factor=4.0, low_freq_factor=1.0,
                                                        original_max_position_embeddings=8192, rope_type="llama3"))
# TinyLlama-1.1B: no head_dim key, 2048 / 32 = 64, 32:4 heads
TINYLLAMA = dict(model_type="llama", hidden_size=2048, num_attention_heads=32, num_key_value_heads=4,
                 intermediate_size=5632, num_hidden_layers=22, vocab_size=32000, rms_norm_eps=1e-5, rope_theta=10000.0,
                 hidden_act="silu")


def _cfg(tmp_path, d):
    (tmp_path / "config.json").write_text(json.dumps(d))
    return config_from_hf(tmp_path)


def test_config_from_hf_accepts_llama32_1b(tmp_path):
    c = _cfg(tmp_path, LLAMA32_1B)
    assert (c.num_layers, c.hidden, c.q_heads, c.kv_heads, c.head_dim, c.intermediate, c.vocab) == \
           (16, 2048, 32, 8, 64, 8192, 128256)
    assert (c.rope_scaling_type, c.rope_factor, c.rope_original_max_pos) == (2, 32.0, 8192)


def test_config_from_hf_accepts_tinyllama_shape_without_a_head_dim_key(tmp_path):
    c = _cfg(tmp_path, TINYLLAMA)
    assert (c.q_heads, c.kv_heads, c.head_dim) == (32, 4, 64)


def test_config_from_hf_takes_an_explicit_head_dim_that_is_not_hidden_over_heads(tmp_path):
    c = _cfg(tmp_path, dict(BASE, hidden_size=1024, num_attention_heads=8, num_key_value_heads=2, head_dim=64))
    assert (c.hidden, c.q_heads, c.kv_heads, c.head_dim) == (1024, 8, 2, 64)
    c = _cfg(tmp_path, dict(BASE, hidden_size=1024, num_attention_heads=8, num_key_value_heads=8))
    assert c.head_dim == 128


@pytest.mark.parametrize("hd", [80, 96, 256])
def test_config_from_hf_refuses_other_head_sizes(tmp_path, hd):
    with pytest.raises(B200Error, match=rf"head_dim {hd} is not supported \(the kernels serve 64 and 128\)"):
        _cfg(tmp_path, dict(BASE, hidden_size=1024, num_attention_heads=8, num_key_value_heads=2, head_dim=hd))


def test_config_from_hf_refuses_an_odd_q_heads_at_head_dim_64(tmp_path):
    with pytest.raises(B200Error, match=r"head_dim 64 with 5 query heads is not supported \(q_heads \* head_dim must be a "
                                        r"multiple of 128: head_dim 64 needs an even q_heads\)"):
        _cfg(tmp_path, dict(BASE, hidden_size=1024, num_attention_heads=5, num_key_value_heads=1, head_dim=64))


def create_rc(**kw):
    from kubeai_b200 import _lib
    from kubeai_b200.engine import mini_config
    l = _lib.lib()
    e = C.c_void_p()
    rc = l.b200_engine_create(C.byref(mini_config(**kw)), C.byref(e))
    if rc == 0:
        l.b200_engine_destroy(e)
    return rc, l.b200_last_error().decode()


@pytest.mark.parametrize("hq, hkv, hd, ok", [(8, 2, 64, True), (8, 1, 64, True), (2, 1, 64, True), (6, 3, 64, True),
                                             (8, 8, 64, True), (5, 1, 64, False), (3, 3, 64, False), (4, 1, 96, False),
                                             (4, 1, 32, False), (4, 1, 0, True), (4, 1, 128, True)])
def test_create_applies_the_head_dim_rules(hq, hkv, hd, ok):
    """head_dim 64 or 128 (0 = 128) and whole 128-row slabs of q (an even q_heads at 64); an odd kv_heads is fine because
    the qkv epilogue classifies each 64-row half of a slab.  Refusals come before any device work (-5: no device here)."""
    rc, msg = create_rc(hidden=1024, q_heads=hq, kv_heads=hkv, head_dim=hd)
    if ok:
        assert rc in (0, -5), (hq, hkv, hd, rc, msg)
    else:
        assert rc == -1, (hq, hkv, hd, rc, msg)
        assert msg == (f"unsupported head_dim {hd} with {hq} query and {hkv} KV heads (head_dim 64 or 128; q_heads * head_dim "
                       "and (q_heads + 2 * kv_heads) * head_dim must be multiples of 128, so head_dim 64 needs an even "
                       "q_heads)"), msg


def test_cos_sin_cache_at_head_dim_64_with_llama3_scaling_matches_transformers():
    """The oracle's rotary table (the engine builds the same one) equals transformers' for the golden's config after the
    bf16 cast: cos | sin of the D / 2 = 32 frequencies."""
    from oracle.weights import ModelCfg, cos_sin_cache
    from scripts.gen_golden_hd64 import HD64
    cfg = ModelCfg(**HD64)
    cs = torch.from_numpy(cos_sin_cache(cfg)).bfloat16()
    assert cs.shape == (cfg.max_model_len, 64)
    hf = torch.cat([torch.from_numpy(GOLD["hf_cos"][:, :32]), torch.from_numpy(GOLD["hf_sin"][:, :32])], -1).bfloat16()
    assert torch.equal(torch.from_numpy(GOLD["hf_cos"][:, 32:]), torch.from_numpy(GOLD["hf_cos"][:, :32]))
    diff = (cs.float() - hf.float()).abs()
    # fp32 cos / sin of the same fp32 angles: a few entries may land on the other side of a bf16 rounding boundary
    assert (diff == 0).float().mean() >= 0.999 and float(diff.max()) <= 2 ** -8, (float((diff > 0).float().mean()), float(diff.max()))


def test_oracle_at_head_dim_64_with_tied_embeddings_matches_hf():
    from oracle import llama_oracle as O
    from oracle.weights import ModelCfg
    from scripts.gen_golden_gqa import tied_weights
    from scripts.gen_golden_hd64 import HD64
    cfg = ModelCfg(**HD64)
    assert cfg.head_dim == 64 and cfg.q_heads * cfg.head_dim == cfg.hidden
    assert GOLD["cfg"].tolist() == [cfg.num_layers, cfg.hidden, cfg.q_heads, cfg.kv_heads, cfg.head_dim, cfg.intermediate,
                                    cfg.vocab, cfg.max_model_len, cfg.seed]
    o = O.LlamaOracle(cfg, tied_weights(cfg))
    l = o.forward(GOLD["ids"])[0].numpy()
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


def test_config_from_hf_checks_head_dim_against_the_checkpoint(tmp_path):
    """A head_dim 64 checkpoint (hidden 512 = 8 * 64) gives head_dim 64; the same weights under a config.json that says
    128, or that drops head_dim so that hidden / q_heads is taken, are refused with the rows the checkpoint has."""
    from scripts.gen_golden_hd64 import write_checkpoint
    write_checkpoint(tmp_path)
    assert sorted(safetensors_list(tmp_path))[0].startswith("model.")
    c = config_from_hf(tmp_path)
    assert (c.hidden, c.q_heads, c.kv_heads, c.head_dim) == (512, 8, 2, 64)
    d = json.loads((tmp_path / "config.json").read_text())
    (tmp_path / "config.json").write_text(json.dumps(dict(d, head_dim=128)))
    with pytest.raises(B200Error, match=r"head_dim 128 does not match the checkpoint: layer 0 has q_proj / k_proj of "
                                        r"512 / 128 rows, not q_heads \* head_dim = 1024 / kv_heads \* head_dim = 256"):
        config_from_hf(tmp_path)
    (tmp_path / "config.json").write_text(json.dumps(dict(d, head_dim=128, hidden_size=1024)))
    with pytest.raises(B200Error, match="does not match the checkpoint"):
        config_from_hf(tmp_path)
