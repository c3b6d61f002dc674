"""TEST INFRASTRUCTURE — CPU restatement of the reference backend's per-step model math.

The reference (kubeai-project/kubeai) holds no model arithmetic: its backend is the third-party
vLLM pod (`vllm/vllm-openai:v0.10.2`, /root/reference/charts/kubeai/values.yaml:45-46, launched by
/root/reference/internal/modelcontroller/engine_vllm.go:82-100).  This file restates the published
vLLM Llama forward with its rounding points (paths inside the vllm 0.22.0 wheel of this image, the
closest available version):

  rms_norm                        vllm/ir/ops/layernorm.py:9-21
  fused_add_rms_norm              vllm/_custom_ops.py:323-327 (_C CUDA op: bf16 sum, then norm of the rounded sum)
  neox RoPE, bf16 cos/sin cache   vllm/model_executor/layers/rotary_embedding/base.py:70-92,140-198
                                  vllm/model_executor/layers/rotary_embedding/common.py:144-183
  SiluAndMul                      vllm/model_executor/layers/activation.py:117-148
  decoder layer / MLP / attention vllm/model_executor/models/llama.py:81-121,223-233,316-340
  greedy sampling                 vllm/v1/sample/sampler.py:91,235-236

Pinning: the reference's own tests hold NO vector for model math (SURVEY.md §8c "parity unpinned"
at the reference level); this restatement is pinned against HF transformers 5.5 LlamaForCausalLM
run in this container (oracle/gen_golden.py -> tests/golden/llama_mini.npz).

Every tensor here is a float32 torch tensor whose values are bf16-representable wherever the
backend would hold bf16 ("r(x)" rounds to bf16 and returns float32).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .weights import ModelCfg, bf16_bits_to_f32, cos_sin_cache


def r(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (nearest-even), keep float32 storage."""
    return x.to(torch.bfloat16).to(torch.float32)


def to_torch(bits: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(bf16_bits_to_f32(bits).copy())


def gemm(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """bf16 x bf16 -> fp32 accumulate -> bf16 (linear without bias, weight [N, K])."""
    return r(x @ w.t())


def rms_norm(x, w, eps):
    var = x.pow(2).mean(dim=-1, keepdim=True)
    y = x * torch.rsqrt(var + eps)
    return r(r(y) * w)


def fused_add_rms_norm(x, residual, w, eps):
    """residual += x in bf16, then RMSNorm of the ROUNDED sum — the semantics of vLLM's CUDA op
    (vllm/_custom_ops.py:323-327 -> torch.ops._C.fused_add_rms_norm: `z = input + residual` in scalar_t,
    variance and normalisation from z) and of HF transformers (modeling_llama.py:325,328-329 + :62-67).
    vLLM's python IR op (vllm/ir/ops/layernorm.py:42-60) keeps the fp32 sum instead; the two differ by one
    double rounding of the normalised value.  The engine follows the CUDA-op form because its GEMM residual-add epilogue
    stores the summed residual in bf16 and the next RMSNorm normalises that (gemm_wgmma.cu)."""
    z = r(x + residual)
    var = z.pow(2).mean(dim=-1, keepdim=True)
    y = z * torch.rsqrt(var + eps)
    return r(r(y) * w), z


def rope_neox(x, positions, cs_bf16):
    """x: [T, heads, D]; cs_bf16: [max_pos, D] (cos|sin) already rounded to bf16 (D = 128 in the engine)."""
    cs = cs_bf16[positions]
    h = x.shape[-1] // 2
    cos, sin = cs[:, None, :h], cs[:, None, h:]
    x1, x2 = x[..., :h], x[..., h:]
    o1 = r(r(x1 * cos) - r(x2 * sin))
    o2 = r(r(x2 * cos) + r(x1 * sin))
    return torch.cat([o1, o2], dim=-1)


def silu_and_mul(gu):
    d = gu.shape[-1] // 2
    g, u = gu[..., :d], gu[..., d:]
    return r(r(g / (1.0 + torch.exp(-g))) * u)


def attention(q, k, v, q_pos, scale):
    """q: [Tq, Hq, 128], k/v: [Tk, Hkv, 128] (positions 0..Tk-1), causal by absolute position."""
    Tq, Hq, _ = q.shape
    Tk, Hkv, _ = k.shape
    g = Hq // Hkv
    kk = k.repeat_interleave(g, dim=1)
    vv = v.repeat_interleave(g, dim=1)
    s = torch.einsum("qhd,khd->hqk", q, kk) * scale
    mask = torch.arange(Tk, device=q.device)[None, :] > q_pos[:, None]
    s = s.masked_fill(mask[None], float("-inf"))
    p = torch.softmax(s, dim=-1)
    return r(torch.einsum("hqk,khd->qhd", p, vv))


class LlamaOracle:
    def __init__(self, cfg: ModelCfg, weights: dict):
        self.cfg = cfg
        self.w = {k: to_torch(v) for k, v in weights.items()}
        self.cs = r(torch.from_numpy(cos_sin_cache(cfg)))

    @torch.no_grad()
    def forward(self, ids, kv_prefix=None, pos0: int = 0):
        """Logits [n, V] for the tokens `ids` appended after `pos0` cached positions.
        kv_prefix: list per layer of (k [pos0, Hkv, 128], v) or None.  Returns (logits, kv)."""
        c = self.cfg
        D = c.head_dim
        ids = torch.as_tensor(ids, dtype=torch.long)
        n = ids.numel()
        pos = torch.arange(pos0, pos0 + n)
        scale = 1.0 / math.sqrt(D)
        hidden = self.w["embed"][ids]
        residual = None
        kv_out = []
        for l in range(c.num_layers):
            p = f"layers.{l}."
            if residual is None:
                residual = hidden
                h = rms_norm(hidden, self.w[p + "norm1"], c.rms_eps)
            else:
                h, residual = fused_add_rms_norm(hidden, residual, self.w[p + "norm1"], c.rms_eps)
            qkv = gemm(h, self.w[p + "wqkv"])
            q = qkv[:, : c.q_heads * D].reshape(n, c.q_heads, D)
            k = qkv[:, c.q_heads * D: (c.q_heads + c.kv_heads) * D].reshape(n, c.kv_heads, D)
            v = qkv[:, (c.q_heads + c.kv_heads) * D:].reshape(n, c.kv_heads, D)
            q = rope_neox(q, pos, self.cs)
            k = rope_neox(k, pos, self.cs)
            if kv_prefix is not None:
                k_all = torch.cat([kv_prefix[l][0], k], dim=0)
                v_all = torch.cat([kv_prefix[l][1], v], dim=0)
            else:
                k_all, v_all = k, v
            kv_out.append((k_all, v_all))
            a = attention(q, k_all, v_all, pos, scale).reshape(n, c.q_heads * D)
            hidden = gemm(a, self.w[p + "wo"])
            h, residual = fused_add_rms_norm(hidden, residual, self.w[p + "norm2"], c.rms_eps)
            gu = gemm(h, self.w[p + "wgu"])
            act = silu_and_mul(gu)
            hidden = gemm(act, self.w[p + "wdown"])
        h, _ = fused_add_rms_norm(hidden, residual, self.w["final_norm"], c.rms_eps)
        logits = gemm(h, self.w["lm_head"])
        return logits, kv_out

    @torch.no_grad()
    def generate(self, prompt, max_tokens: int):
        """Greedy decode with a KV cache; returns (tokens, per-step logits of the sampled row)."""
        logits, kv = self.forward(prompt)
        toks, rows = [], []
        pos = len(prompt)
        for _ in range(max_tokens):
            row = logits[-1]
            t = int(torch.argmax(row))  # lowest index wins ties (torch semantics)
            toks.append(t)
            rows.append(row.clone())
            logits, kv = self.forward([t], kv_prefix=kv, pos0=pos)
            pos += 1
        return toks, rows
