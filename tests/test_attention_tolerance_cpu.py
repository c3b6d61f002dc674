"""The per-(row, head) attention bound of the GPU suite (max |err| <= RMS_C * rms(want), test_attention_exact_gpu.py) on
the CPU: it accepts the attention kernels' rounding (P rounded to bf16 before P . V, fp32 sums, one bf16 rounding of the
output) and rejects a single wrong token in 1-8K tokens of context, which vLLM's bf16 tolerance alone lets through."""
import pytest
import torch

from oracle import llama_oracle as O
from test_attention_exact_gpu import RMS_C, rms_ratio

Hq, Hkv, D = 32, 8, 128
SCALE = D ** -0.5


def bf16_p_attention(q, k, v):
    """The kernels' rounding: fp32 scores and exponentials, P rounded to bf16 for P . V, the fp32 row sum unrounded."""
    kk, vv = k.repeat_interleave(Hq // Hkv, 1), v.repeat_interleave(Hq // Hkv, 1)
    s = torch.einsum("qhd,khd->hqk", q, kk) * SCALE
    p = torch.exp(s - s.max(-1, keepdim=True).values)
    return O.r(torch.einsum("hqk,khd->qhd", O.r(p), vv) / p.sum(-1).transpose(0, 1)[..., None])


def _case(L, seed, q_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    k = O.r(torch.randn(L + 16, Hkv, D, generator=g))
    v = O.r(torch.randn(L + 16, Hkv, D, generator=g))
    q = O.r(q_scale * torch.randn(1, Hq, D, generator=g))
    want = O.attention(q.double(), k[:L].double(), v[:L].double(), torch.tensor([L - 1]), SCALE).float()
    return q, k, v, want


def _worst(got, want):
    err, rms = rms_ratio(got, want)
    return float((err / rms).max())


@pytest.mark.parametrize("q_scale", [1.0, 4.0])
@pytest.mark.parametrize("L", [1023, 2048, 8192])
def test_bound_accepts_the_kernels_rounding(L, q_scale):
    for seed in range(4):
        q, k, v, want = _case(L, seed, q_scale)
        worst = _worst(bf16_p_attention(q, k[:L], v[:L]), want)
        assert worst <= 0.75 * RMS_C, f"ctx {L} seed {seed} q x{q_scale}: bf16-P rounding uses {worst / RMS_C:.2f} of the bound"


@pytest.mark.parametrize("L", [1023, 2048, 8192])
def test_bound_rejects_single_token_errors(L):
    pos = torch.tensor([L - 1])
    for seed in range(4):
        q, k, v, want = _case(L, 100 + seed)
        j = L // 2 + 3
        ks = k.clone()
        ks[[j, j + 1]] = ks[[j + 1, j]]
        vw = v.clone()
        vw[j] = v[L + 3]                  # one V row read from a wrong slot
        mutants = {
            "two K rows swapped": O.attention(q, ks[:L], v[:L], pos, SCALE),
            "one V row from a wrong slot": O.attention(q, k[:L], vw[:L], pos, SCALE),
            "one token past the end unmasked": O.attention(q, k[:L + 1], v[:L + 1], torch.tensor([L]), SCALE),
            "newest token dropped": O.attention(q, k[:L - 1], v[:L - 1], torch.tensor([L - 2]), SCALE),
        }
        for name, got in mutants.items():
            worst = _worst(got, want)
            assert worst > RMS_C, f"ctx {L} seed {seed}: '{name}' stays inside the bound ({worst:.3f} <= {RMS_C})"
