"""Steps of more than 128 tokens through the projection GEMM (kubeai_b200/csrc/gemm_wgmma.cu): a token's output row must not
depend on where the token sits in the step.  The ragged last token tile runs a narrower wgmma than the full tiles, and the
CTAs of one weight slab run next to each other; neither may change a bit of any row."""
import math

import pytest
import torch

from test_gemm3_gpu import close, ref_gemm, rnd

pytestmark = pytest.mark.gpu

# Llama-3-8B projections (N, K); gate_up is the interleaved gate/up weight of the fused SiLU epilogue
QKV, O, GATE_UP, DOWN = (6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)


def test_ragged_last_tile_rows_equal_full_tile_rows():
    """Every residue of T mod 256 from 1 to 255, stepping by 7: reversing the rows of X moves the ragged last tile's
    tokens into the first (full) tile of a launch with the same T, hence the same schedule and the same K-splits."""
    from kubeai_b200 import ops
    N, K = 512, 512
    x_all, w = rnd(512, K, seed=51), rnd(N, K, scale=1 / math.sqrt(K), seed=52)
    for T in range(257, 513, 7):
        x = x_all[:T].contiguous()
        got, sch = ops.gemm3(x, w)
        flipped, sch2 = ops.gemm3(x.flip(0).contiguous(), w)
        torch.cuda.synchronize()
        assert sch == sch2
        same = got.view(torch.int16) == flipped.flip(0).view(torch.int16)
        assert bool(same.all()), f"T={T} ({sch}): {int((~same).sum())} outputs differ between the ragged and a full tile"


def test_gate_up_burst_rows_equal_single_tile_rows():
    """T = 1340 on gate_up (224 slabs x 6 token tiles, no K-split) against 256-row single-tile launches of the same rows."""
    from kubeai_b200 import ops
    (N, K), T = GATE_UP, 1340
    x, w = rnd(T, K, seed=53), rnd(N, K, scale=1 / math.sqrt(K), seed=54)
    got, sch = ops.gemm3(x, w)
    assert sch[0] == 1
    for r0 in (0, 512, T - 256):
        part, sch1 = ops.gemm3(x[r0:r0 + 256].contiguous(), w)
        torch.cuda.synchronize()
        assert sch1[0] == 1
        same = got[r0:r0 + 256].view(torch.int16) == part.view(torch.int16)
        assert bool(same.all()), f"rows {r0}..{r0 + 255}: {int((~same).sum())} outputs differ from the single-tile launch"


@pytest.mark.parametrize("shape", [QKV, O, GATE_UP, DOWN], ids=["qkv", "o", "gate_up", "down"])
def test_llama_projection_at_1340_tokens_matches_oracle(shape):
    from kubeai_b200 import ops
    (N, K), T = shape, 1340
    x, w = rnd(T, K, seed=55), rnd(N, K, scale=1 / math.sqrt(K), seed=56)
    got, sch = ops.gemm3(x, w)
    torch.cuda.synchronize()
    close(got, ref_gemm(x, w), f"T={T} N={N} K={K} schedule {sch}")
