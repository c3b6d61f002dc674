"""The checkers of tests/kernel_numerics.py on CPU emulations of the elementwise kernels: each accepts an emulation that
rounds where the kernel rounds and rejects ones that are subtly wrong (a rounding point, eps, the squared values or the
mean's count moved), so the GPU tests in test_elementwise_exact_gpu.py would catch such a kernel."""
import numpy as np
import pytest
import torch

from kernel_numerics import (bf16, check_rmsnorm, check_silu, f32_bits, fp32_between, norm_launch, rope_expected,
                             warp_sum)
from oracle import llama_oracle as O
from oracle.weights import ModelCfg, cos_sin_cache

EPS = 1e-5


def _rows(H, n, seed):
    """n rows of N(0, 1) after the hard rows the GPU test uses: eps-dominated, constant, a few massive channels."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, H, generator=g)
    x[0] = torch.randn(H, generator=g) * 1e-4
    x[1] = 0.75
    x[2, torch.randperm(H, generator=g)[:4]] = torch.tensor([1e4, -1e4, 3e3, -7e3])
    return bf16(x)


def emu_rmsnorm(x, w, res=None, variant=None):
    """rmsnorm_kernel in torch fp32.  variant: None (faithful), "no_round" (no bf16 rounding before the weight multiply),
    "eps_outside" (1 / (sqrt(mean) + eps)), "unrounded_sq" (squares of the unrounded fused sum), "h_minus_8" (mean over
    H - 8)."""
    z = x + res if res is not None else x
    v = bf16(z)
    sq = z if variant == "unrounded_sq" else v
    H = v.shape[-1]
    ms = (sq * sq).sum(-1, dtype=torch.float32) / (H - 8 if variant == "h_minus_8" else H)
    inv = 1 / (ms.sqrt() + EPS) if variant == "eps_outside" else (ms + EPS).rsqrt()
    y = v * inv[:, None]
    return bf16(y * w) if variant == "no_round" else bf16(bf16(y) * w)


@pytest.mark.parametrize("H", [256, 4096])
@pytest.mark.parametrize("variant", [None, "no_round", "eps_outside", "unrounded_sq", "h_minus_8"])
def test_rmsnorm_checker_accepts_the_kernel_and_rejects_each_wrong_variant(H, variant):
    x = _rows(H, 24, seed=H)
    res = _rows(H, 24, seed=H + 1) * 0.5
    w = bf16(1 + 0.1 * torch.randn(H, generator=torch.Generator().manual_seed(3)))
    for r in (None, res):
        v = bf16(x + r) if r is not None else x
        ok, _ = check_rmsnorm(v, w, emu_rmsnorm(x, w, r, variant), EPS)
        if variant is None:
            assert bool(ok.all()), (~ok).nonzero().flatten().tolist()
        elif r is not None or variant != "unrounded_sq":      # without a residual the fused sum is the row itself
            assert not bool(ok.all()), f"{variant} passed the check"


def test_rmsnorm_checker_finds_an_inv_other_than_the_nearest():
    """A kernel inv a few ulps from float64 passes through a non-nearest candidate; one at 2^-16 relative (10 RMS_DELTA)
    fails on most rows where the shift moves a rounding.  A bf16 row has at most 128 distinct mantissas, so on some rows it
    moves none, and on some the first rounding it moves already moves inside the interval."""
    x = _rows(4096, 64, seed=7)
    w = bf16(1 + 0.1 * torch.randn(4096, generator=torch.Generator().manual_seed(8)))
    inv64 = (x.double().pow(2).mean(-1) + float(np.float32(EPS))).rsqrt()
    near = inv64.float() * (1 + 3 * 2.0 ** -23)
    ok, nonnearest = check_rmsnorm(x, w, bf16(bf16(x * near[:, None]) * w), EPS)
    assert bool(ok.all()) and nonnearest > 0
    far = inv64.float() * (1 + 2.0 ** -16)
    nearest = bf16(bf16(x * inv64.float()[:, None]) * w)
    out = bf16(bf16(x * far[:, None]) * w)
    ok, _ = check_rmsnorm(x, w, out, EPS)
    moved = (out != nearest).any(-1)
    assert int(moved.sum()) > 10 and not bool(ok[~moved].logical_not().any()) and int((~ok).sum()) > moved.sum() // 2


def emu_silu(g, u, variant=None):
    """silu_mul_kernel in torch fp32, with __fdividef's flush to 0 past a 2^126 denominator.  variant "no_round": s not
    rounded to bf16 before the multiply by up."""
    d = 1 + torch.exp(-g)
    s = torch.where(d > 2.0 ** 126, g * 0, g / d)
    return bf16(s * u) if variant == "no_round" else bf16(bf16(s) * u)


@pytest.mark.parametrize("variant", [None, "no_round"])
def test_silu_checker_accepts_the_kernel_and_rejects_an_unrounded_silu(variant):
    gen = torch.Generator().manual_seed(11)
    g = bf16(torch.cat([torch.rand(20000, generator=gen) * 160 - 80, torch.randn(20000, generator=gen) * 4,
                        -87.5 - torch.rand(500, generator=gen) * 200]))
    u = bf16(torch.randn(g.numel(), generator=gen))
    ok, straddle = check_silu(g, u, emu_silu(g, u, variant))
    if variant is None:
        assert bool(ok.all()), g[~ok][:8].tolist()
        assert straddle < 0.01 * g.numel()
    else:
        assert not bool(ok.all())


def test_silu_checker_rejects_a_silu_one_bf16_step_off():
    gen = torch.Generator().manual_seed(12)
    g = bf16(torch.rand(20000, generator=gen) * 160 - 80)
    u = bf16(torch.randn(g.numel(), generator=gen))
    s = bf16(g / (1 + torch.exp(-g)))
    s_up = (s.to(torch.bfloat16).view(torch.int16) + 1).view(torch.bfloat16).float()     # one step away from zero
    off = bf16(s_up * u)
    changed = off != emu_silu(g, u)
    ok, _ = check_silu(g, u, off)
    # only where the float64 interval straddles a boundary may the neighbour be accepted
    assert int(changed.sum()) > 0.9 * g.numel() and float(ok[changed].float().mean()) < 0.01


def emu_rope(qkv, pos, cs, Hq, Hkv, D, rounded=True):
    """rope_kv_kernel's rotation of the q and k heads in torch fp32; rounded=False drops the bf16 rounding of the four
    products."""
    T = qkv.shape[0]
    p = pos.long().clamp(0, cs.shape[0] - 1)
    x = qkv[:, :(Hq + Hkv) * D].reshape(T, Hq + Hkv, D)
    a, b = x[..., :D // 2], x[..., D // 2:]
    c, s = cs[p][:, None, :D // 2], cs[p][:, None, D // 2:]
    rr = bf16 if rounded else (lambda t: t)
    return torch.cat([bf16(rr(a * c) - rr(b * s)), bf16(rr(b * c) + rr(a * s))], dim=-1)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("rounded", [True, False])
def test_rope_checker_accepts_the_kernel_and_rejects_unrounded_products(D, rounded):
    Hq, Hkv, max_pos = 4, 2, 300
    cs = O.r(torch.from_numpy(cos_sin_cache(ModelCfg(max_model_len=max_pos, head_dim=D))))
    gen = torch.Generator().manual_seed(D)
    qkv = bf16(torch.randn(40, (Hq + 2 * Hkv) * D, generator=gen) * 3)
    pos = torch.randint(0, max_pos, (40,), generator=gen, dtype=torch.int32)
    pos[:4] = torch.tensor([0, max_pos - 1, -5, max_pos + 3])
    same = torch.equal(f32_bits(emu_rope(qkv, pos, cs, Hq, Hkv, D, rounded)), f32_bits(rope_expected(qkv, pos, cs, Hq, Hkv, D)))
    assert same == rounded


def test_fp32_between_lists_every_value_of_the_interval():
    one = np.float32(1.0)
    got = fp32_between(1.0, float(np.nextafter(np.nextafter(one, np.float32(2)), np.float32(2)))).numpy()
    assert got.tolist() == [1.0, float(np.nextafter(one, np.float32(2))), float(np.nextafter(np.nextafter(one, np.float32(2)), np.float32(2)))]
    assert fp32_between(1.0 + 2.0 ** -30, 1.0 + 2.0 ** -24).numel() == 0        # strictly between two fp32 values
    z = fp32_between(-2e-45, 2e-45).numpy()                                     # both zeros and the smallest subnormals
    assert z.size == 4 and (z[:2] < 0).sum() == 1 and np.signbit(z[1]) and not np.signbit(z[2])
    r = fp32_between(0.1, 0.1 * (1 + 2.0 ** -20)).numpy()
    assert r[0] >= 0.1 and float(r[-1]) <= 0.1 * (1 + 2.0 ** -20) and (np.diff(r.view(np.int32)) == 1).all()


def test_norm_launch_and_warp_sum():
    assert norm_launch(511, 8192) == (1024, 1) and norm_launch(512, 8192) == (256, 4)
    assert norm_launch(1500, 3072) == (384, 1) and norm_launch(600, 6144) == (256, 3) and norm_launch(512, 256) == (32, 1)
    v = np.arange(32, dtype=np.float32)
    assert warp_sum(v) == np.float32(496)
