"""Paged attention pinned to answers that are exact, so that a gather, masking or merge error on a single token fails by
O(1) instead of hiding inside a bf16 tolerance.

Inputs:
  * a page pool in which everything the kernels must not use is poisoned.  Blocks no block table names are NaN, and so are
    the block-table entries past a sequence's last page (they point at a NaN block): one NaN in an output means a page
    outside the table was read.  Rows past the last token of the last page are finite poison (the engine only promises
    that they are finite): K a large multiple of a random direction, V +-512;
  * V rows of magnitude [1, 2) with random signs, all distinct, so that an output row names the pool row it came from;
  * needles: query head h is bf16(GAMMA * k[target_h, h // 4]).  Where the fp64 softmax puts less than 2^-12 on the other
    tokens, the output must be V[target] bit for bit (the other tokens move it by under 2^-10, a quarter of a bf16 ulp);
  * duplicate keys (the output is the mean of the copies' V rows, to one bf16 ulp), a dominant key in the first or last
    tile, and queries aimed at tokens the kernel must mask (compared with the fp64 oracle).

Every case runs on the decode kernel (one CTA per (sequence, KV head), split-KV with 2..64 parts, and the engine's split
rule) and on the wgmma prefill kernel (64-query work items).  Each launch writes into a sentinel-filled output wider
than the heads; rows and columns outside the work items must keep it.

RMS_C is the bound for random data: max |err| over a (row, head) <= RMS_C * rms(want[row, head]).  The kernels' own error
(P rounded to bf16, fp32 sums) reached 0.033 of the rms over the GPU suite on an H100 80GB HBM3 (0.028 for a CPU emulation
of the same rounding); one wrong token in 1-8K tokens of context moves the output by more than 0.05 of it
(tests/test_attention_tolerance_cpu.py).
"""
import math
from functools import lru_cache

import pytest
import torch

from oracle import llama_oracle as O

pytestmark = pytest.mark.gpu

D = 128
SCALE = D ** -0.5
GAMMA = 4.0
LEAK_MAX = 2.0 ** -12
RMS_C = 0.04
POISON_K = 8.0                  # |K| of rows past the end, in units of a Gaussian row
POISON_V = 512.0
OUT_SENTINEL = -7776.0          # exactly representable in bf16; no attention output here comes near it
PRODUCTION_BLOCKS = 128 * 129 + 64
CONTEXTS = [1, 15, 16, 17, 63, 64, 65, 1023, 2047, 2048, 4097, 8192, 32768]
DECODE_VARIANTS = ["unsplit", "engine", 2, 3, 7, 32, 64]
PREFILL_KERNELS = ["wgmma"]


# ------------------------------------------------------------------------------------------------------------ bounds
def ulp_bf16(x):
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -20))) - 7)


def rms_ratio(got, want):
    """Per (row, head): max |got - want| over the 128 dims, and rms(want).  got, want: [rows, H * 128] or [rows, H, 128]."""
    got = got.double().reshape(got.shape[0], -1, D)
    want = want.double().reshape(want.shape[0], -1, D)
    return (got - want).abs().amax(-1), want.pow(2).mean(-1).sqrt()


def assert_rms_close(got, want, what, c=RMS_C):
    err, rms = rms_ratio(got.float().cpu(), want.float().cpu())
    ratio = err / rms.clamp_min(1e-30)
    worst = float(ratio.max())
    print(f"{what}: max err/rms {worst:.4f}")
    bad = err > c * rms
    if bad.any():
        r, h = (int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} (row, head) pairs with max|err| > {c} rms; worst "
                             f"{worst:.3f}; first at row {r} head {h} (err {float(err[r, h]):.4g}, rms {float(rms[r, h]):.4g})")
    return worst


# ------------------------------------------------------------------------------------------------------------ the pool
class Pool:
    """K/V of `lens` sequences in a shuffled page pool [blocks][K|V][kv head][16][128], NaN wherever the kernels must not
    read.  k[s] / v[s] hold every row of sequence s's pages (past-the-end poison included) as fp32 on the device."""

    def __init__(self, lens, Hkv, seed, top=False):
        dev = "cuda"
        g = torch.Generator(device=dev).manual_seed(seed)
        self.lens, self.Hkv = list(lens), Hkv
        nbs = [(L + 15) // 16 for L in lens]
        used = sum(nbs)
        nblocks = max(used + 8, PRODUCTION_BLOCKS if top else 0)
        perm = torch.randperm(used + 8, generator=torch.Generator().manual_seed(seed)) + (nblocks - used - 8)
        self.nan_block = int(perm[-1])
        self.kv = torch.full((nblocks, 2, Hkv, 16, D), float("nan"), dtype=torch.bfloat16, device=dev)
        self.max_blocks = max(nbs) + 3
        btab = torch.full((len(lens), self.max_blocks), self.nan_block, dtype=torch.int32)
        self.blocks, self.k, self.v = [], [], []
        pos = 0
        for s, L in enumerate(lens):
            nb = nbs[s]
            blocks = perm[pos:pos + nb]
            pos += nb
            btab[s, :nb] = blocks.int()
            k = torch.randn(nb * 16, Hkv, D, generator=g, device=dev)
            sign = torch.randint(0, 2, (nb * 16, Hkv, D), generator=g, device=dev) * 2 - 1
            v = sign * (1 + torch.rand(nb * 16, Hkv, D, generator=g, device=dev))
            k[L:] *= POISON_K
            v[L:] = sign[L:] * POISON_V
            k, v = O.r(k), O.r(v)
            self.kv[blocks.to(dev), 0] = k.bfloat16().reshape(nb, 16, Hkv, D).permute(0, 2, 1, 3)
            self.kv[blocks.to(dev), 1] = v.bfloat16().reshape(nb, 16, Hkv, D).permute(0, 2, 1, 3)
            self.blocks.append(blocks.tolist())
            self.k.append(k)
            self.v.append(v)
        self.btab = btab.to(dev)

    def set_rows(self, s, pos, kvh, k=None, v=None):
        """Overwrite token `pos` of sequence s, KV head kvh, in the pool and in the mirrors."""
        blk, row = self.blocks[s][pos // 16], pos % 16
        if k is not None:
            self.k[s][pos, kvh] = O.r(k)
            self.kv[blk, 0, kvh, row] = k.bfloat16()
        if v is not None:
            self.v[s][pos, kvh] = O.r(v)
            self.kv[blk, 1, kvh, row] = v.bfloat16()

    def locate(self, row):
        """(block, row, kv head) of every V row of the pool equal to `row` [128]."""
        hits = (self.kv[:, 1] == row.to(self.kv.device, torch.bfloat16)).all(-1).nonzero().tolist()
        return [(b, r, h) for b, h, r in hits]

    def where(self, s, pos):
        return self.blocks[s][pos // 16], pos % 16


def ref64(pool, s, q, pos, tgt=None):
    """fp64 attention on the device of q [n, Hq, 128] at positions pos [n] over sequence s's tokens 0..pos.  Returns the
    bf16-rounded output [n, Hq, 128] and, given targets tgt [n, Hq], the softmax weight on every token but the target."""
    Hkv = pool.Hkv
    L = pool.lens[s]
    k, v = pool.k[s][:L].double(), pool.v[s][:L].double()
    n = q.shape[0]
    outs, leaks = [], []
    step = max(1, (1 << 26) // (4 * Hkv * L))
    for i in range(0, n, step):
        qc = q[i:i + step].double().reshape(-1, Hkv, 4, D)
        sc = torch.einsum("ngjd,lgd->ngjl", qc, k) * SCALE
        sc.masked_fill_(torch.arange(L, device=q.device)[None, None, None, :] > pos[i:i + step, None, None, None], float("-inf"))
        p = torch.softmax(sc, dim=-1)
        outs.append(O.r(torch.einsum("ngjl,lgd->ngjd", p, v).float()).reshape(-1, 4 * Hkv, D))
        if tgt is not None:
            t = tgt[i:i + step].reshape(-1, Hkv, 4, 1)
            leaks.append((1 - p.gather(-1, t)).reshape(-1, 4 * Hkv))
    return torch.cat(outs), (torch.cat(leaks) if tgt is not None else None)


# ------------------------------------------------------------------------------------------------------------ launches
def _sentinel_out(rows, Hq):
    return torch.full((rows, Hq * D + 64), OUT_SENTINEL, dtype=torch.bfloat16, device="cuda")


def run_decode(pool, q, work, variant):
    """Decode attention of the work items [n, 4] (q_tok0, 1, q_pos0, seq) with rows of q [T, Hq * 128]; variant: "unsplit",
    "engine" (launches of 8 items, split by the engine's rule) or a split count.  Returns the sentinel-checked output."""
    from kubeai_b200 import lib, ops
    Hq = 4 * pool.Hkv
    out = _sentinel_out(q.shape[0], Hq)
    n = work.shape[0]
    if variant == "engine":
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        for i in range(0, n, 8):
            w = work[i:i + 8]
            split = lib().b200_attn_split_query(w.shape[0], pool.Hkv, int(w[:, 2].max()) + 1, sms)
            ops.paged_attn(q, pool.kv, pool.btab, w, Hq, pool.Hkv, decode=True, out=out, split=split if split > 1 else 0)
    else:
        per = 1024 if variant == "unsplit" else 256
        for i in range(0, n, per):
            ops.paged_attn(q, pool.kv, pool.btab, work[i:i + per], Hq, pool.Hkv, decode=True, out=out,
                           split=0 if variant == "unsplit" else variant)
    return _check_sentinel(out, work, Hq)


def run_prefill(pool, q, work):
    from kubeai_b200 import ops
    Hq = 4 * pool.Hkv
    out = _sentinel_out(q.shape[0], Hq)
    ops.paged_attn_prefill_tc(q, pool.kv, pool.btab, work, Hq, pool.Hkv, out=out)
    return _check_sentinel(out, work, Hq)


def run(pool, q, work, path):
    return run_prefill(pool, q, work) if path in PREFILL_KERNELS else run_decode(pool, q, work, path)


def _check_sentinel(out, work, Hq):
    torch.cuda.synchronize()
    written = torch.zeros(out.shape[0], dtype=torch.bool, device=out.device)
    for t0, cnt, _, _ in work.tolist():
        written[t0:t0 + cnt] = True
    sent = out == OUT_SENTINEL
    assert sent[:, Hq * D:].all(), "a column past the last head was written"
    assert sent[~written].all(), "a row outside the work items was written"
    got = out[:, :Hq * D]
    assert not torch.isnan(got[written]).any(), "NaN in the output: a page outside the block table was read"
    return got.float()


# ------------------------------------------------------------------------------------------------------------ needles
@lru_cache(maxsize=None)
def needle_pool(Hkv, L, top=False):
    return Pool([L], Hkv, seed=1000 * Hkv + L % 997 + (7 if top else 0), top=top)


def _needle_q(pool, tgt):
    """q [n, Hq * 128] with head h = bf16(GAMMA * k[tgt[:, h], h // 4])."""
    n, Hq = tgt.shape
    kvh = torch.arange(Hq, device=tgt.device) // 4
    return O.r(GAMMA * pool.k[0][tgt, kvh[None, :].expand(n, Hq)]).bfloat16().reshape(n, Hq * D).contiguous()


def _with_gaps(q, rows, total, seed):
    """q's rows placed at `rows` of a [total, ...] tensor whose other rows are random queries no work item names."""
    full = torch.randn(total, q.shape[1], generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda").bfloat16()
    full[rows] = q
    return full


@lru_cache(maxsize=None)
def decode_needles(Hkv, L, top=False):
    """Work items at position L - 1 whose 4 * Hkv heads together aim at every (position, KV head) of the context."""
    pool = needle_pool(Hkv, L, top)
    gen = torch.Generator().manual_seed(L + 31 * Hkv)
    n = (L + 3) // 4
    tgt = torch.empty(n, 4 * Hkv, dtype=torch.long)
    for h in range(Hkv):
        perm = torch.randperm(L, generator=gen)
        idx = (torch.arange(4)[None, :] * n + torch.arange(n)[:, None]) % L     # the group's heads: different tokens
        tgt[:, 4 * h:4 * h + 4] = perm[idx]
    for h in range(Hkv):
        assert set(tgt[:, 4 * h:4 * h + 4].flatten().tolist()) == set(range(L)), "every position is a target"
    if L >= 4:
        assert all(len(set(r)) == 4 for r in tgt.reshape(n, Hkv, 4).reshape(-1, 4).tolist())
    tgt = tgt.cuda()
    q = _needle_q(pool, tgt)
    pos = torch.full((n,), L - 1, dtype=torch.long, device="cuda")
    _, leak = ref64(pool, 0, q.float().reshape(n, -1, D), pos, tgt)
    rows = torch.arange(n) + torch.arange(n) // 64 + 1           # row 0 and every 65th row belong to no work item
    work = torch.tensor([[int(r), 1, L - 1, 0] for r in rows], dtype=torch.int32, device="cuda")
    rows = rows.cuda()
    return _with_gaps(q, rows, n + n // 64 + 2, L), work, tgt, pos, leak, rows


@lru_cache(maxsize=None)
def prefill_needles(Hkv, L, Q, top=False):
    """Prefill work items of up to Q queries (q_pos0 at every residue mod 64, some ragged) whose heads aim at every
    (position, KV head) of the context; each query aims at a token at or before its own position."""
    pool = needle_pool(Hkv, L, top)
    gen = torch.Generator().manual_seed(7 * L + Hkv + Q)
    n_items = max(64, math.ceil(1.5 * L / (4 * Q)))
    work, tok, row = [], 0, 1
    for i in range(n_items):
        p0 = max(0, L - Q - i % 64)
        cnt = min(Q if i % 5 != 2 else 1 + (i * 7) % Q, L - p0)      # every fifth item ragged
        work.append([row, cnt, p0, 0])
        tok += cnt
        row += cnt + (i % 9 == 0)                                    # now and then a row no work item names
    pos = torch.cat([torch.arange(p0, p0 + c) for _, c, p0, _ in work])
    rows = torch.cat([torch.arange(r, r + c) for r, c, _, _ in work]).cuda()
    Hq = 4 * Hkv
    tgt = torch.empty(tok, Hq, dtype=torch.long)
    for h in range(Hkv):
        # slots (row, head of the group), highest position first, matched with the targets in descending order
        slot_pos = pos[:, None].expand(tok, 4).reshape(-1)
        order = torch.randperm(slot_pos.numel(), generator=gen)
        order = order[torch.argsort(slot_pos[order], descending=True, stable=True)]
        want = torch.randperm(L, generator=gen).sort(descending=True).values
        assert order.numel() >= L
        t = torch.empty(slot_pos.numel(), dtype=torch.long)
        t[order[:L]] = want
        rest = order[L:]
        t[rest] = (torch.rand(rest.numel(), generator=gen) * (slot_pos[rest] + 1)).long()
        assert (t <= slot_pos).all(), "a needle aimed past its query's position"
        tgt[:, 4 * h:4 * h + 4] = t.reshape(tok, 4)
        assert set(t.tolist()) == set(range(L)), "every position is a target"
    assert {p0 % 64 for _, _, p0, _ in work} == set(range(64)) or L < Q + 63
    tgt, pos = tgt.cuda(), pos.cuda()
    q = _needle_q(pool, tgt)
    _, leak = ref64(pool, 0, q.float().reshape(tok, -1, D), pos, tgt)
    return _with_gaps(q, rows, row + 1, L + Q), torch.tensor(work, dtype=torch.int32, device="cuda"), tgt, pos, leak, rows


def check_needles(pool, got, tgt, pos, leak, what):
    assert float(leak.max()) < LEAK_MAX, f"{what}: construction: weight {float(leak.max()):.2e} off a needle's target"
    n, Hq = tgt.shape
    kvh = torch.arange(Hq, device=tgt.device) // 4
    want = pool.v[0][tgt, kvh[None, :].expand(n, Hq)]
    got = got.reshape(n, Hq, D)
    bad = (got != want).any(-1).nonzero().tolist()
    if bad:
        lines = []
        for r, h in bad[:6]:
            t = int(tgt[r, h])
            b, row = pool.where(0, t)
            hits = pool.locate(got[r, h].bfloat16())
            seen = ", ".join(f"block {hb} row {hr} kv head {hh}" for hb, hr, hh in hits[:3]) or \
                f"no V row (max err {float((got[r, h] - want[r, h]).abs().max()):.3g})"
            lines.append(f"query row {r} (position {int(pos[r])}) head {h}: aimed at position {t} (block {b} row {row}), read {seen}")
        raise AssertionError(f"{what}: {len(bad)} of {n * Hq} needles missed\n  " + "\n  ".join(lines))


DECODE_CASES = [(8, L) for L in CONTEXTS] + [(h, L) for h in (1, 2) for L in (1, 17, 65, 2048, 4097)]


@pytest.mark.parametrize("variant", DECODE_VARIANTS)
@pytest.mark.parametrize("Hkv,L,top", [(h, L, False) for h, L in DECODE_CASES] + [(8, 2048, True)])
def test_decode_needles_read_exactly_their_target(Hkv, L, top, variant):
    pool = needle_pool(Hkv, L, top)
    q, work, tgt, pos, leak, rows = decode_needles(Hkv, L, top)
    got = run_decode(pool, q, work, variant)
    check_needles(pool, got[rows], tgt, pos, leak, f"decode {variant} Hkv {Hkv} ctx {L}{' top of pool' if top else ''}")


@pytest.mark.parametrize("kernel", PREFILL_KERNELS)
@pytest.mark.parametrize("Hkv,L,top", [(h, L, False) for h, L in DECODE_CASES] + [(8, 2048, True)])
def test_prefill_needles_read_exactly_their_target(Hkv, L, top, kernel):
    pool = needle_pool(Hkv, L, top)
    q, work, tgt, pos, leak, rows = prefill_needles(Hkv, L, 64, top)
    got = run_prefill(pool, q, work)
    check_needles(pool, got[rows], tgt, pos, leak, f"prefill {kernel} Hkv {Hkv} ctx {L}{' top of pool' if top else ''}")


# ------------------------------------------------------------------------------------------------------------ duplicates
def _dup_sets(L):
    """Positions of 2-4 copies of one key, crossing the decode kernel's merge boundaries: one 16-token warp strip, two
    strips of one 64-token tile, two tiles, split slices (empty ones too when the split is large), first and last token."""
    t = (L // 2) // 64 * 64
    sets = [(t + 18, t + 29), (t + 3, t + 55), (5, L - 40), (0, L // 3, 2 * L // 3, L - 1), (0, L - 1),
            (L - 70, L - 66, L - 2), (63, 64), (15, 16, 1000)]
    return [s for s in sets if len(set(s)) == len(s) and min(s) >= 0 and max(s) < L]


@lru_cache(maxsize=None)
def dup_case():
    """Sequences of 17..4097 tokens, Hkv 8; KV head g of each sequence carries one set of copies, and the 4 query heads of
    the group aim at it.  Returns the pool and, per sequence, the sets."""
    lens = [4097, 2048, 300, 65, 17]
    pool = Pool(lens, 8, seed=55)
    gen = torch.Generator(device="cuda").manual_seed(56)
    sets = []
    for s, L in enumerate(lens):
        cand = _dup_sets(L)
        per = [cand[g % len(cand)] for g in range(8)]
        for g, ps in enumerate(per):
            sign = torch.randint(0, 2, (D,), generator=gen, device="cuda") * 2 - 1
            for p in ps:
                pool.set_rows(s, p, g, k=pool.k[s][ps[0], g].clone(),
                              v=sign * (1 + torch.rand(D, generator=gen, device="cuda")))
        sets.append(per)
    return pool, sets


def _dup_queries(path):
    """(q, work, positions, seq of each row): decode rows at the last position; prefill items of Q rows at the end, whose
    earlier rows see only the copies at or before their position."""
    pool, sets = dup_case()
    Q = _q_rows(path)
    rows, work, pos, seq = [], [], [], []
    for s, L in enumerate(pool.lens):
        qs = torch.stack([O.r(GAMMA * pool.k[s][sets[s][h // 4][0], h // 4]) for h in range(32)])
        cnt = min(Q, L)
        work.append([len(rows), cnt, L - cnt, s])
        for r in range(cnt):
            rows.append(qs)
            pos.append(L - cnt + r)
            seq.append(s)
    q = torch.stack(rows).reshape(len(rows), -1).bfloat16().contiguous()
    return pool, sets, q, torch.tensor(work, dtype=torch.int32, device="cuda"), pos, seq


@pytest.mark.parametrize("path", DECODE_VARIANTS + PREFILL_KERNELS)
def test_duplicate_keys_average_their_values_to_one_ulp(path):
    pool, sets, q, work, pos, seq = _dup_queries(path)
    got = run(pool, q, work, path).reshape(q.shape[0], 32, D)
    checked = 0
    for s in range(len(pool.lens)):
        rs = [r for r, x in enumerate(seq) if x == s]
        vis = [[[c for c in sets[s][g] if c <= pos[r]] for g in range(8)] for r in rs]
        tgt = torch.tensor([[(vis[i][h // 4] or [0])[0] for h in range(32)] for i in range(len(rs))], device="cuda")
        _, leak = ref64(pool, s, q[rs].float().reshape(len(rs), 32, D), torch.tensor([pos[r] for r in rs], device="cuda"), tgt)
        for i, r in enumerate(rs):
            for g in range(8):
                vg = vis[i][g]
                if not vg:
                    continue
                off = float(leak[i, 4 * g:4 * g + 4].max()) - (len(vg) - 1) / len(vg)
                assert off < LEAK_MAX, f"construction: weight {off:.2e} off the copies"
                mean = pool.v[s][vg, g].double().mean(0)
                err = (got[r, 4 * g:4 * g + 4].double() - mean).abs()
                ulp = ulp_bf16(mean)
                assert (err <= ulp).all(), (f"{path}: seq {s} (ctx {pool.lens[s]}) row at position {pos[r]}, kv head {g}: copies "
                                            f"at {sets[s][g]}, {len(vg)} visible; max err {float((err / ulp).max()):.2f} ulp")
                checked += 1
    assert checked >= 40


# ------------------------------------------------------------------------------------------------------------ rescaling, masking
@lru_cache(maxsize=None)
def sink_case(where):
    """Random queries over 2048- and 4097-token contexts with one key per KV head that dominates the softmax (about 9
    nats above the rest), in the first or in the last 64-token tile."""
    lens = [2048, 4097]
    pool = Pool(lens, 8, seed=77 if where == "first" else 78)
    gen = torch.Generator(device="cuda").manual_seed(79)
    qs = O.r(torch.randn(len(lens), 32, D, generator=gen, device="cuda"))
    for s, L in enumerate(lens):
        p = 3 if where == "first" else L - 2
        for g in range(8):
            grp = qs[s, 4 * g:4 * g + 4]
            k = grp.sum(0)
            a = 9.0 / float((grp @ k).mean() * SCALE)
            pool.set_rows(s, p, g, k=a * k)
    return pool, qs


def _row_queries(pool, qs, Q):
    """Every sequence's query vectors repeated on the last Q positions (Q = 1: decode)."""
    rows, work, pos, seq = [], [], [], []
    for s, L in enumerate(pool.lens):
        cnt = min(Q, L)
        work.append([len(rows), cnt, L - cnt, s])
        rows += [qs[s]] * cnt
        pos += list(range(L - cnt, L))
        seq += [s] * cnt
    q = torch.stack(rows).reshape(len(rows), -1).bfloat16().contiguous()
    return q, torch.tensor(work, dtype=torch.int32, device="cuda"), pos, seq


def _against_fp64(pool, q, got, pos, seq, what):
    want = torch.empty_like(got)
    for s in set(seq):
        rows = [i for i, x in enumerate(seq) if x == s]
        ri = torch.tensor(rows, device="cuda")
        want[ri] = ref64(pool, s, q[ri].float().reshape(len(rows), -1, D), torch.tensor(pos, device="cuda")[ri])[0].reshape(len(rows), -1)
    err = (got - want).abs()
    assert bool((err <= 4e-3 + 1.6e-2 * want.abs()).all()), f"{what}: max err {float(err.max()):.4g} (vLLM tolerance)"
    assert_rms_close(got, want, what)


def _q_rows(path):
    return 1 if path not in PREFILL_KERNELS else 64


@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("path", DECODE_VARIANTS + PREFILL_KERNELS)
def test_dominant_key_rescales_in_both_directions(path, where):
    pool, qs = sink_case(where)
    q, work, pos, seq = _row_queries(pool, qs, _q_rows(path))
    _against_fp64(pool, q, run(pool, q, work, path), pos, seq, f"{path} sink in the {where} tile")


@lru_cache(maxsize=None)
def mask_case():
    """Contexts that end inside a page; decode queries aim at the poisoned rows past the end."""
    lens = [17, 1000, 2047, 4097, 333]
    pool = Pool(lens, 8, seed=91)
    qs = []
    for s, L in enumerate(lens):
        pad = 16 - L % 16
        qs.append(torch.stack([O.r(GAMMA / POISON_K * pool.k[s][L + h % pad, h // 4]) for h in range(32)]))
    return pool, torch.stack(qs)


@pytest.mark.parametrize("path", DECODE_VARIANTS)
def test_decode_masks_the_poisoned_rows_it_loads(path):
    pool, qs = mask_case()
    q, work, pos, seq = _row_queries(pool, qs, 1)
    _against_fp64(pool, q, run(pool, q, work, path), pos, seq, f"decode {path} aimed past the end")


@pytest.mark.parametrize("kernel", PREFILL_KERNELS)
def test_prefill_masks_future_and_past_the_end_tokens(kernel):
    """Each query aims at a token it must not see: the next position (inside the chunk, or the first token past the
    work item's end) or a poisoned row past the end of the sequence."""
    pool, _ = mask_case()
    Q = 64
    rows, work, pos, seq = [], [], [], []
    for s, L in enumerate(pool.lens):
        for p0 in sorted({L - min(Q, L), max(0, L - Q - 37), L // 2}):
            cnt = min(Q, L - p0)
            work.append([len(rows), cnt, p0, s])
            for r in range(cnt):
                p = p0 + r
                heads = []
                for h in range(32):
                    t = p + 1 + (h % 4 if p + 1 >= L else 0)
                    t = min(t, (L + 15) // 16 * 16 - 1)
                    heads.append(O.r(GAMMA * (pool.k[s][t, h // 4] / (POISON_K if t >= L else 1.0))))
                rows.append(torch.stack(heads))
                pos.append(p)
                seq.append(s)
    q = torch.stack(rows).reshape(len(rows), -1).bfloat16().contiguous()
    wt = torch.tensor(work, dtype=torch.int32, device="cuda")
    _against_fp64(pool, q, run_prefill(pool, q, wt), pos, seq, f"prefill {kernel} aimed at masked tokens")

