"""Host-side scheduling rules of the projection GEMM and of split-KV decode attention, through the C ABI without a GPU
(b200_schedule_query / b200_attn_split_query are pure host functions).  These are the decisions DESIGN.md §4 describes for
Llama-3-8B on a 132-SM H100; the test pins them so that a change of a threshold shows up as a diff here and not as a silent
few percent in the bench."""
import ctypes as C

import pytest

from kubeai_b200._lib import lib

SMS = 132
QKV, O, GATE_UP, DOWN, LM_HEAD = (6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336), (128256, 4096)


def q(shape, T, sms=SMS):
    out = (C.c_int32 * 8)()
    assert lib().b200_schedule_query(shape[0], shape[1], T, sms, out) == 0
    keys = ("block_n", "token_tiles", "tiles", "splits", "ctas", "rule")
    return dict(zip(keys, list(out)[:6]))


def test_decode_step_splits_k_until_the_device_is_full():
    # o_proj / down_proj: 32 slabs of 128 rows -> 4 K-splits = 128 CTAs on 132 SMs
    for shape in (O, DOWN):
        s = q(shape, 128)
        assert (s["block_n"], s["tiles"], s["splits"], s["ctas"], s["rule"]) == (128, 32, 4, 128, 1), (shape, s)
    # qkv: 48 slabs -> 2 splits (3 would need a second wave of 12 CTAs)
    assert (q(QKV, 128)["splits"], q(QKV, 128)["ctas"]) == (2, 96)
    # gate_up and lm_head have more slabs than SMs: whole-K tiles, the split count is the device's choice
    for shape in (GATE_UP, LM_HEAD):
        s = q(shape, 77)
        assert (s["splits"], s["rule"]) == (1, 1), (shape, s)


def test_prefill_burst_of_1340_tokens():
    # the token tile follows the step size; a 1340-token burst is 6 tiles of 256 per slab, more tiles than SMs: no split
    assert [q(O, T)["block_n"] for T in (1, 64, 65, 128, 129, 2048)] == [64, 64, 128, 128, 256, 256]
    s = q(O, 1340)
    assert (s["token_tiles"], s["tiles"], s["splits"], s["rule"]) == (6, 192, 1, 2)


def test_every_split_keeps_at_least_four_k_blocks():
    s = q((256, 512), 16)            # 2 slabs would take 66 splits; 8 k-blocks allow 2
    assert (s["splits"], s["ctas"]) == (2, 4)
    assert q((256, 128), 16)["splits"] == 1


def test_split_count_scales_with_the_device():
    assert q(O, 128, sms=148)["splits"] == 4 and q(O, 128, sms=64)["splits"] == 2 and q(QKV, 128, sms=16)["splits"] == 1


@pytest.mark.parametrize("nwork,ctx,want", [(128, 450, 1), (19, 2000, 1), (1, 2000, 16), (1, 100, 1), (4, 2000, 10), (16, 2000, 3),
                                            (1, 300, 3), (8, 1000, 5)])
def test_split_kv_parts(nwork, ctx, want):
    # about two CTAs per SM, at least two 64-token tiles per part, never when the grid already fills the device (a pure
    # function of the SM count: pinned for 148 SMs; the H100's 132 gives 9 parts instead of 10 for 4 sequences)
    assert lib().b200_attn_split_query(nwork, 8, ctx, 148) == want
    assert lib().b200_attn_split_query(4, 8, 2000, SMS) == 9
