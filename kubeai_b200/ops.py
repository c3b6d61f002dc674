"""Op-level drivers over the C ABI (b200_op_*): torch is used only to own device memory and the
stream; every call goes straight into the hand-written CUDA kernels.  There is no fallback: without
the library or a GPU these raise."""
from __future__ import annotations

import ctypes as C

import torch

from ._lib import check, lib


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk(t, dtype=torch.bfloat16):
    assert t.is_cuda and t.is_contiguous() and t.dtype == dtype, (t.device, t.dtype, t.is_contiguous())


def gemm(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """out[t, n] = sum_k x[t, k] w[n, k]; bf16 in, fp32 accumulate, bf16 out."""
    _chk(x), _chk(w)
    T, K = x.shape
    N = w.shape[0]
    out = torch.empty(T, N, dtype=torch.bfloat16, device=x.device)
    check(lib().b200_op_gemm(_p(w), _p(x), _p(out), N, T, K, _stream()))
    return out


def gemm_deferred(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """The engine's form of the product (split-K sized to the device whatever the variant; N % 8 == 0)."""
    _chk(x), _chk(w)
    T, K = x.shape
    N = w.shape[0]
    out = torch.empty(T, N, dtype=torch.bfloat16, device=x.device)
    check(lib().b200_op_gemm_deferred(_p(w), _p(x), _p(out), N, T, K, _stream()))
    return out


PRO_NONE, PRO_NORM = 0, 1
EPI_PLAIN, EPI_RESADD, EPI_SILU, EPI_ROPE_KV, EPI_ARGMAX = 0, 1, 2, 3, 4


def gemm3(x, w, T=None, pro=PRO_NONE, epi=EPI_PLAIN, force=0, ssq_in=None, norm_w=None, eps=1e-5, out=None, ssq_out=None,
          positions=None, slots=None, cos_sin=None, kv_layer=None, q_heads=0, kv_heads=0, argmax_out=None, n_valid=0,
          normed_out=None, norm_w_out=None):
    """The fused projection GEMM (b200_op_gemm3).  x: [rows >= T, K] activations (or the residual for PRO_NORM),
    w: [N, K].  Returns (out, schedule) with schedule = (K-splits per tile, rule that chose them: 0 given by `force`,
    1 device-filling for one token tile, 2 device-filling over several token tiles (T > 128), CTAs)."""
    from ._lib import Gemm3Args
    _chk(x), _chk(w)
    T = x.shape[0] if T is None else T
    N, K = w.shape
    a = Gemm3Args(N=N, T=T, K=K, x_rows=x.shape[0], pro=pro, epi=epi, force=force, w=w.data_ptr(), x=x.data_ptr(), eps=eps,
                  q_heads=q_heads, kv_heads=kv_heads, n_valid=n_valid)
    if pro == PRO_NORM:
        _chk(norm_w), _chk(ssq_in, torch.float32)
        a.ssq_in, a.ssq_slabs, a.norm_w = ssq_in.data_ptr(), ssq_in.shape[1], norm_w.data_ptr()
    if epi == EPI_PLAIN:
        out = torch.empty(T, N, dtype=torch.bfloat16, device=x.device) if out is None else out
    elif epi == EPI_RESADD:
        _chk(out)                                               # the residual, updated in place
        ssq_out = torch.zeros(T, N // 128, dtype=torch.float32, device=x.device) if ssq_out is None else ssq_out
        a.ssq_out = ssq_out.data_ptr()
        if norm_w_out is not None:                              # fused RMSNorm of the new residual for the next projection
            _chk(norm_w_out)
            normed_out = torch.empty(T, N, dtype=torch.bfloat16, device=x.device) if normed_out is None else normed_out
            a.normed_out, a.norm_w_out = normed_out.data_ptr(), norm_w_out.data_ptr()
    elif epi == EPI_SILU:
        out = torch.empty(T, N // 2, dtype=torch.bfloat16, device=x.device) if out is None else out
    elif epi == EPI_ROPE_KV:
        _chk(out), _chk(positions, torch.int32), _chk(slots, torch.int32), _chk(cos_sin), _chk(kv_layer)
        a.positions, a.slots, a.cos_sin, a.kv_layer = positions.data_ptr(), slots.data_ptr(), cos_sin.data_ptr(), kv_layer.data_ptr()
        a.max_pos = cos_sin.shape[0]
    elif epi == EPI_ARGMAX:
        argmax_out = torch.empty(T, dtype=torch.int32, device=x.device) if argmax_out is None else argmax_out
        a.argmax_out = argmax_out.data_ptr()
    if out is not None:
        a.out, a.ldo = out.data_ptr(), out.stride(0)
    sch = (C.c_int32 * 3)()
    check(lib().b200_op_gemm3(C.byref(a), _stream(), sch))
    res = argmax_out if epi == EPI_ARGMAX else (out, ssq_out, normed_out) if (epi == EPI_RESADD and norm_w_out is not None) \
        else (out, ssq_out) if epi == EPI_RESADD else out
    return res, tuple(sch)


def embed(table, ids):
    _chk(table), _chk(ids, torch.int32)
    out = torch.empty(ids.numel(), table.shape[1], dtype=torch.bfloat16, device=table.device)
    check(lib().b200_op_embed(_p(table), _p(ids), _p(out), ids.numel(), table.shape[1], table.shape[0], _stream()))
    return out


def rmsnorm(x, w, eps, residual=None, row_index=None):
    """Returns normed output; `residual` (if given) is updated in place unless row_index is given."""
    _chk(x), _chk(w)
    rows = row_index.numel() if row_index is not None else x.shape[0]
    out = torch.empty(rows, x.shape[1], dtype=torch.bfloat16, device=x.device)
    check(lib().b200_op_rmsnorm(_p(x), _p(residual), _p(w), _p(out), _p(row_index), rows, x.shape[1], eps, _stream()))
    return out


def rope_kvwrite(qkv, positions, slots, cos_sin, kv_layer, q_heads, kv_heads):
    _chk(qkv), _chk(positions, torch.int32), _chk(slots, torch.int32), _chk(cos_sin), _chk(kv_layer)
    check(lib().b200_op_rope_kvwrite(_p(qkv), _p(positions), _p(slots), _p(cos_sin), _p(kv_layer), qkv.shape[0],
                                     q_heads, kv_heads, cos_sin.shape[0], _stream()))


def silu_mul(gu):
    _chk(gu)
    T, I2 = gu.shape
    out = torch.empty(T, I2 // 2, dtype=torch.bfloat16, device=gu.device)
    check(lib().b200_op_silu_mul(_p(gu), _p(out), T, I2 // 2, _stream()))
    return out


def argmax(logits):
    _chk(logits)
    out = torch.empty(logits.shape[0], dtype=torch.int32, device=logits.device)
    check(lib().b200_op_argmax(_p(logits), _p(out), logits.shape[0], logits.shape[1], logits.stride(0), _stream()))
    return out


def paged_attn(qkv, kv_layer, block_tables, work, q_heads, kv_heads, decode: bool, out=None, split: int = 0):
    """qkv: [T, (Hq+2Hkv)*128] (q read from it), work: int32 [n, 4] = (q_tok0, q_count, q_pos0, seq).
    split >= 1 (decode only): split-KV form with that many CTAs per (work item, KV head)."""
    _chk(qkv), _chk(kv_layer), _chk(block_tables, torch.int32), _chk(work, torch.int32)
    T = qkv.shape[0]
    if out is None:
        out = torch.zeros(T, q_heads * 128, dtype=torch.bfloat16, device=qkv.device)
    if split:
        assert decode
        check(lib().b200_op_paged_attn_decode_split(_p(qkv), qkv.shape[1], _p(out), out.shape[1], _p(kv_layer), _p(block_tables),
                                                    block_tables.shape[1], _p(work), work.shape[0], q_heads, kv_heads,
                                                    128 ** -0.5, split, _stream()))
        return out
    check(lib().b200_op_paged_attn(_p(qkv), qkv.shape[1], _p(out), out.shape[1], _p(kv_layer), _p(block_tables),
                                   block_tables.shape[1], _p(work), work.shape[0], q_heads, kv_heads,
                                   128 ** -0.5, 1 if decode else 0, _stream()))
    return out


def paged_attn_prefill_tc(qkv, kv_layer, block_tables, work, q_heads, kv_heads, out=None):
    """wgmma chunked-prefill attention; work: int32 [n, 4] = (q_tok0, q_count <= 64, q_pos0, seq)."""
    _chk(qkv), _chk(kv_layer), _chk(block_tables, torch.int32), _chk(work, torch.int32)
    T = qkv.shape[0]
    if out is None:
        out = torch.zeros(T, q_heads * 128, dtype=torch.bfloat16, device=qkv.device)
    check(lib().b200_op_paged_attn_prefill_tc(_p(qkv), T, qkv.shape[1], _p(out), out.shape[1], _p(kv_layer), _p(block_tables),
                                              block_tables.shape[1], _p(work), work.shape[0], q_heads, kv_heads, 128 ** -0.5, _stream()))
    return out


def init_uniform(n, seed, scale, offset, device="cuda"):
    out = torch.empty(n, dtype=torch.bfloat16, device=device)
    check(lib().b200_op_init_uniform(_p(out), n, seed & 0xFFFFFFFF, scale, offset, _stream()))
    return out
