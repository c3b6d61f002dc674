"""Op-level drivers over the C ABI (b200_op_*): torch is used only to own device memory and the
stream; every call goes straight into the hand-written CUDA kernels.  There is no fallback: without
the library or a GPU these raise."""
from __future__ import annotations

import ctypes as C

import numpy as np
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
          normed_out=None, norm_w_out=None, head_dim=0):
    """The fused projection GEMM (b200_op_gemm3).  x: [rows >= T, K] activations (or the residual for PRO_NORM),
    w: [N, K].  Returns (out, schedule) with schedule = (K-splits per tile, rule that chose them: 0 given by `force`,
    1 device-filling for one token tile, 2 device-filling over several token tiles (T > 128), CTAs).  head_dim (EPI_ROPE_KV):
    64 or 128, 0 = 128."""
    from ._lib import Gemm3Args
    _chk(x), _chk(w)
    T = x.shape[0] if T is None else T
    N, K = w.shape
    a = Gemm3Args(N=N, T=T, K=K, x_rows=x.shape[0], pro=pro, epi=epi, force=force, w=w.data_ptr(), x=x.data_ptr(), eps=eps,
                  q_heads=q_heads, kv_heads=kv_heads, n_valid=n_valid, head_dim=head_dim)
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


def score_rows(hidden, norm_w, score_w, row_index, flags, activation=0, eps=1e-5):
    """A score head's tail (b200_op_score_rows): fp32 [rows, L] logits score_w [L, H] . rmsnorm(hidden[row_index[s]]),
    with the activation (0 by label count, 1 sigmoid, 2 softmax, 3 none) on the rows whose flag is set."""
    _chk(hidden), _chk(norm_w), _chk(score_w), _chk(row_index, torch.int32), _chk(flags, torch.int32)
    rows, (L, H) = row_index.numel(), score_w.shape
    out = torch.empty(rows, L, dtype=torch.float32, device=hidden.device)
    check(lib().b200_op_score_rows(_p(hidden), _p(norm_w), _p(score_w), _p(row_index), _p(flags), rows, H, L, activation, eps,
                                   _p(out), _stream()))
    return out


def rope_kvwrite(qkv, positions, slots, cos_sin, kv_layer, q_heads, kv_heads, head_dim=None):
    """head_dim None: b200_op_rope_kvwrite (D = 128); 64 or 128: b200_op_rope_kvwrite_hd."""
    _chk(qkv), _chk(positions, torch.int32), _chk(slots, torch.int32), _chk(cos_sin), _chk(kv_layer)
    args = (_p(qkv), _p(positions), _p(slots), _p(cos_sin), _p(kv_layer), qkv.shape[0], q_heads, kv_heads, cos_sin.shape[0])
    if head_dim is None:
        check(lib().b200_op_rope_kvwrite(*args, _stream()))
    else:
        check(lib().b200_op_rope_kvwrite_hd(*args, head_dim, _stream()))


def silu_mul(gu, interleaved=False):
    """gu: [T, 2 I] as [gate | up], or with interleaved=True gate and up columns alternating in 64-column blocks (the
    engine's layout)."""
    _chk(gu)
    T, I2 = gu.shape
    out = torch.empty(T, I2 // 2, dtype=torch.bfloat16, device=gu.device)
    check(lib().b200_op_silu_mul_il(_p(gu), _p(out), T, I2 // 2, int(interleaved), _stream()))
    return out


def argmax(logits):
    _chk(logits)
    out = torch.empty(logits.shape[0], dtype=torch.int32, device=logits.device)
    check(lib().b200_op_argmax(_p(logits), _p(out), logits.shape[0], logits.shape[1], logits.stride(0), _stream()))
    return out


def sample(logits, temperature, top_k=0, top_p=1.0, seed=0, n=0, min_p=0.0):
    """Token per row of bf16 logits [S, V] (b200_op_sample).  Each parameter is a scalar or one value per row:
    temperature < 1e-5 = greedy; top_k 0 / -1 / >= V, top_p 1 and min_p 0 = off; seed (uint64) keys the row's Philox
    stream and n (the index of the token being generated) counts it."""
    _chk(logits)
    S = logits.shape[0]
    rows = np.empty(S, dtype=[("temperature", "<f4"), ("top_k", "<i4"), ("top_p", "<f4"), ("seed_lo", "<u4"),
                              ("seed_hi", "<u4"), ("n", "<i4"), ("min_p", "<f4")])
    seed = np.broadcast_to(np.asarray(seed, dtype=object), (S,))
    rows["temperature"] = np.broadcast_to(np.asarray(temperature, dtype=np.float32), (S,))
    rows["top_k"] = np.broadcast_to(np.asarray(top_k, dtype=np.int32), (S,))
    rows["top_p"] = np.broadcast_to(np.asarray(top_p, dtype=np.float32), (S,))
    rows["seed_lo"] = [int(s) & 0xFFFFFFFF for s in seed]
    rows["seed_hi"] = [(int(s) >> 32) & 0xFFFFFFFF for s in seed]
    rows["n"] = np.broadcast_to(np.asarray(n, dtype=np.int32), (S,))
    rows["min_p"] = np.broadcast_to(np.asarray(min_p, dtype=np.float32), (S,))
    rows_dev = torch.from_numpy(rows.view(np.int32).reshape(S, 7).copy()).to(logits.device)
    out = torch.empty(S, dtype=torch.int32, device=logits.device)
    check(lib().b200_op_sample(_p(logits), logits.stride(0), _p(rows_dev), S, logits.shape[1], _p(out), _stream()))
    return out


def penalize(logits, rows, restore=True):
    """The engine's logits edits on bf16 logits [S, V] (b200_op_penalize), one dict per row with any of presence_penalty,
    frequency_penalty, repetition_penalty (1 or 0 = off), min_tokens, prompt, output, logit_bias ({id: bias}) and stop_ids.
    restore=True: returns the edited rows and puts the raw values back into `logits`; False: edits `logits` in place and
    returns it."""
    _chk(logits)
    S, V = logits.shape
    keep, arr = _penalty_rows(rows)
    edited = torch.empty_like(logits) if restore else None
    check(lib().b200_op_penalize(_p(logits), logits.stride(0), S, V, arr, _p(edited), _stream()))
    return edited if restore else logits


def _penalty_rows(rows):
    """(the numpy arrays the rows point into, ctypes PenaltyRow array) of penalize()'s row dicts."""
    from ._lib import PenaltyRow
    keep, arr = [], (PenaltyRow * max(len(rows), 1))()

    def ptr(a, ct):
        keep.append(a)
        return a.ctypes.data_as(C.POINTER(ct)) if len(a) else None
    for s, r in enumerate(rows):
        prompt = np.ascontiguousarray(r.get("prompt", ()), dtype=np.int32)
        output = np.ascontiguousarray(r.get("output", ()), dtype=np.int32)
        stops = np.ascontiguousarray(r.get("stop_ids", ()), dtype=np.int32)
        bias = dict(r.get("logit_bias") or {})
        bid = np.ascontiguousarray(list(bias.keys()), dtype=np.int32)
        bval = np.ascontiguousarray(list(bias.values()), dtype=np.float32)
        arr[s] = PenaltyRow(presence_penalty=r.get("presence_penalty", 0.0), frequency_penalty=r.get("frequency_penalty", 0.0),
                            repetition_penalty=r.get("repetition_penalty", 1.0), min_tokens=r.get("min_tokens", 0),
                            num_prompt=len(prompt), prompt=ptr(prompt, C.c_int32), num_output=len(output),
                            output=ptr(output, C.c_int32), num_logit_bias=len(bid), logit_bias_ids=ptr(bid, C.c_int32),
                            logit_bias_values=ptr(bval, C.c_float), num_stop_ids=len(stops), stop_ids=ptr(stops, C.c_int32))
    return keep, arr


def penalty_lists(n_slots, cap, device="cuda"):
    """Record lists for penalty_list / penalize_update / penalize_slots: (recs int32 [n_slots, cap, 4], each record
    (id, count, bias as fp32 bits, flags), lens int32 [n_slots]), zeroed."""
    return (torch.zeros(n_slots, cap, 4, dtype=torch.int32, device=device),
            torch.zeros(n_slots, dtype=torch.int32, device=device))


def penalty_list(recs, lens, slot, V, row):
    """Build list `slot` of (recs, lens) from one penalize() row dict, as the engine does when it admits the request
    (b200_op_penalty_list)."""
    _chk(recs, torch.int32), _chk(lens, torch.int32)
    keep, arr = _penalty_rows([row])
    check(lib().b200_op_penalty_list(arr, V, _p(recs), _p(lens), recs.shape[0], recs.shape[1], slot, _stream()))


_SLOT_ROW = np.dtype([("row", "<i4"), ("slot", "<i4"), ("presence", "<f4"), ("frequency", "<f4"), ("repetition", "<f4"),
                      ("n_generated", "<i4"), ("min_tokens", "<i4"), ("history", "<i4")])


def _slot_rows(rows):
    """b200_penalty_slot_rows of (row, slot, presence, frequency, repetition, n_generated, min_tokens, history) tuples."""
    return np.array([tuple(r) for r in rows], dtype=_SLOT_ROW)


def penalize_update(recs, lens, rows, sampled, V):
    """One penalize_update launch (b200_op_penalize_update): for each (row, slot, presence, frequency, repetition,
    n_generated, min_tokens, history) tuple with history, sampled[row] (host ints, one per logits row) joins list `slot`."""
    _chk(recs, torch.int32), _chk(lens, torch.int32)
    a = _slot_rows(rows)
    s = np.ascontiguousarray(sampled, dtype=np.int32)
    check(lib().b200_op_penalize_update(a.ctypes.data, len(a), s.ctypes.data_as(C.POINTER(C.c_int32)), len(s), V, _p(recs),
                                        _p(lens), recs.shape[0], recs.shape[1], _stream()))


def penalize_slots(logits, rows, recs, lens, restore=True):
    """penalize() on the lists of (recs, lens) (b200_op_penalize_slots): each (row, slot, ...) tuple, as in
    penalize_update, edits logits row `row` from list `slot`.  restore as in penalize()."""
    _chk(logits), _chk(recs, torch.int32), _chk(lens, torch.int32)
    S, V = logits.shape
    a = _slot_rows(rows)
    edited = torch.empty_like(logits) if restore else None
    check(lib().b200_op_penalize_slots(_p(logits), logits.stride(0), S, V, a.ctypes.data, len(a), _p(recs), _p(lens),
                                       recs.shape[0], recs.shape[1], _p(edited), _stream()))
    return edited if restore else logits


def logprobs(logits, tokens, top_n):
    """Log-probabilities of bf16 logits [S, V] (b200_op_logprobs): returns (lp float32 [S] of tokens[s], top_ids int32
    [S, 20], top_lp float32 [S, 20]); row s's first top_n[s] entries (scalar or per row, 0..20) are its most likely tokens,
    the rest stay zero."""
    _chk(logits)
    S, V = logits.shape
    dev = logits.device
    tok = torch.as_tensor(np.broadcast_to(np.asarray(tokens, dtype=np.int32), (S,)).copy()).to(dev)
    n = torch.as_tensor(np.broadcast_to(np.asarray(top_n, dtype=np.int32), (S,)).copy()).to(dev)
    lp = torch.zeros(S, dtype=torch.float32, device=dev)
    top_ids = torch.zeros(S, 20, dtype=torch.int32, device=dev)
    top_lp = torch.zeros(S, 20, dtype=torch.float32, device=dev)
    check(lib().b200_op_logprobs(_p(logits), logits.stride(0), S, V, _p(tok), _p(n), _p(lp), _p(top_ids), _p(top_lp),
                                 _stream()))
    return lp, top_ids, top_lp


def logprobs_rank(logits, tokens, top_n):
    """logprobs() plus the rank of tokens[s] (b200_op_logprobs_rank): returns (lp, rank int32 [S], top_ids, top_lp); the
    rank is the number of tokens whose logit is >= tokens[s]'s."""
    _chk(logits)
    S, V = logits.shape
    dev = logits.device
    tok = torch.as_tensor(np.broadcast_to(np.asarray(tokens, dtype=np.int32), (S,)).copy()).to(dev)
    n = torch.as_tensor(np.broadcast_to(np.asarray(top_n, dtype=np.int32), (S,)).copy()).to(dev)
    lp = torch.zeros(S, dtype=torch.float32, device=dev)
    rank = torch.zeros(S, dtype=torch.int32, device=dev)
    top_ids = torch.zeros(S, 20, dtype=torch.int32, device=dev)
    top_lp = torch.zeros(S, 20, dtype=torch.float32, device=dev)
    check(lib().b200_op_logprobs_rank(_p(logits), logits.stride(0), S, V, _p(tok), _p(n), _p(lp), _p(rank), _p(top_ids),
                                      _p(top_lp), _stream()))
    return lp, rank, top_ids, top_lp


def paged_attn(qkv, kv_layer, block_tables, work, q_heads, kv_heads, decode: bool, out=None, split: int = 0, head_dim=None):
    """qkv: [T, (Hq+2Hkv)*D] (q read from it), work: int32 [n, 4] = (q_tok0, q_count, q_pos0, seq).
    split >= 1 (decode only): split-KV form with that many CTAs per (work item, KV head).
    head_dim None: the entry points without _hd (D = 128); 64 or 128: their _hd siblings."""
    _chk(qkv), _chk(kv_layer), _chk(block_tables, torch.int32), _chk(work, torch.int32)
    T = qkv.shape[0]
    D = 128 if head_dim is None else head_dim
    if out is None:
        out = torch.zeros(T, q_heads * D, dtype=torch.bfloat16, device=qkv.device)
    args = (_p(qkv), qkv.shape[1], _p(out), out.shape[1], _p(kv_layer), _p(block_tables), block_tables.shape[1], _p(work),
            work.shape[0], q_heads, kv_heads, D ** -0.5)
    hd = () if head_dim is None else (head_dim,)
    if split:
        assert decode
        fn = lib().b200_op_paged_attn_decode_split if head_dim is None else lib().b200_op_paged_attn_decode_split_hd
        check(fn(*args, split, *hd, _stream()))
        return out
    fn = lib().b200_op_paged_attn if head_dim is None else lib().b200_op_paged_attn_hd
    check(fn(*args, 1 if decode else 0, *hd, _stream()))
    return out


def paged_attn_prefill_tc(qkv, kv_layer, block_tables, work, q_heads, kv_heads, out=None, head_dim=None):
    """wgmma chunked-prefill attention; work: int32 [n, 4] = (q_tok0, q_count <= 64, q_pos0, seq).  head_dim as paged_attn."""
    _chk(qkv), _chk(kv_layer), _chk(block_tables, torch.int32), _chk(work, torch.int32)
    T = qkv.shape[0]
    D = 128 if head_dim is None else head_dim
    if out is None:
        out = torch.zeros(T, q_heads * D, dtype=torch.bfloat16, device=qkv.device)
    args = (_p(qkv), T, qkv.shape[1], _p(out), out.shape[1], _p(kv_layer), _p(block_tables), block_tables.shape[1], _p(work),
            work.shape[0], q_heads, kv_heads, D ** -0.5)
    if head_dim is None:
        check(lib().b200_op_paged_attn_prefill_tc(*args, _stream()))
    else:
        check(lib().b200_op_paged_attn_prefill_tc_hd(*args, head_dim, _stream()))
    return out


def init_uniform(n, seed, scale, offset, device="cuda"):
    out = torch.empty(n, dtype=torch.bfloat16, device=device)
    check(lib().b200_op_init_uniform(_p(out), n, seed & 0xFFFFFFFF, scale, offset, _stream()))
    return out


def kv_copy_blocks(kv, num_layers, layer_stride_bytes, block_bytes, src, dst):
    """The fork's page copy (b200_op_kv_copy_blocks) on a KV pool tensor `kv` (any dtype, contiguous): for each pair i and
    layer l, the block_bytes at byte l * layer_stride_bytes + src[i] * block_bytes go to dst[i]'s page.  In place."""
    assert kv.is_cuda and kv.is_contiguous()
    s = torch.as_tensor(np.asarray(src, dtype=np.int32), device=kv.device)
    d = torch.as_tensor(np.asarray(dst, dtype=np.int32), device=kv.device)
    check(lib().b200_op_kv_copy_blocks(_p(kv), num_layers, layer_stride_bytes, block_bytes, _p(s), _p(d), len(s), _stream()))
    return kv
