"""Thin Python wrappers over the C ABI: torch tensors in, raw pointers + sizes across the boundary.

torch is used here only for device memory, streams and shape bookkeeping.
"""
import ctypes

import torch

from . import _lib
from ._lib import (ACT_NONE, ACT_RELU, AUX_ADD, AUX_MASK_NZ, AUX_NONE, PK_BF16, PK_F32, SEL_KZ, SEL_ZB0, SEL_ZB1,  # noqa: F401  (re-exported: engine uses K.ACT_RELU ...)
                   SEL_ZERO, GemmDesc, View4, check, lib)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dt(t):
    if t.dtype == torch.bfloat16:
        return PK_BF16
    if t.dtype == torch.float32:
        return PK_F32
    raise TypeError("unsupported dtype %s" % t.dtype)


def _P(t):
    """a tensor's device address, or NULL for None"""
    return t.data_ptr() if t is not None else None


def _fill_view(v, t):
    """torch view with <= 4 dims, last dim contiguous -> View4 (dim[0] = contiguous extent)."""
    assert t.is_cuda and t.dim() >= 1 and t.dim() <= 4, "views must be CUDA tensors with 1..4 dims"
    assert t.stride(-1) == 1 or t.shape[-1] == 1, "innermost dimension must be contiguous"
    shape = list(t.shape)[::-1]
    strides = list(t.stride())[::-1]
    v.ptr = t.data_ptr()
    for i in range(4):
        v.dim[i] = shape[i] if i < len(shape) else 1
    for i in range(3):
        v.stride[i] = strides[i + 1] if i + 1 < len(strides) else 0
    return v


def gemm(a, b, c, a_mn=False, b_mn=False, a_sel=(SEL_ZB0, SEL_ZB1), b_sel=(SEL_ZB0, SEL_ZB1), kz_count=1,
         a_row_off=None, b_row_off=None, alpha=1.0, bias=None, act=ACT_NONE, drop_p=0.0, drop_seed=0,
         aux=None, aux_mode=AUX_NONE, aux_scale=1.0, accumulate=False, block_n=0, k_splits=0, row_lse=None, a_rows_dev=None):
    """C = epilogue(alpha * sum_p A_p @ B_p^T) on the wgmma tensor cores (include/pika_b200.h).

    a, b: a bf16 view or a list of views (pairs).  Views are torch tensors of <= 4 dims laid out
    (z3, z2, rows, contiguous):  K-major A = (.., M, K), MN-major A = (.., K, M); same for B with N.
    c: (zb1, zb0, M, N) view, bf16 or f32.  aux: tensor broadcast-compatible with c's logical shape,
    given as a view with the same number of dims as c.
    a_rows_dev: int32 device tensor [1]; only that many leading rows of A take part (pk_gemm_desc.a_rows_dev).
    """
    a = a if isinstance(a, (list, tuple)) else [a]
    b = b if isinstance(b, (list, tuple)) else [b]
    assert len(a) == len(b) and 1 <= len(a) <= _lib.MAX_PAIRS
    d = GemmDesc()
    d.n_pairs = len(a)
    for i, (ai, bi) in enumerate(zip(a, b)):
        assert ai.dtype == torch.bfloat16 and bi.dtype == torch.bfloat16, "GEMM operands must be bf16"
        _fill_view(d.a[i], ai)
        _fill_view(d.b[i], bi)
        d.a_row_off[i] = a_row_off[i] if a_row_off else 0
        d.b_row_off[i] = b_row_off[i] if b_row_off else 0
    d.a_mn_major, d.b_mn_major = int(a_mn), int(b_mn)
    # selectors only matter for dims that exist (extent > 1); default maps z2<-zb0, z3<-zb1
    d.a_sel2, d.a_sel3 = a_sel
    d.b_sel2, d.b_sel3 = b_sel
    d.kz_count = kz_count
    _fill_view(d.c, c)
    d.c_dtype = _dt(c)
    d.c_accumulate = int(accumulate)
    d.alpha = alpha
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous()
        d.bias = bias.data_ptr()
    d.act = act
    d.drop_p = drop_p
    d.drop_seed = drop_seed & 0xFFFFFFFF
    if aux is not None:
        assert aux.dim() == c.dim() and aux.stride(-1) == 1
        d.aux_mode = aux_mode
        d.aux = aux.data_ptr()
        d.aux_dtype = _dt(aux)
        st = list(aux.stride())[::-1]          # (n, m, zb0, zb1)
        for i in range(3):
            d.aux_stride[i] = st[i + 1] if i + 1 < len(st) else 0
        d.aux_scale = aux_scale
    d.block_n = block_n
    d.k_splits = k_splits
    if row_lse is not None:
        assert row_lse.dtype == torch.float32 and row_lse.is_contiguous() and c.dim() == 2
        assert tuple(row_lse.shape) == (row_lse_parts(c.shape[-2], c.shape[-1], block_n), c.shape[-2], 2)
        d.row_lse = row_lse.data_ptr()
    if a_rows_dev is not None:
        assert a_rows_dev.dtype == torch.int32 and a_rows_dev.is_cuda
        d.a_rows_dev = a_rows_dev.data_ptr()
    check(lib.pk_gemm_bf16(d, _stream()), "pk_gemm_bf16")
    return c


def row_lse_parts(M, N, block_n=0):
    """number of per-row (max, sum-exp) partials the GEMM writes into ``row_lse`` for an [M, N] output: one per N tile
    (every row's columns are owned by one CTA)"""
    return int(lib.pk_gemm_row_lse_parts(M, N, block_n))


def _emission_reg(fastemit_lambda, delay_penalty):
    """-> the two floats, or None when both are 0 (the plain entry points run)"""
    lf, ld = float(fastemit_lambda), float(delay_penalty)
    return None if lf == 0.0 and ld == 0.0 else (lf, ld)


def rnnt_loss_fwd_bwd(logits, labels, frame_lens, label_lens, V=None, grad_scale=None, dlogits=None, want_grad=True, colsum=None,
                      row_lse=None, fastemit_lambda=0.0, delay_penalty=0.0):
    """logits [B,T,U1,ldv] (bf16|f32) -> (costs [B] f32, dlogits).  dlogits may alias logits.
    row_lse [n_parts, B*T*U1, 2]: per-row log-sum-exp partials written by the producing GEMM (skips the first pass).
    fastemit_lambda, delay_penalty: emission regularisation (include/pika_b200.h, *_reg); both 0 is the plain loss."""
    B, T, U1, ldv = logits.shape
    V = ldv if V is None else V
    assert logits.is_contiguous() and labels.dtype == torch.int32 and labels.dim() == 2
    assert frame_lens.dtype == torch.int32 and label_lens.dtype == torch.int32
    reg = _emission_reg(fastemit_lambda, delay_penalty)
    ws_bytes = int(lib.pk_rnnt_loss_workspace_bytes(B, T, U1))
    if colsum is not None:
        ws_bytes += int(lib.pk_rnnt_loss_colsum_workspace_bytes(B, T, U1, ldv))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=logits.device)
    costs = torch.empty(B, dtype=torch.float32, device=logits.device)
    if want_grad and dlogits is None:
        dlogits = torch.empty_like(logits)
    args = (_P(logits), _dt(logits), _P(labels), _P(frame_lens), _P(label_lens), B, T, U1, V, ldv, max(labels.stride(0), 1), _P(grad_scale),
            _P(costs), _P(dlogits if want_grad else None), _P(colsum), _P(ws), ws_bytes)
    if row_lse is not None:
        assert row_lse.dtype == torch.float32 and row_lse.is_contiguous() and tuple(row_lse.shape[1:]) == (B * T * U1, 2)
        args += (_P(row_lse), int(row_lse.shape[0]))
        if reg is None:
            check(lib.pk_rnnt_loss_fwd_bwd_lse(*args, _stream()), "pk_rnnt_loss_fwd_bwd_lse")
        else:
            check(lib.pk_rnnt_loss_fwd_bwd_lse_reg(*args, *reg, _stream()), "pk_rnnt_loss_fwd_bwd_lse_reg")
        return costs, dlogits
    if reg is None:
        check(lib.pk_rnnt_loss_fwd_bwd(*args, _stream()), "pk_rnnt_loss_fwd_bwd")
    else:
        check(lib.pk_rnnt_loss_fwd_bwd_reg(*args, *reg, _stream()), "pk_rnnt_loss_fwd_bwd_reg")
    return costs, dlogits


def rnnt_loss_compact(logits, labels, frame_lens, label_lens, h, V=None, colsum=None, row_lse=None, fastemit_lambda=0.0, delay_penalty=0.0):
    """bf16 logits [B,T,U1,ldv], joint activations h [B*T*U1, H] -> (costs [B], dz_c [R, ldv], h_c [R, H], row_map [R], row_count [1]).
    Only the rows whose gradient is not all zeros are stored: dz_c / h_c rows [0, row_count) hold them in row order, row_map[r] is the
    row's index there or -1.  dz_c is a new buffer as large as the logits (the two are alive together while the gradient is formed)."""
    B, T, U1, ldv = logits.shape
    V = ldv if V is None else V
    R, H = B * T * U1, h.shape[-1]
    assert logits.is_contiguous() and logits.dtype == torch.bfloat16 and labels.dtype == torch.int32 and labels.dim() == 2
    assert frame_lens.dtype == torch.int32 and label_lens.dtype == torch.int32
    assert h.is_contiguous() and h.dtype == torch.bfloat16 and h.numel() == R * H
    ws_bytes = int(lib.pk_rnnt_loss_workspace_bytes(B, T, U1))
    if colsum is not None:
        ws_bytes += int(lib.pk_rnnt_loss_colsum_workspace_bytes(B, T, U1, ldv))
    dev = logits.device
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    costs = torch.empty(B, dtype=torch.float32, device=dev)
    dz_c = torch.empty(R, ldv, dtype=torch.bfloat16, device=dev)
    h_c = torch.empty(R, H, dtype=torch.bfloat16, device=dev)
    row_map = torch.empty(R, dtype=torch.int32, device=dev)
    row_count = torch.empty(1, dtype=torch.int32, device=dev)
    if row_lse is not None:
        assert row_lse.dtype == torch.float32 and row_lse.is_contiguous() and tuple(row_lse.shape[1:]) == (R, 2)
    args = (_P(logits), PK_BF16, _P(labels), _P(frame_lens), _P(label_lens), B, T, U1, V, ldv, max(labels.stride(0), 1), None, _P(costs),
            _P(dz_c), _P(colsum), _P(ws), ws_bytes, _P(row_lse), int(row_lse.shape[0]) if row_lse is not None else 0, _P(h), H, _P(h_c),
            _P(row_map), _P(row_count))
    reg = _emission_reg(fastemit_lambda, delay_penalty)
    if reg is None:
        check(lib.pk_rnnt_loss_fwd_bwd_compact(*args, _stream()), "pk_rnnt_loss_fwd_bwd_compact")
    else:
        check(lib.pk_rnnt_loss_fwd_bwd_compact_reg(*args, *reg, _stream()), "pk_rnnt_loss_fwd_bwd_compact_reg")
    return costs, dz_c, h_c, row_map, row_count


# ------------------------------------------------------------------------------------------------
# thin wrappers for the memory-bound kernels


def cast_split(src, hi, lo=None, cols_pad=None, scale=1.0):
    """src [rows, cols] (f32|bf16, row stride free) -> hi (and lo) bf16 [rows, cols_pad]."""
    rows, cols = src.shape
    cols_pad = cols_pad or cols
    assert hi.shape[-1] == cols_pad and hi.stride(-1) == 1 and src.stride(-1) == 1
    check(lib.pk_cast_split(_P(src), _dt(src), src.stride(0), _P(hi), _P(lo), hi.stride(0), rows, cols, cols_pad, scale, _stream()),
          "pk_cast_split")


def attention_lse_stride(T):
    """row pitch of the per-(batch, head) lse / D vectors (64-element aligned so that tiles of them are bulk-copy sources)"""
    return int(lib.pk_attention_lse_stride(T))


def attention_keep_bits(B, T, heads, drop_p, device):
    """the dropout keep-bit buffer attention_fwd fills and attention_bwd reads (None when drop_p == 0: nothing is dropped)"""
    if drop_p <= 0:
        return None
    return torch.empty(int(lib.pk_attention_keep_bits_bytes(B, T, heads)) // 4, dtype=torch.int32, device=device)


def attention_chunk_admits_all(T, chunk):
    """True when the chunk mask ``chunk`` = (chunk_len, chunk_off, left_chunks) lets every query of a T-frame sequence see every key"""
    rc = int(lib.pk_attention_chunk_admits_all(T, *chunk))
    check(min(rc, 0), "pk_attention_chunk_admits_all")
    return rc == 1


def attention_fwd(qkv, out, lse, heads, alpha, drop_p=0.0, seed=0, keep_bits=None, chunk=None):
    """qkv [B,T,3D] bf16 (q | k | v column blocks) -> out [B,T,D], lse [B*heads*T] f32 (fused attention, head dim 64).
    keep_bits (attention_keep_bits): also write the dropout decisions there, for attention_bwd to read.  chunk = (chunk_len,
    chunk_off, left_chunks): the chunk mask of pk_attention_fwd_chunk (keep_bits then needed whenever drop_p > 0)."""
    B, T, D3 = qkv.shape
    D = D3 // 3
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and out.is_contiguous() and out.shape == (B, T, D)
    assert lse.dtype == torch.float32 and lse.numel() == B * heads * attention_lse_stride(T)
    base, es = qkv.data_ptr(), 2
    args = (base, base + D * es, base + 2 * D * es, D3, _P(out), D, _P(lse), B, T, heads, D // heads, alpha, drop_p, seed & 0xFFFFFFFF)
    if chunk is not None:
        check(lib.pk_attention_fwd_chunk(*args, _P(keep_bits), *chunk, _stream()), "pk_attention_fwd_chunk")
        return
    if keep_bits is None:
        check(lib.pk_attention_fwd(*args, _stream()), "pk_attention_fwd")
        return
    assert keep_bits.is_contiguous() and keep_bits.numel() * keep_bits.element_size() >= lib.pk_attention_keep_bits_bytes(B, T, heads)
    check(lib.pk_attention_fwd_bits(*args, _P(keep_bits), _stream()), "pk_attention_fwd_bits")


def attention_bwd(qkv, out, dout, lse, dqkv, heads, alpha, drop_p=0.0, seed=0, keep_bits=None, chunk=None):
    """dqkv <- gradient of attention_fwd; with keep_bits (the forward's) the mask is read from them, otherwise drawn from seed.
    chunk: the forward's chunk mask (pk_attention_bwd_chunk; reads keep_bits)."""
    B, T, D3 = qkv.shape
    D = D3 // 3
    assert dout.is_contiguous() and dqkv.is_contiguous() and dqkv.shape == qkv.shape and dout.dtype == torch.bfloat16
    ws = torch.zeros(B * heads * attention_lse_stride(T), dtype=torch.float32, device=qkv.device)     # D scratch (the kernel writes its padding too)
    base, gb, es = qkv.data_ptr(), dqkv.data_ptr(), 2
    args = (base, base + D * es, base + 2 * D * es, D3, _P(out), D, _P(dout), D, _P(lse), _P(ws),
            gb, gb + D * es, gb + 2 * D * es, D3, B, T, heads, D // heads, alpha, drop_p)
    if chunk is not None:
        check(lib.pk_attention_bwd_chunk(*args, _P(keep_bits), *chunk, _stream()), "pk_attention_bwd_chunk")
    elif keep_bits is None:
        check(lib.pk_attention_bwd(*args, seed & 0xFFFFFFFF, _stream()), "pk_attention_bwd")
    else:
        check(lib.pk_attention_bwd_bits(*args, _P(keep_bits), _stream()), "pk_attention_bwd_bits")


_col_ws = {}


def col_ws(C, device):
    """persistent scratch for the two-stage column reductions (per device, per C)"""
    key = (C, str(device))
    if key not in _col_ws:
        _col_ws[key] = torch.empty(int(lib.pk_colstats_ws_floats(C)) + 2 * C, dtype=torch.float32, device=device)
    return _col_ws[key]


def bn_fwd(x, y, w, b, eps, train, momentum, run_mean, run_var, mean, rstd, ws=None):
    rows, C = x.shape
    ws = col_ws(C, x.device)
    check(lib.pk_bn_fwd(_P(x), _P(y), _dt(x), rows, C, _P(w), _P(b), eps, int(train), momentum,
                        _P(run_mean), _P(run_var), _P(mean), _P(rstd), _P(ws), _stream()), "pk_bn_fwd")


def bn_bwd(dy, x, dx, w, mean, rstd, train, relu_mask, dw, db):
    rows, C = x.shape
    check(lib.pk_bn_bwd(_P(dy), _P(x), _P(dx), _dt(x), rows, C, _P(w), _P(mean), _P(rstd), int(train),
                        int(relu_mask), _P(dw), _P(db), _P(col_ws(C, x.device)), _stream()), "pk_bn_bwd")


def colsum(x, out):
    rows, C = x.shape
    assert x.is_contiguous()
    check(lib.pk_colsum(_P(x), _dt(x), rows, C, _P(out), _P(col_ws(C, x.device)), _stream()), "pk_colsum")


def layernorm_fwd(x, y, w, b, eps, mean, rstd):
    rows, C = x.shape
    check(lib.pk_layernorm_fwd(_P(x), _P(y), _dt(x), rows, C, _P(w), _P(b), eps, _P(mean), _P(rstd), _stream()), "pk_layernorm_fwd")


def layernorm_bwd(dy, x, dx, w, mean, rstd, dw, db):
    rows, C = x.shape
    check(lib.pk_layernorm_bwd(_P(dy), _P(x), _P(dx), _dt(x), rows, C, _P(w), _P(mean), _P(rstd), _P(dw), _P(db), _stream()),
          "pk_layernorm_bwd")


def softmax_fwd(S, P, Pd, n, drop_p, seed):
    rows = S.numel() // S.shape[-1]
    check(lib.pk_softmax_fwd(_P(S), S.shape[-1], _P(P), _P(Pd), _dt(P), P.shape[-1], rows, n, drop_p, seed & 0xFFFFFFFF, _stream()),
          "pk_softmax_fwd")


def softmax_masked_fwd(S, P, Pd, n, q_len, heads, causal, key_pad, drop_p, seed):
    """rows of S = (sequence, head, query); key c of query i is dropped when c > i (causal) or key_pad[sequence, c] != 0"""
    rows = S.numel() // S.shape[-1]
    if key_pad is not None:
        assert key_pad.dtype == torch.uint8 and key_pad.is_contiguous() and key_pad.shape[-1] == n
    check(lib.pk_softmax_masked_fwd(_P(S), S.shape[-1], _P(P), _P(Pd), _dt(P), P.shape[-1], rows, n, q_len, heads, int(bool(causal)),
                                    _P(key_pad), drop_p, seed & 0xFFFFFFFF, _stream()), "pk_softmax_masked_fwd")


def softmax_chunk_fwd(S, P, Pd, n, chunk, drop_p, seed):
    """rows of S = (sequence, head, query i < n); query i keeps the keys its chunk allows (chunk = (chunk_len, chunk_off, left_chunks),
    the mask of pk_attention_fwd_chunk)"""
    rows = S.numel() // S.shape[-1]
    check(lib.pk_softmax_chunk_fwd(_P(S), S.shape[-1], _P(P), _P(Pd), _dt(P), P.shape[-1], rows, n, *chunk, drop_p, seed & 0xFFFFFFFF,
                                   _stream()), "pk_softmax_chunk_fwd")


def softmax_bwd(dPd, P, dS, n, drop_p, seed):
    rows = P.numel() // P.shape[-1]
    check(lib.pk_softmax_bwd(_P(dPd), dPd.shape[-1], _P(P), P.shape[-1], _P(dS), _dt(P), rows, n, drop_p, seed & 0xFFFFFFFF, _stream()),
          "pk_softmax_bwd")


def softmax_masked_relpos_fwd(S, QR, P, Pd, Pb, n, heads, causal, key_pad, max_rel, drop_p, seed):
    """pk_softmax_masked_fwd with the relative-position key terms QR [sequences*n*heads, ld_r] added along the band; writes the bucket
    sums Pb (same shape) of Pd.  Rows of S are (sequence, head, query), rows of QR / Pb (sequence, query, head)."""
    rows = S.numel() // S.shape[-1]
    if key_pad is not None:
        assert key_pad.dtype == torch.uint8 and key_pad.is_contiguous() and key_pad.shape[-1] == n
    assert QR.dtype == torch.float32 and Pb.dtype == torch.float32 and QR.stride(-1) == 1 and Pb.stride() == QR.stride()
    check(lib.pk_softmax_masked_relpos_fwd(_P(S), S.shape[-1], _P(QR), QR.stride(0), _P(P), _P(Pd), _dt(P), P.shape[-1],
                                           rows, n, n, heads, int(bool(causal)), _P(key_pad), max_rel, _P(Pb),
                                           drop_p, seed & 0xFFFFFFFF, _stream()), "pk_softmax_masked_relpos_fwd")


def softmax_relpos_bwd(dPd, G, P, dS, dSb, n, heads, max_rel, drop_p, seed):
    """pk_softmax_bwd with the relative-position value terms G = dO R^T added along the band; writes the bucket sums dSb of dS"""
    rows = P.numel() // P.shape[-1]
    assert G.dtype == torch.float32 and dSb.dtype == torch.float32 and G.stride(-1) == 1 and dSb.stride() == G.stride()
    check(lib.pk_softmax_relpos_bwd(_P(dPd), dPd.shape[-1], _P(G), G.stride(0), _P(P), P.shape[-1], _P(dS), _dt(P),
                                    rows, n, n, heads, max_rel, _P(dSb), drop_p, seed & 0xFFFFFFFF, _stream()),
          "pk_softmax_relpos_bwd")


def dropout(x, y, p, seed):
    check(lib.pk_dropout(_P(x), _P(y), _dt(x), x.numel(), p, seed & 0xFFFFFFFF, _stream()), "pk_dropout")


def mask_nz(dy, y, dx, scale):
    check(lib.pk_mask_nz(_P(dy), _P(y), _P(dx), _dt(y), y.numel(), scale, _stream()), "pk_mask_nz")


def add(a, b, o):
    check(lib.pk_add(_P(a), _P(b), _P(o), _dt(a), a.numel(), _stream()), "pk_add")


def log_softmax(x, y, n, scale=1.0):
    rows = x.numel() // x.shape[-1]
    check(lib.pk_log_softmax(_P(x), _dt(x), x.shape[-1], _P(y), rows, n, scale, _stream()), "pk_log_softmax")


def joint_gate_fwd(ex, py, h, B, T, U1, H):
    check(lib.pk_joint_gate_fwd(_P(ex), _P(py), _P(h), _dt(ex), B, T, U1, H, h.stride(0), _stream()), "pk_joint_gate_fwd")


def joint_gate_bwd(ex, py, dh, dex, dpy, B, T, U1, H, dh_map=None):
    """dh_map [B*T*U1] int32 (rnnt_loss_compact): dh holds the kept rows only, row r of the joint is dh[dh_map[r]] or zeros"""
    check(lib.pk_joint_gate_bwd(_P(ex), _P(py), _P(dh), _P(dh_map), _P(dex), _P(dpy), _dt(ex), B, T, U1, H, _stream()), "pk_joint_gate_bwd")


def lstm_cell_fwd(gx, gh, c_prev, c_out, h_out, gates_save, B, H):
    check(lib.pk_lstm_cell_fwd(_P(gx), gx.stride(0), _P(gh), gh.stride(0) if gh is not None else 0, _P(c_prev), _P(c_out), _P(h_out),
                               _dt(h_out), h_out.stride(0), _P(gates_save), B, H, _stream()), "pk_lstm_cell_fwd")


def lstm_cell_bwd(dh_out, dh_rec, dc_next, gates, c, c_prev, dgates, dc_prev, B, H):
    check(lib.pk_lstm_cell_bwd(_P(dh_out), dh_out.stride(0) if dh_out is not None else 0, _P(dh_rec), _P(dc_next), _P(gates), _P(c),
                               _P(c_prev), _P(dgates), _dt(dgates), _P(dc_prev), B, H, _stream()), "pk_lstm_cell_bwd")


def embedding_fwd(idx, table, out):
    n, ld = out.shape
    check(lib.pk_embedding_fwd(_P(idx), _P(table), table.shape[1], _P(out), _dt(out), ld, n, _stream()), "pk_embedding_fwd")


def embedding_bwd(idx, dout, dtable, padding_idx):
    n, ld = dout.shape
    check(lib.pk_embedding_bwd(_P(idx), _P(dout), _dt(dout), ld, dtable.shape[1], _P(dtable), n,
                               padding_idx if padding_idx is not None else -1, _stream()), "pk_embedding_bwd")


def absmax(x, out, nan_flag=None):
    check(lib.pk_absmax(_P(x), x.numel(), _P(out), _P(nan_flag), _stream()), "pk_absmax")


def sgd_nesterov_clip(p, g, buf, lr, momentum, max_norm, absmax_t, first, nan_flag=None):
    check(lib.pk_sgd_nesterov_clip(_P(p), _P(g), _P(buf), p.numel(), lr, momentum, max_norm, _P(absmax_t), _P(nan_flag), int(first),
                                   _stream()), "pk_sgd_nesterov_clip")


def bmuf_delta(glob, local, delta):
    check(lib.pk_bmuf_delta(_P(glob), _P(local), _P(delta), glob.numel(), _stream()), "pk_bmuf_delta")


def bmuf_update(glob, local, delta_prev, delta_sum, world, bm, blr):
    check(lib.pk_bmuf_update(_P(glob), _P(local), _P(delta_prev), _P(delta_sum), glob.numel(), world, bm, blr, _stream()),
          "pk_bmuf_update")


def adam_clip(p, g, exp_avg, exp_avg_sq, lr, betas, eps, step, max_norm=-1.0, absmax_t=None, nan_flag=None, p_out2=None):
    """clip (when max_norm > 0, from pk_absmax's absmax_t / nan_flag) + one Adam step at ``step`` (the already-incremented,
    possibly fractional step count); the bias corrections are formed here in double, as torch.optim.Adam forms them"""
    for t in (g, exp_avg, exp_avg_sq) + ((p_out2,) if p_out2 is not None else ()):
        assert t.numel() == p.numel() and t.dtype == torch.float32 and t.is_contiguous()
    beta1, beta2 = betas
    bc1 = 1 - beta1 ** step
    bc2_sqrt = (1 - beta2 ** step) ** 0.5
    on = max_norm > 0
    check(lib.pk_adam_clip(_P(p), _P(g), _P(exp_avg), _P(exp_avg_sq), _P(p_out2), p.numel(), lr, beta1, beta2, eps, bc1, bc2_sqrt,
                           max_norm, _P(absmax_t if on else None), _P(nan_flag if on else None), _stream()), "pk_adam_clip")


def bmuf_adam_update(glob, local, delta_prev, exp_avg_g, exp_avg_sq_g, msg, world, bm, blr, beta1_tau, beta1_rho, beta2_tau,
                     beta2_rho):
    """msg: [delta_sum; exp_avg_sum; exp_avg_sq_sum] (3n); the powers of beta are formed by the caller in double"""
    n = glob.numel()
    assert msg.numel() == 3 * n and all(t.numel() == n for t in (local, delta_prev, exp_avg_g, exp_avg_sq_g))
    check(lib.pk_bmuf_adam_update(_P(glob), _P(local), _P(delta_prev), _P(exp_avg_g), _P(exp_avg_sq_g), _P(msg), n, world, bm, blr,
                                  beta1_tau, beta1_rho, beta2_tau, beta2_rho, _stream()), "pk_bmuf_adam_update")


_lstm_ws = {}


def _lstm_scratch(H, device):
    key = (H, str(device))
    if key not in _lstm_ws:
        _lstm_ws[key] = torch.zeros(int(lib.pk_lstm_seq_workspace_bytes(H)), dtype=torch.uint8, device=device)
    return _lstm_ws[key]


def _lens_arg(lens, B):
    assert lens is None or (lens.dtype == torch.int32 and lens.is_contiguous() and lens.numel() == B)
    return _P(lens)


def lstm_seq_fwd_ex(gx, w_hh, out, gates_save, cs, lens=None, reverse=False):
    """gx [n_dir,B,U,4H] f32; w_hh bf16 [n_dir*4H,H]; out [B,U,ldo] (a column-slice view is fine: direction d writes columns
    [d*H, (d+1)*H) of it); gates_save [n_dir,U,B,4H], cs [n_dir,U,B,H]; lens int32 [B] or None."""
    n_dir, B, U, G4 = gx.shape
    H = G4 // 4
    assert gx.is_contiguous() and w_hh.dtype == torch.bfloat16 and w_hh.is_contiguous() and w_hh.shape[0] == n_dir * G4
    assert out.stride(2) == 1 and out.stride(0) == U * out.stride(1) and out.shape[-1] == n_dir * H
    check(lib.pk_lstm_seq_fwd_ex(_P(gx), _P(w_hh), _P(out), _dt(out), out.stride(1), _P(gates_save), _P(cs), _lens_arg(lens, B),
                                 B, U, H, n_dir, int(reverse), _P(_lstm_scratch(n_dir * H, gx.device)), _stream()),
          "pk_lstm_seq_fwd_ex")


def lstm_seq_bwd_ex(dout, gates_save, cs, w_hh, dG, lens=None, reverse=False):
    """dout [B,U,ldo] (column-slice views as in lstm_seq_fwd_ex) -> dG bf16 [n_dir,U,B,4H]."""
    n_dir, U, B, G4 = dG.shape
    H = G4 // 4
    assert dout.stride(2) == 1 and dout.stride(0) == U * dout.stride(1) and dout.shape[-1] == n_dir * H
    assert dG.dtype == torch.bfloat16 and dG.is_contiguous() and w_hh.shape[0] == n_dir * G4
    check(lib.pk_lstm_seq_bwd_ex(_P(dout), _dt(dout), dout.stride(1), _P(gates_save), _P(cs), _P(w_hh), _P(dG), _lens_arg(lens, B),
                                 B, U, H, n_dir, int(reverse), _P(_lstm_scratch(n_dir * H, dout.device)), _stream()),
          "pk_lstm_seq_bwd_ex")


def gather_rows(src, idx, dst):
    rows, C = dst.shape
    check(lib.pk_gather_rows(_P(src), _P(idx), _P(dst), _dt(src), rows, C, _stream()), "pk_gather_rows")


def scatter_add_rows(src, idx, dst):
    rows, C = src.shape
    assert dst.dtype == torch.float32
    check(lib.pk_scatter_add_rows(_P(src), _P(idx), _P(dst), _dt(src), rows, C, _stream()), "pk_scatter_add_rows")


def beam_xf_taps(st, layer, embed, x_cur, taps):
    """taps [rows, 5 * ldc]: the causal conv's im2col row of every row's new position (layer 0: embedding rows of ``embed`` f32)"""
    assert embed.dtype == torch.float32 and embed.is_contiguous() and taps.is_contiguous()
    check(lib.pk_beam_xf_taps(st, layer, _P(embed), embed.shape[1], _P(x_cur), _P(taps), taps.shape[1] // 5,
                              _stream()), "pk_beam_xf_taps")


def beam_xf_attn(st, layer, qkv, heads, rel, out):
    """qkv [rows, 3D] -> out [rows, D]: single-query attention over each row's cached positions; rel: f32 [2m+1, 64] or None"""
    assert qkv.is_contiguous() and out.is_contiguous() and (rel is None or (rel.dtype == torch.float32 and rel.is_contiguous()))
    check(lib.pk_beam_xf_attn(st, layer, _P(qkv), heads, _P(rel), 0 if rel is None else rel.shape[0] // 2, _P(out),
                              _stream()), "pk_beam_xf_attn")


def beam_xf_select(st, x, h):
    check(lib.pk_beam_xf_select(st, _P(x), _P(h), h.shape[-1], _stream()), "pk_beam_xf_select")


def beam_xf_slots(st, prev_ks, K):
    check(lib.pk_beam_xf_slots(st, _P(prev_ks), K, _stream()), "pk_beam_xf_slots")


def ce_grad(z, tok, coef, scale, dz, n):
    rows, ld = z.shape
    check(lib.pk_ce_grad(_P(z), _dt(z), ld, _P(tok), _P(coef), scale, _P(dz), rows, n, _stream()), "pk_ce_grad")


def conv_same_f64(x, n_len, h, m_len, y=None):
    """scipy.signal.fftconvolve(x[b, :n_len[b]], h[b, :m_len[b]], "same") per row, float64 (pk_conv_same_f64).
    x [B, n] f64, h [B, m] f64, n_len / m_len int32 [B] on the device; host-side bounds are the row widths.  -> y [B, n] f64
    (entries past n_len[b] are left untouched)."""
    assert x.dtype == torch.float64 and h.dtype == torch.float64 and x.stride(1) == 1 and h.stride(1) == 1
    B, n = x.shape
    m = h.shape[1]
    if y is None:
        y = torch.zeros_like(x)
    need = int(lib.pk_conv_same_f64_workspace_bytes(B, n, m))
    if need < 0:
        raise ValueError("pk_conv_same_f64: RIR width %d outside [1, 65536]" % m)
    ws = torch.empty(need, dtype=torch.uint8, device=x.device)
    check(lib.pk_conv_same_f64(_P(x), x.stride(0), _P(n_len), _P(h), h.stride(0), _P(m_len), B, n, m, _P(y), y.stride(0), _P(ws), need,
                               _stream()), "pk_conv_same_f64")
    return y


# ------------------------------------------------------------------------------------------------
# pruned RNN-T loss (include/pika_b200.h, "Pruned RNN-T loss")


def _ws_query(fn, name, *dims):
    """a workspace size returned through a long long* out-parameter"""
    out = ctypes.c_longlong(0)
    check(fn(*dims, ctypes.addressof(out)), name)
    return int(out.value)


def rnnt_lattice(lpb_skew, lpl_skew, frame_lens, label_lens, B, T, U1, grad_scale=None, fastemit_lambda=0.0, delay_penalty=0.0):
    """log-prob tables in the lattice's skewed layout [B, T+U1-1, U1] -> (costs [B], gb [B,T,U1], gl [B,T,U1])"""
    dev = lpb_skew.device
    ws_bytes = _ws_query(lib.pk_rnnt_lattice_workspace, "pk_rnnt_lattice_workspace", B, T, U1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    costs = torch.empty(B, dtype=torch.float32, device=dev)
    gb = torch.empty(B, T, U1, dtype=torch.float32, device=dev)
    gl = torch.empty_like(gb)
    args = (_P(frame_lens), _P(label_lens), B, T, U1, _P(lpb_skew), _P(lpl_skew), _P(grad_scale), _P(costs), _P(gb), _P(gl), _P(ws), ws_bytes)
    reg = _emission_reg(fastemit_lambda, delay_penalty)
    if reg is None:
        check(lib.pk_rnnt_lattice(*args, _stream()), "pk_rnnt_lattice")
    else:
        check(lib.pk_rnnt_lattice_reg(*args, *reg, _stream()), "pk_rnnt_lattice_reg")
    return costs, gb, gl


def rnnt_simple_prep(src, V, nb, n_in, n_out, hi, lo=None):
    """src f32 [nb*n_in, ld] -> hi (, lo) bf16 [nb*n_out, ld_out] = exp(src - rowmax) with zero padding; returns rowmax [nb*n_in]"""
    assert src.dtype == torch.float32 and src.stride(-1) == 1 and hi.dtype == torch.bfloat16 and hi.is_contiguous()
    rmax = torch.empty(nb * n_in, dtype=torch.float32, device=src.device)
    check(lib.pk_rnnt_simple_prep(_P(src), src.stride(0), V, nb, n_in, n_out, _P(hi), _P(lo), hi.shape[-1], _P(rmax), _stream()),
          "pk_rnnt_simple_prep")
    return rmax


def rnnt_simple_tables(am, lm, am_max, lm_max, S, labels, frame_lens, label_lens, B, T, U1):
    """-> (lpb_skew, lpl_skew) [B, T+U1-1, U1] f32 of the simple joiner"""
    dev = am.device
    lpb = torch.empty(B, T + U1 - 1, U1, dtype=torch.float32, device=dev)
    lpl = torch.empty_like(lpb)
    check(lib.pk_rnnt_simple_tables(_P(am), _P(lm), am.stride(0), _P(am_max), _P(lm_max), _P(S), S.shape[-1], _P(labels),
                                    max(labels.stride(0), 1), _P(frame_lens), _P(label_lens), B, T, U1, _P(lpb), _P(lpl), _stream()),
          "pk_rnnt_simple_tables")
    return lpb, lpl


def rnnt_simple_w(gb, gl, S, frame_lens, label_lens, scale, w_hi, w_lo=None):
    B, T, U1 = gb.shape
    check(lib.pk_rnnt_simple_w(_P(gb), _P(gl), _P(S), S.shape[-1], _P(frame_lens), _P(label_lens), _P(scale), B, T, U1, _P(w_hi), _P(w_lo),
                               w_hi.shape[-1], _stream()), "pk_rnnt_simple_w")


def rnnt_simple_grad(src, V, rmax, G, n_g, axis, gb, gl, labels, frame_lens, label_lens, scale, out):
    """out [rows, ldv] (f32 | bf16): d am (axis 0, rows over t) or d lm (axis 1, rows over u) of the simple loss"""
    B, T, U1 = gb.shape
    assert out.is_contiguous() and out.shape[-1] == src.stride(0) and G.stride(-1) == 1
    check(lib.pk_rnnt_simple_grad(_P(src), src.stride(0), V, _P(rmax), _P(G), G.shape[-1], n_g, axis, _P(gb), _P(gl), _P(labels),
                                  max(labels.stride(0), 1), _P(frame_lens), _P(label_lens), _P(scale), B, T, U1, _P(out), _dt(out),
                                  _stream()), "pk_rnnt_simple_grad")


def rnnt_simple_smooth_stats(am, lm, V, am_max, lm_max, frame_lens, label_lens, B, T, U1):
    """the smoothing terms' statistics -> (Nl [B*U1], logq [ldv], Na [B*T]) f32; rows past the lengths are 0"""
    assert am.dtype == lm.dtype == torch.float32 and am.is_contiguous() and lm.is_contiguous() and am.shape[1] == lm.shape[1]
    ldv = am.shape[1]
    dev = am.device
    ws_bytes = _ws_query(lib.pk_rnnt_simple_smooth_stats_workspace, "pk_rnnt_simple_smooth_stats_workspace", B, U1, ldv)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    Nl = torch.empty(B * U1, dtype=torch.float32, device=dev)
    logq = torch.empty(ldv, dtype=torch.float32, device=dev)
    Na = torch.empty(B * T, dtype=torch.float32, device=dev)
    check(lib.pk_rnnt_simple_smooth_stats(_P(am), _P(lm), ldv, V, _P(am_max), _P(lm_max), _P(frame_lens), _P(label_lens), B, T, U1, _P(Nl),
                                          _P(logq), _P(Na), _P(ws), ws_bytes, _stream()), "pk_rnnt_simple_smooth_stats")
    return Nl, logq, Na


def rnnt_simple_tables_smooth(am, lm, am_max, lm_max, S, labels, frame_lens, label_lens, B, T, U1, Nl, logq, Na, lm_only_scale,
                              am_only_scale):
    """-> (lpb_skew, lpl_skew) [B, T+U1-1, U1] f32 of the simple joiner smoothed with the LM-only / AM-only terms"""
    dev = am.device
    lpb = torch.empty(B, T + U1 - 1, U1, dtype=torch.float32, device=dev)
    lpl = torch.empty_like(lpb)
    check(lib.pk_rnnt_simple_tables_smooth(_P(am), _P(lm), am.stride(0), _P(am_max), _P(lm_max), _P(S), S.shape[-1], _P(labels),
                                           max(labels.stride(0), 1), _P(frame_lens), _P(label_lens), B, T, U1, _P(Nl), _P(logq), _P(Na),
                                           float(lm_only_scale), float(am_only_scale), _P(lpb), _P(lpl), _stream()),
          "pk_rnnt_simple_tables_smooth")
    return lpb, lpl


def rnnt_simple_grad_smooth(src, V, rmax, G, n_g, axis, gb, gl, labels, frame_lens, label_lens, scale, logq, lse, lm_only_scale,
                            am_only_scale, out):
    """rnnt_simple_grad of the smoothed simple loss (G formed with the scale mu * scale, lse = Na on axis 0, Nl on axis 1)"""
    B, T, U1 = gb.shape
    assert out.is_contiguous() and out.shape[-1] == src.stride(0) and G.stride(-1) == 1
    check(lib.pk_rnnt_simple_grad_smooth(_P(src), src.stride(0), V, _P(rmax), _P(G), G.shape[-1], n_g, axis, _P(gb), _P(gl), _P(labels),
                                         max(labels.stride(0), 1), _P(frame_lens), _P(label_lens), _P(scale), _P(logq), _P(lse),
                                         float(lm_only_scale), float(am_only_scale), B, T, U1, _P(out), _dt(out), _stream()),
          "pk_rnnt_simple_grad_smooth")


def rnnt_prune_bounds(ga, gb, frame_lens, label_lens, R):
    """occupancy -(ga + gb) [B,T,U1] (gb may be None) -> bounds [B,T] int32"""
    B, T, U1 = ga.shape
    bounds = torch.empty(B, T, dtype=torch.int32, device=ga.device)
    check(lib.pk_rnnt_prune_bounds(_P(ga), _P(gb), _P(frame_lens), _P(label_lens), B, T, U1, R, _P(bounds), _stream()),
          "pk_rnnt_prune_bounds")
    return bounds


def joint_gate_pruned_fwd(ex, py, bounds, h, B, T, U1, R, H):
    check(lib.pk_joint_gate_pruned_fwd(_P(ex), _P(py), _P(bounds), _P(h), _dt(ex), B, T, U1, R, H, _stream()), "pk_joint_gate_pruned_fwd")


def joint_gate_pruned_bwd(ex, py, bounds, dh, dex, dpy, B, T, U1, R, H):
    check(lib.pk_joint_gate_pruned_bwd(_P(ex), _P(py), _P(bounds), _P(dh), _P(dex), _P(dpy), _dt(ex), B, T, U1, R, H, _stream()),
          "pk_joint_gate_pruned_bwd")


def rnnt_pruned_loss(logits, labels, frame_lens, label_lens, bounds, U1, R, V, grad_scale=None, dlogits=None, colsum=None, row_lse=None,
                     fastemit_lambda=0.0, delay_penalty=0.0):
    """logits [B*T*R, ldv] (row (b,t,r) = node (t, bounds[b,t] + r)) -> costs [B]; dlogits (may alias logits) and colsum [ldv] filled
    when given"""
    B, T = bounds.shape
    rows, ldv = logits.shape
    assert rows == B * T * R and logits.is_contiguous() and labels.dtype == torch.int32 and bounds.dtype == torch.int32
    ws_bytes = _ws_query(lib.pk_rnnt_pruned_loss_workspace, "pk_rnnt_pruned_loss_workspace", B, T, U1, R, ldv)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=logits.device)
    costs = torch.empty(B, dtype=torch.float32, device=logits.device)
    if row_lse is not None:
        assert row_lse.dtype == torch.float32 and row_lse.is_contiguous() and tuple(row_lse.shape[1:]) == (rows, 2)
    args = (_P(logits), _dt(logits), _P(labels), _P(frame_lens), _P(label_lens), _P(bounds), B, T, U1, R, V, ldv, max(labels.stride(0), 1),
            _P(grad_scale), _P(costs), _P(dlogits), _P(colsum), _P(ws), ws_bytes, _P(row_lse),
            int(row_lse.shape[0]) if row_lse is not None else 0)
    reg = _emission_reg(fastemit_lambda, delay_penalty)
    if reg is None:
        check(lib.pk_rnnt_pruned_loss(*args, _stream()), "pk_rnnt_pruned_loss")
    else:
        check(lib.pk_rnnt_pruned_loss_reg(*args, *reg, _stream()), "pk_rnnt_pruned_loss_reg")
    return costs


# ------------------------------------------------------------------------------------------------
# forced alignment (include/pika_b200.h, "RNN-T forced alignment")


def rnnt_tables(logits, labels, frame_lens, label_lens, V=None, row_lse=None):
    """logits [B,T,U1,ldv] (bf16|f32) -> (lpb_skew, lpl_skew) [B, T+U1-1, U1] f32: the loss's first pass without the lattice.
    row_lse [n_parts, B*T*U1, 2]: the producing GEMM's row partials (the logits are then not re-read)"""
    B, T, U1, ldv = logits.shape
    V = ldv if V is None else V
    assert logits.is_contiguous() and labels.dtype == torch.int32 and labels.dim() == 2
    assert frame_lens.dtype == torch.int32 and label_lens.dtype == torch.int32
    dev = logits.device
    lse = torch.empty(B * T * U1, dtype=torch.float32, device=dev)
    lpb = torch.empty(B, T + U1 - 1, U1, dtype=torch.float32, device=dev)
    lpl = torch.empty_like(lpb)
    if row_lse is not None:
        assert row_lse.dtype == torch.float32 and row_lse.is_contiguous() and tuple(row_lse.shape[1:]) == (B * T * U1, 2)
    check(lib.pk_rnnt_tables(_P(logits), _dt(logits), _P(labels), _P(frame_lens), _P(label_lens), B, T, U1, V, ldv, max(labels.stride(0), 1),
                             _P(row_lse), int(row_lse.shape[0]) if row_lse is not None else 0, _P(lse), _P(lpb), _P(lpl), _stream()),
          "pk_rnnt_tables")
    return lpb, lpl


def rnnt_pruned_tables(logits, labels, frame_lens, label_lens, bounds, U1, R, V, row_lse=None):
    """pruned logits [B*T*R, ldv] (row (b,t,r) = node (t, bounds[b,t] + r)) -> (lpb_skew, lpl_skew) [B, T+U1-1, U1] f32, -inf outside
    the windows"""
    B, T = bounds.shape
    rows, ldv = logits.shape
    assert rows == B * T * R and logits.is_contiguous() and labels.dtype == torch.int32 and bounds.dtype == torch.int32
    dev = logits.device
    lse = torch.empty(rows, dtype=torch.float32, device=dev)
    lpb = torch.empty(B, T + U1 - 1, U1, dtype=torch.float32, device=dev)
    lpl = torch.empty_like(lpb)
    if row_lse is not None:
        assert row_lse.dtype == torch.float32 and row_lse.is_contiguous() and tuple(row_lse.shape[1:]) == (rows, 2)
    check(lib.pk_rnnt_pruned_tables(_P(logits), _dt(logits), _P(labels), _P(frame_lens), _P(label_lens), _P(bounds), B, T, U1, R, V, ldv,
                                    max(labels.stride(0), 1), _P(row_lse), int(row_lse.shape[0]) if row_lse is not None else 0, _P(lse),
                                    _P(lpb), _P(lpl), _stream()), "pk_rnnt_pruned_tables")
    return lpb, lpl


def rnnt_lattice_costs(lpb_skew, lpl_skew, frame_lens, label_lens, B, T, U1):
    """rnnt_lattice without the gradient coefficients -> costs [B] = -log P(y | x)"""
    dev = lpb_skew.device
    ws_bytes = _ws_query(lib.pk_rnnt_lattice_workspace, "pk_rnnt_lattice_workspace", B, T, U1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    costs = torch.empty(B, dtype=torch.float32, device=dev)
    check(lib.pk_rnnt_lattice_costs(_P(frame_lens), _P(label_lens), B, T, U1, _P(lpb_skew), _P(lpl_skew), _P(costs), _P(ws), ws_bytes,
                                    _stream()), "pk_rnnt_lattice_costs")
    return costs


def rnnt_viterbi(lpb_skew, lpl_skew, frame_lens, label_lens, B, T, U1, ld_emit=None, want_decisions=False):
    """best path through the lattice -> (score [B] f32, emit_frames [B, ld_emit] int32 (default U1 - 1)[, decisions
    [B, T+U1-1, ceil(U1/32)] int32 words: the label-arc bits, see include/pika_b200.h])"""
    dev = lpb_skew.device
    ld = U1 - 1 if ld_emit is None else int(ld_emit)
    ws_bytes = _ws_query(lib.pk_rnnt_viterbi_workspace, "pk_rnnt_viterbi_workspace", B, T, U1)
    ws = torch.empty(ws_bytes // 4, dtype=torch.int32, device=dev)
    score = torch.empty(B, dtype=torch.float32, device=dev)
    emit = torch.empty(B, ld, dtype=torch.int32, device=dev)
    check(lib.pk_rnnt_viterbi(_P(frame_lens), _P(label_lens), B, T, U1, _P(lpb_skew), _P(lpl_skew), _P(score), _P(emit), ld, _P(ws), ws_bytes,
                              _stream()), "pk_rnnt_viterbi")
    if want_decisions:
        return score, emit, ws.view(B, T + U1 - 1, (U1 + 31) // 32)
    return score, emit
