"""The chunk-masked attention kernels (pk_attention_fwd_chunk / pk_attention_bwd_chunk, pk_softmax_chunk_fwd) against float64
restatements of the same bf16 inputs: out, lse, dQ, dK and dV element by element under the bounds of test_attention_kernels_gpu.py,
with the chunk mask of tests/chunk_oracle.py.  Sequence lengths on both sides of the 64-row tiles and 128-row blocks; chunk lengths of
1, 3, 64, 128, non-multiples of 64 and longer than the sequence; offsets 0, 6 and 24 (the encoder's layers); left_chunks -1, 0 and 2.
Dropout decisions are read back from the forward's keep bits.  A mask that admits every key gives the unmasked kernels' bits, and bad
arguments launch nothing."""
import ctypes
import math

import pytest
import torch
from chunk_oracle import allowed
from test_attention_keep_bits_gpu import decode_keep_bits
from test_attention_kernels_gpu import (ALPHA, DTYPES, _bh, _check, _gen, _outbuf, _rows_two_passes, _scores, _tail_intact,
                                        attention_tols, drop_mask, drop_params, ref_attention_bwd, ref_softmax, tol_p)

pytestmark = pytest.mark.gpu


def _k():
    from pika_b200 import kernels
    return kernels


def _inputs(B, T, heads, seed):
    gen = _gen(seed)
    D = heads * 64
    qkv = (torch.randn(B, T, 3 * D, device="cuda", generator=gen) * 1.5).to(torch.bfloat16)
    dout = torch.randn(B, T, D, device="cuda", generator=gen).to(torch.bfloat16)
    return qkv, dout


def _run_chunk(qkv, dout, heads, chunk, p, seed):
    """forward + backward through the chunk entry points; lse starts as NaN so that every entry, padding included, must be written"""
    K = _k()
    B, T, D3 = qkv.shape
    lse = torch.full((B * heads * K.attention_lse_stride(T),), math.nan, device="cuda")
    out = torch.empty(B, T, D3 // 3, dtype=torch.bfloat16, device="cuda")
    bits = K.attention_keep_bits(B, T, heads, p, qkv.device)
    K.attention_fwd(qkv, out, lse, heads, ALPHA, p, seed, keep_bits=bits, chunk=chunk)
    dqkv = torch.empty_like(qkv)
    K.attention_bwd(qkv, out, dout, lse, dqkv, heads, ALPHA, p, seed, keep_bits=bits, chunk=chunk)
    torch.cuda.synchronize()
    return out, lse, dqkv, bits


def _check_chunk(tag, qkv, dout, heads, chunk, p, seed):
    B, T = qkv.shape[:2]
    D = heads * 64
    out, lse, dqkv, bits = _run_chunk(qkv, dout, heads, chunk, p, seed)
    assert bool(torch.isfinite(lse).all()), "lse: an entry (padding included) left unwritten or not finite"
    A = allowed(T, *chunk).cuda()
    q, k, v = (_bh(qkv[..., i * D:(i + 1) * D], heads) for i in range(3))
    M, scale = None, 1.0
    if p:
        keep = decode_keep_bits(bits, B * heads, T)
        # the decisions of every allowed pair are the shared generator's (row (b*heads + h)*T + t), as without the mask
        ref_keep = drop_mask(B * heads * T, T, p, seed).view(B * heads, T, T)
        assert torch.equal(keep & A, ref_keep & A), "keep bits of allowed pairs differ from the shared dropout mask"
        M, scale = (keep & A).double(), drop_params(p)[1]
    s = (ALPHA * q @ k.transpose(1, 2)).masked_fill(~A, -math.inf)
    lse_ref = torch.logsumexp(s, -1)
    P = torch.exp(s - lse_ref[..., None])
    Pd = P if M is None else P * M * scale
    O = Pd @ v
    O_k = _bh(out, heads)
    tol_o, tol_lse = attention_tols(P, Pd, v, O, lse_ref)
    _check("chunk O" + tag, O_k, O, tol_o)
    _check("chunk lse" + tag, lse.view(B * heads, -1)[:, :T], lse_ref, tol_lse)
    grads = ref_attention_bwd(q, k, v, P, Pd, _bh(dout, heads), O_k, ALPHA, M, scale)
    for name, got, (ref, tol) in zip(("dQ", "dK", "dV"), (dqkv[..., :D], dqkv[..., D:2 * D], dqkv[..., 2 * D:]), grads):
        _check("chunk %s%s" % (name, tag), _bh(got, heads), ref, tol)


CHUNK_T = [1, 63, 64, 65, 128, 129, 994]
# (chunk_len, chunk_off, left_chunks): the encoder's per-layer masks at C = 1 and 16 ((4C, 6), (4C, 24), (C, 10)), single-frame
# chunks, 3-frame chunks, tile-aligned and not, and chunks longer than any sequence here (with a lower limit that never binds)
CHUNKS = [(1, 0, 0), (1, 0, -1), (3, 6, 2), (4, 6, 2), (4, 24, -1), (1, 10, 0), (64, 6, -1), (64, 0, 2), (128, 24, 0), (100, 6, 2),
          (40, 24, -1), (16, 10, 2), (2048, 0, 0)]


@pytest.mark.parametrize("chunk", CHUNKS, ids=["len%d-off%d-left%d" % c for c in CHUNKS])
@pytest.mark.parametrize("T", CHUNK_T)
def test_chunk_attention_fwd_bwd(T, chunk):
    B, heads = 2, 3
    qkv, dout = _inputs(B, T, heads, seed=T * 131 + chunk[0] * 7 + chunk[1] * 3 + chunk[2])
    _check_chunk("", qkv, dout, heads, chunk, 0.0, 0)


DROP_CASES = [(65, (3, 6, 2)), (129, (64, 24, 0)), (994, (64, 6, -1)), (994, (16, 10, 2)), (994, (128, 24, 0)), (333, (1, 0, 0))]


@pytest.mark.parametrize("T,chunk", DROP_CASES, ids=["T%d-len%d-off%d-left%d" % ((t,) + c) for t, c in DROP_CASES])
def test_chunk_attention_dropout(T, chunk):
    """dropout decisions read back from keep_bits; the dK/dV kernel reads the bits of the blocks the forward wrote"""
    B, heads, p, seed = 2, 3, 0.15, 777
    qkv, dout = _inputs(B, T, heads, seed=T + chunk[0])
    _check_chunk(" drop", qkv, dout, heads, chunk, p, seed)


def test_chunk_attention_many_heads_at_the_encoder_shape():
    """B * heads = 64 (batch, head) pairs of 994 frames under layer 0's mask at C = 16 with two left chunks"""
    qkv, dout = _inputs(4, 994, 16, seed=5)
    _check_chunk(" enc", qkv, dout, 16, (64, 6, 2), 0.0, 0)


@pytest.mark.parametrize("p", [0.0, 0.2])
@pytest.mark.parametrize("T,chunk", [(994, (2048, 0, -1)), (129, (160, 24, 3)), (64, (64, 0, 0)), (1, (1, 0, 0))])
def test_admit_all_mask_is_bit_identical_to_unmasked(T, chunk, p):
    K = _k()
    assert K.attention_chunk_admits_all(T, chunk)
    B, heads, seed = 2, 3, 99
    qkv, dout = _inputs(B, T, heads, seed=T)
    out_c, lse_c, dq_c, bits_c = _run_chunk(qkv, dout, heads, chunk, p, seed)
    lse = torch.zeros(B * heads * K.attention_lse_stride(T), device="cuda")
    out = torch.empty_like(out_c)
    bits = K.attention_keep_bits(B, T, heads, p, qkv.device)
    K.attention_fwd(qkv, out, lse, heads, ALPHA, p, seed, keep_bits=bits)        # pk_attention_fwd_bits (pk_attention_fwd at p = 0)
    dq = torch.empty_like(qkv)
    K.attention_bwd(qkv, out, dout, lse, dq, heads, ALPHA, p, seed, keep_bits=bits)
    torch.cuda.synchronize()
    assert torch.equal(out, out_c) and torch.equal(lse, lse_c) and torch.equal(dq, dq_c)
    if p:
        assert torch.equal(decode_keep_bits(bits, B * heads, T), decode_keep_bits(bits_c, B * heads, T))


def test_admits_all_rule():
    K = _k()
    for T in (1, 63, 64, 65, 994):
        for chunk in CHUNKS:
            A = allowed(T, *chunk)
            assert K.attention_chunk_admits_all(T, chunk) == bool(A.all()), (T, chunk)


# ------------------------------------------------------------------------------------------------ the materialised path
@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("n,chunk", [(1, (1, 0, 0)), (63, (3, 6, 2)), (248, (16, 10, 2)), (248, (64, 24, -1)), (1031, (100, 6, 0)),
                                     (2048, (40, 24, 2))])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_softmax_chunk_fwd(n, chunk, dtype, p):
    """rows (sequence, head, query i = row % n): P is the masked softmax, Pd its dropout with the shared mask; pk_softmax_bwd is the
    backward (checked by test_attention_kernels_gpu.py on any P)"""
    K, dt = _k(), DTYPES[dtype]
    heads, seed = 2, 4242
    rows = _rows_two_passes(heads * n) if n <= 248 else 2 * heads * n
    ld_p = (n + 7) // 8 * 8
    gen = _gen(n * 17 + chunk[0])
    S = _scores(rows, ld_p + 8, n, gen)
    Pb, Pdb = _outbuf(rows, ld_p, dt), _outbuf(rows, ld_p, dt)
    K.softmax_chunk_fwd(S, Pb[:rows], Pdb[:rows], n, chunk, p, seed)
    torch.cuda.synchronize()
    P, Pd = _tail_intact(Pb, rows, "P"), _tail_intact(Pdb, rows, "Pd")
    assert bool((P[:, n:] == 0).all()) and bool((Pd[:, n:] == 0).all()), "row padding of P / Pd must be 0"
    keep = allowed(n, *chunk).cuda().repeat(rows // n, 1)
    ref = ref_softmax(S[:, :n], keep)
    _check("chunk softmax P %s" % dtype, P[:, :n], ref, tol_p(ref, dt))
    assert bool((P[:, :n][~keep] == 0).all())
    if p == 0:
        assert torch.equal(P, Pd)
    else:
        M = drop_mask(rows, n, p, seed)
        scale = drop_params(p)[1]
        exp = torch.where(M, (P[:, :n].float() * scale).to(dt), torch.zeros((), dtype=dt, device="cuda"))
        assert torch.equal(Pd[:, :n], exp)


# ------------------------------------------------------------------------------------------------ argument checks
def test_bad_arguments_launch_nothing():
    from pika_b200 import _lib
    lib = _lib.lib
    B, T, heads = 2, 65, 3
    qkv, dout = _inputs(B, T, heads, seed=1)
    D = heads * 64
    out = torch.empty(B, T, D, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(B * heads * 128, device="cuda")
    ws = torch.zeros_like(lse)
    dq = torch.empty_like(qkv)
    bits = _k().attention_keep_bits(B, T, heads, 0.1, qkv.device)
    P = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off * t.element_size()) if t is not None else ctypes.c_void_p(0)
    Lg, I, F, U = ctypes.c_longlong, ctypes.c_int, ctypes.c_float, ctypes.c_uint32
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def fwd(drop, kb, cl, co, lc):
        return lib.pk_attention_fwd_chunk(P(qkv), P(qkv, D), P(qkv, 2 * D), Lg(3 * D), P(out), Lg(D), P(lse), I(B), I(T), I(heads), I(64),
                                          F(ALPHA), F(drop), U(1), P(kb), I(cl), I(co), I(lc), st)

    def bwd(drop, kb, cl, co, lc):
        return lib.pk_attention_bwd_chunk(P(qkv), P(qkv, D), P(qkv, 2 * D), Lg(3 * D), P(out), Lg(D), P(dout), Lg(D), P(lse), P(ws),
                                          P(dq), P(dq, D), P(dq, 2 * D), Lg(3 * D), I(B), I(T), I(heads), I(64), F(ALPHA), F(drop),
                                          P(kb), I(cl), I(co), I(lc), st)

    S = torch.zeros(heads * T, 72, device="cuda")
    Pm = torch.empty(heads * T, 72, device="cuda")

    def sm(cl, co, lc, rows=heads * T):
        return lib.pk_softmax_chunk_fwd(P(S), Lg(72), P(Pm), P(Pm), I(1), Lg(72), Lg(rows), I(T), I(cl), I(co), I(lc), F(0.0), U(0), st)

    torch.cuda.synchronize()
    before = _lib.launch_count()
    for args in ((0.0, None, 0, 0, -1), (0.0, None, 4, -1, -1), (0.0, None, 4, 0, -2), (0.1, None, 4, 6, 2)):
        assert fwd(*args) < 0 and bwd(*args) < 0, args
    for args in ((0, 0, -1), (4, -1, -1), (4, 0, -2)):
        assert sm(*args) < 0, args
    assert sm(4, 0, -1, rows=heads * T + 1) < 0
    assert lib.pk_attention_chunk_admits_all(T, 0, 0, -1) < 0 and lib.pk_attention_chunk_admits_all(0, 4, 0, -1) < 0
    assert _lib.launch_count() == before
    # the same buffers with good arguments do launch
    assert fwd(0.1, bits, 4, 6, 2) == 0 and bwd(0.1, bits, 4, 6, 2) == 0 and sm(4, 0, -1) == 0
    torch.cuda.synchronize()
    assert _lib.launch_count() > before
