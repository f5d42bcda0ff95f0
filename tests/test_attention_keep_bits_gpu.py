"""The fused attention's dropout keep bits (pk_attention_keep_bits_bytes, pk_attention_fwd_bits / pk_attention_bwd_bits): the
forward writes the shared generator's mask in the documented layout, the backward reads it and agrees bit for bit with the
seeded pk_attention_bwd, and a missing buffer is rejected before anything launches."""
import ctypes
import math

import pytest
import torch
from test_attention_kernels_gpu import ALPHA, SENT, F, I, L, U, _abi, _attn_inputs, _attn_run, _check_attention, _strided, drop_mask

pytestmark = pytest.mark.gpu


def _k():
    from pika_b200 import kernels
    return kernels


def _ptr_off(t, nbytes):
    return ctypes.c_void_p(t.data_ptr() + nbytes)


def decode_keep_bits(bits, BH, T):
    """bool [BH, T, T] (query, key) from the layout of include/pika_b200.h: blocks [BH][n][n] of 128 words, (r, c) of a block in
    word (r >> 4) * 32 + ((c & 7) >> 1) * 8 + (r & 7), bit ((r >> 3) & 1) * 16 + (c >> 3) * 2 + (c & 1)"""
    n = (T + 127) // 128 * 2
    words = bits.view(BH, n, n, 128).long() & 0xFFFFFFFF
    r = torch.arange(64, device=bits.device).view(64, 1)
    c = torch.arange(64, device=bits.device).view(1, 64)
    widx = ((r >> 4) * 32 + ((c & 7) >> 1) * 8 + (r & 7)).expand(64, 64)
    bit = ((r >> 3) & 1) * 16 + (c >> 3) * 2 + (c & 1)
    blk = (words[..., widx.reshape(-1)].view(BH, n, n, 64, 64) >> bit) & 1      # [BH, qb, kb, r, c]
    return blk.permute(0, 1, 3, 2, 4).reshape(BH, n * 64, n * 64)[:, :T, :T] != 0


def test_keep_bits_size_query():
    from pika_b200 import _lib
    size = _lib.lib.pk_attention_keep_bits_bytes
    for T, n in ((1, 2), (128, 2), (129, 4), (976, 16), (994, 16), (2048, 32)):
        assert size(3, T, 5) == 3 * 5 * n * n * 512
    assert size(32, 994, 16) == 32 * 16 * 16 * 16 * 512            # 64 MiB at the encoder's shape
    assert size(4096, 4096, 15) > 2 ** 32                          # no 32-bit overflow


@pytest.mark.parametrize("T", [1, 65, 129, 333, 1000])
def test_keep_bits_are_the_shared_mask(T):
    """the bits the forward writes are pk_softmax_fwd's mask of row (b*heads + h)*T + t, bit for bit"""
    B, heads, p, seed = 2, 3, 0.2, 2024
    qkv, _ = _attn_inputs(B, T, heads, seed=T + 7)
    K = _k()
    out = torch.empty(B, T, heads * 64, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(B * heads * K.attention_lse_stride(T), device="cuda")
    bits = K.attention_keep_bits(B, T, heads, p, qkv.device)
    K.attention_fwd(qkv, out, lse, heads, ALPHA, p, seed, keep_bits=bits)
    torch.cuda.synchronize()
    M = drop_mask(B * heads * T, T, p, seed).view(B * heads, T, T)
    assert torch.equal(decode_keep_bits(bits, B * heads, T), M)


def test_backward_reads_the_given_keep_bits():
    """pk_attention_bwd_bits takes its mask from keep_bits, not from a seed: the bits of seed 6 give exactly the gradients the seeded
    backward draws for seed 6, and the forward + backward through the bits match the float64 reference"""
    B, T, heads, p = 2, 200, 3, 0.2
    D = heads * 64
    K = _k()
    qkv, dout = _attn_inputs(B, T, heads, seed=41)
    out, lse, dqkv = _attn_run(qkv, dout, heads, p, 5)
    other = K.attention_keep_bits(B, T, heads, p, qkv.device)
    K.attention_fwd(qkv, torch.empty_like(out), torch.empty_like(lse), heads, ALPHA, p, 6, keep_bits=other)
    d2 = torch.empty_like(qkv)
    K.attention_bwd(qkv, out, dout, lse, d2, heads, ALPHA, p, 5, keep_bits=other)
    d6 = torch.empty_like(qkv)
    K.attention_bwd(qkv, out, dout, lse, d6, heads, ALPHA, p, 6)
    torch.cuda.synchronize()
    assert torch.equal(d2, d6) and not torch.equal(d2, dqkv)
    bits = K.attention_keep_bits(B, T, heads, p, qkv.device)
    out_b, lse_b, dq_b = torch.empty_like(out), torch.zeros_like(lse), torch.empty_like(qkv)
    K.attention_fwd(qkv, out_b, lse_b, heads, ALPHA, p, 5, keep_bits=bits)
    K.attention_bwd(qkv, out_b, dout, lse_b, dq_b, heads, ALPHA, p, 5, keep_bits=bits)
    torch.cuda.synchronize()
    assert torch.equal(out_b, out) and torch.equal(lse_b, lse) and torch.equal(dq_b, dqkv)
    _check_attention(" bits", qkv, dout, heads, out_b, lse_b, dq_b[..., :D], dq_b[..., D:2 * D], dq_b[..., 2 * D:], p, 5)


def test_rejects_missing_keep_bits_with_dropout():
    """keep_bits may be NULL only when drop_p == 0; a NULL or misaligned buffer with dropout is rejected and nothing launches"""
    from pika_b200 import _lib
    buf = torch.zeros(1 << 20, device="cuda")
    fwd = lambda p, kb: _abi("pk_attention_fwd_bits", buf, buf, buf, L(192), buf, L(64), buf, I(1), I(8), I(1), I(64), F(ALPHA), F(p), U(0),
                             kb)
    bwd = lambda p, kb: _abi("pk_attention_bwd_bits", buf, buf, buf, L(192), buf, L(64), buf, L(64), buf, buf, buf, buf, buf, L(192),
                             I(1), I(8), I(1), I(64), F(ALPHA), F(p), kb)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    for call in (fwd, bwd):
        for kb in (None, _ptr_off(buf, 4)):
            assert call(0.1, kb) < 0
            assert "keep_bits" in _lib.lib.pk_last_error().decode()
    assert _lib.launch_count() == before
    assert fwd(0.0, None) == 0 and bwd(0.0, None) == 0          # no dropout: no bits needed
    torch.cuda.synchronize()


def test_attention_strided_abi_keep_bits():
    """separate q / k / v with a padded row stride, padded ld_out / ld_dout, ld_dqkv != ld_qkv, dropout through a caller's
    keep-bit buffer: the same bits as the fused layout with the seeded calls, and nothing outside the [T, heads*64] views is
    written"""
    B, T, heads = 2, 129, 5
    D = heads * 64
    qkv, dout = _attn_inputs(B, T, heads, seed=3)
    out_ref, lse_ref, dqkv_ref = _attn_run(qkv, dout, heads, 0.1, 11)
    ld_qkv, ld_out, ld_dout, ld_dqkv = D + 24, D + 16, D + 8, D + 40
    q, k, v = (_strided(qkv[..., i * D:(i + 1) * D], ld_qkv, math.nan) for i in range(3))
    do = _strided(dout, ld_dout, math.nan)
    out = torch.full((B * T + 1, ld_out), SENT, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros_like(lse_ref)
    bits = _k().attention_keep_bits(B, T, heads, 0.1, qkv.device)
    assert _abi("pk_attention_fwd_bits", q, k, v, L(ld_qkv), out, L(ld_out), lse, I(B), I(T), I(heads), I(64), F(ALPHA), F(0.1), U(11),
                bits) == 0
    grads = [torch.full((B * T + 1, ld_dqkv), SENT, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
    ws = torch.zeros_like(lse)
    assert _abi("pk_attention_bwd_bits", q, k, v, L(ld_qkv), out, L(ld_out), do, L(ld_dout), lse, ws, *grads, L(ld_dqkv), I(B), I(T), I(heads),
                I(64), F(ALPHA), F(0.1), bits) == 0
    torch.cuda.synchronize()
    assert torch.equal(out[:B * T, :D], out_ref.view(B * T, D)) and torch.equal(lse, lse_ref)
    assert bool((out[:B * T, D:] == SENT).all()) and bool((out[B * T] == SENT).all())
    for i, g in enumerate(grads):
        assert torch.equal(g[:B * T, :D], dqkv_ref.view(B * T, 3 * D)[:, i * D:(i + 1) * D])
        assert bool((g[:B * T, D:] == SENT).all()) and bool((g[B * T] == SENT).all())
