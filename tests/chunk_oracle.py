"""Chunk-limited self-attention restated on the CPU: the chunk mask, masked attention in any float dtype, and the TDNN-Transformer
encoder with a chunk mask on each attention layer, built from oracle.model's primitives (batchnorm, tdnn, layernorm, linear).
Dropout off.  DESIGN.md "Chunked attention" states the rule."""
import math

import torch
import torch.nn.functional as F

from oracle import model as om


def allowed(T, chunk_len, chunk_off, left_chunks):
    """bool [T, T]: query i (row) may attend to key j (column)"""
    c = (torch.arange(T) + chunk_off) // chunk_len
    ci, cj = c[:, None], c[None, :]
    ok = cj <= ci
    if left_chunks >= 0:
        ok &= cj >= ci - left_chunks
    return ok


def attention(q, k, v, alpha, mask=None, keep=None, drop_scale=1.0):
    """q, k, v [..., T, dh] -> (out [..., T, dh], lse [..., T]); mask bool [T, T] (True = allowed), keep [..., T, T] dropout decisions"""
    s = alpha * (q @ k.transpose(-1, -2))
    if mask is not None:
        s = s.masked_fill(~mask, -math.inf)
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    if keep is not None:
        p = p * keep.to(p.dtype) * drop_scale
    return p @ v, lse


def mha(x, sd, name, heads, mask=None):
    """oracle.model.mha in the dtype of x (no cast of the scores), mask bool [T, T] True = allowed"""
    B, T, D = x.shape
    dh = D // heads

    def shape(z):
        return z.view(B, T, heads, dh).transpose(1, 2)

    q, k, v = (shape(om.linear(x, sd, name + n)) for n in (".linear_query", ".linear_keys", ".linear_values"))
    ctx, _ = attention(q, k, v, 1.0 / math.sqrt(dh), mask)
    return om.linear(ctx.transpose(1, 2).reshape(B, T, D), sd, name + ".final_linear")


def transformer_layer(x, sd, name, heads, mask=None):
    h = mha(om.layernorm(x, sd, name + ".layer_norm"), sd, name + ".self_attn", heads, mask) + x
    ff = name + ".feed_forward"
    inter = F.relu(om.linear(om.layernorm(h, sd, ff + ".layer_norm"), sd, ff + ".w_1"))
    return om.linear(inter, sd, ff + ".w_2") + h


def encoder_forward(sd, x, train=True, chunks=None, prefix="encoder."):
    """oracle.model.encoder_forward with attention layer l under the chunk mask chunks[l] = (chunk_len, chunk_off, left_chunks), or
    full context where chunks is None or chunks[l] is None"""
    B = x.shape[0]
    C = sd[prefix + "fc_in.weight"].shape[0]
    h = F.relu(om.linear(x, sd, prefix + "fc_in")).reshape(-1, C)
    h = om.batchnorm(h, sd, prefix + "bn_in", train).view(B, -1, C)
    for l, (dil, stride) in enumerate(om.TDNN_DIL_STRIDE):
        h = F.relu(om.tdnn(h, sd, prefix + "hidden_conv.%d" % l, dil, stride))
        T = h.shape[1]
        h = om.batchnorm(h.reshape(-1, C), sd, prefix + "hidden_bn.%d" % l, train).view(B, T, C)
        if (l + 1) % 3 == 0:
            ch = chunks[l // 3] if chunks is not None else None
            h = transformer_layer(h, sd, prefix + "transformer.%d" % (l // 3), om.HEADS[l // 3], allowed(T, *ch) if ch else None)
    T = h.shape[1]
    h = om.batchnorm(h.reshape(-1, C), sd, prefix + "bn_final", train)
    return om.linear(h, sd, prefix + "fc_out").view(B, T, -1)


def dependency_end(t_out, W, s_total=4, o_total=42):
    """input frames [0, end) that encoder output frame t_out may depend on under chunks of W input frames"""
    return W * ((s_total * t_out + o_total) // W + 1)
