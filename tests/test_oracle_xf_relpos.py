"""Relative-position self-attention (Shaw et al.; trainer/model/modules/multi_headed_attn.py:9-41,105-108,186-229) in the
transformer prediction net, on the CPU: a restatement of the reference's attention with torch-CPU fp32 primitives over a plain
``state_dict``, pinned in forward and backward to tests/golden/model_xf_relpos.npz, which make_golden_relpos.py produced by executing
the reference's own modules (m = 3, where the end buckets collect several keys, and m = 16, where none does; label rows of unequal
length padded with the padding id).  Also: a seeded construction of the drop-in reproduces the reference's initial weights and
state_dict keys."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_oracle_xf_prednet import xf_args, xf_inputs


def build_xf_relpos(V, m, seed=778):
    from pika_b200.model.transducer import Net
    torch.manual_seed(seed)
    a = xf_args(V)
    a.max_relative_positions = m
    return Net(a, 240, V)


# ------------------------------------------------------------------------------------------------ the restatement
def relative_buckets(L, m):
    """bucket of query i and key j: clamp(j - i, -m, m) + m  (multi_headed_attn.py:14-23, non-cache branch)"""
    j = torch.arange(L)
    return (j[None, :] - j[:, None]).clamp(-m, m) + m


def relpos_mha(x, sd, name, heads, mask, m):
    """MultiHeadedAttention.forward, self-attention with relative positions, no cache, dropout off: the table R serves as key and
    value relations; scores = (q/sqrt(d)).k_j + (q/sqrt(d)).R[b(i,j)], masked with -1e18, softmax, out = sum_j P_ij (v_j + R[b(i,j)])"""
    from oracle import model as om
    B, L, D = x.shape
    dh = D // heads

    def shape(z):
        return z.view(B, L, heads, dh).transpose(1, 2)

    k = shape(om.linear(x, sd, name + ".linear_keys"))
    v = shape(om.linear(x, sd, name + ".linear_values"))
    q = shape(om.linear(x, sd, name + ".linear_query")) / math.sqrt(dh)
    rel = sd[name + ".relative_positions_embeddings.weight"][relative_buckets(L, m)]          # [L, L, dh]
    scores = torch.matmul(q, k.transpose(2, 3)) + torch.einsum("bhid,ijd->bhij", q, rel)
    attn = torch.softmax(scores.masked_fill(mask.unsqueeze(1), -1e18), dim=-1)
    ctx = torch.matmul(attn, v) + torch.einsum("bhij,ijd->bhid", attn, rel)
    return om.linear(ctx.transpose(1, 2).reshape(B, L, D), sd, name + ".final_linear")


def relpos_prednet_forward(sd, y, m, heads=8):
    """SOS prepend + the convolutional-transformer prediction net (trainer/model/rnnt_conv_transformer_lm.py:59-80) with relative
    positions in every layer; oracle/model.py:conv_transformer_lm_forward otherwise.  y [B,U] int64 -> [B,U+1,H]"""
    from oracle import model as om
    src = torch.cat((torch.zeros(y.shape[0], 1, dtype=torch.long), y.long()), 1)
    emb_w = sd["embed.weight"]
    pad = emb_w.shape[0] - 1
    out = F.embedding(src, emb_w, padding_idx=pad)
    B, L = src.shape
    mask = src.eq(pad).unsqueeze(1).expand(B, L, L) | torch.triu(torch.ones(L, L, dtype=torch.bool), diagonal=1).unsqueeze(0)
    l = 0
    while "decoder.conv.%d.weight" % l in sd:
        w, b = sd["decoder.conv.%d.weight" % l], sd["decoder.conv.%d.bias" % l]
        out = F.relu(F.conv1d(out.transpose(1, 2), w, b, padding=w.shape[2] - 1)[:, :, :-(w.shape[2] - 1)]).transpose(1, 2)
        name = "decoder.transformer.%d" % l
        h = relpos_mha(om.layernorm(out, sd, name + ".layer_norm"), sd, name + ".self_attn", heads, mask, m) + out
        ff = name + ".feed_forward"
        out = om.linear(F.relu(om.linear(om.layernorm(h, sd, ff + ".layer_norm"), sd, ff + ".w_1")), sd, ff + ".w_2") + h
        l += 1
    return om.linear(om.layernorm(out, sd, "decoder.layer_norm"), sd, "decoder.linear_out")


# ------------------------------------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def fix(golden_dir):
    return np.load(os.path.join(golden_dir, "model_xf_relpos.npz"))


def test_fixture_covers_clipped_and_unclipped_buckets(fix):
    V, B, Tp, U = [int(v) for v in fix["dims"]]
    ms = [int(m) for m in fix["ms"]]
    assert min(ms) < U + 1 <= max(ms)
    assert len(set(fix["ulens"].tolist())) == B


@pytest.mark.parametrize("m", [3, 16])
def test_drop_in_relpos_init_matches_reference_weights_and_keys(fix, m):
    V = int(fix["dims"][0])
    model = build_xf_relpos(V, m)
    sd = model.state_dict()
    keys = [k for k in sd if not k.startswith("encoder.")]
    assert keys == fix["m%d_keys" % m].tolist()
    rel_keys = [k for k in keys if k.endswith("relative_positions_embeddings.weight")]
    assert len(rel_keys) == 2 and all(tuple(sd[k].shape) == (2 * m + 1, 64) for k in rel_keys)
    for k in keys:
        if not sd[k].dtype.is_floating_point:
            continue
        v = sd[k]
        fp = np.array([v.double().sum().item(), v.double().abs().sum().item(), float(v.flatten()[0]), float(v.flatten()[-1])])
        np.testing.assert_allclose(fp, fix["m%d_w_%s" % (m, k)], rtol=1e-12, atol=0, err_msg=k)
    # the encoder's transformer layers never carry a table (trainer/model/rnnt_tdnn_transformer.py:66)
    assert not any("relative_positions" in k for k in sd if k.startswith("encoder."))


@pytest.mark.parametrize("m", [3, 16])
def test_oracle_relpos_prednet_forward_backward_matches_reference(fix, m):
    from fixture_utils import grad_fingerprint
    from oracle import model as om
    from oracle import rnnt as orc
    V, B, Tp, U = [int(v) for v in fix["dims"]]
    model = build_xf_relpos(V, m)
    trained = [k for k, _ in model.named_parameters() if not k.startswith("encoder.")]          # the shared embedding once
    sd = {k: v.detach().clone().requires_grad_(k in trained) for k, v in model.state_dict().items()}
    y = torch.from_numpy(fix["y"])
    enc = torch.from_numpy(xf_inputs(int(fix["seed"]), B, Tp)).requires_grad_(True)
    pred = relpos_prednet_forward(sd, y, m)
    np.testing.assert_allclose(pred.detach().numpy(), fix["m%d_pred" % m], rtol=0, atol=2e-5)
    logits = om.joint_forward(sd, enc, pred, softmax=False)
    yl = fix["y"].copy()
    yl[yl == V] = 0
    costs, dz = orc.rnnt_loss_from_logits(logits.detach().numpy(), yl.astype(np.int32), fix["tlens"], fix["ulens"])
    np.testing.assert_allclose(costs, fix["m%d_costs" % m], rtol=1e-5)
    logits.backward(torch.from_numpy(np.asarray(dz, np.float32)))
    n = 0
    for k in trained:
        p = sd[k]
        ref = fix["m%d_gs_%s" % (m, k)]
        got = grad_fingerprint(p.grad if p.grad is not None else torch.zeros_like(p), 512)
        if ref[2] < 1e-6:          # analytically zero (the keys bias under the softmax's shift invariance): rounding noise on both sides
            assert got[2] < 1e-6, k
            continue
        assert abs(got[2] - ref[2]) <= 1e-4 * ref[2], (k, got[2], ref[2])
        assert np.linalg.norm(got[3:] - ref[3:]) <= 1e-4 * np.linalg.norm(ref[3:]), k
        n += 1
    assert n > 40
    for l in range(2):
        k = "decoder.transformer.%d.self_attn.relative_positions_embeddings.weight" % l
        assert fix["m%d_gs_%s" % (m, k)][2] > 1e-3                    # the table is trained: its gradient is pinned, not empty
    got = grad_fingerprint(enc.grad, 512)
    ref = fix["m%d_denc" % m]
    assert np.linalg.norm(got[3:] - ref[3:]) <= 1e-4 * np.linalg.norm(ref[3:])


def test_relative_buckets_band_layout():
    """the band the kernels rely on: bucket r in (0, 2m) holds the single key j = i - m + r; 0 collects j <= i - m, 2m j >= i + m"""
    L, m = 12, 3
    b = relative_buckets(L, m)
    for i in range(L):
        for j in range(L):
            r = int(b[i, j])
            assert (r == 0) == (j <= i - m) and (r == 2 * m) == (j >= i + m)
            if 0 < r < 2 * m:
                assert j == i - m + r

