"""Layer-level GPU parity: every autograd Function of pika_b200.engine (forward AND backward,
through the C ABI) against plain torch fp32 modules on the same inputs.  fp32-class mode
(split-bf16 tensor-core products): 1e-3 norm-relative, the north star's stated tolerance."""
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
TOL = 1e-3
# the torch references must be real fp32 (cuDNN convolutions default to TF32, whose 1e-3 error flips
# ReLU masks at near-zero pre-activations)
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.fixture(autouse=True)
def fp32_mode():
    from pika_b200 import engine
    engine.set_precision("fp32")
    engine.set_dropout_enabled(True)
    yield
    engine.set_precision("bf16")


def g(*shape, seed=0, scale=1.0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=gen) * scale


def test_linear_relu_residual():
    from pika_b200 import engine as E
    lin = nn.Linear(240, 328).cuda()
    x = g(260, 240, seed=1).requires_grad_(True)
    res = g(260, 328, seed=2).requires_grad_(True)
    y = E.linear(x, lin.weight, lin.bias, act=False, residual=res)
    ref = F.linear(x, lin.weight, lin.bias) + res
    assert rel(y, ref) < TOL
    dy = g(260, 328, seed=3)
    gx, gr, gw, gb = torch.autograd.grad(ref, [x, res, lin.weight, lin.bias], dy)
    lin.weight.grad = lin.bias.grad = None
    y.backward(dy)
    assert rel(x.grad, gx) < TOL
    assert rel(res.grad, gr) < TOL
    assert rel(lin.weight.grad, gw) < TOL
    assert rel(lin.bias.grad, gb) < TOL
    # relu variant
    x2 = g(100, 240, seed=4).requires_grad_(True)
    y2 = E.linear(x2, lin.weight, lin.bias, act=True)
    ref2 = F.relu(F.linear(x2, lin.weight, lin.bias))
    assert rel(y2, ref2) < TOL
    dy2 = g(100, 328, seed=5)
    gx2, gw2 = torch.autograd.grad(ref2, [x2, lin.weight], dy2)
    lin.weight.grad = None
    y2.backward(dy2)
    assert rel(x2.grad, gx2) < TOL
    assert rel(lin.weight.grad, gw2) < TOL


def test_linear_concatenated_qkv():
    from pika_b200 import engine as E
    ls = [nn.Linear(256, 256).cuda() for _ in range(3)]
    x = g(70, 256, seed=6).requires_grad_(True)
    y = E.linear(x, [l.weight for l in ls], [l.bias for l in ls])
    ref = torch.cat([l(x) for l in ls], 1)
    assert rel(y, ref) < TOL
    dy = g(70, 768, seed=7)
    gs = torch.autograd.grad(ref, [x] + [l.weight for l in ls] + [l.bias for l in ls], dy)
    for l in ls:
        l.weight.grad = l.bias.grad = None
    y.backward(dy)
    assert rel(x.grad, gs[0]) < TOL
    for i, l in enumerate(ls):
        assert rel(l.weight.grad, gs[1 + i]) < TOL
        assert rel(l.bias.grad, gs[4 + i]) < TOL


@pytest.mark.parametrize("dil,stride", [(1, 1), (3, 1), (3, 4)])
def test_tdnn(dil, stride):
    from pika_b200 import engine as E
    C = 256
    conv = nn.Conv2d(1, C, (3, C), dilation=(dil, 1), stride=(stride, 1)).cuda()
    x = g(3, 90, C, seed=8).requires_grad_(True)
    y = E.TdnnFn.apply(x, conv.weight, conv.bias, dil, stride)
    pre = conv(x.unsqueeze(1)).squeeze(-1).transpose(1, 2)
    assert y.shape == pre.shape and rel(y, F.relu(pre)) < TOL
    ref = pre * (y.detach() > 0)          # same ReLU mask on both sides (ties at |pre| ~ 1e-7 are arbitrary)
    dy = g(*ref.shape, seed=9)
    gx, gw, gb = torch.autograd.grad(ref, [x, conv.weight, conv.bias], dy)
    conv.weight.grad = conv.bias.grad = None
    y.backward(dy)
    assert rel(x.grad, gx) < TOL
    assert rel(conv.weight.grad, gw) < TOL
    assert rel(conv.bias.grad, gb) < TOL


@pytest.mark.parametrize("train", [True, False])
def test_batchnorm(train):
    from pika_b200 import engine as E
    bn, ref_bn = nn.BatchNorm1d(256).cuda(), nn.BatchNorm1d(256).cuda()
    with torch.no_grad():
        bn.weight.copy_(g(256, seed=10) * 0.2 + 1); bn.bias.copy_(g(256, seed=11) * 0.2)
        bn.running_mean.copy_(g(256, seed=12) * 0.1); bn.running_var.copy_(g(256, seed=13).abs() + 0.5)
    ref_bn.load_state_dict(bn.state_dict())
    bn.train(train); ref_bn.train(train)
    x = (g(333, 256, seed=14) * 2 + 0.5).requires_grad_(True)
    y = E.BatchNormFn.apply(x, bn, train, bn.weight, bn.bias)
    ref = ref_bn(x)
    assert rel(y, ref) < TOL
    dy = g(333, 256, seed=15)
    gx, gw, gb = torch.autograd.grad(ref, [x, ref_bn.weight, ref_bn.bias], dy)
    y.backward(dy)
    assert rel(x.grad, gx) < TOL
    assert rel(bn.weight.grad, gw) < TOL
    assert rel(bn.bias.grad, gb) < TOL
    assert rel(bn.running_mean, ref_bn.running_mean) < 1e-4
    assert rel(bn.running_var, ref_bn.running_var) < 1e-4


def test_layernorm():
    from pika_b200 import engine as E
    ln = nn.LayerNorm(1024, eps=1e-6).cuda()
    with torch.no_grad():
        ln.weight.copy_(g(1024, seed=16) * 0.2 + 1); ln.bias.copy_(g(1024, seed=17) * 0.2)
    x = (g(75, 1024, seed=18) * 3 + 1).requires_grad_(True)
    y = E.LayerNormFn.apply(x, ln, ln.weight, ln.bias)
    ref = ln(x)
    assert rel(y, ref) < TOL
    dy = g(75, 1024, seed=19)
    gx, gw, gb = torch.autograd.grad(ref, [x, ln.weight, ln.bias], dy)
    ln.weight.grad = ln.bias.grad = None
    y.backward(dy)
    assert rel(x.grad, gx) < TOL
    assert rel(ln.weight.grad, gw) < TOL
    assert rel(ln.bias.grad, gb) < TOL


@pytest.mark.parametrize("heads,T", [(4, 50), (2, 77)])
def test_attention(heads, T):
    from pika_b200 import engine as E
    B, D = 2, 256
    dh = D // heads
    qkv = g(B, T, 3 * D, seed=20).requires_grad_(True)
    out = E.AttentionFn.apply(qkv, heads, 0.0, 0)
    q, k, v = (qkv[:, :, i * D:(i + 1) * D].view(B, T, heads, dh).transpose(1, 2) for i in range(3))
    s = torch.matmul(q / math.sqrt(dh), k.transpose(2, 3))
    ref = torch.matmul(torch.softmax(s, -1), v).transpose(1, 2).reshape(B, T, D)
    assert rel(out, ref) < TOL
    dy = g(B, T, D, seed=21)
    (gq,) = torch.autograd.grad(ref, [qkv], dy)
    out.backward(dy)
    assert rel(qkv.grad, gq) < TOL


def test_attention_dropout_consistency():
    """With dropout the backward must use the same mask as the forward: check against autograd on an
    explicit mask recovered from the forward."""
    from pika_b200 import engine as E
    B, T, D, heads = 1, 40, 128, 2
    dh = D // heads
    qkv = g(B, T, 3 * D, seed=22).requires_grad_(True)
    out = E.AttentionFn.apply(qkv, heads, 0.3, 777)
    out2 = E.AttentionFn.apply(qkv, heads, 0.3, 777)
    assert torch.equal(out, out2)
    q, k, v = (qkv[:, :, i * D:(i + 1) * D].view(B, T, heads, dh).transpose(1, 2) for i in range(3))
    p = torch.softmax(torch.matmul(q / math.sqrt(dh), k.transpose(2, 3)), -1)
    # recover the mask: solve out = (p*mask/0.7) v per head using the saved dropped probabilities is not
    # exposed; instead verify gradient by finite differences along a random direction
    dy = g(B, T, D, seed=23)
    out.backward(dy)
    d = g(B, T, 3 * D, seed=24)
    eps = 1e-2
    with torch.no_grad():
        f1 = (E.AttentionFn.apply(qkv + eps * d, heads, 0.3, 777) * dy).sum()
        f0 = (E.AttentionFn.apply(qkv - eps * d, heads, 0.3, 777) * dy).sum()
    fd = ((f1 - f0) / (2 * eps)).item()
    an = (qkv.grad * d).sum().item()
    assert abs(fd - an) / max(abs(fd), 1e-6) < 2e-2


def test_lstm_and_embedding():
    from pika_b200 import engine as E
    V, Ed, H, B, U = 30, 100, 128, 3, 9
    emb = nn.Embedding(V + 1, Ed, padding_idx=V).cuda()
    lstm = nn.LSTM(Ed, H, num_layers=2, batch_first=True, dropout=0.0).cuda()
    y = torch.randint(1, V, (B, U), device="cuda")

    class M(nn.Module):
        pass
    m = M(); m.embed = emb; m.decoder = lstm
    lstm.train()
    out = E.prednet_forward_act(m, y)
    yy = torch.cat((torch.zeros(B, 1, dtype=torch.long, device="cuda"), y), 1)
    ref, _ = lstm(emb(yy))
    assert rel(out, ref) < TOL
    dy = g(B, U + 1, H, seed=25)
    params = [emb.weight] + list(lstm.parameters())
    gs = torch.autograd.grad(ref, params, dy)
    for p in params:
        p.grad = None
    out.backward(dy)
    for p, gr, name in zip(params, gs, ["emb"] + [n for n, _ in lstm.named_parameters()]):
        assert rel(p.grad, gr) < 2e-3, name


def test_joint_and_fused_loss():
    _joint_and_fused_loss(128, 11, 4)         # the channel-sliced gate forward and the fused gate backward


# each fallback of the gate kernels to the frame-major forward / two-pass backward: H % 32 != 0 (both), T < 8 (forward
# only), U+1 > 160 (both)
@pytest.mark.parametrize("H,T,U", [(200, 9, 4), (128, 5, 4), (128, 9, 170)])
def test_joint_and_fused_loss_gate_fallbacks(H, T, U):
    _joint_and_fused_loss(H, T, U)


def _joint_and_fused_loss(H, T, U):
    from pika_b200 import engine as E
    import numpy as np
    from oracle import rnnt as orc
    V, B = 45, 2

    class M(nn.Module):
        pass
    m = M()
    m.fc1, m.fc_gate, m.fc2 = nn.Linear(2 * H, H).cuda(), nn.Linear(2 * H, H).cuda(), nn.Linear(H, V).cuda()
    enc = g(B, T, H, seed=26).requires_grad_(True)
    pred = g(B, U + 1, H, seed=27).requires_grad_(True)
    logits = E.JointFn.apply(enc, pred, m)
    z = torch.cat((enc.unsqueeze(2).expand(-1, -1, U + 1, -1), pred.unsqueeze(1).expand(-1, T, -1, -1)), -1)
    ref = m.fc2(torch.tanh(m.fc1(z)) * torch.sigmoid(m.fc_gate(z)))
    assert rel(logits[..., :V], ref) < TOL
    assert torch.all(logits[..., V:] == 0)
    dy = torch.zeros_like(logits)
    dy[..., :V] = g(B, T, U + 1, V, seed=28)
    params = [enc, pred] + [p for l in (m.fc1, m.fc_gate, m.fc2) for p in l.parameters()]
    gs = torch.autograd.grad(ref, params, dy[..., :V], retain_graph=True)
    for p in params:
        p.grad = None
    logits.backward(dy)
    for p, gr in zip(params, gs):
        assert rel(p.grad, gr) < TOL
    # fused joint + loss vs oracle
    labels = torch.randint(1, V, (B, U), device="cuda")
    fl = torch.tensor([T, T - 2], dtype=torch.int32, device="cuda")
    ll = torch.tensor([U, U - 1], dtype=torch.int32, device="cuda")
    for p in params:
        p.grad = None
    costs = E.JointLossFn.apply(enc, pred, m, labels.int(), fl, ll)
    costs.sum().backward()
    c_ref, dz = orc.rnnt_loss_from_logits(ref.detach().cpu().numpy(), labels.cpu().numpy(), fl.cpu().numpy(), ll.cpu().numpy())
    np.testing.assert_allclose(costs.detach().cpu().numpy(), c_ref, rtol=1e-3)
    gs2 = torch.autograd.grad(ref, params, torch.from_numpy(dz).float().cuda())
    for p, gr in zip(params, gs2):
        assert rel(p.grad, gr) < 2e-3


def test_dropout_linear_backward_uses_forward_mask():
    from pika_b200 import engine as E
    lin = nn.Linear(128, 192).cuda()
    x = g(64, 128, seed=29).requires_grad_(True)
    E.set_seed(5)
    y = E.linear(x, lin.weight, lin.bias, act=True, drop_p=0.25)
    pre = F.relu(F.linear(x, lin.weight, lin.bias))
    mask = (y != 0) | (pre == 0)
    assert abs((y != 0).float().sum().item() / (pre != 0).float().sum().item() - 0.75) < 0.03
    ref = pre * mask / 0.75
    assert rel(y, ref) < TOL
    dy = g(64, 192, seed=30)
    (gx,) = torch.autograd.grad(ref, [x], dy)
    y.backward(dy)
    assert rel(x.grad, gx) < TOL
    # dropout without relu, with residual (final_linear / w_2 form)
    x2 = g(64, 128, seed=31).requires_grad_(True)
    r2 = g(64, 192, seed=32)
    y2 = E.linear(x2, lin.weight, lin.bias, drop_p=0.25, residual=r2)
    lin_out = F.linear(x2, lin.weight, lin.bias)
    m2 = ((y2 - r2).abs() > 1e-6)
    ref2 = lin_out * m2 / 0.75 + r2
    assert rel(y2, ref2) < TOL
    (gx2,) = torch.autograd.grad(ref2, [x2], dy)
    y2.backward(dy)
    assert rel(x2.grad, gx2) < TOL


@pytest.mark.parametrize("B,U,H", [(5, 12, 128), (32, 40, 256), (64, 20, 256), (45, 9, 128),    # > 32 sequences: one cooperative launch per 32
                                   (32, 150, 1024)])                                          # the benchmark's prediction net: 128 CTAs
def test_lstm_persistent_kernel_bf16(B, U, H):
    """bf16 production path: the cooperative persistent LSTM kernels (lstm_seq.cu) vs torch fp32 nn.LSTM with
    bf16-rounded weights; bf16 activations/recurrent operands -> 2e-2 outputs, 6e-2 gradients (norm-relative)."""
    from pika_b200 import engine as E
    E.set_precision("bf16")
    V, Ed = 30, 100
    emb = nn.Embedding(V + 1, Ed, padding_idx=V).cuda()
    lstm = nn.LSTM(Ed, H, num_layers=2, batch_first=True, dropout=0.0).cuda()
    with torch.no_grad():
        for p in list(lstm.parameters()) + [emb.weight]:
            p.copy_(p.to(torch.bfloat16).float())
    y = torch.randint(1, V, (B, U), device="cuda")

    class M(nn.Module):
        pass
    m = M(); m.embed = emb; m.decoder = lstm
    lstm.train()
    out = E.prednet_forward_act(m, y)
    assert out.dtype == torch.bfloat16
    yy = torch.cat((torch.zeros(B, 1, dtype=torch.long, device="cuda"), y), 1)
    ref, _ = lstm(emb(yy))
    assert rel(out, ref) < 2e-2
    dy = g(B, U + 1, H, seed=40)
    params = [emb.weight] + list(lstm.parameters())
    gs = torch.autograd.grad(ref, params, dy)
    for p in params:
        p.grad = None
    out.backward(dy.to(torch.bfloat16))
    for p, gr, name in zip(params, gs, ["emb"] + [n for n, _ in lstm.named_parameters()]):
        assert rel(p.grad, gr) < 6e-2, (name, rel(p.grad, gr))


def test_fused_lse_joint_loss_matches_separate_first_pass():
    """bf16 production path: the fc2 GEMM's row-LSE partials + rnnt_rowfinish must reproduce the stand-alone first pass
    (same rounded logits, only the fp32 summation order differs)."""
    from pika_b200 import engine as E
    H, V, B, T, U = 128, 520, 3, 13, 5
    prev, was = E.get_precision(), E._FUSED_LSE
    E.set_precision("bf16")
    # the weights and labels come from the global RNG: seed it, so that they do not depend on what earlier tests drew from it
    # (on some draws the two first passes round a few bf16 gradient entries differently, which moves the joint's weight
    # gradients by up to a few 1e-4 norm-relative, around the bound below)
    torch.manual_seed(0)
    try:
        class M(nn.Module):
            pass
        m = M()
        m.fc1, m.fc_gate, m.fc2 = nn.Linear(2 * H, H).cuda(), nn.Linear(2 * H, H).cuda(), nn.Linear(H, V).cuda()
        labels = torch.randint(1, V, (B, U), device="cuda").int()
        fl = torch.tensor([T, T - 2, T - 5], dtype=torch.int32, device="cuda")
        ll = torch.tensor([U, U - 1, 0], dtype=torch.int32, device="cuda")
        res = []
        for fused in (True, False):
            E._FUSED_LSE = fused
            enc = g(B, T, H, seed=26).bfloat16().requires_grad_(True)
            pred = g(B, U + 1, H, seed=27).bfloat16().requires_grad_(True)
            params = [enc, pred] + [p for l in (m.fc1, m.fc_gate, m.fc2) for p in l.parameters()]
            for p in params:
                p.grad = None
            costs = E.JointLossFn.apply(enc, pred, m, labels, fl, ll)
            costs.sum().backward()
            res.append((costs.detach().clone(), [p.grad.detach().float().clone() for p in params]))
        assert torch.allclose(res[0][0], res[1][0], rtol=1e-5, atol=1e-4)
        for a, b in zip(res[0][1], res[1][1]):
            assert rel(a, b) < 5e-3          # bf16 activation grads re-round; parameter grads agree far tighter
        for a, b in zip(res[0][1][2:], res[1][1][2:]):
            assert rel(a, b) < 2e-4
    finally:
        E._FUSED_LSE = was
        E.set_precision(prev)


@pytest.mark.parametrize("heads,T,B", [(4, 50, 2), (2, 200, 2), (16, 333, 1), (1, 64, 1), (3, 129, 2)])
def test_fused_attention_bf16_matches_torch(heads, T, B):
    """bf16 production path, head dim 64: attention_tc.cu (scores stay on chip) vs fp32 torch on the same bf16 inputs."""
    from pika_b200 import engine as E
    D = heads * 64
    prev = E.get_precision()
    E.set_precision("bf16")
    try:
        assert E._FUSED_ATTN
        qkv = g(B, T, 3 * D, seed=40).bfloat16().requires_grad_(True)
        out = E.AttentionFn.apply(qkv, heads, 0.0, 0)
        x = qkv.detach().float().requires_grad_(True)
        q, k, v = (x[:, :, i * D:(i + 1) * D].view(B, T, heads, 64).transpose(1, 2) for i in range(3))
        ref = torch.matmul(torch.softmax(torch.matmul(q / 8.0, k.transpose(2, 3)), -1), v).transpose(1, 2).reshape(B, T, D)
        assert rel(out, ref) < 1e-2
        dy = g(B, T, D, seed=41).bfloat16()
        (gx,) = torch.autograd.grad(ref, [x], dy.float())
        out.backward(dy)
        for i, name in enumerate("qkv"):
            assert rel(qkv.grad[:, :, i * D:(i + 1) * D], gx[:, :, i * D:(i + 1) * D]) < 2e-2, name
    finally:
        E.set_precision(prev)


@pytest.mark.parametrize("drop_p", [0.0, 0.25])
def test_fused_attention_matches_materialised_path(drop_p):
    """same dropout masks (counter-based, indexed over the [B*heads*T, T] probability matrix) in both implementations"""
    from pika_b200 import engine as E
    B, T, heads = 2, 150, 4
    D = heads * 64
    prev = E.get_precision()
    E.set_precision("bf16")
    try:
        res = []
        for fused in (True, False):
            E._FUSED_ATTN = fused
            qkv = g(B, T, 3 * D, seed=42).bfloat16().requires_grad_(True)
            out = E.AttentionFn.apply(qkv, heads, drop_p, 4242)
            out.backward(g(B, T, D, seed=43).bfloat16())
            res.append((out.detach().float(), qkv.grad.float()))
        assert rel(res[0][0], res[1][0]) < 1e-2
        assert rel(res[0][1], res[1][1]) < 2e-2
    finally:
        E._FUSED_ATTN = True
        E.set_precision(prev)
