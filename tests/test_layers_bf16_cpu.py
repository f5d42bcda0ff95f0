"""The float64 references of tests/layers_bf16_oracle.py against torch.nn modules and autograd in float64 on the CPU, at small shapes,
so that the bf16 layer tests' reference is trusted without a GPU.  Each bound is also checked to hold for the same operation computed
in fp32 from bf16 operands and stored in bf16, as the engine computes it."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import layers_bf16_oracle as O


def gen(seed):
    return torch.Generator().manual_seed(seed)


def bf(*shape, seed, scale=1.0):
    """bf16-representable float64 values"""
    return O.bf16r(torch.randn(*shape, generator=gen(seed), dtype=torch.float64) * scale)


def close(a, b, tol=1e-10):
    assert a.shape == b.shape
    err = float((a - b).abs().max())
    assert err <= tol * max(1.0, float(b.abs().max())), err


def within(got, ref, bound):
    assert O.worst(got, ref, bound) <= 1.0


def test_half_ulp_bounds_the_rounding():
    x = torch.randn(100000, generator=gen(0), dtype=torch.float64) * 10.0 ** torch.randint(-6, 6, (100000,), generator=gen(1))
    assert bool(((O.bf16r(x) - x).abs() <= O.half_ulp(x, torch.bfloat16)).all())
    assert bool(((x.float().double() - x).abs() <= O.half_ulp(x, torch.float32)).all())
    assert float(O.half_ulp(torch.tensor([1.0], dtype=torch.float64), torch.bfloat16)) == 2.0 ** -8


@pytest.mark.parametrize("relu,p,res,mask", [(False, 0.0, False, False), (True, 0.0, False, False), (True, 0.2, False, False),
                                             (False, 0.2, True, True)])
def test_linear_reference(relu, p, res, mask):
    M, K, N = 37, 48, 20
    lin = nn.Linear(K, N).double()
    with torch.no_grad():
        lin.weight.copy_(O.bf16r(lin.weight))
    x = bf(M, K, seed=2)
    if mask:
        x = x.clamp_min(0)
    x.requires_grad_(True)
    keep = (torch.rand(M, N, generator=gen(3)) >= p).double() / (1 - p)
    r = bf(M, N, seed=4)
    pre = lin(x)
    ref = (F.relu(pre) if relu else pre) * keep + (r if res else 0)
    y, inner = O.linear_fwd(x.detach(), lin.weight.detach(), lin.bias.detach(), relu, keep, r if res else None)
    close(y, ref.detach())
    # fp32 accumulation from the bf16 operands, stored in bf16, lies within the bound
    y32 = (x.detach().float() @ lin.weight.detach().float().t() + lin.bias.detach().float())
    y32 = (y32.clamp_min(0) if relu else y32) * keep.float() + (r.float() if res else 0)
    within(y32.bfloat16(), y, O.stored(y, inner, torch.bfloat16))
    dy = bf(M, N, seed=5)
    gx, gw, gb = torch.autograd.grad(ref, [x, lin.weight, lin.bias], dy)
    # d(pre) as LinearFn forms it: ReLU mask from y != 0 and the keep scale, or the keep mask alone
    dpre = dy * (y != 0) * (1 / (1 - p)) if relu else dy * keep
    xm = (x.detach() != 0) * 1.0 if mask else None
    (dx, _), (dw, _), (db, _) = O.linear_bwd(dpre, x.detach(), lin.weight.detach(), xm)
    close(dx, gx * (xm if mask else 1))
    close(dw, gw)
    close(db, gb)


@pytest.mark.parametrize("dil,stride", [(1, 1), (3, 1), (3, 4)])
def test_tdnn_reference(dil, stride):
    B, T, C, N = 2, 40, 16, 12
    conv = nn.Conv2d(1, N, (3, C), dilation=(dil, 1), stride=(stride, 1)).double()
    x = bf(B, T, C, seed=6).requires_grad_(True)
    ref = conv(x.unsqueeze(1)).squeeze(-1).transpose(1, 2)
    w = conv.weight.detach().view(N, 3, C)
    pre, inner = O.tdnn_fwd(x.detach(), w, conv.bias.detach(), dil, stride)
    close(pre, ref.detach())
    assert bool((inner > 0).all())
    dy = bf(*ref.shape, seed=7)
    gx, gw, gb = torch.autograd.grad(ref, [x, conv.weight, conv.bias], dy)
    (dx, _), (dw, _), (db, _) = O.tdnn_bwd(dy, x.detach(), w, dil, stride)
    close(dx, gx)
    close(dw, gw.view(N, 3, C))
    close(db, gb)


def test_causal_conv_reference():
    B, T, C, N, Kw = 2, 13, 10, 6, 5
    conv = nn.Conv1d(C, N, Kw, padding=Kw - 1).double()
    x = bf(B, T, C, seed=8).requires_grad_(True)
    ref = conv(x.transpose(1, 2))[..., :T].transpose(1, 2)
    pre, _ = O.causal_conv_fwd(x.detach(), conv.weight.detach(), conv.bias.detach())
    close(pre, ref.detach())
    dy = bf(B, T, N, seed=9)
    gx, gw, gb = torch.autograd.grad(ref, [x, conv.weight, conv.bias], dy)
    (dx, _), (dw, _), (db, _) = O.causal_conv_bwd(dy, x.detach(), conv.weight.detach())
    close(dx, gx)
    close(dw, gw)
    close(db, gb)


def _affine(mod, seed):
    with torch.no_grad():
        mod.weight.copy_(1 + 0.2 * torch.randn(mod.weight.shape, generator=gen(seed), dtype=torch.float64))
        mod.bias.copy_(0.2 * torch.randn(mod.bias.shape, generator=gen(seed + 1), dtype=torch.float64))


def test_layernorm_reference():
    ln = nn.LayerNorm(64, eps=1e-6).double()
    _affine(ln, 10)
    x = (bf(23, 64, seed=12) * 2 + 0.5).requires_grad_(True)
    ref = ln(x)
    y, inner, st = O.norm_fwd(x.detach(), ln.weight.detach(), ln.bias.detach(), ln.eps, 1)
    close(y, ref.detach())
    y32 = F.layer_norm(x.detach().float(), (64,), ln.weight.detach().float(), ln.bias.detach().float(), ln.eps)
    within(y32.bfloat16(), y, O.stored(y, inner, torch.bfloat16))
    dy = bf(23, 64, seed=13)
    gx, gw, gb = torch.autograd.grad(ref, [x, ln.weight, ln.bias], dy)
    (dx, dxi), (dw, _), (db, _) = O.norm_bwd(dy, st, ln.weight.detach(), 1, True)
    close(dx, gx)
    close(dw, gw)
    close(db, gb)
    x32 = x.detach().float().requires_grad_(True)
    (gx32,) = torch.autograd.grad(F.layer_norm(x32, (64,), ln.weight.detach().float(), ln.bias.detach().float(), ln.eps), [x32],
                                  dy.float())
    within(gx32.bfloat16(), dx, O.stored(dx, dxi, torch.bfloat16))


@pytest.mark.parametrize("train", [True, False])
def test_batchnorm_reference(train):
    bn = nn.BatchNorm1d(32).double()
    _affine(bn, 14)
    with torch.no_grad():
        bn.running_mean.copy_(0.1 * torch.randn(32, generator=gen(16), dtype=torch.float64))
        bn.running_var.copy_(0.5 + torch.rand(32, generator=gen(17), dtype=torch.float64))
    stats = (bn.running_mean.clone(), bn.running_var.clone())
    bn.train(train)
    x = (bf(57, 32, seed=18) * 2 + 0.5).requires_grad_(True)
    ref = bn(x)
    if train:
        y, _, st = O.norm_fwd(x.detach(), bn.weight.detach(), bn.bias.detach(), bn.eps, 0)
    else:
        y, _, st = O.norm_fwd(x.detach(), bn.weight.detach(), bn.bias.detach(), bn.eps, 0, stats[0][None], stats[1][None])
    close(y, ref.detach())
    dy = bf(57, 32, seed=19)
    gx, gw, gb = torch.autograd.grad(ref, [x, bn.weight, bn.bias], dy)
    (dx, _), (dw, _), (db, _) = O.norm_bwd(dy, st, bn.weight.detach(), 0, train)
    close(dx, gx)
    close(dw, gw)
    close(db, gb)


def test_joint_gate_reference():
    H = 16
    ex = bf(5, 1, 2 * H, seed=20).requires_grad_(True)
    py = bf(1, 7, 2 * H, seed=21).requires_grad_(True)
    a, g = ex[..., :H] + py[..., :H], ex[..., H:] + py[..., H:]
    ref = torch.tanh(a) * torch.sigmoid(g)
    h, inner = O.joint_gate(ex.detach(), py.detach())
    close(h, ref.detach())
    # the approximate tanh at its stated error, in either direction, stays inside the bound
    a32, g32 = a.detach().float(), g.detach().float()
    for sgn in (1.0, -1.0):
        t = torch.tanh(a32) * (1 + sgn * O.EPS_TANH)
        s = 0.5 * torch.tanh(0.5 * g32) * (1 - sgn * O.EPS_TANH) + 0.5
        within((t * s).bfloat16(), h, O.stored(h, inner, torch.bfloat16))
    dh = bf(5, 7, H, seed=22)
    gex, gpy = torch.autograd.grad(ref, [ex, py], dh)
    d, _ = O.joint_gate_bwd(ex.detach(), py.detach(), dh)
    close(d.sum(1, keepdim=True), gex)
    close(d.sum(0, keepdim=True), gpy)


def test_rnnt_reference_matches_the_numpy_oracle():
    from oracle import rnnt as orc
    T, U1, V = 9, 5, 13
    z = torch.randn(T, U1, V, generator=gen(23), dtype=torch.float64)
    labels = torch.randint(1, V, (U1 - 1,), generator=gen(24), dtype=torch.int32)
    for Tb, Ub in ((T, U1 - 1), (6, 2), (4, 0)):
        cost, dz, occ = O.rnnt_from_logits(z, labels, Tb, Ub)
        c_ref, dz_ref = orc.rnnt_loss_from_logits(z[None, :Tb, :Ub + 1].numpy(), labels[None, :Ub].numpy(), np.array([Tb]),
                                                  np.array([Ub]))
        assert abs(cost - c_ref[0]) < 1e-9
        close(dz[:Tb, :Ub + 1], torch.from_numpy(dz_ref[0]))
        assert bool((dz[Tb:] == 0).all()) and bool((dz[:, Ub + 1:] == 0).all())
        assert bool((occ >= 0).all())
