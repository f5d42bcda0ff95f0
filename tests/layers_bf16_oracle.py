"""float64 references of the engine's autograd Functions in the bf16 training precision, and the element-wise error bounds the bf16
layer tests hold them to (tests/test_layers_bf16_gpu.py; the references themselves are pinned to torch.nn in float64 by
tests/test_layers_bf16_cpu.py).

Every reference takes the operands the engine actually used: activations and incoming gradients as the engine's bf16 tensors, weights
rounded to bf16 as ``engine.stage_weight`` rounds them (``w.bfloat16().double()``), masks as the engine drew them.  It then differs from
the engine only by the engine's fp32 accumulation and its final rounding, which the bounds below state:

  * a contraction of length K whose terms are exact products of bf16 operands, summed in fp32 in any order, is within
    gamma_K = K u32 of the exact sum, relative to the sum of the terms' magnitudes (|A||B|); C_ACC = 2 leaves room for the two
    roundings per step that a fused multiply-add chain or a split-K reduce-add can take;
  * a result stored in bf16 (or f32) is then rounded once more: half an ulp of the stored type at the result's magnitude;
  * a bf16 operand the engine forms itself (a masked or dropout-scaled gradient, a stored activation) is rounded by the reference at
    the same point, so it is the same value on both sides.
"""
import math

import torch

U24 = 2.0 ** -24            # f32 unit roundoff
C_ACC = 2.0
MANT = {torch.float32: 24, torch.bfloat16: 8}
TINY = 1e-37


def half_ulp(x, dtype):
    """half an ulp of ``dtype`` at |x| (the largest round-to-nearest error of a value of that magnitude)"""
    m, e = torch.frexp(x.abs())
    return torch.where(m == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - 1 - MANT[dtype]))


def bf16r(x):
    """round to bf16, back in float64"""
    return x.float().bfloat16().double()


def acc(K, mag):
    """bound on the fp32 accumulation error of K terms whose magnitudes sum to ``mag``"""
    return C_ACC * K * U24 * mag


def stored(ref, inner, dtype):
    """bound on |got - ref| for a value within ``inner`` of ``ref`` before it is stored in ``dtype``"""
    return inner + half_ulp(ref.abs() + inner, dtype) + TINY


def worst(got, ref, bound):
    """largest |got - ref| / bound (NaN anywhere in ``got`` counts as infinite)"""
    err = (got.double() - ref).abs()
    if bool(torch.isnan(err).any()):
        return math.inf
    return float((err / bound).max())


def norm_rel(got, ref):
    return float((got.double() - ref).norm() / ref.norm().clamp_min(1e-300))


# ------------------------------------------------------------------------------------------------ Linear
def linear_fwd(x, w, b=None, relu=False, keep=None, residual=None):
    """y = keep * act(x w^T + b) + residual (LinearFn's epilogue order); keep: the dropout keep mask times its scale, or None.
    -> (y, inner bound before the bf16 store)"""
    y = x @ w.t()
    mag = x.abs() @ w.abs().t()
    if b is not None:
        y = y + b
        mag = mag + b.abs()
    inner = acc(x.shape[1] + 1, mag)
    if relu:
        y = y.clamp_min(0)
    if keep is not None:
        y, inner = y * keep, inner * keep + U24 * (y * keep).abs()             # the keep scale's f32 multiply rounds once
    if residual is not None:
        y = y + residual
        inner = inner + 2 * U24 * (y.abs() + residual.abs())
    return y, inner


def linear_bwd(dpre, x, w, x_mask_scale=None):
    """gradients of y = x w^T + b for d(pre-activation) ``dpre`` -> ((dx, inner), (dw, inner), (db, inner)); x_mask_scale: the
    AUX_MASK_NZ epilogue's (x != 0) * scale applied to dx"""
    M, N = dpre.shape
    dx = dpre @ w
    dx_in = acc(N, dpre.abs() @ w.abs())
    if x_mask_scale is not None:
        dx, dx_in = dx * x_mask_scale, dx_in * x_mask_scale
    dw = dpre.t() @ x
    dw_in = acc(M, dpre.abs().t() @ x.abs())
    db = dpre.sum(0)
    db_in = acc(M, dpre.abs().sum(0))
    return (dx, dx_in), (dw, dw_in), (db, db_in)


# ------------------------------------------------------------------------------------------------ TDNN / causal convolution
def tdnn_fwd(x, w, b, dil, stride):
    """relu-free Conv2d(1, N, (3, C), dilation=(dil, 1), stride=(stride, 1)) on x [B, T, C]; w [N, 3, C] -> (pre [B, T', N], inner)"""
    B, T, C = x.shape
    t_out = (T - 2 * dil - 1) // stride + 1
    span = (t_out - 1) * stride + 1
    taps = [x[:, k * dil:k * dil + span:stride] for k in range(3)]
    pre = sum(taps[k] @ w[:, k].t() for k in range(3)) + b
    mag = sum(taps[k].abs() @ w[:, k].abs().t() for k in range(3)) + b.abs()
    return pre, acc(3 * C + 1, mag)


def tdnn_bwd(dpre, x, w, dil, stride):
    """-> ((dx, inner), (dw [N, 3, C], inner), (db, inner))"""
    B, T, C = x.shape
    t_out = dpre.shape[1]
    span = (t_out - 1) * stride + 1
    dx = torch.zeros_like(x)
    dx_mag = torch.zeros_like(x)
    for k in range(3):
        dx[:, k * dil:k * dil + span:stride] += dpre @ w[:, k]
        dx_mag[:, k * dil:k * dil + span:stride] += dpre.abs() @ w[:, k].abs()
    d2 = dpre.reshape(-1, dpre.shape[-1])
    dw = torch.stack([d2.t() @ x[:, k * dil:k * dil + span:stride].reshape(-1, C) for k in range(3)], 1)
    dw_mag = torch.stack([d2.abs().t() @ x[:, k * dil:k * dil + span:stride].reshape(-1, C).abs() for k in range(3)], 1)
    rows = d2.shape[0]
    return (dx, acc(3 * dpre.shape[-1], dx_mag)), (dw, acc(rows, dw_mag)), (d2.sum(0), acc(rows, d2.abs().sum(0)))


def causal_conv_fwd(x, w, b):
    """Conv1d(C, N, Kw, padding=Kw-1) keeping the first T outputs (the causal convolution), x [B, T, C], w [N, C, Kw] -> (pre, inner)"""
    B, T, C = x.shape
    Kw = w.shape[2]
    xp = torch.cat([x.new_zeros(B, Kw - 1, C), x], 1)
    pre = sum(xp[:, k:k + T] @ w[:, :, k].t() for k in range(Kw)) + b
    mag = sum(xp[:, k:k + T].abs() @ w[:, :, k].abs().t() for k in range(Kw)) + b.abs()
    return pre, acc(Kw * C + 1, mag)


def causal_conv_bwd(dpre, x, w):
    """-> ((dx, inner), (dw [N, C, Kw], inner), (db, inner))"""
    B, T, C = x.shape
    Kw = w.shape[2]
    N = w.shape[0]
    xp = torch.cat([x.new_zeros(B, Kw - 1, C), x], 1)
    dxp = torch.zeros_like(xp)
    mag = torch.zeros_like(xp)
    for k in range(Kw):
        dxp[:, k:k + T] += dpre @ w[:, :, k]
        mag[:, k:k + T] += dpre.abs() @ w[:, :, k].abs()
    d2 = dpre.reshape(-1, N)
    dw = torch.stack([d2.t() @ xp[:, k:k + T].reshape(-1, C) for k in range(Kw)], 2)
    dw_mag = torch.stack([d2.abs().t() @ xp[:, k:k + T].reshape(-1, C).abs() for k in range(Kw)], 2)
    rows = d2.shape[0]
    return ((dxp[:, Kw - 1:], acc(Kw * N, mag[:, Kw - 1:])), (dw, acc(rows, dw_mag)), (d2.sum(0), acc(rows, d2.abs().sum(0))))


# ------------------------------------------------------------------------------------------------ normalisations
def _norm_stats(x, dim):
    n = x.shape[dim]
    mean = x.mean(dim, keepdim=True)
    var = ((x - mean) ** 2).mean(dim, keepdim=True)
    # fp32 sums of n terms: the mean to gamma_n of mean |x|, the variance to gamma_n of the mean square (shifted or not); rsqrt adds a
    # few ulp
    e_mean = acc(n, x.abs().mean(dim, keepdim=True))
    e_var = acc(n, (x ** 2).mean(dim, keepdim=True)) + 2 * (x - mean).abs().mean(dim, keepdim=True) * e_mean
    return mean, var, e_mean, e_var


def norm_fwd(x, w, b, eps, dim, mean=None, var=None):
    """(x - mean) rstd w + b with the statistics over ``dim`` (0: BatchNorm over rows, 1: LayerNorm over columns), or the given ones
    (BatchNorm eval) -> (y, inner, st); st holds xhat, rstd and the error bounds of xhat (absolute) and rstd (relative)"""
    if mean is None:
        mean, var, e_mean, e_var = _norm_stats(x, dim)
    else:
        e_mean, e_var = torch.zeros_like(mean), torch.zeros_like(var)
    rstd = 1.0 / torch.sqrt(var + eps)
    e_r = 0.5 * e_var / (var + eps) + 8 * U24
    xhat = (x - mean) * rstd
    e_xhat = rstd * e_mean + xhat.abs() * e_r + 4 * U24 * xhat.abs()
    y = xhat * w + b
    # the kernels may fold the affine map into y = x (rstd w) + (b - mean rstd w): then x and mean are each rounded relative to
    # their own magnitude, not to |x - mean|
    inner = w.abs() * e_xhat + 4 * U24 * (xhat * w).abs() + 2 * U24 * y.abs() + 4 * U24 * rstd * w.abs() * (x.abs() + mean.abs())
    return y, inner, dict(xhat=xhat, rstd=rstd, e_xhat=e_xhat, e_r=e_r)


def norm_bwd(dy, st, w, dim, train):
    """backward of norm_fwd for ``dy``; train: the statistics depend on x.  -> ((dx, inner), (dw, inner), (db, inner))"""
    xhat, rstd, e_xhat, e_r = st["xhat"], st["rstd"], st["e_xhat"], st["e_r"]
    g = dy * w
    n = xhat.shape[dim]
    if train:
        m1 = g.mean(dim, keepdim=True)
        m2 = (g * xhat).mean(dim, keepdim=True)
        core = g - m1 - xhat * m2
        e_m1 = acc(n, g.abs().mean(dim, keepdim=True))
        e_m2 = acc(n, (g * xhat).abs().mean(dim, keepdim=True)) + (g.abs() * e_xhat).mean(dim, keepdim=True)
        e_core = e_m1 + xhat.abs() * e_m2 + e_xhat * m2.abs() + 4 * U24 * (g.abs() + m1.abs() + (xhat * m2).abs())
    else:
        core, e_core = g, U24 * g.abs()
    dx = rstd * core
    dx_in = rstd * e_core + e_r * dx.abs() + 2 * U24 * dx.abs()
    rows = xhat.shape[0]                 # the affine parameters are per column in both norms
    dw = (dy * xhat).sum(0)
    dw_in = acc(rows, (dy * xhat).abs().sum(0)) + (dy.abs() * e_xhat).sum(0)
    db = dy.sum(0)
    return (dx, dx_in), (dw, dw_in), (db, acc(rows, dy.abs().sum(0)))


# ------------------------------------------------------------------------------------------------ gated joint
# the bf16 gate evaluates tanh with tanh.approx.f32 and sigmoid as 0.5 tanh(x / 2) + 0.5; the PTX ISA states a maximum relative error
# of 2^-11 for tanh.approx.f32 over the full range
EPS_TANH = 2.0 ** -11


def joint_gate(ex, py):
    """ex, py [.., 2H] (fc1 | fc_gate halves) -> h = tanh(a) sigmoid(g), a = ex1 + py1, g = exg + pyg, and the bound of the bf16 path's
    fp32 evaluation before the bf16 store: the sums round once (tanh' <= 1, sigmoid' <= 1/4), the approximate tanh is within
    EPS_TANH |t| and the sigmoid within EPS_TANH |2s - 1| / 2, and the product rounds once"""
    H = ex.shape[-1] // 2
    a = ex[..., :H] + py[..., :H]
    g = ex[..., H:] + py[..., H:]
    t, s = torch.tanh(a), torch.sigmoid(g)
    h = t * s
    inner = (U24 * a.abs() * s + U24 * g.abs() * t.abs() / 4 + EPS_TANH * t.abs() * (s + 0.5 * (2 * s - 1).abs()) * (1 + 1e-3)
             + U24 * h.abs())
    return h, inner


def joint_gate_bwd(ex, py, dh):
    """-> (d[a | g] [.., 2H], the bf16 path's per-element bound): the gradient of h = tanh(a) sigmoid(g), the same for ex and py.
    With the approximate tanh and sigmoid, |d (1 - t'^2) s' - d (1 - t^2) s| <= 2.5 EPS_TANH |d| and |d t' s' (1 - s') - d t s (1 - s)|
    <= 0.75 EPS_TANH |d|"""
    H = ex.shape[-1] // 2
    a = ex[..., :H] + py[..., :H]
    g = ex[..., H:] + py[..., H:]
    t, s = torch.tanh(a), torch.sigmoid(g)
    d = torch.cat([dh * s * (1 - t * t), dh * t * s * (1 - s)], -1)
    return d, torch.cat([2.5 * EPS_TANH * dh.abs(), 0.75 * EPS_TANH * dh.abs()], -1) + 4 * U24 * d.abs()


# ------------------------------------------------------------------------------------------------ RNN-T loss
def rnnt_from_logits(z, labels, T, U):
    """float64 RNN-T cost and d cost / d logits of one utterance from its logits z [T', U1, V] (rows past T / U ignored) ->
    (cost, dz [T', U1, V], occupancy bound per row [T', U1]).  The lattice is oracle/rnnt.py's."""
    import numpy as np
    from oracle import rnnt as orc
    lp = torch.log_softmax(z, -1)
    y = labels[:U].long()
    lpb = lp[:T, :U + 1, 0]
    lpl = lp[:T, torch.arange(U, device=z.device), y] if U > 0 else lp.new_zeros(T, 0)          # [T, U]
    alpha, beta = orc.rnnt_alpha_beta(lpb.cpu().numpy(), lpl.cpu().numpy(), T, U)
    ll = beta[0, 0]
    bn = np.full((T, U + 1), -np.inf)
    bn[:T - 1] = beta[1:]
    bn[T - 1, U] = 0.0
    with np.errstate(invalid="ignore"):
        gb = -np.exp(alpha + bn + lpb.cpu().numpy() - ll)
        gl = -np.exp(alpha[:, :U] + beta[:, 1:] + lpl.cpu().numpy() - ll) if U > 0 else np.zeros((T, 0))
    gb, gl = np.nan_to_num(gb), np.nan_to_num(gl)
    g = torch.zeros_like(z)
    g[:T, :U + 1, 0] = torch.from_numpy(gb).to(z)
    if U > 0:
        g[:T, torch.arange(U, device=z.device), y] += torch.from_numpy(gl).to(z)
    dz = g - lp.exp() * g.sum(-1, keepdim=True)
    occ = g.abs().sum(-1)
    return -ll, dz, occ
