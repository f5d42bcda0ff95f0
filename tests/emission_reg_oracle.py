"""float64 restatement of the RNN-T emission regularisation (DESIGN.md "FastEmit and delay penalty"), in the style of
tests/pruned_rnnt_oracle.py.

Per utterance: T frames, U labels y, blank 0; lpb [T, U+1] and lpl [T, U] the blank / label log-probs of the lattice.
  delay_term       lam_d * ((T - 1)/2 - t) for every label arc (t, u), [T, U]
  lattice          the penalised alpha, beta [T, U+1], the cost -log P (penalised) and the coefficients gb, gl = d cost / d lpb,
                   d cost / d lpl (<= 0), gl times 1 + lam_f (FastEmit), as the lattice kernel emits them
  row_grad         one joint row's d / d logits from (gb, gl), as the row passes form it
  dense_loss       a whole utterance from logits [T, U+1, V]: (cost, dlogits)
  pruned_loss      the lattice over tables with every node outside the windows at -inf
  simple_loss      the simple joiner's loss (smoothed when lam_l or lam_a > 0) on the penalised lattice: (cost, dam, dlm, gb, gl);
                   FastEmit never applies to it
"""
import numpy as np

import pruned_rnnt_oracle as P
import pruned_smoothed_oracle as PS
from oracle.rnnt import log_softmax


def delay_term(T, U, lam_d):
    """[T, U]: the delay penalty's addend to lpl(t, u)"""
    return np.repeat((lam_d * ((T - 1) / 2.0 - np.arange(T, dtype=np.float64)))[:, None], U, 1)


def lattice(lpb, lpl, T, U, lam_f=0.0, lam_d=0.0):
    """-> (cost, gb [T, U+1], gl [T, U+1], alpha, beta) on the delay-penalised lattice, gl scaled by 1 + lam_f"""
    lpb = np.asarray(lpb, np.float64)[:T, :U + 1]
    lpl = np.asarray(lpl, np.float64)[:T, :U] + delay_term(T, U, lam_d)
    alpha, beta = P.alpha_beta_diag(lpb, lpl, T, U)
    cost, gb, gl = P.occupancy(lpb, lpl, T, U, fast=True)
    return cost, gb, gl * (1.0 + lam_f), alpha, beta


def row_grad(lp_row, gb, gl, y):
    """d / d logits of one row with log-softmax lp_row [V]: gb at blank, gl at label y (-1: none), minus softmax * (gb + gl)"""
    g = np.zeros(lp_row.shape[0])
    g[0] += gb
    if y >= 0:
        g[y] += gl
    return g - np.exp(lp_row) * g.sum()


def dense_loss(logits, y, lam_f=0.0, lam_d=0.0):
    """logits [T, U+1, V] of one utterance, y [U] -> (cost, dlogits [T, U+1, V])"""
    lp = log_softmax(np.asarray(logits, np.float64))
    T, U1, V = lp.shape
    U = U1 - 1
    lpb = lp[:, :, 0]
    lpl = lp[:, np.arange(U), y] if U > 0 else np.zeros((T, 0))
    cost, gb, gl, _, _ = lattice(lpb, lpl, T, U, lam_f, lam_d)
    d = np.zeros_like(lp)
    for t in range(T):
        for u in range(U1):
            d[t, u] = row_grad(lp[t, u], gb[t, u], gl[t, u], y[u] if u < U else -1)
    return cost, d


def pruned_loss(lpb, lpl, s, R, lam_f=0.0, lam_d=0.0):
    """tables of one utterance [T, U+1] / [T, U] and window starts s [T] -> (cost, gb, gl) with the nodes outside the windows at -inf"""
    T, U1 = lpb.shape
    U = U1 - 1
    m = P.window_mask(s, T, U, R)
    pb = np.where(m, lpb, -np.inf)
    pl = np.where(m[:, :U], lpl, -np.inf) if U > 0 else lpl
    cost, gb, gl, _, _ = lattice(pb, pl, T, U, lam_f, lam_d)
    return cost, gb, gl


def simple_loss(am, lm, y, lam_d=0.0, logq=None, lam_l=0.0, lam_a=0.0):
    """the simple joiner's loss of one utterance on the delay-penalised lattice -> (cost, dam [T, V], dlm [U+1, V], gb, gl).
    lam_l / lam_a > 0: smoothed with the batch unigram logq (tests/pruned_smoothed_oracle.py).  The delay term is a constant of the
    tables, so the projections' gradients are pruned_smoothed_oracle.simple_loss's formulas fed the penalised occupancies."""
    am = np.asarray(am, np.float64)
    lm = np.asarray(lm, np.float64)
    T, U = am.shape[0], len(y)
    if logq is None:
        logq = np.zeros(am.shape[1])
    lpb, lpl, S, clamped, Nl, Na = PS.smoothed_tables(am, lm, y, logq, lam_l, lam_a)
    cost, gb, gl, _, _ = lattice(lpb, lpl, T, U, 0.0, lam_d)
    mu = 1.0 - lam_l - lam_a
    E = np.exp(am - am.max(1, keepdims=True))
    Pm = np.exp(lm - lm.max(1, keepdims=True))
    gamma = -(gb + gl)
    W = np.where(clamped, 0.0, mu * gamma / np.where(clamped, 1.0, S))
    dam = E * (W @ Pm)
    dlm = Pm * (W.T @ E)
    if lam_a:
        dam += lam_a * gamma.sum(1)[:, None] * np.exp(am + logq[None, :] - Na[:, None])
    if lam_l:
        dlm += lam_l * gamma.sum(0)[:, None] * np.exp(lm - Nl[:, None])
    ka, kl = mu + lam_a, mu + lam_l
    dam[:, 0] += ka * gb.sum(1)
    dlm[:, 0] += kl * gb.sum(0)
    for u in range(U):
        dam[:, y[u]] += ka * gl[:, u]
        dlm[u, y[u]] += kl * gl[:, u].sum()
    return cost, dam, dlm, gb, gl
