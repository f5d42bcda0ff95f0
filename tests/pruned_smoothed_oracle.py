"""float64 restatement of the pruned RNN-T loss's smoothed simple loss (DESIGN.md "Pruned RNN-T"), built on pruned_rnnt_oracle.py.

Per utterance: am [T, V], lm [U+1, V], y [U]; lam_l = lm_only_scale, lam_a = am_only_scale, mu = 1 - lam_l - lam_a.
  lp(t,u,k) = mu * lp_full(t,u,k) + lam_l * (lm[u,k] - Nl(u)) + lam_a * (am[t,k] + log q_k - Na(t))   for k = 0 and k = y_{u+1}
with Nl(u) = logsumexp lm[u], Na(t) = logsumexp (am[t] + log q) and q the mean of softmax(lm[b, u]) over the batch's valid rows
(+ 1e-10), a constant of the step: no gradient flows through it.  The batch is needed for q only.
"""
import numpy as np

import pruned_rnnt_oracle as P

Q_EPS = 1e-10


def _lse(x):
    m = x.max(1, keepdims=True)
    return (m + np.log(np.exp(x - m).sum(1, keepdims=True)))[:, 0]


def unigram_logq(lms):
    """lms: the valid [U_b+1, V] rows of every utterance -> log q [V]"""
    rows = np.concatenate([np.asarray(l, np.float64) for l in lms])
    sm = np.exp(rows - _lse(rows)[:, None])
    return np.log(sm.sum(0) / rows.shape[0] + Q_EPS)


def smoothed_tables(am, lm, y, logq, lam_l, lam_a):
    """-> (lpb [T, U+1], lpl [T, U], S, clamped, Nl [U+1], Na [T])"""
    am = np.asarray(am, np.float64)
    lm = np.asarray(lm, np.float64)
    lpb, lpl, S, clamped = P.simple_tables(am, lm, y)
    Nl, Na = _lse(lm), _lse(am + logq[None, :])
    if lam_l == 0.0 and lam_a == 0.0:
        return lpb, lpl, S, clamped, Nl, Na
    mu = 1.0 - lam_l - lam_a
    lpb = mu * lpb + lam_l * (lm[None, :, 0] - Nl[None, :]) + lam_a * (am[:, None, 0] + logq[0] - Na[:, None])
    lpl = lpl.copy()
    for u in range(len(y)):
        k = y[u]
        lpl[:, u] = mu * lpl[:, u] + lam_l * (lm[u, k] - Nl[u]) + lam_a * (am[:, k] + logq[k] - Na)
    return lpb, lpl, S, clamped, Nl, Na


def simple_loss(am, lm, y, logq, lam_l, lam_a):
    """one utterance with q given -> (cost, dam [T, V], dlm [U+1, V], gb, gl).  lam_l = lam_a = 0 is pruned_rnnt_oracle.simple_loss."""
    am = np.asarray(am, np.float64)
    lm = np.asarray(lm, np.float64)
    T, U = am.shape[0], len(y)
    lpb, lpl, S, clamped, Nl, Na = smoothed_tables(am, lm, y, logq, lam_l, lam_a)
    cost, gb, gl = P.occupancy(lpb, lpl, T, U)
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


def batch_simple_loss(ams, lms, ys, lam_l, lam_a):
    """per-utterance lists am [T_b, V], lm [U_b+1, V], y [U_b] -> (logq, [(cost, dam, dlm, gb, gl)] per utterance)"""
    logq = unigram_logq(lms)
    return logq, [simple_loss(a, l, y, logq, lam_l, lam_a) for a, l, y in zip(ams, lms, ys)]
