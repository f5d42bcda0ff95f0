"""float64 restatement of the pruned RNN-T loss (DESIGN.md "Pruned RNN-T"), built on oracle/rnnt.py's lattice.

Per utterance: am [T, V], lm [U+1, V] (the simple joiner's projections), y [U] labels, blank = 0.
  simple_loss      the RNN-T loss of z[t,u] = am[t] + lm[u] with the normaliser N = log(max(E.P^T, 2^-100)) + the row maxes,
                   and its gradients dam, dlm (the clamped nodes' normaliser is constant, as in the kernels)
  prune_bounds     the integer window starts s[t] from a float32 occupancy gamma [T, U+1]
  pruned_cost      the RNN-T loss over log-prob tables with every node outside the windows at -inf
The ``fast`` forms (alpha_beta_diag, prune_bounds_fast, fast=True) compute the same values with numpy vectorised over one
anti-diagonal (lattice) or over every window start (bounds), for production sizes such as T = 240, U = 150.
"""
import numpy as np

from oracle.rnnt import rnnt_alpha_beta

NEG_INF = -np.inf
FLOOR = 2.0 ** -100


def alpha_beta_diag(lpb, lpl, T, U):
    """oracle.rnnt.rnnt_alpha_beta with each anti-diagonal t + u = d in one numpy step -> alpha, beta [T, U+1]"""
    lpb = np.asarray(lpb, np.float64)
    lpl = np.asarray(lpl, np.float64).reshape(T, U)
    alpha = np.full((T, U + 1), NEG_INF)
    beta = np.full((T, U + 1), NEG_INF)
    alpha[0, 0] = 0.0
    for d in range(1, T + U):
        u = np.arange(max(0, d - T + 1), min(d, U) + 1)
        t = d - u
        a = np.full(u.size, NEG_INF)
        c = np.full(u.size, NEG_INF)
        m = t > 0
        a[m] = alpha[t[m] - 1, u[m]] + lpb[t[m] - 1, u[m]]
        m = u > 0
        c[m] = alpha[t[m], u[m] - 1] + lpl[t[m], u[m] - 1]
        alpha[t, u] = np.logaddexp(a, c)
    beta[T - 1, U] = lpb[T - 1, U]
    for d in range(T + U - 2, -1, -1):
        u = np.arange(max(0, d - T + 1), min(d, U) + 1)
        t = d - u
        a = np.full(u.size, NEG_INF)
        c = np.full(u.size, NEG_INF)
        m = t < T - 1
        a[m] = beta[t[m] + 1, u[m]] + lpb[t[m], u[m]]
        m = u < U
        c[m] = beta[t[m], u[m] + 1] + lpl[t[m], u[m]]
        beta[t, u] = np.logaddexp(a, c)
    return alpha, beta


def occupancy(lpb, lpl, T, U, fast=False):
    """-> (cost, gb [T, U+1], gl [T, U+1]) with gb / gl = d cost / d lpb, d cost / d lpl (<= 0), as the lattice kernel emits them"""
    alpha, beta = (alpha_beta_diag if fast else rnnt_alpha_beta)(lpb, lpl, T, U)
    ll = beta[0, 0]
    bn = np.full((T, U + 1), NEG_INF)
    bn[:T - 1] = beta[1:]
    bn[T - 1, U] = 0.0
    with np.errstate(invalid="ignore", over="ignore"):
        gb = -np.exp(alpha + bn + lpb - ll)
        gl = np.zeros((T, U + 1))
        if U > 0:
            gl[:, :U] = -np.exp(alpha[:, :U] + beta[:, 1:] + lpl - ll)
    gb[~np.isfinite(gb)] = 0.0
    gl[~np.isfinite(gl)] = 0.0
    return -ll, gb, gl


def simple_tables(am, lm, y):
    """-> (lpb [T, U+1], lpl [T, U], S [T, U+1] = E.P^T, clamped mask)"""
    am = np.asarray(am, np.float64)
    lm = np.asarray(lm, np.float64)
    ma, ml = am.max(1), lm.max(1)
    E, P = np.exp(am - ma[:, None]), np.exp(lm - ml[:, None])
    S = E @ P.T
    clamped = S < FLOOR
    N = np.log(np.maximum(S, FLOOR)) + ma[:, None] + ml[None, :]
    lpb = am[:, None, 0] + lm[None, :, 0] - N
    U = len(y)
    lpl = np.zeros((am.shape[0], U))
    for u in range(U):
        lpl[:, u] = am[:, y[u]] + lm[u, y[u]] - N[:, u]
    return lpb, lpl, S, clamped


def simple_loss(am, lm, y, fast=False):
    """-> (cost, dam [T, V], dlm [U+1, V], gb, gl)"""
    am = np.asarray(am, np.float64)
    lm = np.asarray(lm, np.float64)
    T, U = am.shape[0], len(y)
    lpb, lpl, S, clamped = simple_tables(am, lm, y)
    cost, gb, gl = occupancy(lpb, lpl, T, U, fast)
    E = np.exp(am - am.max(1, keepdims=True))
    P = np.exp(lm - lm.max(1, keepdims=True))
    W = np.where(clamped, 0.0, -(gb + gl) / np.where(clamped, 1.0, S))
    dam = E * (W @ P)
    dlm = P * (W.T @ E)
    dam[:, 0] += gb.sum(1)
    dlm[:, 0] += gb.sum(0)
    for u in range(U):
        dam[:, y[u]] += gl[:, u]
        dlm[u, y[u]] += gl[:, u].sum()
    return cost, dam, dlm, gb, gl


def prune_bounds(gamma, T, U, R):
    """gamma [>= T, >= U+1] float32 occupancy -> s [T] int (the kernel's algorithm, same f64 sums in the same order)"""
    if U > T * (R - 1):
        raise ValueError("U = %d > T (R - 1) = %d: no path fits in windows of %d" % (U, T * (R - 1), R))
    g = np.asarray(gamma, np.float32)
    S = max(U - R + 1, 0)
    s = np.zeros(T, np.int64)
    for t in range(T):
        best, best_c = 0, -1.0
        for st in range(S + 1):
            c = 0.0
            for u in range(st, min(st + R - 1, U) + 1):
                c = c + float(g[t, u])
            if c > best_c:
                best, best_c = st, c
        lo = max(0, U - R + 1 - (T - 1 - t) * (R - 1))
        hi = min(t * (R - 1), S)
        s[t] = min(max(best, lo), hi)
    s = np.maximum.accumulate(s)
    for t in range(T - 2, -1, -1):
        s[t] = max(s[t], s[t + 1] - (R - 1))
    return s


def prune_bounds_fast(gamma, T, U, R):
    """prune_bounds with the window sums of every start s formed at once: the same f64 additions in the same (ascending u) order"""
    if U > T * (R - 1):
        raise ValueError("U = %d > T (R - 1) = %d: no path fits in windows of %d" % (U, T * (R - 1), R))
    g = np.asarray(gamma, np.float32)[:T, :U + 1].astype(np.float64)
    S = max(U - R + 1, 0)
    c = np.zeros((T, S + 1))
    st = np.arange(S + 1)
    for k in range(R):
        u = st + k
        ok = u <= U
        c[:, ok] = c[:, ok] + g[:, u[ok]]
    best = np.where(c.max(1) > -1.0, c.argmax(1), 0)          # argmax: the smallest start on a tie
    t = np.arange(T)
    lo = np.maximum(0, U - R + 1 - (T - 1 - t) * (R - 1))
    hi = np.minimum(t * (R - 1), S)
    s = np.minimum(np.maximum(best, lo), hi)
    s = np.maximum.accumulate(s)
    for t in range(T - 2, -1, -1):
        s[t] = max(s[t], s[t + 1] - (R - 1))
    return s


def window_mask(s, T, U, R):
    """[T, U+1] bool: node (t, u) lies in frame t's window [s_t, s_t + R - 1]"""
    u = np.arange(U + 1)[None, :]
    return (u >= np.asarray(s)[:T, None]) & (u < np.asarray(s)[:T, None] + R)


def pruned_cost(lpb, lpl, s, R, fast=False):
    """RNN-T cost over the tables with the nodes outside the windows at -inf -> (cost, gb, gl)"""
    T, U1 = lpb.shape
    U = U1 - 1
    m = window_mask(s, T, U, R)
    pb = np.where(m, lpb, NEG_INF)
    pl = np.where(m[:, :U], lpl, NEG_INF) if U > 0 else lpl
    return occupancy(pb, pl, T, U, fast)


def check_bounds_properties(s, T, U, R):
    s = np.asarray(s)[:T]
    assert s[0] == 0
    assert (np.diff(s) >= 0).all()
    assert (np.diff(s) <= R - 1).all()
    assert s[-1] + R - 1 >= U
    assert (s >= 0).all() and (s <= max(U - R + 1, 0)).all()
