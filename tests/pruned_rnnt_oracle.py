"""float64 restatement of the pruned RNN-T loss (DESIGN.md "Pruned RNN-T"), built on oracle/rnnt.py's lattice.

Per utterance: am [T, V], lm [U+1, V] (the simple joiner's projections), y [U] labels, blank = 0.
  simple_loss      the RNN-T loss of z[t,u] = am[t] + lm[u] with the normaliser N = log(max(E.P^T, 2^-100)) + the row maxes,
                   and its gradients dam, dlm (the clamped nodes' normaliser is constant, as in the kernels)
  prune_bounds     the integer window starts s[t] from a float32 occupancy gamma [T, U+1]
  pruned_cost      the RNN-T loss over log-prob tables with every node outside the windows at -inf
"""
import numpy as np

from oracle.rnnt import rnnt_alpha_beta

NEG_INF = -np.inf
FLOOR = 2.0 ** -100


def occupancy(lpb, lpl, T, U):
    """-> (cost, gb [T, U+1], gl [T, U+1]) with gb / gl = d cost / d lpb, d cost / d lpl (<= 0), as the lattice kernel emits them"""
    alpha, beta = rnnt_alpha_beta(lpb, lpl, T, U)
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


def simple_loss(am, lm, y):
    """-> (cost, dam [T, V], dlm [U+1, V], gb, gl)"""
    am = np.asarray(am, np.float64)
    lm = np.asarray(lm, np.float64)
    T, U = am.shape[0], len(y)
    lpb, lpl, S, clamped = simple_tables(am, lm, y)
    cost, gb, gl = occupancy(lpb, lpl, T, U)
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


def window_mask(s, T, U, R):
    """[T, U+1] bool: node (t, u) lies in frame t's window [s_t, s_t + R - 1]"""
    u = np.arange(U + 1)[None, :]
    return (u >= np.asarray(s)[:T, None]) & (u < np.asarray(s)[:T, None] + R)


def pruned_cost(lpb, lpl, s, R):
    """RNN-T cost over the tables with the nodes outside the windows at -inf -> (cost, gb, gl)"""
    T, U1 = lpb.shape
    U = U1 - 1
    m = window_mask(s, T, U, R)
    pb = np.where(m, lpb, NEG_INF)
    pl = np.where(m[:, :U], lpl, NEG_INF) if U > 0 else lpl
    return occupancy(pb, pl, T, U)


def check_bounds_properties(s, T, U, R):
    s = np.asarray(s)[:T]
    assert s[0] == 0
    assert (np.diff(s) >= 0).all()
    assert (np.diff(s) <= R - 1).all()
    assert s[-1] + R - 1 >= U
    assert (s >= 0).all() and (s <= max(U - R + 1, 0)).all()
