"""float64 numpy restatement of the RNN-T forced alignment (pk_rnnt_viterbi; DESIGN.md "Forced alignment"), plus brute force over
every monotone path and the conversions between the natural [T, U1] tables and the lattice's skewed layout."""
import itertools

import numpy as np

NEG_INF = -np.inf


def viterbi(lpb, lpl, T, U):
    """lpb [>= T, >= U+1], lpl [>= T, >= U] log-probs (f32 values, summed in f64) -> (score, dec [T, U+1] bool, frames [U] int).
    delta(t,u) = max(delta(t-1,u) + lpb(t-1,u), delta(t,u-1) + lpl(t,u-1)); the label arc only when strictly greater.
    frames[u-1] = t of the label arc into (t, u); all -1 when the score is -inf."""
    lpb = np.asarray(lpb, np.float64)
    lpl = np.asarray(lpl, np.float64)
    delta = np.full((T, U + 1), NEG_INF)
    dec = np.zeros((T, U + 1), bool)
    delta[0, 0] = 0.0
    for t in range(T):
        for u in range(U + 1):
            if t == 0 and u == 0:
                continue
            a = delta[t - 1, u] + lpb[t - 1, u] if t > 0 else NEG_INF
            lab = delta[t, u - 1] + lpl[t, u - 1] if u > 0 else NEG_INF
            dec[t, u] = lab > a
            delta[t, u] = lab if dec[t, u] else a
    score = delta[T - 1, U] + lpb[T - 1, U]
    frames = np.full(U, -1, np.int64)
    if score > NEG_INF:
        t, u = T - 1, U
        while t + u > 0:
            if dec[t, u]:
                frames[u - 1] = t
                u -= 1
            else:
                t -= 1
    return score, dec, frames


def path_score(lpb, lpl, arcs):
    """arcs: 0 = blank, 1 = label, from (0, 0) to (T-1, U), then the final blank; summed in path order"""
    t = u = 0
    s = 0.0
    for a in arcs:
        if a:
            s = s + float(lpl[t, u])
            u += 1
        else:
            s = s + float(lpb[t, u])
            t += 1
    return s + float(lpb[t, u])


def path_frames(arcs, U):
    t = u = 0
    frames = np.full(U, -1, np.int64)
    for a in arcs:
        if a:
            frames[u] = t
            u += 1
        else:
            t += 1
    return frames


def brute_force(lpb, lpl, T, U):
    """every monotone path -> (best score, frames of the best path under the tie rule).  The tie rule of the back-trace (blank
    preferred at a tied node, walking back from the end) picks, among the best paths, the one whose arc sequence read from the end
    has blank at the first position where they differ."""
    n = T - 1 + U
    paths = []
    for pos in itertools.combinations(range(n), U):
        arcs = [0] * n
        for p in pos:
            arcs[p] = 1
        paths.append((path_score(lpb, lpl, arcs), arcs))
    best = max(s for s, _ in paths)
    if best == NEG_INF:
        return best, np.full(U, -1, np.int64)
    arcs = min((a for s, a in paths if s == best), key=lambda a: a[::-1])
    return best, path_frames(arcs, U)


def to_skew(nat, T, U1):
    """[B, T, U1] -> [B, T+U1-1, U1] with node (t, u) at diagonal t+u (other entries 0)"""
    B = nat.shape[0]
    out = np.zeros((B, T + U1 - 1, U1), nat.dtype)
    for t in range(T):
        out[:, t + np.arange(U1), np.arange(U1)] = nat[:, t, :]
    return out


def from_skew(sk, T, U1):
    B = sk.shape[0]
    out = np.zeros((B, T, U1), sk.dtype)
    for t in range(T):
        out[:, t, :] = sk[:, t + np.arange(U1), np.arange(U1)]
    return out


def decision_bits(words, T, U):
    """the kernel's packed decisions of one utterance [T+U1-1, ceil(U1/32)] -> [T, U+1] bool"""
    w = np.asarray(words).view(np.uint32)
    out = np.zeros((T, U + 1), bool)
    for t in range(T):
        for u in range(U + 1):
            out[t, u] = (int(w[t + u, u // 32]) >> (u % 32)) & 1
    return out
