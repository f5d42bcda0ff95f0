"""The emission-regularisation oracle (tests/emission_reg_oracle.py) against independent computations: torchaudio's RNN-T loss on
delay-penalised log-probs, brute force over every path, central differences, and FastEmit formed from torchaudio's gradient.  Plus
the properties the two options promise, and the command-line flags."""
import math

import numpy as np
import pytest
import torch

import emission_reg_oracle as E
import pruned_rnnt_oracle as P
import pruned_smoothed_oracle as PS
from oracle.rnnt import log_softmax, rnnt_brute_force


def _case(seed, T, U, V):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((T, U + 1, V)) * 2.0, rng.integers(1, V, U)


def _penalised_log_probs(logits, y, lam_d):
    """log-softmax with lam_d ((T-1)/2 - t) added at [t, u, y_{u+1}], u < U"""
    lp = log_softmax(np.asarray(logits, np.float64))
    T, U1, _ = lp.shape
    pen = E.delay_term(T, U1 - 1, lam_d)
    for u in range(U1 - 1):
        lp[:, u, y[u]] += pen[:, u]
    return lp


def _torchaudio(lp, y, T, U):
    """torchaudio's RNN-T loss on given log-probs (f32: its CPU kernel has no f64) -> (cost, d cost / d log-probs)"""
    import torchaudio.functional as F
    x = torch.tensor(lp[None], dtype=torch.float32, requires_grad=True)
    c = F.rnnt_loss(x, torch.tensor(np.asarray(y)[None], dtype=torch.int32), torch.tensor([T], dtype=torch.int32),
                    torch.tensor([U], dtype=torch.int32), blank=0, reduction="none", fused_log_softmax=False)
    c.sum().backward()
    return float(c.detach()[0]), x.grad[0].double().numpy()


@pytest.mark.parametrize("lam_d", [0.0, 0.01, 0.3, 2.0])
@pytest.mark.parametrize("T,U,V", [(7, 4, 9), (1, 0, 5), (5, 0, 6), (3, 5, 7)])
def test_delay_cost_matches_torchaudio_and_brute_force(T, U, V, lam_d):
    logits, y = _case(T * 100 + U, T, U, V)
    c, _ = E.dense_loss(logits, y, 0.0, lam_d)
    lp = _penalised_log_probs(logits, y, lam_d)
    ref, _ = _torchaudio(lp, y, T, U)
    assert abs(c - ref) <= 2e-5 * max(1.0, abs(c)), (c, ref)
    if T + U <= 10:
        assert abs(c - rnnt_brute_force(lp, y, T, U)) <= 1e-10 * max(1.0, abs(c))
    if U == 0:                           # no label arcs: the penalty has nothing to act on
        assert c == E.dense_loss(logits, y)[0]


@pytest.mark.parametrize("lam_d", [0.05, 1.0])
def test_delay_gradient_matches_central_differences(lam_d):
    T, U, V = 5, 3, 6
    logits, y = _case(7, T, U, V)
    _, d = E.dense_loss(logits, y, 0.0, lam_d)
    h = 1e-6
    num = np.zeros_like(logits)
    for idx in np.ndindex(*logits.shape):
        zp, zm = logits.copy(), logits.copy()
        zp[idx] += h
        zm[idx] -= h
        num[idx] = (E.dense_loss(zp, y, 0.0, lam_d)[0] - E.dense_loss(zm, y, 0.0, lam_d)[0]) / (2 * h)
    np.testing.assert_allclose(d, num, atol=1e-7)


@pytest.mark.parametrize("lam_f,lam_d", [(0.0, 0.0), (0.01, 0.0), (0.5, 0.0), (0.01, 0.2), (1.0, 1.0)])
@pytest.mark.parametrize("T,U,V", [(8, 5, 11), (4, 0, 5), (1, 3, 6)])
def test_fastemit_gradient_matches_scaled_torchaudio_gradient(T, U, V, lam_f, lam_d):
    """torchaudio's d cost / d log-probs with the label entries scaled by 1 + lam_f, chained through the log-softmax"""
    logits, y = _case(T + 31 * U, T, U, V)
    c, d = E.dense_loss(logits, y, lam_f, lam_d)
    lp = _penalised_log_probs(logits, y, lam_d)
    ref_c, g = _torchaudio(lp, y, T, U)
    for u in range(U):
        g[:, u, y[u]] *= 1.0 + lam_f
    sm = np.exp(log_softmax(logits))
    ref = g - sm * g.sum(-1, keepdims=True)
    np.testing.assert_allclose(d, ref, atol=1e-5)             # torchaudio runs in f32
    assert abs(c - ref_c) <= 2e-5 * max(1.0, abs(c))
    assert c == E.dense_loss(logits, y, 0.0, lam_d)[0]          # FastEmit does not change the cost


def _mean_and_var_emit_time(logits, y, lam_d):
    """posterior mean and variance of sum_u t_u (t_u = the frame label u is emitted on), by enumeration of every path"""
    import itertools
    lp = _penalised_log_probs(logits, y, lam_d)
    T, U1, _ = lp.shape
    U = U1 - 1
    scores, times = [], []
    for pos in itertools.combinations(range(T + U - 1), U):
        pos, t, u, s, st = set(pos), 0, 0, 0.0, 0
        for i in range(T + U - 1):
            if i in pos:
                s += lp[t, u, y[u]]
                st += t
                u += 1
            else:
                s += lp[t, u, 0]
                t += 1
        scores.append(s + lp[T - 1, U, 0])
        times.append(st)
    w = np.exp(np.array(scores) - np.logaddexp.reduce(scores))
    times = np.array(times, np.float64)
    m = float((w * times).sum())
    return m, float((w * (times - m) ** 2).sum())


def test_posterior_emission_time_falls_with_the_delay_penalty():
    """d/d lam_d E[sum_u t_u] = -Var(sum_u t_u) <= 0; the oracle's label occupancies give the same mean as the enumeration"""
    T, U, V = 6, 3, 5
    logits, y = _case(3, T, U, V)
    lams = [0.0, 0.05, 0.2, 0.5, 1.0, 3.0]
    means = []
    for lam in lams:
        m, var = _mean_and_var_emit_time(logits, y, lam)
        lp = log_softmax(logits)
        _, _, gl, _, _ = E.lattice(lp[:, :, 0], lp[:, np.arange(U), y], T, U, 0.0, lam)
        occ_mean = float((-gl[:, :U] * np.arange(T)[:, None]).sum())
        assert abs(occ_mean - m) < 1e-9
        means.append(m)
        h = 1e-5
        slope = (_mean_and_var_emit_time(logits, y, lam + h)[0] - _mean_and_var_emit_time(logits, y, max(lam - h, 0.0))[0]) / (
            (lam + h) - max(lam - h, 0.0))
        assert abs(slope + var) < 1e-4 * max(1.0, var)
    assert all(b <= a + 1e-12 for a, b in zip(means, means[1:])) and means[-1] < means[0]


def test_pruned_oracle_with_full_windows_is_the_dense_lattice():
    T, U, V, R = 6, 4, 7, 5
    logits, y = _case(9, T, U, V)
    lp = log_softmax(logits)
    lpb, lpl = lp[:, :, 0], lp[:, np.arange(U), y]
    for lam_f, lam_d in ((0.0, 0.0), (0.3, 0.7)):
        c, gb, gl, _, _ = E.lattice(lpb, lpl, T, U, lam_f, lam_d)
        pc, pgb, pgl = E.pruned_loss(lpb, lpl, np.zeros(T, np.int64), R, lam_f, lam_d)
        assert pc == c and np.array_equal(pgb, gb) and np.array_equal(pgl, gl)
    # a tight window: the penalised pruned cost is at least the penalised dense one (fewer paths)
    s = P.prune_bounds_fast(-(gb + gl), T, U, 2)
    assert E.pruned_loss(lpb, lpl, s, 2, 0.0, 0.7)[0] >= E.lattice(lpb, lpl, T, U, 0.0, 0.7)[0] - 1e-12


@pytest.mark.parametrize("lam_l,lam_a", [(0.0, 0.0), (0.25, 0.0), (0.0, 0.1), (0.2, 0.15)])
def test_simple_oracle_at_zero_delay_is_the_existing_oracle(lam_l, lam_a):
    rng = np.random.default_rng(4)
    T, U, V = 7, 4, 9
    am, lm = rng.standard_normal((T, V)) * 2, rng.standard_normal((U + 1, V)) * 2
    y = rng.integers(1, V, U)
    logq = PS.unigram_logq([lm])
    ref = PS.simple_loss(am, lm, y, logq, lam_l, lam_a)
    got = E.simple_loss(am, lm, y, 0.0, logq, lam_l, lam_a)
    assert abs(got[0] - ref[0]) < 1e-10
    for a, b in zip(got[1:], ref[1:]):
        np.testing.assert_allclose(a, b, atol=1e-10)


def test_simple_oracle_gradient_matches_central_differences_with_delay():
    rng = np.random.default_rng(12)
    T, U, V, lam_d = 5, 3, 6, 0.4
    am, lm = rng.standard_normal((T, V)), rng.standard_normal((U + 1, V))
    y = rng.integers(1, V, U)
    _, dam, dlm, _, _ = E.simple_loss(am, lm, y, lam_d)
    h = 1e-6
    for x, d in ((am, dam), (lm, dlm)):
        for idx in np.ndindex(*x.shape):
            x[idx] += h
            cp = E.simple_loss(am, lm, y, lam_d)[0]
            x[idx] -= 2 * h
            cm = E.simple_loss(am, lm, y, lam_d)[0]
            x[idx] += h
            assert abs((cp - cm) / (2 * h) - d[idx]) < 1e-6


def test_cli_flags_default_to_off_and_refuse_bad_values():
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T, train_transducer_mbr_bmuf_otfaug as M
    base = ["transducer", "data.lst", "log", "out"]
    for build in (T.build_parser, M.build_parser):
        a, _ = build().parse_known_args(base)
        assert a.fastemit_lambda == 0.0 and a.delay_penalty == 0.0
        a, _ = build().parse_known_args(base + ["--fastemit_lambda", "0.01", "--delay_penalty", "0.0015"])
        assert a.fastemit_lambda == 0.01 and a.delay_penalty == 0.0015
        T.check_emission_reg_args(build(), a)
    for flag in ("--fastemit_lambda", "--delay_penalty"):
        for bad in ("-0.1", "nan", "inf"):
            p = T.build_parser()
            a, _ = p.parse_known_args(base + [flag, bad])
            with pytest.raises(SystemExit):
                T.check_emission_reg_args(p, a)


def test_engine_and_warp_rnnt_refuse_bad_values():
    from pika_b200 import engine
    from pika_b200.warp_rnnt import RNNTLoss
    assert engine.check_emission_reg(0, 0) == (0.0, 0.0)
    assert engine.check_emission_reg(0.01, 1) == (0.01, 1.0)
    for bad in ((-1e-3, 0.0), (0.0, -1.0), (math.nan, 0.0), (0.0, math.inf)):
        with pytest.raises(ValueError):
            engine.check_emission_reg(*bad)
        with pytest.raises(ValueError):
            RNNTLoss(fastemit_lambda=bad[0], delay_penalty=bad[1])
    loss = RNNTLoss(blank=0, reduction="sum", fastemit_lambda=0.5, delay_penalty=0.25)
    assert (loss.fastemit_lambda, loss.delay_penalty) == (0.5, 0.25)
