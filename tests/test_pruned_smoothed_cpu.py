"""The smoothed simple loss's float64 oracle (tests/pruned_smoothed_oracle.py) against the unsmoothed oracle, torch float64 autograd,
finite differences and brute force, and the trainers' smoothing flags, without a GPU."""
import numpy as np
import pytest
import torch

import pruned_rnnt_oracle as P
import pruned_smoothed_oracle as S
from oracle import rnnt as orc

SCALES = [(0.25, 0.0), (0.0, 0.2), (0.25, 0.1)]


def _batch(rng, Ts, Us, V, spread=2.0):
    ams = [rng.standard_normal((T, V)) * spread for T in Ts]
    lms = [rng.standard_normal((U + 1, V)) * spread for U in Us]
    ys = [rng.integers(1, V, U) for U in Us]
    return ams, lms, ys


def test_zero_scales_are_the_unsmoothed_oracle_exactly():
    rng = np.random.default_rng(0)
    ams, lms, ys = _batch(rng, (6, 1, 4), (3, 0, 4), 11)
    logq, res = S.batch_simple_loss(ams, lms, ys, 0.0, 0.0)
    for (a, l, y), got in zip(zip(ams, lms, ys), res):
        for g, r in zip(got, P.simple_loss(a, l, y)):
            assert np.array_equal(np.asarray(g), np.asarray(r))


def test_unigram_is_the_mean_softmax_over_valid_rows():
    rng = np.random.default_rng(1)
    lms = [rng.standard_normal((U + 1, 9)) for U in (3, 0, 2)]
    q = np.exp(S.unigram_logq(lms))
    rows = np.concatenate(lms)
    ref = (np.exp(rows) / np.exp(rows).sum(1, keepdims=True)).mean(0) + 1e-10
    np.testing.assert_allclose(q, ref, rtol=1e-12)
    assert abs(q.sum() - 1.0 - 9e-10) < 1e-12


def _nll(lpb, lpl, T, U):
    alpha = [[None] * (U + 1) for _ in range(T)]
    for t in range(T):
        for u in range(U + 1):
            if t == 0 and u == 0:
                alpha[t][u] = lpb.new_zeros(())
                continue
            terms = []
            if t > 0:
                terms.append(alpha[t - 1][u] + lpb[t - 1, u])
            if u > 0:
                terms.append(alpha[t][u - 1] + lpl[t, u - 1])
            alpha[t][u] = torch.logsumexp(torch.stack(terms), 0)
    return -(alpha[T - 1][U] + lpb[T - 1, U])


def _torch_cost(am, lm, y, logq, lam_l, lam_a):
    """the definition in float64 torch: N with the 2^-100 floor and detached row maxes (a clamped node's normaliser is constant)"""
    T, U = am.shape[0], len(y)
    ma, ml = am.max(1).values.detach(), lm.max(1).values.detach()
    Sm = torch.exp(am - ma[:, None]) @ torch.exp(lm - ml[:, None]).t()
    N = torch.log(torch.clamp(Sm, min=P.FLOOR)) + ma[:, None] + ml[None, :]
    Nl, Na = torch.logsumexp(lm, 1), torch.logsumexp(am + logq[None, :], 1)
    mu = 1.0 - lam_l - lam_a
    yy = torch.as_tensor(y, dtype=torch.long)
    lpb = mu * (am[:, None, 0] + lm[None, :, 0] - N) + lam_l * (lm[None, :, 0] - Nl[None, :]) + lam_a * (am[:, None, 0] + logq[0] - Na[:, None])
    ar = torch.arange(U)
    lpl = (mu * (am[:, yy] + lm[ar, yy][None, :] - N[:, :U]) + lam_l * (lm[ar, yy] - Nl[:U])[None, :]
           + lam_a * (am[:, yy] + logq[yy][None, :] - Na[:, None]))
    return _nll(lpb, lpl, T, U)


@pytest.mark.parametrize("lam_l,lam_a", SCALES)
def test_oracle_gradients_match_torch_autograd_with_q_detached(lam_l, lam_a):
    rng = np.random.default_rng(int(lam_l * 100 + lam_a * 10))
    ams, lms, ys = _batch(rng, (5, 3, 1), (3, 2, 0), 8)
    lm_t = [torch.tensor(l, requires_grad=True) for l in lms]
    rows = torch.cat(lm_t)
    logq_t = torch.log(torch.softmax(rows, 1).mean(0) + S.Q_EPS).detach()
    logq, res = S.batch_simple_loss(ams, lms, ys, lam_l, lam_a)
    np.testing.assert_allclose(logq_t.numpy(), logq, rtol=0, atol=1e-13)
    for b, (a, y) in enumerate(zip(ams, ys)):
        am_t = torch.tensor(a, requires_grad=True)
        cost = _torch_cost(am_t, lm_t[b], y, logq_t, lam_l, lam_a)
        cost.backward()
        c, dam, dlm, _, _ = res[b]
        assert abs(float(cost.detach()) - c) < 1e-10
        np.testing.assert_allclose(dam, am_t.grad.numpy(), atol=1e-10)
        np.testing.assert_allclose(dlm, lm_t[b].grad.numpy(), atol=1e-10)


@pytest.mark.parametrize("lam_l,lam_a", SCALES)
def test_oracle_gradients_match_finite_differences_with_q_fixed(lam_l, lam_a):
    rng = np.random.default_rng(7)
    ams, lms, ys = _batch(rng, (4, 3), (3, 1), 6, spread=1.0)
    logq, res = S.batch_simple_loss(ams, lms, ys, lam_l, lam_a)
    am, lm, y = ams[0], lms[0], ys[0]
    _, dam, dlm, _, _ = res[0]
    eps = 1e-6
    for arr, d in ((am, dam), (lm, dlm)):
        for idx in [(0, 0), (1, int(y[0])), (2, 3), (3, 5)]:
            keep = arr[idx]
            arr[idx] = keep + eps
            cp = S.simple_loss(am, lm, y, logq, lam_l, lam_a)[0]
            arr[idx] = keep - eps
            cm = S.simple_loss(am, lm, y, logq, lam_l, lam_a)[0]
            arr[idx] = keep
            assert abs((cp - cm) / (2 * eps) - d[idx]) < 1e-6, (idx, (cp - cm) / (2 * eps), d[idx])


@pytest.mark.parametrize("T,U", [(1, 0), (2, 1), (3, 2), (4, 3), (2, 4)])
@pytest.mark.parametrize("lam_l,lam_a", SCALES)
def test_oracle_cost_is_the_brute_force_sum_over_alignments(T, U, lam_l, lam_a):
    rng = np.random.default_rng(T * 10 + U)
    ams, lms, ys = _batch(rng, (T, 3), (U, 2), 7)
    logq, res = S.batch_simple_loss(ams, lms, ys, lam_l, lam_a)
    lpb, lpl, _, _, _, _ = S.smoothed_tables(ams[0], lms[0], ys[0], logq, lam_l, lam_a)
    lp = np.full((T, U + 1, 7), np.nan)
    lp[:, :, 0] = lpb
    for u in range(U):
        lp[:, u, ys[0][u]] = lpl[:, u]
    assert abs(orc.rnnt_brute_force(lp, ys[0], T, U) - res[0][0]) < 1e-10


def test_smoothed_oracle_stays_finite_at_the_floor():
    am = np.array([[0.0, 120.0, 0.0], [0.0, 120.0, 0.0]])
    lm = np.array([[0.0, 0.0, 120.0], [0.0, 0.0, 120.0]])
    logq, res = S.batch_simple_loss([am], [lm], [np.array([2])], 0.25, 0.1)
    c, dam, dlm, _, _ = res[0]
    assert np.isfinite(c) and np.isfinite(dam).all() and np.isfinite(dlm).all() and np.isfinite(logq).all()


def test_engine_refuses_out_of_range_scales():
    from pika_b200 import engine
    for bad in [(-0.1, 0.0), (0.0, -1e-3), (0.6, 0.4), (1.0, 0.0), (float("nan"), 0.0), (0.0, float("inf"))]:
        with pytest.raises(ValueError):
            engine.check_smoothing_scales(*bad)
    assert engine.check_smoothing_scales(0.25, 0.1) == (0.25, 0.1)
    # transducer_loss_pruned checks the scales before it touches the model or the lengths
    with pytest.raises(ValueError, match="lm_only_scale"):
        engine.transducer_loss_pruned(None, None, None, None, None, 4, 0.5, 1.0, lm_only_scale=0.7, am_only_scale=0.3)


def _argv(tmp_path, *extra):
    return ["transducer", str(tmp_path / "data.lst"), str(tmp_path / "log"), str(tmp_path), *extra]


@pytest.mark.parametrize("extra,msg", [
    (["--lm_only_scale", "0.25"], "need --prune_range"),
    (["--am_only_scale", "0.1"], "need --prune_range"),
    (["--prune_range", "4", "--lm_only_scale", "-0.1"], "sum < 1"),
    (["--prune_range", "4", "--lm_only_scale", "0.5", "--am_only_scale", "0.5"], "sum < 1"),
    (["--prune_range", "4", "--am_only_scale", "nan"], "sum < 1"),
])
def test_trainer_refuses_bad_smoothing_flags(tmp_path, capsys, extra, msg):
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    with pytest.raises(SystemExit) as e:
        T.main(_argv(tmp_path, *extra))
    assert e.value.code == 2 and msg in capsys.readouterr().err


def test_trainer_smoothing_flags_default_to_off():
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    from pika_b200.trainer.step import smoothing_scales
    a = T.build_parser().parse_known_args(["transducer", "d", "l", "o"])[0]
    assert (a.lm_only_scale, a.am_only_scale) == (0.0, 0.0)
    assert smoothing_scales(a) == dict(lm_only_scale=0.0, am_only_scale=0.0)
    a = T.build_parser().parse_known_args(["transducer", "d", "l", "o", "--prune_range", "4", "--lm_only_scale", "0.25"])[0]
    assert smoothing_scales(a) == dict(lm_only_scale=0.25, am_only_scale=0.0)


@pytest.mark.parametrize("flag", ["--lm_only_scale", "--am_only_scale"])
def test_mbr_trainer_refuses_the_smoothing_flags(tmp_path, capsys, flag):
    from pika_b200.trainer import train_transducer_mbr_bmuf_otfaug as M
    with pytest.raises(SystemExit) as e:
        M.main(_argv(tmp_path, "--prune_range", "4", flag, "0.1"))
    assert e.value.code == 2 and "MBR trainer has no simple loss" in capsys.readouterr().err
