"""The pruned RNN-T loss's float64 oracle (tests/pruned_rnnt_oracle.py) against oracle/rnnt.py, the pruning bounds' guarantees, and the
model / trainer surface of the feature, without a GPU."""
import types

import numpy as np
import pytest
import torch

import pruned_rnnt_oracle as P
from oracle import rnnt as orc


def _utt(rng, T, U, V, scale=1.0):
    am = rng.standard_normal((T, V)) * scale
    lm = rng.standard_normal((U + 1, V)) * scale
    y = rng.integers(1, V, U)
    return am, lm, y


@pytest.mark.parametrize("T,U,V", [(1, 0, 7), (1, 3, 9), (5, 0, 11), (6, 4, 13), (9, 7, 31)])
def test_simple_cost_is_dense_rnnt_of_am_plus_lm(T, U, V):
    rng = np.random.default_rng(T * 100 + U)
    am, lm, y = _utt(rng, T, U, V, scale=2.0)
    cost, dam, dlm, _, _ = P.simple_loss(am, lm, y)
    z = am[:, None, :] + lm[None, :, :]
    ref, g = orc.rnnt_loss(orc.log_softmax(z)[None], y[None], [T], [U])
    assert abs(cost - ref[0]) < 1e-10
    # the gradient identity: d/dz of the dense loss summed over u (am) and over t (lm)
    _, dz = orc.rnnt_loss_from_logits(z[None], y[None], [T], [U])
    np.testing.assert_allclose(dam, dz[0].sum(1), atol=1e-10)
    np.testing.assert_allclose(dlm, dz[0].sum(0), atol=1e-10)


def test_simple_loss_gradient_matches_finite_differences():
    rng = np.random.default_rng(3)
    am, lm, y = _utt(rng, 4, 3, 6)
    _, dam, dlm, _, _ = P.simple_loss(am, lm, y)
    eps = 1e-6
    for (arr, d) in ((am, dam), (lm, dlm)):
        for idx in [(0, 0), (1, int(y[0])), (2, 3)]:
            a = arr.copy()
            arr[idx] += eps
            cp = P.simple_loss(am, lm, y)[0]
            arr[idx] -= 2 * eps
            cm = P.simple_loss(am, lm, y)[0]
            arr[:] = a
            assert abs((cp - cm) / (2 * eps) - d[idx]) < 1e-6


def test_simple_loss_floor_keeps_everything_finite():
    am = np.array([[0.0, 120.0, 0.0], [0.0, 120.0, 0.0]])
    lm = np.array([[0.0, 0.0, 120.0], [0.0, 0.0, 120.0]])
    cost, dam, dlm, _, _ = P.simple_loss(am, lm, np.array([2]))
    assert np.isfinite(cost) and np.isfinite(dam).all() and np.isfinite(dlm).all()


@pytest.mark.parametrize("T,U,R", [(6, 3, 4), (7, 5, 6), (3, 2, 3), (1, 0, 2), (4, 0, 5)])
def test_pruned_cost_with_full_windows_is_dense(T, U, R):
    rng = np.random.default_rng(T + 10 * U)
    am, lm, y = _utt(rng, T, U, 9)
    lp = orc.log_softmax(rng.standard_normal((T, U + 1, 9)))
    lpb = lp[:, :, 0]
    lpl = lp[:, np.arange(U), y] if U else np.zeros((T, 0))
    dense = orc.rnnt_loss(lp[None], y[None], [T], [U])[0][0]
    assert R >= U + 1
    cost = P.pruned_cost(lpb, lpl, np.zeros(T, np.int64), R)[0]
    assert abs(cost - dense) < 1e-10


@pytest.mark.parametrize("seed", range(6))
def test_pruned_cost_is_an_upper_bound_and_brute_force_agrees(seed):
    rng = np.random.default_rng(seed)
    T, U, R = int(rng.integers(2, 5)), int(rng.integers(1, 4)), int(rng.integers(2, 4))
    if U > T * (R - 1):
        U = T * (R - 1)
    V = 6
    y = rng.integers(1, V, U)
    lp = orc.log_softmax(rng.standard_normal((T, U + 1, V)))
    lpb, lpl = lp[:, :, 0], lp[:, np.arange(U), y]
    gamma = rng.random((T, U + 1)).astype(np.float32)
    s = P.prune_bounds(gamma, T, U, R)
    P.check_bounds_properties(s, T, U, R)
    cost = P.pruned_cost(lpb, lpl, s, R)[0]
    dense = orc.rnnt_loss(lp[None], y[None], [T], [U])[0][0]
    assert np.isfinite(cost) and cost >= dense - 1e-12
    m = P.window_mask(s, T, U, R)
    lpm = lp.copy()
    lpm[:, :, 0] = np.where(m, lpb, -np.inf)
    for u in range(U):
        lpm[:, u, y[u]] = np.where(m[:, u], lpl[:, u], -np.inf)
    assert abs(orc.rnnt_brute_force(lpm, y, T, U) - cost) < 1e-10


def _adversarial(T, U, R, kind, rng):
    g = np.zeros((T, U + 1), np.float32)
    if kind == "onehot_end":
        g[:, U] = 1.0
    elif kind == "ties":
        g[:] = 0.5
    elif kind == "onehot_start":
        g[:, 0] = 1.0
    elif kind == "zigzag":
        for t in range(T):
            g[t, (t * 7) % (U + 1)] = 1.0
    else:
        g[:] = rng.random((T, U + 1)).astype(np.float32)
    return g


@pytest.mark.parametrize("kind", ["onehot_end", "ties", "onehot_start", "zigzag", "random"])
@pytest.mark.parametrize("T,U,R", [(8, 5, 3), (5, 0, 4), (4, 12, 4), (1, 0, 2), (1, 3, 4), (12, 30, 5), (20, 7, 32), (6, 6, 2)])
def test_bounds_properties(kind, T, U, R):
    g = _adversarial(T, U, R, kind, np.random.default_rng(T * U + R))
    s = P.prune_bounds(g, T, U, R)
    P.check_bounds_properties(s, T, U, R)


def test_bounds_exact_fit_follows_the_only_path():
    T, R = 5, 3
    U = T * (R - 1)
    s = P.prune_bounds(np.zeros((T, U + 1), np.float32), T, U, R)
    np.testing.assert_array_equal(s, [0, 2, 4, 6, 8])


def test_bounds_refuse_infeasible():
    with pytest.raises(ValueError):
        P.prune_bounds(np.zeros((3, 8), np.float32), 3, 7, 3)


def test_engine_refuses_infeasible_utterance_by_name():
    from pika_b200 import engine
    with pytest.raises(ValueError, match=r"\[1\]"):
        engine.check_prune_feasible(torch.tensor([5, 3, 4]), torch.tensor([4, 7, 6]), 3)
    engine.check_prune_feasible(torch.tensor([5, 3, 4]), torch.tensor([8, 6, 8]), 3)
    with pytest.raises(ValueError):
        engine.check_prune_feasible(torch.tensor([5]), torch.tensor([1]), 1)


@pytest.mark.parametrize("encoder_type,decoder_type", [("transformer", "rnn"), ("rnn", "transformer")])
def test_seeded_net_keeps_the_reference_weights(encoder_type, decoder_type):
    from pika_b200.model.transducer import Net

    def build(prune_range):
        torch.manual_seed(777)
        o = types.SimpleNamespace(rnn_size=256, local_rank=0, decoder_type=decoder_type, brnn=True, encoder_type=encoder_type, embd_dim=64,
                                  padding_idx=30, dropout=0.0, dec_layers=1, enc_layers=2, prune_range=prune_range)
        return Net(o, 80, 30)
    dense, pruned = build(0).state_dict(), build(4).state_dict()
    extra = set(pruned) - set(dense)
    assert extra == {"simple_am_proj.weight", "simple_am_proj.bias", "simple_lm_proj.weight", "simple_lm_proj.bias"}
    assert set(dense) <= set(pruned)
    for k, v in dense.items():
        assert torch.equal(v, pruned[k]), k
    assert pruned["simple_am_proj.weight"].shape == (30, 256)


def test_loss_scales_warmup():
    from pika_b200.trainer.step import prune_loss_scales
    a = types.SimpleNamespace(prune_warmup_batches=0, simple_loss_scale=0.5)
    assert prune_loss_scales(a, 0) == (0.5, 1.0)
    a.prune_warmup_batches = 4
    assert prune_loss_scales(a, 0) == (1.0, pytest.approx(0.1))
    assert prune_loss_scales(a, 2) == (0.75, pytest.approx(0.55))
    assert prune_loss_scales(a, 9) == (0.5, 1.0)


def test_trainer_flags():
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    a = T.build_parser().parse_known_args(["transducer", "d", "l", "o"])[0]
    assert (a.prune_range, a.simple_loss_scale, a.prune_warmup_batches) == (0, 0.5, 0)


@pytest.mark.parametrize("T,U,windows", [(1, 0, None), (1, 4, None), (6, 0, None), (9, 7, None), (13, 11, 3), (17, 5, 2), (8, 7, 1)])
def test_diagonal_lattice_equals_the_node_loop(T, U, windows):
    """alpha_beta_diag (numpy over anti-diagonals) against oracle.rnnt.rnnt_alpha_beta (a loop over nodes), on random tables and on
    tables that are -inf outside R-wide windows (R = 1: every node off the windows, so no path and an all -inf beta)"""
    rng = np.random.default_rng(T * 31 + U)
    lpb = rng.standard_normal((T, U + 1)) * 3 - 2
    lpl = rng.standard_normal((T, U)) * 3 - 2
    if windows is not None:
        R = windows
        s = np.minimum(np.arange(T) * max(R - 1, 1) // 2, max(U - R + 1, 0))
        m = P.window_mask(s, T, U, R)
        lpb = np.where(m, lpb, -np.inf)
        lpl = np.where(m[:, :U], lpl, -np.inf)
    a0, b0 = orc.rnnt_alpha_beta(lpb, lpl, T, U)
    a1, b1 = P.alpha_beta_diag(lpb, lpl, T, U)
    for x, y in ((a0, a1), (b0, b1)):
        assert np.array_equal(np.isneginf(x), np.isneginf(y))
        f = np.isfinite(x)
        np.testing.assert_allclose(y[f], x[f], rtol=1e-12, atol=1e-12)
    c0, gb0, gl0 = P.occupancy(lpb, lpl, T, U)
    c1, gb1, gl1 = P.occupancy(lpb, lpl, T, U, fast=True)
    assert c0 == c1 or abs(c0 - c1) < 1e-11 * max(1.0, abs(c0))
    np.testing.assert_allclose(gb1, gb0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(gl1, gl0, rtol=0, atol=1e-12)


@pytest.mark.parametrize("T,U,R", [(1, 0, 2), (7, 0, 3), (9, 12, 3), (12, 11, 2), (20, 17, 5), (6, 3, 9), (30, 60, 4)])
def test_vectorised_bounds_equal_the_scalar_oracle(T, U, R):
    rng = np.random.default_rng(T + 7 * U + R)
    for g in (rng.random((T, U + 1)).astype(np.float32), np.full((T, U + 1), 0.25, np.float32),
              (rng.random((T, U + 1)) < 0.2).astype(np.float32)):
        if U > T * (R - 1):
            with pytest.raises(ValueError):
                P.prune_bounds_fast(g, T, U, R)
            continue
        np.testing.assert_array_equal(P.prune_bounds_fast(g, T, U, R), P.prune_bounds(g, T, U, R))
