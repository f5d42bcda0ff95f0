"""The float64 Adam / BMUF-Adam / block-Adam restatements (tests/adam_oracle.py) against torch.optim.Adam on the CPU and
against the reference formulas of trainer/bmuf.py, including a fractional step count, the inf-norm clip (inactive, active,
NaN) and lengths that are not a multiple of 4."""
import numpy as np
import pytest
import torch

import adam_oracle as ao


def _rand(n, seed, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(n) * scale).astype(np.float32)


@pytest.mark.parametrize("n", [1, 7, 4099])
@pytest.mark.parametrize("clip", [-1.0, 50.0, 0.3])
@pytest.mark.parametrize("frac", [0.0, 2.7])
def test_adam_step_matches_torch_adam(n, clip, frac):
    """three steps; ``frac`` is added to state['step'] after the first one, as a BMUF-Adam sync does (trainer/bmuf.py:311)"""
    lr, betas, eps = 1e-2, (0.9, 0.999), 1e-8
    p0 = _rand(n, 1)
    tp = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adam([tp], lr, betas=betas, eps=eps)
    p, m, v, step = p0.astype(np.float64), np.zeros(n), np.zeros(n), 0.0
    for it in range(3):
        g = _rand(n, 10 + it, 0.5 if it != 1 else 2.0)
        tp.grad = torch.from_numpy(g.copy())
        if clip > 0:
            torch.nn.utils.clip_grad_norm_([tp], clip, norm_type=float("inf"))
        opt.step()
        step = float(np.float32(step + 1))
        p, m, v = ao.adam_step(p, ao.clip_inf(g, clip).astype(np.float64), m, v, lr, betas, eps, step)
        if it == 0 and frac:
            opt.state[tp]["step"] += frac
            step = float(np.float32(np.float32(step) + np.float32(frac)))
        assert float(opt.state[tp]["step"]) == step
        np.testing.assert_allclose(opt.state[tp]["exp_avg"].numpy(), m, rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(opt.state[tp]["exp_avg_sq"].numpy(), v, rtol=1e-5, atol=1e-9)
        np.testing.assert_allclose(tp.detach().numpy(), p, rtol=0, atol=4 * np.spacing(np.float32(np.abs(p).max())))


def test_clip_nan_turns_every_parameter_nan_like_torch():
    g = _rand(9, 3)
    g[4] = np.nan
    tp = torch.nn.Parameter(torch.from_numpy(_rand(9, 4)))
    tp.grad = torch.from_numpy(g.copy())
    torch.nn.utils.clip_grad_norm_([tp], 1.0, norm_type=float("inf"))
    torch.optim.Adam([tp], 1e-3).step()
    p, _, _ = ao.adam_step(_rand(9, 4).astype(np.float64), ao.clip_inf(g, 1.0).astype(np.float64), np.zeros(9), np.zeros(9),
                           1e-3, (0.9, 0.999), 1e-8, 1.0)
    assert bool(torch.isnan(tp).all()) and np.isnan(p).all()


def test_bmuf_adam_sync_restates_the_reference_update():
    """the moment filter of trainer/bmuf.py:283-295 written out in torch, against the oracle, for two consecutive syncs"""
    n, world, bm, blr, tau, betas = 11, 3, 0.9, 1.0, 4, (0.9, 0.999)
    rng = np.random.default_rng(0)
    glob, dprev, m_g, v_g, rho = rng.standard_normal(n), np.zeros(n), np.zeros(n), np.zeros(n), 0.0
    tg, tdp, tm, tv = (torch.from_numpy(x.copy()) for x in (glob, dprev, m_g, v_g))
    trho = 0.0
    for _ in range(2):
        ds, ms, vs = rng.standard_normal(n), rng.standard_normal(n) * 0.1, rng.random(n) * 0.01
        glob, dprev, m_g, v_g, rho = ao.bmuf_adam_sync(glob, dprev, m_g, v_g, ds, ms, vs, world, bm, blr, betas, tau, rho)
        trho = bm * trho + tau
        vec = torch.from_numpy(np.concatenate([ds, ms, vs])) / float(world)
        tdp = bm * tdp + blr * (1 - bm) * vec[:n]
        tg = tg - (1 + bm) * tdp
        b1t, b2t, b1r, b2r = betas[0] ** tau, betas[1] ** tau, betas[0] ** (trho * bm), betas[1] ** (trho * bm)
        tm = (b1t * (b1r - 1) * tm + (1 - b1t * b1r) * vec[n:2 * n]) / (1 - b1t)
        tv = (b2t * (b2r - 1) * tv + (1 - b2t * b2r) * vec[2 * n:]) / (1 - b2t)
        assert rho == trho
        for a, b in ((glob, tg), (dprev, tdp), (m_g, tm), (v_g, tv)):
            np.testing.assert_allclose(a, b.numpy(), rtol=1e-13, atol=1e-15)


def test_block_adam_sync_is_adam_on_the_summed_delta():
    n = 6
    glob = _rand(n, 1).astype(np.float64)
    tp = torch.nn.Parameter(torch.from_numpy(glob.copy()))
    opt = torch.optim.Adam([tp], 0.05, weight_decay=0.0)
    m, v, step = np.zeros(n), np.zeros(n), 0.0
    for it in range(3):
        dsum = _rand(n, 20 + it).astype(np.float64) + _rand(n, 30 + it)
        tp.grad = torch.from_numpy(dsum.copy())
        opt.step()
        glob, m, v, step = ao.block_adam_sync(glob, m, v, step, dsum, 0.05)
        np.testing.assert_allclose(tp.detach().numpy(), glob, rtol=1e-13)
    assert step == 3
