"""The pruned RNN-T loss's simple loss smoothed with LM-only / AM-only terms on the GPU (pk_rnnt_simple_smooth_stats,
pk_rnnt_simple_tables_smooth, pk_rnnt_simple_grad_smooth through engine.simple_loss and engine.transducer_loss_pruned) against the
float64 oracle (tests/pruned_smoothed_oracle.py), in both precision modes."""
import os

import numpy as np
import pytest
import torch

import pruned_rnnt_oracle as P
import pruned_smoothed_oracle as S
from test_pruned_rnnt_gpu import _batch, _nll, _place, _simple_inputs, _small_net

pytestmark = pytest.mark.gpu

PRECS = ["bf16", "fp32"]
SCALES = [(0.25, 0.0), (0.0, 0.2), (0.25, 0.1)]
TOL = dict(bf16=(2e-2, 3e-2), fp32=(1e-4, 2e-4))


@pytest.fixture
def prec(request):
    from pika_b200 import engine
    old = engine.get_precision()
    engine.set_precision(request.param)
    yield request.param
    engine.set_precision(old)


def _lens(*v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def _args(am, lm, V, y, Ts, Us, R):
    """engine.simple_loss's positional arguments up to R"""
    B, T, ldv = am.shape
    U1 = lm.shape[1]
    return (torch.from_numpy(am).cuda().view(B * T, ldv), torch.from_numpy(lm).cuda().view(B * U1, ldv), V, B, T, U1,
            torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us), R)


@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("lam_l,lam_a", SCALES)
@pytest.mark.parametrize("V,spike", [(60, None), (61, None), (6000, None), (60, 120.0)])
def test_smoothed_simple_loss_against_oracle(prec, lam_l, lam_a, V, spike):
    from pika_b200 import engine
    rng = np.random.default_rng(V + int(100 * lam_l) + int(10 * lam_a))
    Ts, Us, R = (7, 1, 5), (4, 0, 2), 3
    am, lm, y = _simple_inputs(rng, Ts, Us, V, spike=spike)
    B, T, ldv = am.shape
    U1 = lm.shape[1]
    costs, bounds, dam, dlm = engine.simple_loss(*_args(am, lm, V, y, Ts, Us, R), 0.7, lm_only_scale=lam_l, am_only_scale=lam_a)
    dam = dam.float().view(B, T, ldv).cpu().numpy()
    dlm = dlm.float().view(B, U1, ldv).cpu().numpy()
    bounds = bounds.cpu().numpy()
    assert np.isfinite(dam).all() and np.isfinite(dlm).all() and bool(torch.isfinite(costs).all())
    _, ref = S.batch_simple_loss([am[b, :Tb, :V] for b, Tb in enumerate(Ts)], [lm[b, :Ub + 1, :V] for b, Ub in enumerate(Us)],
                                 [y[b, :Ub] for b, Ub in enumerate(Us)], lam_l, lam_a)
    tol = TOL[prec]
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        c, da, dl, _, _ = ref[b]
        assert abs(float(costs[b]) - c) <= tol[0] * max(1.0, abs(c)), (b, float(costs[b]), c)
        np.testing.assert_allclose(dam[b, :Tb, :V], 0.7 * da, atol=tol[1])
        np.testing.assert_allclose(dlm[b, :Ub + 1, :V], 0.7 * dl, atol=tol[1])
        assert not dam[b, Tb:].any() and not dam[b, :, V:].any() and not dlm[b, :, V:].any() and not dlm[b, Ub + 1:].any()
        P.check_bounds_properties(bounds[b], Tb, Ub, R)


def test_smooth_stats_against_float64_and_padding_never_enters_a_sum():
    from pika_b200 import engine, kernels as K
    rng = np.random.default_rng(6000)
    Ts, Us, V = (9, 3, 6), (5, 0, 7), 6000
    B, T, U1 = len(Ts), max(Ts), max(Us) + 1
    ldv = engine._ldv(V)
    am = np.zeros((B, T, ldv), np.float32)
    lm = np.zeros((B, U1, ldv), np.float32)
    am[:, :, :V] = rng.standard_normal((B, T, V)) * 3
    lm[:, :, :V] = rng.standard_normal((B, U1, V)) * 3

    def stats(am, lm):
        a, l = torch.from_numpy(am).cuda().view(B * T, ldv), torch.from_numpy(lm).cuda().view(B * U1, ldv)
        E = torch.empty(B * T, ldv, dtype=torch.bfloat16, device="cuda")
        Pm = torch.empty(B * U1, ldv, dtype=torch.bfloat16, device="cuda")
        am_max = K.rnnt_simple_prep(a, V, B, T, T, E)
        lm_max = K.rnnt_simple_prep(l, V, B, U1, U1, Pm)
        return [x.cpu().numpy() for x in K.rnnt_simple_smooth_stats(a, l, V, am_max, lm_max, _lens(*Ts), _lens(*Us), B, T, U1)]
    Nl, logq, Na = stats(am, lm)
    Nl, Na = Nl.reshape(B, U1), Na.reshape(B, T)
    ref_q = S.unigram_logq([lm[b, :Ub + 1, :V] for b, Ub in enumerate(Us)])
    np.testing.assert_allclose(logq[:V], ref_q, rtol=0, atol=2e-5)
    assert not logq[V:].any()
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        np.testing.assert_allclose(Nl[b, :Ub + 1], S._lse(lm[b, :Ub + 1, :V].astype(np.float64)), rtol=2e-6)
        np.testing.assert_allclose(Na[b, :Tb], S._lse(am[b, :Tb, :V].astype(np.float64) + ref_q[None]), rtol=2e-6)
        assert not Nl[b, Ub + 1:].any() and not Na[b, Tb:].any()
    # other values in the padded rows and frames (and large ones in the padding columns) change nothing
    am2, lm2 = am.copy(), lm.copy()
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        am2[b, Tb:, :V] = 50.0 + rng.standard_normal((T - Tb, V))
        lm2[b, Ub + 1:, :V] = 50.0 + rng.standard_normal((U1 - Ub - 1, V))
    am2[:, :, V:] = 1e4
    lm2[:, :, V:] = 1e4
    Nl2, logq2, Na2 = stats(am2, lm2)
    assert np.array_equal(logq2, logq)
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        assert np.array_equal(Nl2.reshape(B, U1)[b, :Ub + 1], Nl[b, :Ub + 1])
        assert np.array_equal(Na2.reshape(B, T)[b, :Tb], Na[b, :Tb])


@pytest.mark.parametrize("prec", PRECS, indirect=True)
def test_smoothed_simple_loss_is_deterministic(prec):
    from pika_b200 import engine
    rng = np.random.default_rng(5)
    Ts, Us, V, R = (9, 4, 7), (6, 0, 3), 6000, 3
    am, lm, y = _simple_inputs(rng, Ts, Us, V)
    a = _args(am, lm, V, y, Ts, Us, R)
    r1 = engine.simple_loss(*a, 1.0, lm_only_scale=0.25, am_only_scale=0.1)
    r2 = engine.simple_loss(*a, 1.0, lm_only_scale=0.25, am_only_scale=0.1)
    for x, z in zip(r1, r2):
        assert torch.equal(x, z)


@pytest.mark.parametrize("prec", PRECS, indirect=True)
def test_zero_scales_are_bit_equal_to_the_unsmoothed_call(prec):
    """transducer_loss_pruned with both scales 0 runs the same launches and gives the same costs and the same gradients of the
    parameters its two loss Functions form, bit for bit"""
    from pika_b200 import _lib, engine
    V, R, Ts, Us = 60, 3, (9, 6), (7, 4)
    x, y, fl, ll = _batch(V, Ts, Us)
    engine.set_dropout_enabled(False)
    try:
        m = _small_net("rnn", "rnn", V, R)
        res = []
        for kw in ({}, {}, dict(lm_only_scale=0.0, am_only_scale=0.0)):          # the first call also stages the weights: not counted
            m.zero_grad(set_to_none=True)
            n0 = _lib.launch_count()
            simple, pruned = engine.transducer_loss_pruned(m, x, y, fl, ll, R, 0.5, 1.0, x_len=fl, **kw)
            (0.5 * simple + pruned).sum().backward()
            torch.cuda.synchronize()
            res.append((_lib.launch_count() - n0, simple, pruned, {k: p.grad.clone() for k, p in m.named_parameters()
                                                                    if k.startswith(("fc1", "fc_gate", "fc2", "simple_"))}))
    finally:
        engine.set_dropout_enabled(True)
    (n1, s1, p1, g1), (n2, s2, p2, g2) = res[1:]
    assert n1 == n2 and torch.equal(s1, s2) and torch.equal(p1, p2)
    assert g1.keys() == g2.keys() and all(torch.equal(g1[k], g2[k]) for k in g1)


@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("decoder_type", ["rnn", "transformer"])
@pytest.mark.parametrize("V", [61, 64, 520])
def test_smoothed_pruned_step_gradients_match_float64_restatement(V, prec, decoder_type):
    """one step of transducer_loss_pruned (sigma_s = 0.5, sigma_p = 1, lam_l = 0.25, lam_a = 0.1) against float64 torch given the same
    encoder / prediction-net outputs and the GPU's bounds, the unigram q held constant: joint, fc2 and simple-projection gradients"""
    from pika_b200 import engine
    R, lam_l, lam_a = 3, 0.25, 0.1
    Ts, Us = (9, 6), (7, 4)
    x, y, fl, ll = _batch(V, Ts, Us)
    engine.set_dropout_enabled(False)
    try:
        m = _small_net("rnn", decoder_type, V, R)
        simple, pruned = engine.transducer_loss_pruned(m, x, y, fl, ll, R, 0.5, 1.0, x_len=fl, lm_only_scale=lam_l, am_only_scale=lam_a)
        (0.5 * simple + pruned).sum().backward()
        with torch.no_grad():
            enc = engine.model_encoder_forward_act(m, x, fl).double()
            pred = engine.prednet_forward_act(m, y).double()
            _, bounds = engine.SimpleLossFn.apply(enc.to(engine.act_dtype()), pred.to(engine.act_dtype()), m, y.int(), fl, ll, R, 0.5,
                                                  False, lam_l, lam_a)
    finally:
        engine.set_dropout_enabled(True)
    ps = {k: p.detach().double().requires_grad_(True) for k, p in m.named_parameters() if k.startswith(("fc1", "fc_gate", "fc2", "simple_"))}
    B, T, H = enc.shape
    U1 = pred.shape[1]
    lin = lambda v, n: v @ ps[n + ".weight"].t() + ps[n + ".bias"]                  # noqa: E731
    ex1, exg = enc @ ps["fc1.weight"][:, :H].t() + ps["fc1.bias"], enc @ ps["fc_gate.weight"][:, :H].t() + ps["fc_gate.bias"]
    py1, pyg = pred @ ps["fc1.weight"][:, H:].t(), pred @ ps["fc_gate.weight"][:, H:].t()
    s = bounds.long()
    u = (s[:, :, None] + torch.arange(R, device="cuda")).clamp(max=U1 - 1)
    bi = torch.arange(B, device="cuda")[:, None, None]
    h = torch.tanh(ex1[:, :, None] + py1[bi, u]) * torch.sigmoid(exg[:, :, None] + pyg[bi, u])
    lp = torch.log_softmax(lin(h, "fc2"), -1)                                        # [B, T, R, V]
    am, lm = lin(enc, "simple_am_proj"), lin(pred, "simple_lm_proj")
    valid = torch.cat([lm[b, :Us[b] + 1] for b in range(B)])
    logq = torch.log(torch.softmax(valid, -1).mean(0) + S.Q_EPS).detach()           # a constant of the step
    mu = 1.0 - lam_l - lam_a
    total = 0.0
    for b in range(B):
        Tb, Ub = Ts[b], Us[b]
        yb = y[b, :Ub]
        lsz = torch.log_softmax(am[b, :Tb, None] + lm[b, None, :Ub + 1], -1)        # [Tb, Ub+1, V]
        llm = torch.log_softmax(lm[b, :Ub + 1], -1)                                  # [Ub+1, V]
        lam_ = torch.log_softmax(am[b, :Tb] + logq, -1)                              # [Tb, V]
        ar = torch.arange(Ub, device="cuda")
        sb = mu * lsz[:, :, 0] + lam_l * llm[None, :, 0] + lam_a * lam_[:, None, 0]
        sl = mu * lsz[:, ar, yb] + lam_l * llm[ar, yb][None, :] + lam_a * lam_[:, yb]
        total = total + 0.5 * _nll(sb, sl, Tb, Ub)
        pb = torch.full((Tb, Ub + 1), -1e30, dtype=torch.float64, device="cuda")
        pl = torch.full((Tb, max(Ub, 1)), -1e30, dtype=torch.float64, device="cuda")
        rows_b, rows_l = [], []
        for t in range(Tb):
            for r in range(R):
                uu = int(s[b, t]) + r
                if uu <= Ub:
                    rows_b.append((t, uu, lp[b, t, r, 0]))
                    if uu < Ub:
                        rows_l.append((t, uu, lp[b, t, r, yb[uu]]))
        total = total + _nll(_place(pb, rows_b), _place(pl, rows_l)[:, :Ub], Tb, Ub)
    total.backward()
    tol = 6e-2 if prec == "bf16" else 2e-3
    for k, p in ps.items():
        g = m.get_parameter(k).grad.double()
        err = float((g - p.grad).norm() / p.grad.norm().clamp(min=1e-12))
        assert err < tol, (k, err)


def test_train_cli_pruned_smoothed(tmp_path):
    """the trainer with --prune_range 4 --lm_only_scale 0.25 --am_only_scale 0.1 logs a finite Loss and Simple every epoch"""
    from test_loader_cpu import make_dataset
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    lst, utts = make_dataset(tmp_path, n_utts=8, shards=1, n_lo=14000, n_hi=22000)
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--window-type=hamming\n--sample-frequency=16000\n--dither=1\n--low-freq=40\n--high-freq=-200\n--num-mel-bins=80\n")
    out = tmp_path / "out"
    out.mkdir()
    log = tmp_path / "log.WORKER-ID"
    argv = ["transducer", lst, str(log), str(out), "--cuda", "--local_rank", "0", "--encoder_type", "transformer",
            "--decoder_type", "rnn", "--rnn_size", "1024", "--embd_dim", "100", "--output_dim", "60", "--padding_idx", "60", "--padding_tgt", "60",
            "--dec_layers", "2", "--dropout", "0.0", "--brnn", "--model_lctx", "21", "--model_rctx", "21", "--model_stride", "4",
            "--lctx", "1", "--rctx", "1", "--feats_dim", "80", "--feat_config", str(cfg), "--cmn", "--batch_size", "4",
            "--num_workers", "1", "--batch_first", "--max_len", "1600", "--TU_limit", "50000", "--gain_range", "25,25", "--speed_rate", "1.0",
            "--grad_clip", "3.0", "--initial_lr", "0.002", "--final_lr", "0.001", "--momentum", "0.9", "--num_epochs", "3",
            "--num_batches_per_epoch", "2", "--sync_period", "1", "--block_momentum", "0.9", "--block_lr", "1.0", "--seed", "777",
            "--prune_range", "4", "--lm_only_scale", "0.25", "--am_only_scale", "0.1"]
    os.environ.setdefault("WORLD_SIZE", "1")
    T.main(argv)
    text = open(str(log).replace("WORKER-ID", "0")).read()
    assert "Training Finished" in text
    lines = [l for l in text.splitlines() if "Overall Avg Loss" in l]
    losses = [float(l.split("Loss:")[1].split()[0]) for l in lines]
    simple = [float(l.split("Simple:")[1].split()[0]) for l in lines]
    print("pruned losses per epoch", losses, "smoothed simple", simple)
    assert len(losses) == 3 and np.isfinite(losses).all() and np.isfinite(simple).all() and min(simple) > 0
