"""Pruned RNN-T loss on the GPU (pk_rnnt_simple_*, pk_rnnt_lattice, pk_rnnt_prune_bounds, pk_joint_gate_pruned_*, pk_rnnt_pruned_loss
and engine.transducer_loss_pruned) against the float64 oracle (tests/pruned_rnnt_oracle.py) and the dense path, in both precision modes."""
import os
import types

import numpy as np
import pytest
import torch

import pruned_rnnt_oracle as P

pytestmark = pytest.mark.gpu

PRECS = ["bf16", "fp32"]


@pytest.fixture
def prec(request):
    from pika_b200 import engine
    old = engine.get_precision()
    engine.set_precision(request.param)
    yield request.param
    engine.set_precision(old)


def _lens(*v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def _simple_inputs(rng, Ts, Us, V, spread=3.0, spike=None):
    from pika_b200 import engine
    B, T, U1 = len(Ts), max(Ts), max(Us) + 1
    ldv = engine._ldv(V)
    am = np.zeros((B, T, ldv), np.float32)
    lm = np.zeros((B, U1, ldv), np.float32)
    am[:, :, :V] = rng.standard_normal((B, T, V)) * spread
    lm[:, :, :V] = rng.standard_normal((B, U1, V)) * spread
    if spike is not None:                    # disjoint 120-nat peaks: E.P underflows on those nodes
        am[0, :, 1] += spike
        lm[0, :, 2] += spike
    y = rng.integers(1, V, (B, max(max(Us), 1))).astype(np.int32)
    return am, lm, y


@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("V,spike", [(60, None), (61, None), (6000, None), (60, 120.0)])
def test_simple_loss_against_oracle(prec, V, spike):
    from pika_b200 import engine
    rng = np.random.default_rng(V)
    Ts, Us = (7, 1, 5), (4, 0, 2)
    am, lm, y = _simple_inputs(rng, Ts, Us, V, spike=spike)
    B, T, ldv = am.shape
    U1 = lm.shape[1]
    costs, _, dam, dlm = engine.simple_loss(torch.from_numpy(am).cuda().view(B * T, ldv), torch.from_numpy(lm).cuda().view(B * U1, ldv), V,
                                            B, T, U1, torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us), 0, 0.7)
    dam = dam.float().view(B, T, ldv).cpu().numpy()
    dlm = dlm.float().view(B, U1, ldv).cpu().numpy()
    assert np.isfinite(dam).all() and np.isfinite(dlm).all() and bool(torch.isfinite(costs).all())
    tol = dict(bf16=(2e-2, 3e-2), fp32=(1e-4, 2e-4))[prec]
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        c, da, dl, _, _ = P.simple_loss(am[b, :Tb, :V], lm[b, :Ub + 1, :V], y[b, :Ub])
        assert abs(float(costs[b]) - c) <= tol[0] * max(1.0, abs(c)), (b, float(costs[b]), c)
        np.testing.assert_allclose(dam[b, :Tb, :V], 0.7 * da, atol=tol[1])
        np.testing.assert_allclose(dlm[b, :Ub + 1, :V], 0.7 * dl, atol=tol[1])
        assert not dam[b, Tb:].any() and not dam[b, :, V:].any() and not dlm[b, :, V:].any()


def _gamma_cases(rng):
    T, U1 = 9, 13
    cases = []
    for kind in ("random", "ties", "onehot_end", "onehot_start"):
        g = np.zeros((4, T, U1), np.float32)
        Ts, Us = [9, 1, 6, 4], [12, 0, 5, 12]
        for b in range(4):
            g[b, :Ts[b], :Us[b] + 1] = {"random": rng.random((Ts[b], Us[b] + 1)), "ties": np.full((Ts[b], Us[b] + 1), 0.25),
                                        "onehot_end": np.eye(1, Us[b] + 1, Us[b])[[0] * Ts[b]],
                                        "onehot_start": np.eye(1, Us[b] + 1, 0)[[0] * Ts[b]]}[kind]
        cases.append((g, Ts, Us))
    return cases


@pytest.mark.parametrize("R", [2, 4, 5, 32])
def test_prune_bounds_bit_equal_to_oracle(R):
    from pika_b200 import kernels as K
    rng = np.random.default_rng(R)
    for g, Ts, Us in _gamma_cases(rng):
        Us = [min(u, t * (R - 1)) for t, u in zip(Ts, Us)]
        s = K.rnnt_prune_bounds(torch.from_numpy(-g).cuda(), None, _lens(*Ts), _lens(*Us), R).cpu().numpy()
        for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
            ref = P.prune_bounds(g[b], Tb, Ub, R)
            np.testing.assert_array_equal(s[b, :Tb], ref)
            assert (s[b, Tb:] == ref[-1]).all()
            P.check_bounds_properties(s[b], Tb, Ub, R)
        s2 = K.rnnt_prune_bounds(torch.from_numpy(-g).cuda(), None, _lens(*Ts), _lens(*Us), R).cpu().numpy()
        assert np.array_equal(s, s2)
    # an infeasible utterance gets -1 everywhere (the loss is then +inf, never a wrong finite value)
    s = K.rnnt_prune_bounds(torch.zeros(1, 3, 9, device="cuda"), None, _lens(3), _lens(8), 3)
    assert (s == -1).all()


def _gate_ref(ex, py, s, B, T, U1, R, H):
    ex, py = ex.double().view(B, T, 2 * H), py.double().view(B, U1, 2 * H)
    u = (s.long().clamp(min=0)[:, :, None] + torch.arange(R, device=s.device)).clamp(max=U1 - 1)
    pu = py[torch.arange(B, device=s.device)[:, None, None], u]                    # [B, T, R, 2H]
    a = torch.tanh(ex[:, :, None, :H] + pu[..., :H])
    g = torch.sigmoid(ex[:, :, None, H:] + pu[..., H:])
    return a, g, u


@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("R", [2, 5, 32])
def test_joint_gate_pruned_against_float64(prec, R):
    from pika_b200 import engine, kernels as K
    torch.manual_seed(R)
    B, T, U1, H = 3, 11, 40, 256
    dt = engine.act_dtype()
    ex = torch.randn(B * T, 2 * H, device="cuda").to(dt)
    py = torch.randn(B * U1, 2 * H, device="cuda").to(dt)
    steps = torch.tensor([[0, 0, 1, 1, 1, 3, 3, 3, 3, 4, 5], [0, R - 1, R - 1, 2 * (R - 1), 2 * (R - 1), 2 * (R - 1), 3 * (R - 1),
                                                              3 * (R - 1), 3 * (R - 1), 4 * (R - 1), 4 * (R - 1)], [0] * 11])
    s = steps.clamp(max=U1 - 1).int().cuda()
    h = torch.empty(B * T * R, H, device="cuda", dtype=dt)
    K.joint_gate_pruned_fwd(ex, py, s, h, B, T, U1, R, H)
    a, g, u = _gate_ref(ex, py, s, B, T, U1, R, H)
    atol = 2e-2 if prec == "bf16" else 1e-5
    torch.testing.assert_close(h.double().view(B, T, R, H), a * g, atol=atol, rtol=0)
    raw = s.long()[:, :, None] + torch.arange(R, device="cuda")
    dh = torch.randn(B, T, R, H, device="cuda").to(dt)
    dh[raw > U1 - 1] = 0                                                             # clamped rows carry no gradient (masked by the loss)
    dex = torch.empty_like(ex)
    dpy = torch.empty_like(py)
    K.joint_gate_pruned_bwd(ex, py, s, dh.view(-1, H), dex, dpy, B, T, U1, R, H)
    d = dh.double()
    d1, dg = d * g * (1 - a * a), d * a * g * (1 - g)
    rex = torch.cat((d1.sum(2), dg.sum(2)), -1)
    rpy = torch.zeros(B, U1, 2 * H, dtype=torch.float64, device="cuda")
    rpy.scatter_add_(1, u.view(B, T * R, 1).expand(-1, -1, 2 * H), torch.cat((d1, dg), -1).view(B, T * R, 2 * H))
    scale = float(R) ** 0.5
    torch.testing.assert_close(dex.double().view(B, T, 2 * H), rex, atol=atol * scale * 3, rtol=0)
    torch.testing.assert_close(dpy.double().view(B, U1, 2 * H), rpy, atol=atol * scale * 3, rtol=0)
    h2, dex2, dpy2 = torch.empty_like(h), torch.empty_like(ex), torch.empty_like(py)
    K.joint_gate_pruned_fwd(ex, py, s, h2, B, T, U1, R, H)
    K.joint_gate_pruned_bwd(ex, py, s, dh.view(-1, H), dex2, dpy2, B, T, U1, R, H)
    assert torch.equal(h, h2) and torch.equal(dex, dex2) and torch.equal(dpy, dpy2)


@pytest.mark.parametrize("prec", PRECS, indirect=True)
def test_simple_and_pruned_loss_kernels_are_deterministic(prec):
    from pika_b200 import engine, kernels as K
    rng = np.random.default_rng(5)
    Ts, Us, V, R = (9, 4, 7), (6, 0, 3), 64, 3
    am, lm, y = _simple_inputs(rng, Ts, Us, V)
    B, T, ldv = am.shape
    U1 = lm.shape[1]
    args = (torch.from_numpy(am).cuda().view(B * T, ldv), torch.from_numpy(lm).cuda().view(B * U1, ldv), V, B, T, U1,
            torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us), R, 1.0)
    r1, r2 = engine.simple_loss(*args), engine.simple_loss(*args)
    for a, b in zip(r1, r2):
        assert torch.equal(a, b)
    bounds = r1[1]
    dt = engine.act_dtype()
    logits = torch.randn(B * T * R, ldv, device="cuda").to(dt)
    outs = []
    for _ in range(2):
        dl, cs = torch.empty_like(logits), torch.empty(ldv, device="cuda")
        c = K.rnnt_pruned_loss(logits, torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us), bounds, U1, R, V, dlogits=dl, colsum=cs)
        outs.append((c, dl, cs))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("prec", PRECS, indirect=True)
def test_pruned_loss_kernel_against_oracle(prec):
    """pk_rnnt_pruned_loss on given logits and bounds: costs and dlogits against the float64 pruned lattice"""
    from pika_b200 import engine, kernels as K
    from oracle import rnnt as orc
    rng = np.random.default_rng(11)
    Ts, Us, V, R = (6, 3, 5), (5, 0, 2), 61, 3
    B, T, U1 = 3, 6, 6
    ldv = engine._ldv(V)
    y = rng.integers(1, V, (B, 5)).astype(np.int32)
    s = np.zeros((B, T), np.int32)
    s[0] = [0, 1, 1, 2, 3, 3]
    s[2] = [0, 0, 1, 1, 1, 1]
    z = np.zeros((B * T * R, ldv), np.float32)
    z[:, :V] = rng.standard_normal((B * T * R, V)) * 2
    dt = engine.act_dtype()
    zt = torch.from_numpy(z).cuda().to(dt)
    zq = zt.float().cpu().numpy()
    dl, cs = torch.empty_like(zt), torch.empty(ldv, device="cuda")
    costs = K.rnnt_pruned_loss(zt, torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us), torch.from_numpy(s).cuda(), U1, R, V, dlogits=dl,
                               colsum=cs)
    dl = dl.float().cpu().numpy().reshape(B, T, R, ldv)
    ref_cs = np.zeros(ldv)
    for b in range(B):
        Tb, Ub = Ts[b], Us[b]
        lp = orc.log_softmax(zq.reshape(B, T, R, ldv)[b, :, :, :V])                # [T, R, V]
        lpb = np.full((Tb, Ub + 1), -np.inf)
        lpl = np.full((Tb, Ub), -np.inf)
        for t in range(Tb):
            for r in range(R):
                u = s[b, t] + r
                if u <= Ub:
                    lpb[t, u] = lp[t, r, 0]
                    if u < Ub:
                        lpl[t, u] = lp[t, r, y[b, u]]
        c, gb, gl = P.pruned_cost(lpb, lpl, s[b], R)
        assert abs(float(costs[b]) - c) < 1e-3 * max(1, abs(c))
        for t in range(T):
            for r in range(R):
                u = s[b, t] + r
                ref = np.zeros(ldv)
                if t < Tb and u <= Ub:
                    g = np.zeros(V)
                    g[0] += gb[t, u]
                    if u < Ub:
                        g[y[b, u]] += gl[t, u]
                    ref[:V] = g - np.exp(lp[t, r]) * g.sum()
                np.testing.assert_allclose(dl[b, t, r], ref, atol=1e-2 if prec == "bf16" else 1e-5)
                ref_cs += ref
    np.testing.assert_allclose(cs.cpu().numpy(), ref_cs, atol=5e-2 if prec == "bf16" else 1e-4)


def _small_net(encoder_type, decoder_type, V, prune_range):
    from pika_b200.model.transducer import Net
    torch.manual_seed(777)
    o = types.SimpleNamespace(rnn_size=256, local_rank=0, decoder_type=decoder_type, brnn=True, encoder_type=encoder_type, embd_dim=64,
                              padding_idx=V, dropout=0.0, dec_layers=1, enc_layers=2, prune_range=prune_range)
    return Net(o, 40, V).cuda().train()


def _batch(V, Ts, Us, D=40):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(len(Ts), max(Ts), D, generator=g).cuda()
    y = torch.randint(1, V, (len(Us), max(Us)), generator=g).cuda()
    return x, y, _lens(*Ts), _lens(*Us)


@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("decoder_type", ["rnn", "transformer"])
def test_pruned_loss_with_full_windows_matches_dense(prec, decoder_type):
    """R = U_max + 1 keeps every node: costs and every shared parameter gradient equal the dense transducer_loss's"""
    from pika_b200 import engine
    V, Ts, Us = 60, (17, 12, 9), (6, 3, 0)
    R = max(Us) + 1
    x, y, fl, ll = _batch(V, Ts, Us)
    engine.set_dropout_enabled(False)
    try:
        m = _small_net("rnn", decoder_type, V, R)
        dense = engine.transducer_loss(m, x, y, fl, ll, x_len=fl)
        dense.sum().backward()
        g_dense = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None and not k.startswith("simple_")}
        m.zero_grad(set_to_none=True)
        simple, pruned = engine.transducer_loss_pruned(m, x, y, fl, ll, R, 0.0, 1.0, x_len=fl)
        (0.0 * simple + pruned).sum().backward()
    finally:
        engine.set_dropout_enabled(True)
    rtol = 2e-2 if prec == "bf16" else 1e-4
    torch.testing.assert_close(pruned, dense, rtol=rtol, atol=rtol)
    for k, gd in g_dense.items():
        gp = m.get_parameter(k).grad
        err = float((gp - gd).norm() / gd.norm().clamp(min=1e-3))          # floor: gradients that are zero in exact arithmetic (key bias)
        assert err < (5e-2 if prec == "bf16" else 1e-3), (k, err)
    assert float(m.simple_am_proj.weight.grad.abs().max()) == 0.0


@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("decoder_type", ["rnn", "transformer"])
@pytest.mark.parametrize("V", [61, 64, 520])
def test_pruned_step_gradients_match_float64_restatement(V, prec, decoder_type):
    """one step of transducer_loss_pruned (sigma_s = 0.5, sigma_p = 1) against float64 torch given the same encoder / prediction-net
    outputs and the GPU's bounds: joint, fc2 and simple-projection gradients"""
    from pika_b200 import engine
    R = 3
    Ts, Us = (9, 6), (7, 4)
    x, y, fl, ll = _batch(V, Ts, Us)
    engine.set_dropout_enabled(False)
    try:
        m = _small_net("rnn", decoder_type, V, R)
        simple, pruned = engine.transducer_loss_pruned(m, x, y, fl, ll, R, 0.5, 1.0, x_len=fl)
        (0.5 * simple + pruned).sum().backward()
        with torch.no_grad():
            enc = engine.model_encoder_forward_act(m, x, fl).double()
            pred = engine.prednet_forward_act(m, y).double()
            _, bounds = engine.SimpleLossFn.apply(enc.to(engine.act_dtype()), pred.to(engine.act_dtype()), m, y.int(), fl, ll, R, 0.5, False)
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
    total = 0.0
    for b in range(B):
        Tb, Ub = Ts[b], Us[b]
        yb = y[b, :Ub]
        lsz = torch.log_softmax(am[b, :Tb, None] + lm[b, None, :Ub + 1], -1)
        full_b = lsz[:, :, 0]
        full_l = lsz[:, torch.arange(Ub), yb]
        total = total + 0.5 * _nll(full_b, full_l, Tb, Ub)
        # nodes outside the windows: a finite -1e30 instead of -inf, so that autograd through logsumexp stays finite (exp gives 0)
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
        pb = _place(pb, rows_b)
        pl = _place(pl, rows_l)
        total = total + _nll(pb, pl[:, :Ub], Tb, Ub)
    total.backward()
    tol = 6e-2 if prec == "bf16" else 2e-3
    for k, p in ps.items():
        g = m.get_parameter(k).grad.double()
        err = float((g - p.grad).norm() / p.grad.norm().clamp(min=1e-12))
        assert err < tol, (k, err)


def _place(base, entries):
    out = base.clone()
    for t, u, v in entries:
        out = out.index_put((torch.tensor([t], device="cuda"), torch.tensor([u], device="cuda")), v.reshape(1))
    return out


def _nll(lpb, lpl, T, U):
    """differentiable float64 RNN-T NLL over [T, U+1] / [T, U] tables"""
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


def test_infeasible_utterance_raises_before_any_result():
    from pika_b200 import engine
    V = 60
    x, y, fl, ll = _batch(V, (5, 9), (6, 8))                                        # utterance 0: U = 6 > T (R - 1) = 5
    m = _small_net("rnn", "rnn", V, 2)
    with pytest.raises(ValueError, match=r"\[0\]"):
        engine.transducer_loss_pruned(m, x, y, fl, ll, 2, 0.5, 1.0, x_len=fl)


def test_train_cli_pruned(tmp_path):
    """the trainer with --prune_range 4 --prune_warmup_batches 2: the pruned Loss falls, Simple is logged and finite, the pickles reload
    and decode to the same hypotheses as the same model without the simple joiner"""
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
            "--grad_clip", "3.0", "--initial_lr", "0.002", "--final_lr", "0.001", "--momentum", "0.9", "--num_epochs", "5",
            "--num_batches_per_epoch", "2", "--sync_period", "1", "--block_momentum", "0.9", "--block_lr", "1.0", "--seed", "777",
            "--prune_range", "4", "--prune_warmup_batches", "2"]
    os.environ.setdefault("WORLD_SIZE", "1")
    T.main(argv)
    text = open(str(log).replace("WORKER-ID", "0")).read()
    assert "Training Finished" in text
    lines = [l for l in text.splitlines() if "Overall Avg Loss" in l]
    losses = [float(l.split("Loss:")[1].split()[0]) for l in lines]
    simple = [float(l.split("Simple:")[1].split()[0]) for l in lines]
    print("pruned losses per epoch", losses, "simple", simple)
    assert len(losses) == 5 and np.isfinite(losses).all() and np.isfinite(simple).all() and min(losses[-2:]) < losses[0]
    m = torch.load(str(out / "model.epoch.4.0"), weights_only=False)
    assert hasattr(m, "simple_am_proj") and bool(torch.isfinite(m.fc2.weight).all())
    # decoding ignores the simple joiner: the same greedy hypotheses with it deleted
    from pika_b200 import engine
    m = m.cuda().eval()
    x, y, fl, ll = _batch(60, (80, 64), (3, 2), D=240)
    with torch.no_grad():
        a = engine.transducer_forward(m, x, y).argmax(-1)
        del m.simple_am_proj, m.simple_lm_proj
        b = engine.transducer_forward(m, x, y).argmax(-1)
    assert torch.equal(a, b)
