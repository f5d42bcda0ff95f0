"""FastEmit and the delay penalty on the GPU: every *_reg entry point (include/pika_b200.h) against the float64 oracle
(tests/emission_reg_oracle.py), the plain entry points' outputs and launches at (0, 0), the engine's losses and gradients, and the
trainers' flags."""
import os
import types

import numpy as np
import pytest
import torch

import emission_reg_oracle as E
import pruned_rnnt_oracle as P
import pruned_smoothed_oracle as PS
from oracle.rnnt import log_softmax

pytestmark = pytest.mark.gpu

REGS = [(0.3, 0.0), (0.0, 0.05), (0.5, 0.02)]
LOG2E = 1.4426950408889634


def _lens(*v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def _row_lse(z, V):
    """one (max, sum-exp) partial per row in the GEMM's log2 units: [1, rows, 2]"""
    x = z.reshape(-1, z.shape[-1])[:, :V].float() * LOG2E
    m = x.max(-1).values
    return torch.stack((m, torch.exp2(x - m[:, None]).sum(-1)), -1)[None].contiguous()


def _dense_case(dtype, V=61, Ts=(9, 1, 6, 4), Us=(5, 3, 0, 2), seed=0):
    from pika_b200 import engine
    rng = np.random.default_rng(seed)
    B, T, U1 = len(Ts), max(Ts), max(Us) + 1
    ldv = engine._ldv(V)
    z = np.zeros((B, T, U1, ldv), np.float32)
    z[..., :V] = rng.standard_normal((B, T, U1, V)) * 2
    y = rng.integers(1, V, (B, max(U1 - 1, 1))).astype(np.int32)
    zt = torch.from_numpy(z).cuda().to(dtype).contiguous()
    return zt, zt.float().cpu().numpy(), y, Ts, Us, V


def _oracle_dense(zq, y, Ts, Us, V, lam_f, lam_d, gs):
    B, T, U1, ldv = zq.shape
    costs, dl = np.zeros(B), np.zeros((B, T, U1, ldv))
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        c, d = E.dense_loss(zq[b, :Tb, :Ub + 1, :V], y[b, :Ub], lam_f, lam_d)
        costs[b], dl[b, :Tb, :Ub + 1, :V] = c, d * gs[b]
    return costs, dl


@pytest.mark.parametrize("lam_f,lam_d", REGS)
@pytest.mark.parametrize("dtype,variant", [(torch.float32, "plain"), (torch.float32, "lse"), (torch.bfloat16, "plain"),
                                           (torch.bfloat16, "lse"), (torch.bfloat16, "compact")],      # the compacted gradient is bf16 only
                         ids=["f32-plain", "f32-lse", "bf16-plain", "bf16-lse", "bf16-compact"])
def test_dense_entry_points_against_oracle(dtype, variant, lam_f, lam_d):
    from pika_b200 import kernels as K
    zt, zq, y, Ts, Us, V = _dense_case(dtype, seed=int(lam_f * 10 + lam_d * 100))
    B, T, U1, ldv = zt.shape
    yt, fl, ll = torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us)
    gs = np.array([1.0, 0.5, 2.0, 0.25], np.float32)[:B]
    reg = dict(fastemit_lambda=lam_f, delay_penalty=lam_d)
    row_lse = _row_lse(zt, V) if variant != "plain" else None
    if variant == "compact":
        gs = np.ones(B, np.float32)
        h = torch.randn(B * T * U1, 64, device="cuda").to(torch.bfloat16)
        costs, dz_c, h_c, row_map, cnt = K.rnnt_loss_compact(zt, yt, fl, ll, h, V=V, row_lse=row_lse, **reg)
        rm = row_map.long()
        dl = torch.zeros(B * T * U1, ldv, device="cuda", dtype=torch.bfloat16)
        dl[rm >= 0] = dz_c[rm[rm >= 0]]
        assert torch.equal(h_c[rm[rm >= 0]], h[rm >= 0])
        dense_c, dense_dl = K.rnnt_loss_fwd_bwd(zt, yt, fl, ll, V=V, row_lse=row_lse, **reg)
        assert torch.equal(costs, dense_c) and torch.equal(dl.view_as(zt), dense_dl)
        padded = torch.ones(B, T, U1, dtype=torch.bool)
        for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
            padded[b, :Tb, :Ub + 1] = False
        assert (rm.cpu()[padded.flatten()] < 0).all()           # padded rows stay zero rows
        dl = dl.view_as(zt)
    else:
        costs, dl = K.rnnt_loss_fwd_bwd(zt, yt, fl, ll, V=V, grad_scale=torch.from_numpy(gs).cuda(), row_lse=row_lse, **reg)
    ref_c, ref_dl = _oracle_dense(zq, y, Ts, Us, V, lam_f, lam_d, gs)
    ct = 1e-5 if dtype == torch.float32 and variant == "plain" else 2e-4
    np.testing.assert_allclose(costs.cpu().numpy(), ref_c, rtol=ct, atol=ct)
    np.testing.assert_allclose(dl.float().cpu().numpy(), ref_dl, atol=3e-5 if dtype == torch.float32 else 1e-2)


def _skew(x, U1):
    """[B, T, U1] -> the lattice's skewed layout [B, T+U1-1, U1]; cells outside the lattice hold 0"""
    B, T, _ = x.shape
    out = torch.zeros(B, T + U1 - 1, U1, dtype=torch.float32, device="cuda")
    t = torch.arange(T, device="cuda")[:, None]
    u = torch.arange(U1, device="cuda")[None, :]
    out[:, t + u, u.expand(T, U1)] = x
    return out


@pytest.mark.parametrize("Ts,Us", [((3, 2, 1), (2047, 1500, 0)), ((40, 17, 1), (33, 0, 5)), ((1,), (0,))])
@pytest.mark.parametrize("lam_f,lam_d", REGS)
def test_lattice_entry_point_against_oracle(Ts, Us, lam_f, lam_d):
    """pk_rnnt_lattice_reg on given tables up to U1 = 2048 (the lattice's limit), T_b = 1 and U_b = 0, with per-utterance grad_scale"""
    from pika_b200 import kernels as K
    torch.manual_seed(len(Ts) + max(Us))
    B, T, U1 = len(Ts), max(Ts), max(Us) + 1
    lpb = -torch.rand(B, T, U1, device="cuda") * 3
    lpl = -torch.rand(B, T, U1, device="cuda") * 3
    gs = torch.tensor([1.0, 0.5, 3.0][:B], device="cuda")
    costs, gb, gl = K.rnnt_lattice(_skew(lpb, U1), _skew(lpl, U1), _lens(*Ts), _lens(*Us), B, T, U1, grad_scale=gs, fastemit_lambda=lam_f,
                                   delay_penalty=lam_d)
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        c, rgb, rgl, _, _ = E.lattice(lpb[b].double().cpu().numpy(), lpl[b].double().cpu().numpy(), Tb, Ub, lam_f, lam_d)
        assert abs(float(costs[b]) - c) <= 1e-6 * max(1.0, abs(c)), (b, float(costs[b]), c)
        np.testing.assert_allclose(gb[b, :Tb, :Ub + 1].cpu().numpy(), rgb * float(gs[b]), atol=2e-6)
        np.testing.assert_allclose(gl[b, :Tb, :Ub].cpu().numpy(), rgl[:, :Ub] * float(gs[b]), atol=2e-6)
        assert not gb[b, Tb:].any() and not gb[b, :, Ub + 1:].any() and not gl[b, :, Ub:].any()
        if Ub == 0:                          # no label arcs: the options change nothing
            plain = K.rnnt_lattice(_skew(lpb, U1), _skew(lpl, U1), _lens(*Ts), _lens(*Us), B, T, U1, grad_scale=gs)
            assert float(plain[0][b]) == float(costs[b]) and torch.equal(plain[1][b], gb[b])


def _call(fn, *args):
    from pika_b200 import _lib
    before = _lib.launch_count()
    _lib.check(fn(*args), "")
    torch.cuda.synchronize()
    return _lib.launch_count() - before


def test_reg_entry_points_at_zero_are_the_plain_ones():
    """every *_reg entry point at (0, 0): bit-identical outputs and the same number of launches as the entry point without the suffix"""
    from pika_b200 import _lib, kernels as K
    lib, P_ = _lib.lib, K._P
    zt, _, y, Ts, Us, V = _dense_case(torch.bfloat16)
    B, T, U1, ldv = zt.shape
    yt, fl, ll = torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us)
    gs = torch.tensor([1.0, 0.5, 2.0, 0.25], device="cuda")
    ws_bytes = int(lib.pk_rnnt_loss_workspace_bytes(B, T, U1)) + int(lib.pk_rnnt_loss_colsum_workspace_bytes(B, T, U1, ldv))
    rl = _row_lse(zt, V)
    h = torch.randn(B * T * U1, 64, device="cuda").to(torch.bfloat16)
    st = torch.cuda.current_stream().cuda_stream

    def outs(kind, reg):
        ws = torch.zeros(ws_bytes, dtype=torch.uint8, device="cuda")
        c, cs = torch.empty(B, device="cuda"), torch.empty(ldv, device="cuda")
        common = (P_(zt), K.PK_BF16, P_(yt), P_(fl), P_(ll), B, T, U1, V, ldv, yt.stride(0))
        if kind == "compact":
            dz, hc = torch.empty(B * T * U1, ldv, device="cuda", dtype=torch.bfloat16), torch.empty_like(h)
            rm, rc = torch.empty(B * T * U1, dtype=torch.int32, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
            args = common + (None, P_(c), P_(dz), P_(cs), P_(ws), ws_bytes, P_(rl), 1, P_(h), 64, P_(hc), P_(rm), P_(rc))
            n = _call(lib.pk_rnnt_loss_fwd_bwd_compact_reg if reg else lib.pk_rnnt_loss_fwd_bwd_compact, *args, *((0.0, 0.0) if reg else ()), st)
            return n, (c, cs, rc, rm, dz[:int(rc)], hc[:int(rc)])
        dl = torch.empty_like(zt)
        args = common + (P_(gs), P_(c), P_(dl), P_(cs), P_(ws), ws_bytes) + ((P_(rl), 1) if kind == "lse" else ())
        fn = {"plain": (lib.pk_rnnt_loss_fwd_bwd, lib.pk_rnnt_loss_fwd_bwd_reg),
              "lse": (lib.pk_rnnt_loss_fwd_bwd_lse, lib.pk_rnnt_loss_fwd_bwd_lse_reg)}[kind][int(reg)]
        return _call(fn, *args, *((0.0, 0.0) if reg else ()), st), (c, cs, dl)

    for kind in ("plain", "lse", "compact"):
        n0, a = outs(kind, False)
        n1, b = outs(kind, True)
        assert n0 == n1 and n0 >= 3, (kind, n0, n1)
        for x, z in zip(a, b):
            assert torch.equal(x, z), kind
    # the lattice and the pruned loss
    lpb, lpl = -torch.rand(B, T + U1 - 1, U1, device="cuda"), -torch.rand(B, T + U1 - 1, U1, device="cuda")
    lws = int(K._ws_query(lib.pk_rnnt_lattice_workspace, "", B, T, U1))
    res = []
    for reg in (False, True):
        c, gb, gl = torch.empty(B, device="cuda"), torch.empty(B, T, U1, device="cuda"), torch.empty(B, T, U1, device="cuda")
        ws = torch.empty(lws, dtype=torch.uint8, device="cuda")
        args = (P_(fl), P_(ll), B, T, U1, P_(lpb), P_(lpl), P_(gs), P_(c), P_(gb), P_(gl), P_(ws), lws)
        res.append((_call(lib.pk_rnnt_lattice_reg if reg else lib.pk_rnnt_lattice, *args, *((0.0, 0.0) if reg else ()), st), c, gb, gl))
    assert res[0][0] == res[1][0] == 1 and all(torch.equal(x, z) for x, z in zip(res[0][1:], res[1][1:]))
    R = 3
    s = torch.tensor([[min(t // 2, max(Us[b] - R + 1, 0)) for t in range(T)] for b in range(B)], dtype=torch.int32, device="cuda")
    zp = torch.randn(B * T * R, ldv, device="cuda").to(torch.bfloat16)
    pws = int(K._ws_query(lib.pk_rnnt_pruned_loss_workspace, "", B, T, U1, R, ldv))
    res = []
    for reg in (False, True):
        c, dl, cs = torch.empty(B, device="cuda"), torch.empty_like(zp), torch.empty(ldv, device="cuda")
        ws = torch.empty(pws, dtype=torch.uint8, device="cuda")
        args = (P_(zp), K.PK_BF16, P_(yt), P_(fl), P_(ll), P_(s), B, T, U1, R, V, ldv, yt.stride(0), P_(gs), P_(c), P_(dl), P_(cs), P_(ws), pws,
                None, 0)
        res.append((_call(lib.pk_rnnt_pruned_loss_reg if reg else lib.pk_rnnt_pruned_loss, *args, *((0.0, 0.0) if reg else ()), st), c, dl, cs))
    assert res[0][0] == res[1][0] and all(torch.equal(x, z) for x, z in zip(res[0][1:], res[1][1:]))


@pytest.mark.parametrize("bad", [(-0.1, 0.0), (0.0, -1e-3), (float("nan"), 0.0), (0.0, float("inf"))])
def test_reg_entry_points_refuse_bad_values_before_any_launch(bad):
    from pika_b200 import _lib, kernels as K
    zt, _, y, Ts, Us, V = _dense_case(torch.float32)
    yt, fl, ll = torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us)
    before = _lib.launch_count()
    with pytest.raises(_lib.PikaError, match="fastemit_lambda|delay_penalty"):
        K.rnnt_loss_fwd_bwd(zt, yt, fl, ll, V=V, fastemit_lambda=bad[0], delay_penalty=bad[1])
    B, T, U1, _ = zt.shape
    with pytest.raises(_lib.PikaError, match="fastemit_lambda|delay_penalty"):
        K.rnnt_lattice(_skew(torch.zeros(B, T, U1, device="cuda"), U1), _skew(torch.zeros(B, T, U1, device="cuda"), U1), fl, ll, B, T, U1,
                       fastemit_lambda=bad[0], delay_penalty=bad[1])
    with pytest.raises(_lib.PikaError, match="fastemit_lambda|delay_penalty"):
        K.rnnt_pruned_loss(torch.zeros(B * T * 2, 64, device="cuda"), yt, fl, ll, torch.zeros(B, T, dtype=torch.int32, device="cuda"), U1, 2,
                           V, fastemit_lambda=bad[0], delay_penalty=bad[1])
    assert _lib.launch_count() == before


@pytest.mark.parametrize("lam_f,lam_d", REGS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_pruned_loss_entry_point_against_oracle(dtype, lam_f, lam_d):
    from pika_b200 import engine, kernels as K
    rng = np.random.default_rng(11)
    Ts, Us, V, R = (6, 3, 5, 1), (5, 0, 2, 0), 61, 3
    B, T, U1 = 4, 6, 6
    ldv = engine._ldv(V)
    y = rng.integers(1, V, (B, 5)).astype(np.int32)
    s = np.zeros((B, T), np.int32)
    s[0] = [0, 1, 1, 2, 3, 3]
    s[2] = [0, 0, 1, 1, 1, 1]
    z = np.zeros((B * T * R, ldv), np.float32)
    z[:, :V] = rng.standard_normal((B * T * R, V)) * 2
    zt = torch.from_numpy(z).cuda().to(dtype)
    zq = zt.float().cpu().numpy().reshape(B, T, R, ldv)
    gs = torch.tensor([1.0, 0.5, 2.0, 1.5], device="cuda")
    dl = torch.empty_like(zt)
    costs = K.rnnt_pruned_loss(zt, torch.from_numpy(y).cuda(), _lens(*Ts), _lens(*Us), torch.from_numpy(s).cuda(), U1, R, V, grad_scale=gs,
                               dlogits=dl, fastemit_lambda=lam_f, delay_penalty=lam_d)
    dl = dl.float().cpu().numpy().reshape(B, T, R, ldv)
    for b in range(B):
        Tb, Ub = Ts[b], Us[b]
        lp = log_softmax(zq[b, :, :, :V])
        lpb, lpl = np.full((Tb, Ub + 1), -np.inf), np.full((Tb, Ub), -np.inf)
        for t in range(Tb):
            for r in range(R):
                u = s[b, t] + r
                if u <= Ub:
                    lpb[t, u] = lp[t, r, 0]
                    if u < Ub:
                        lpl[t, u] = lp[t, r, y[b, u]]
        c, gb, gl = E.pruned_loss(lpb, lpl, s[b], R, lam_f, lam_d)
        assert abs(float(costs[b]) - c) < 1e-4 * max(1, abs(c)), (b, float(costs[b]), c)
        for t in range(T):
            for r in range(R):
                u = s[b, t] + r
                ref = np.zeros(ldv)
                if t < Tb and u <= Ub:
                    ref[:V] = E.row_grad(lp[t, r], gb[t, u], gl[t, u], y[b, u] if u < Ub else -1) * float(gs[b])
                np.testing.assert_allclose(dl[b, t, r], ref, atol=1e-2 if dtype == torch.bfloat16 else 3e-5)


@pytest.mark.parametrize("lam_l,lam_a", [(0.0, 0.0), (0.25, 0.1)])
@pytest.mark.parametrize("lam_d", [0.05, 0.5])
def test_simple_loss_and_bounds_on_the_penalised_lattice(lam_d, lam_l, lam_a):
    """engine.simple_loss with the delay penalty: costs and projection gradients against the oracle, and the bounds are the oracle's
    prune_bounds of the penalised lattice's occupancies"""
    from pika_b200 import engine, kernels as K
    old = engine.get_precision()
    engine.set_precision("fp32")
    try:
        rng = np.random.default_rng(int(lam_d * 100))
        Ts, Us, V, R = (9, 1, 6), (7, 0, 4), 60, 3
        B, T, U1 = 3, 9, 8
        ldv = engine._ldv(V)
        am = np.zeros((B, T, ldv), np.float32)
        lm = np.zeros((B, U1, ldv), np.float32)
        am[..., :V] = rng.standard_normal((B, T, V)) * 2
        lm[..., :V] = rng.standard_normal((B, U1, V)) * 2
        y = rng.integers(1, V, (B, U1 - 1)).astype(np.int32)
        fl, ll, yt = _lens(*Ts), _lens(*Us), torch.from_numpy(y).cuda()
        amt, lmt = torch.from_numpy(am).cuda().view(B * T, ldv), torch.from_numpy(lm).cuda().view(B * U1, ldv)
        costs, bounds, dam, dlm = engine.simple_loss(amt, lmt, V, B, T, U1, yt, fl, ll, R, 0.7, True, lam_l, lam_a, delay_penalty=lam_d)
        dam = dam.float().view(B, T, ldv).cpu().numpy()
        dlm = dlm.float().view(B, U1, ldv).cpu().numpy()
        logq = PS.unigram_logq([lm[b, :Us[b] + 1, :V] for b in range(B)])
        for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
            c, da, dl, gb, gl = E.simple_loss(am[b, :Tb, :V], lm[b, :Ub + 1, :V], y[b, :Ub], lam_d, logq, lam_l, lam_a)
            assert abs(float(costs[b]) - c) <= 1e-4 * max(1.0, abs(c)), (b, float(costs[b]), c)
            np.testing.assert_allclose(dam[b, :Tb, :V], 0.7 * da, atol=2e-4)
            np.testing.assert_allclose(dlm[b, :Ub + 1, :V], 0.7 * dl, atol=2e-4)
        # the bounds: the kernel's penalised occupancies through the oracle's algorithm, bit for bit
        _, gb_k, gl_k = _simple_lattice(engine, K, amt, lmt, V, B, T, U1, yt, fl, ll, lam_l, lam_a, lam_d)
        g = -(gb_k + gl_k).cpu().numpy()
        s = bounds.cpu().numpy()
        for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
            np.testing.assert_array_equal(s[b, :Tb], P.prune_bounds(g[b], Tb, Ub, R))
            _, _, _, gb, gl = E.simple_loss(am[b, :Tb, :V], lm[b, :Ub + 1, :V], y[b, :Ub], lam_d, logq, lam_l, lam_a)
            np.testing.assert_allclose(g[b, :Tb, :Ub + 1], -(gb + gl), atol=1e-4)
    finally:
        engine.set_precision(old)


def _simple_lattice(engine, K, am, lm, V, B, T, U1, yt, fl, ll, lam_l, lam_a, lam_d):
    """the simple loss's tables and lattice as engine.simple_loss runs them -> (costs, gb, gl)"""
    ldv = am.shape[1]
    U1p = (U1 + 7) // 8 * 8
    E_ = [torch.empty(B * T, ldv, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    P_ = [torch.empty(B * U1p, ldv, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    am_max = K.rnnt_simple_prep(am, V, B, T, T, E_[0], E_[1])
    lm_max = K.rnnt_simple_prep(lm, V, B, U1, U1p, P_[0], P_[1])
    S = torch.empty(B, T, U1p, dtype=torch.float32, device="cuda")
    engine.gemm_parts([[e.view(B, T, ldv) for e in E_]], [[p.view(B, U1p, ldv) for p in P_]], S)
    if lam_l or lam_a:
        Nl, logq, Na = K.rnnt_simple_smooth_stats(am, lm, V, am_max, lm_max, fl, ll, B, T, U1)
        lpb, lpl = K.rnnt_simple_tables_smooth(am, lm, am_max, lm_max, S.view(B * T, U1p), yt, fl, ll, B, T, U1, Nl, logq, Na, lam_l, lam_a)
    else:
        lpb, lpl = K.rnnt_simple_tables(am, lm, am_max, lm_max, S.view(B * T, U1p), yt, fl, ll, B, T, U1)
    return K.rnnt_lattice(lpb, lpl, fl, ll, B, T, U1, delay_penalty=lam_d)


def _small_net(V, prune_range=0):
    from pika_b200.model.transducer import Net
    torch.manual_seed(777)
    o = types.SimpleNamespace(rnn_size=256, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="rnn", embd_dim=64, padding_idx=V,
                              dropout=0.0, dec_layers=1, enc_layers=2, prune_range=prune_range)
    return Net(o, 40, V).cuda().train()


def _batch(V, Ts, Us):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(len(Ts), max(Ts), 40, generator=g).cuda()
    y = torch.randint(1, V, (len(Us), max(Us)), generator=g).cuda()
    return x, y, _lens(*Ts), _lens(*Us)


def _surrogate(lp_b, lp_l, gb, gl):
    """sum gb * lpb + gl * lpl with (gb, gl) constants: its gradient through the log-probs is the row passes' d / d logits"""
    return (torch.from_numpy(gb).cuda() * lp_b).sum() + (torch.from_numpy(gl).cuda() * lp_l).sum()


@pytest.mark.parametrize("lam_f,lam_d", [(0.3, 0.0), (0.0, 0.05), (0.5, 0.02)])
def test_transducer_loss_against_oracle_composition(lam_f, lam_d):
    """engine.transducer_loss in fp32-class mode: costs and the joint's parameter gradients against float64 torch given the same
    encoder / prediction-net outputs, with the regularised (gb, gl) from the oracle"""
    from pika_b200 import engine
    V, Ts, Us = 60, (11, 7, 1), (6, 0, 3)
    x, y, fl, ll = _batch(V, Ts, Us)
    old = engine.get_precision()
    engine.set_precision("fp32")
    engine.set_dropout_enabled(False)
    try:
        m = _small_net(V)
        costs = engine.transducer_loss(m, x, y, fl, ll, x_len=fl, fastemit_lambda=lam_f, delay_penalty=lam_d)
        costs.sum().backward()
        with torch.no_grad():
            enc = engine.model_encoder_forward_act(m, x, fl).double()
            pred = engine.prednet_forward_act(m, y).double()
    finally:
        engine.set_dropout_enabled(True)
        engine.set_precision(old)
    ps = {k: p.detach().double().requires_grad_(True) for k, p in m.named_parameters() if k.startswith(("fc1", "fc_gate", "fc2"))}
    H = enc.shape[-1]
    h = torch.tanh(enc[:, :, None] @ ps["fc1.weight"][:, :H].t() + ps["fc1.bias"] + (pred @ ps["fc1.weight"][:, H:].t())[:, None]) * \
        torch.sigmoid(enc[:, :, None] @ ps["fc_gate.weight"][:, :H].t() + ps["fc_gate.bias"] + (pred @ ps["fc_gate.weight"][:, H:].t())[:, None])
    lp = torch.log_softmax(h @ ps["fc2.weight"].t() + ps["fc2.bias"], -1)
    total = 0.0
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        yb = y[b, :Ub]
        lpb, lpl = lp[b, :Tb, :Ub + 1, 0], lp[b, :Tb, torch.arange(Ub), yb]
        c, gb, gl, _, _ = E.lattice(lpb.detach().cpu().numpy(), lpl.detach().cpu().numpy(), Tb, Ub, lam_f, lam_d)
        assert abs(float(costs[b].detach()) - c) <= 1e-4 * max(1.0, abs(c)), (b, float(costs[b].detach()), c)
        total = total + _surrogate(lpb, lpl, gb, gl[:, :Ub])
    total.backward()
    for k, p in ps.items():
        g = m.get_parameter(k).grad.double()
        err = float((g - p.grad).norm() / p.grad.norm().clamp(min=1e-12))
        assert err < 2e-3, (k, err)


@pytest.mark.parametrize("lam_f,lam_d", [(0.3, 0.0), (0.0, 0.05), (0.5, 0.02)])
def test_transducer_loss_pruned_against_oracle_composition(lam_f, lam_d):
    """engine.transducer_loss_pruned in fp32-class mode (simple scale 0.5): both losses' costs, the bounds of the penalised simple
    lattice, and the joint / fc2 / simple-projection gradients against float64 torch with the oracle's regularised coefficients"""
    from pika_b200 import engine
    V, R, Ts, Us = 61, 3, (9, 6), (7, 4)
    x, y, fl, ll = _batch(V, Ts, Us)
    old = engine.get_precision()
    engine.set_precision("fp32")
    engine.set_dropout_enabled(False)
    try:
        m = _small_net(V, R)
        simple, pruned = engine.transducer_loss_pruned(m, x, y, fl, ll, R, 0.5, 1.0, x_len=fl, fastemit_lambda=lam_f, delay_penalty=lam_d)
        (0.5 * simple + pruned).sum().backward()
        with torch.no_grad():
            enc = engine.model_encoder_forward_act(m, x, fl).double()
            pred = engine.prednet_forward_act(m, y).double()
            _, bounds = engine.SimpleLossFn.apply(enc.float(), pred.float(), m, y.int(), fl, ll, R, 0.5, False, 0.0, 0.0, lam_d)
    finally:
        engine.set_dropout_enabled(True)
        engine.set_precision(old)
    ps = {k: p.detach().double().requires_grad_(True) for k, p in m.named_parameters() if k.startswith(("fc1", "fc_gate", "fc2", "simple_"))}
    B, T, H = enc.shape
    U1 = pred.shape[1]
    lin = lambda v, n: v @ ps[n + ".weight"].t() + ps[n + ".bias"]                  # noqa: E731
    ex1, exg = enc @ ps["fc1.weight"][:, :H].t() + ps["fc1.bias"], enc @ ps["fc_gate.weight"][:, :H].t() + ps["fc_gate.bias"]
    py1, pyg = pred @ ps["fc1.weight"][:, H:].t(), pred @ ps["fc_gate.weight"][:, H:].t()
    s = bounds.long()
    u = (s[:, :, None] + torch.arange(R, device="cuda")).clamp(max=U1 - 1)
    bi = torch.arange(B, device="cuda")[:, None, None]
    lp = torch.log_softmax(lin(torch.tanh(ex1[:, :, None] + py1[bi, u]) * torch.sigmoid(exg[:, :, None] + pyg[bi, u]), "fc2"), -1)
    am, lm = lin(enc, "simple_am_proj"), lin(pred, "simple_lm_proj")
    total = 0.0
    for b, (Tb, Ub) in enumerate(zip(Ts, Us)):
        yb = y[b, :Ub]
        lsz = torch.log_softmax(am[b, :Tb, None] + lm[b, None, :Ub + 1], -1)
        sb, sl = lsz[:, :, 0], lsz[:, torch.arange(Ub), yb]
        c, gb, gl, _, _ = E.lattice(sb.detach().cpu().numpy(), sl.detach().cpu().numpy(), Tb, Ub, 0.0, lam_d)
        assert abs(float(simple[b].detach()) - c) <= 1e-4 * max(1.0, abs(c)), (b, float(simple[b].detach()), c)
        P.check_bounds_properties(s[b].cpu().numpy(), Tb, Ub, R)
        total = total + 0.5 * _surrogate(sb, sl, gb, gl[:, :Ub])
        pb = torch.full((Tb, Ub + 1), -np.inf, dtype=torch.float64, device="cuda")
        pl = torch.full((Tb, max(Ub, 1)), -np.inf, dtype=torch.float64, device="cuda")
        pb2, pl2 = pb.clone(), pl.clone()
        for t in range(Tb):
            for r in range(R):
                uu = int(s[b, t]) + r
                if uu <= Ub:
                    pb2[t, uu] = lp[b, t, r, 0].detach()
                    if uu < Ub:
                        pl2[t, uu] = lp[b, t, r, yb[uu]].detach()
        c, gbp, glp, _, _ = E.lattice(pb2.cpu().numpy(), pl2[:, :Ub].cpu().numpy(), Tb, Ub, lam_f, lam_d)
        assert abs(float(pruned[b].detach()) - c) <= 1e-4 * max(1.0, abs(c)), (b, float(pruned[b].detach()), c)
        for t in range(Tb):
            for r in range(R):
                uu = int(s[b, t]) + r
                if uu <= Ub:
                    total = total + float(gbp[t, uu]) * lp[b, t, r, 0]
                    if uu < Ub:
                        total = total + float(glp[t, uu]) * lp[b, t, r, yb[uu]]
    total.backward()
    for k, p in ps.items():
        g = m.get_parameter(k).grad.double()
        err = float((g - p.grad).norm() / p.grad.norm().clamp(min=1e-12))
        assert err < 2e-3, (k, err)


def test_pruned_refuses_infeasible_utterance_with_options():
    from pika_b200 import engine
    V = 60
    x, y, fl, ll = _batch(V, (5, 9), (6, 8))                                        # utterance 0: U = 6 > T (R - 1) = 5
    m = _small_net(V, 2)
    with pytest.raises(ValueError, match=r"\[0\]"):
        engine.transducer_loss_pruned(m, x, y, fl, ll, 2, 0.5, 1.0, x_len=fl, fastemit_lambda=0.01, delay_penalty=0.01)
    with pytest.raises(ValueError, match="delay_penalty"):
        engine.transducer_loss(m, x, y, fl, ll, x_len=fl, delay_penalty=-1.0)


def _train_argv(tmp_path, lst, out, extra):
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--window-type=hamming\n--sample-frequency=16000\n--dither=0\n--low-freq=40\n--high-freq=-200\n--num-mel-bins=80\n")
    log = tmp_path / ("log.%s.WORKER-ID" % out.name)
    return str(log), ["transducer", lst, str(log), str(out), "--cuda", "--local_rank", "0", "--encoder_type", "transformer",
                      "--decoder_type", "rnn", "--rnn_size", "1024", "--embd_dim", "100", "--output_dim", "60", "--padding_idx", "60",
                      "--padding_tgt", "60", "--dec_layers", "2", "--dropout", "0.0", "--brnn", "--model_lctx", "21", "--model_rctx", "21",
                      "--model_stride", "4", "--lctx", "1", "--rctx", "1", "--feats_dim", "80", "--feat_config", str(cfg), "--batch_size", "4",
                      "--num_workers", "1", "--batch_first", "--max_len", "1600", "--TU_limit", "50000", "--gain_range", "25,25",
                      "--speed_rate", "1.0", "--grad_clip", "3.0", "--initial_lr", "0.002", "--final_lr", "0.001", "--momentum", "0.9",
                      "--num_epochs", "1", "--num_batches_per_epoch", "2", "--sync_period", "1", "--block_momentum", "0.9", "--block_lr",
                      "1.0", "--seed", "777"] + extra


@pytest.mark.parametrize("pruned", [False, True], ids=["dense", "pruned"])
def test_engine_at_zero_is_bit_identical_to_no_options(pruned):
    """transducer_loss(_pruned) with fastemit_lambda = delay_penalty = 0 against the call without them, on one model and one batch:
    costs and the loss-side parameter gradients (the joint's, and the simple projections'), which are formed in the loss's forward,
    bit for bit"""
    from pika_b200 import engine
    V, R = 61, 3
    x, y, fl, ll = _batch(V, (9, 6), (7, 4))
    engine.set_dropout_enabled(False)
    try:
        m = _small_net(V, R if pruned else 0)
        res = []
        for kw in ({}, dict(fastemit_lambda=0.0, delay_penalty=0.0)):
            m.zero_grad(set_to_none=True)
            if pruned:
                simple, costs = engine.transducer_loss_pruned(m, x, y, fl, ll, R, 0.5, 1.0, x_len=fl, **kw)
                (0.5 * simple + costs).sum().backward()
                costs = torch.cat((simple, costs))
            else:
                costs = engine.transducer_loss(m, x, y, fl, ll, x_len=fl, **kw)
                costs.sum().backward()
            res.append((costs.detach(), {k: p.grad.clone() for k, p in m.named_parameters() if k.startswith(("fc1", "fc_gate", "fc2",
                                                                                                            "simple_"))}))
    finally:
        engine.set_dropout_enabled(True)
    assert torch.equal(res[0][0], res[1][0])
    for k, g in res[0][1].items():
        assert torch.equal(g, res[1][1][k]), k


@pytest.mark.parametrize("pruned", [False, True], ids=["dense", "pruned"])
def test_train_cli_with_the_flags(tmp_path, pruned):
    """one epoch of the trainer with --fastemit_lambda / --delay_penalty (dense and --prune_range 4).  Flags at 0 train as no flags do:
    two runs of the trainer are not bit-identical (the encoder's backward sums in a run-dependent order), so the parameters after two
    steps are compared with the spread of two runs without flags, and the flags on must move them by more"""
    from test_loader_cpu import make_dataset
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    lst, _ = make_dataset(tmp_path, n_utts=8, shards=1, n_lo=14000, n_hi=22000)
    os.environ.setdefault("WORLD_SIZE", "1")
    prune = ["--prune_range", "4"] if pruned else []
    models = {}
    for name, extra in (("none", []), ("none2", []), ("zero", ["--fastemit_lambda", "0", "--delay_penalty", "0"]),
                        ("on", ["--fastemit_lambda", "0.01", "--delay_penalty", "0.002"])):
        out = tmp_path / name
        out.mkdir()
        log, argv = _train_argv(tmp_path, lst, out, prune + extra)
        T.main(argv)
        text = open(log.replace("WORKER-ID", "0")).read()
        assert "Training Finished" in text
        loss = [float(l.split("Loss:")[1].split()[0]) for l in text.splitlines() if "Overall Avg Loss" in l]
        assert len(loss) == 1 and np.isfinite(loss).all()
        models[name] = torch.load(str(out / "model.epoch.0.0"), weights_only=False).state_dict()

    def dist(a):
        return max(float((v.double() - models[a][k].double()).abs().max()) for k, v in models["none"].items() if v.is_floating_point())
    spread = dist("none2")
    assert dist("zero") <= max(2 * spread, 1e-6), (dist("zero"), spread)
    assert dist("on") > 10 * max(spread, 1e-7), (dist("on"), spread)


def test_mbr_train_cli_with_the_flags(tmp_path):
    """the MBR entry point inherits the flags and applies them to its RNN-T branch"""
    from test_loader_cpu import make_dataset
    from pika_b200.model.transducer import Net
    from pika_b200.trainer import train_transducer_mbr_bmuf_otfaug as M
    lst, _ = make_dataset(tmp_path, n_utts=4, shards=1, n_lo=14000, n_hi=18000)
    torch.manual_seed(777)
    margs = types.SimpleNamespace(rnn_size=1024, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="transformer", embd_dim=100,
                                  padding_idx=60, dropout=0.0, dec_layers=2, enc_layers=9)
    init = tmp_path / "init.model"
    torch.save(Net(margs, 240, 60), str(init))
    out = tmp_path / "out"
    out.mkdir()
    log, argv = _train_argv(tmp_path, lst, out, ["--init_model", str(init), "--beam_size", "4", "--rnnt_scale", "0.5", "--sm_scale", "0.8",
                                                 "--fastemit_lambda", "0.01", "--delay_penalty", "0.002"])
    argv[argv.index("--batch_size") + 1] = "2"
    os.environ.setdefault("WORLD_SIZE", "1")
    M.main(argv)
    text = open(log.replace("WORKER-ID", "0")).read()
    assert "Overall Avg RNNT Loss" in text and "Training Finished" in text
    m = torch.load(str(out / "model.epoch.0.0"), weights_only=False)
    assert bool(torch.isfinite(m.fc2.weight).all())
