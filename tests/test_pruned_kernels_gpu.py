"""The pruned RNN-T kernels (include/pika_b200.h, "Pruned RNN-T loss") called directly through pika_b200/kernels.py, at training
shapes and at their documented limits, against float64 restatements built from the same rounded inputs.

Every output that the caller allocates goes into the head of a larger buffer whose tail holds sentinel values that a correct
kernel never writes.  Grid-stride sizes are derived from the device's SM count, so they loop several times on any card:
  simple_tables_kernel, simple_w_kernel, pruned_tables_kernel, pruned_rows_kernel: num_sms * 8 CTAs of 256 threads
  pruned_row_lse_kernel: num_sms * 32 CTAs of 8 warps, one warp per row
"""
import math

import numpy as np
import pytest
import torch

import pruned_rnnt_oracle as P
from test_joint_gate_gpu import EPS_TANH, _ulp_bf16

pytestmark = pytest.mark.gpu

SENT = 77.0                 # exact in bf16
SENT_I = -7777
GUARD = 61
FLOOR32 = np.float32(2.0 ** -100)
LOG2E = 1.0 / math.log(2.0)


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _wrap_nodes(times=3.5):
    """an element count that makes a num_sms * 8 x 256-thread grid-stride loop run more than ``times`` rounds"""
    return int(times * _nsm() * 8 * 256)


def _lens(v):
    return torch.tensor(list(v), dtype=torch.int32, device="cuda")


def _guarded(n, dtype, fill=None):
    """flat device buffer of n + GUARD elements, all sentinel"""
    f = (SENT_I if dtype == torch.int32 else SENT) if fill is None else fill
    return torch.full((n + GUARD,), f, dtype=dtype, device="cuda")


def _tail_ok(buf, n, what):
    torch.cuda.synchronize()
    assert bool((buf[n:] == buf[-1]).all()) and float(buf[-1]) in (SENT, SENT_I), "%s: write past the end" % what


def _raw(name, *args):
    from pika_b200 import _lib, kernels as K
    _lib.check(getattr(_lib.lib, name)(*args, K._stream()), name)


def _ws(name, *dims):
    from pika_b200 import _lib, kernels as K
    return K._ws_query(getattr(_lib.lib, name), name, *dims)


def _ragged(rng, B, T, U, t_min=1):
    """lengths with T_b = T and U_b = U for utterance 0, T_b = 1 and U_b = 0 for utterance 1 when B > 1, the rest random"""
    Ts = rng.integers(t_min, T + 1, B)
    Us = rng.integers(0, U + 1, B)
    Ts[0], Us[0] = T, U
    if B > 1:
        Ts[1], Us[1] = max(t_min, 1), 0
    return Ts.astype(np.int32), Us.astype(np.int32)


def _labels(rng, B, U, V):
    y = rng.integers(1, V, (B, max(U, 1))).astype(np.int32) if V > 1 else np.zeros((B, max(U, 1)), np.int32)
    y[0, 0] = V - 1
    if U >= 3:
        y[0, 2] = y[0, 1]                       # a repeated label
    return y


# ----------------------------------------------------------------------------------------------------------- pk_rnnt_simple_prep
@pytest.mark.parametrize("with_lo", [False, True], ids=["hi", "hi_lo"])
@pytest.mark.parametrize("V", [1, 255, 256, 257, 6000, 51200])
def test_simple_prep(V, with_lo):
    from pika_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(V)
    nb, n_in, n_out = 2, 3, 5
    ld_src, ld_out = V + 13, (V + 7) // 8 * 8 + 8
    src = torch.randn(nb * n_in, ld_src, device="cuda", generator=g) * 4
    src[:, V:] = 1e4                                                          # past V: never read
    src[1, :V] = -200.0
    src[1, V // 2] = 50.0                                                     # one dominant entry
    n = nb * n_out * ld_out
    hb = _guarded(n, torch.bfloat16)
    lb = _guarded(n, torch.bfloat16) if with_lo else None
    hi = hb[:n].view(nb * n_out, ld_out)
    lo = lb[:n].view(nb * n_out, ld_out) if with_lo else None
    rmax = K.rnnt_simple_prep(src, V, nb, n_in, n_out, hi, lo)
    _tail_ok(hb, n, "hi")
    if with_lo:
        _tail_ok(lb, n, "lo")
    x = src[:, :V]
    assert torch.equal(rmax, x.max(1).values)
    e = torch.exp(x.double() - x.double().max(1, keepdim=True).values)      # [nb*n_in, V]
    rows = torch.tensor([b * n_out + i for b in range(nb) for i in range(n_in)], device="cuda")
    pad_rows = torch.tensor([b * n_out + i for b in range(nb) for i in range(n_in, n_out)], device="cuda")
    h = hi[rows, :V].double()
    tiny = 2.0 ** -126                                                         # expf underflowing in f32 (the dominant-entry row)
    assert bool(((h - e).abs() <= _ulp_bf16(e) + tiny).all()), "hi further than 1 bf16 ulp from exp(x - m)"
    for buf in (hi, lo) if with_lo else (hi,):
        assert not buf[rows, V:].any() and not buf[pad_rows].any(), "padding columns / rows not zero"
    if with_lo:
        s = h + lo[rows, :V].double()
        assert bool(((s - e).abs() <= 2.0 ** -16 * e + tiny).all()), "hi + lo further than 2^-16 e from exp(x - m)"
    assert float(hi[rows[1], V // 2]) == 1.0


# ------------------------------------------------------------------------------------------ pk_rnnt_simple_tables[_smooth]
def _tables_inputs(rng, B, T, U1, V, special):
    ldv = (V + 7) // 8 * 8
    U1p = (U1 + 7) // 8 * 8
    Ts, Us = _ragged(rng, B, T, U1 - 1)
    y = _labels(rng, B, U1 - 1, V)
    am = (rng.standard_normal((B * T, ldv)) * 3).astype(np.float32)
    lm = (rng.standard_normal((B * U1, ldv)) * 3).astype(np.float32)
    am_max = (rng.standard_normal(B * T) * 2 + 5).astype(np.float32)
    lm_max = (rng.standard_normal(B * U1) * 2 + 5).astype(np.float32)
    S = np.exp(rng.standard_normal((B * T, U1p)) * 4).astype(np.float32)
    if special:                                 # at valid nodes of utterance 0: 0, a denormal, 2^-100 and its two neighbours
        vals = [0.0, 1e-40, FLOOR32, np.nextafter(FLOOR32, np.float32(1)), np.nextafter(FLOOR32, np.float32(0)), 1e-38]
        for k, v in enumerate(vals):
            S[k % T, k % U1] = v
    return Ts, Us, y, am, lm, am_max, lm_max, S


def _smooth_stats_inputs(rng, B, T, U1, ldv):
    Nl = (rng.standard_normal(B * U1) + 8).astype(np.float32)
    Na = (rng.standard_normal(B * T) + 8).astype(np.float32)
    logq = (-rng.random(ldv) * 9).astype(np.float32)
    return Nl, logq, Na


@pytest.mark.parametrize("smooth", [False, True], ids=["plain", "smooth"])
@pytest.mark.parametrize("size", ["small", "wrap"])
def test_simple_tables(size, smooth):
    rng = np.random.default_rng(7 if size == "small" else 8)
    if size == "small":
        B, T, U1, V = 4, 7, 6, 61
    else:
        T, U1, V = 240, 151, 16
        B = -(-_wrap_nodes() // (T * U1))
        assert B * T * U1 >= 3 * _nsm() * 8 * 256
    Ts, Us, y, am, lm, am_max, lm_max, S = _tables_inputs(rng, B, T, U1, V, special=(size == "small"))
    ldv, U1p = am.shape[1], S.shape[1]
    ND = T + U1 - 1
    n = B * ND * U1
    lpb_b, lpl_b = _guarded(n, torch.float32), _guarded(n, torch.float32)
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    d_am, d_lm, d_amx, d_lmx, d_S, d_y, d_T, d_U = map(c, (am, lm, am_max, lm_max, S, y, Ts, Us))
    lam_l, lam_a = 0.25, 0.125
    if smooth:
        Nl, logq, Na = _smooth_stats_inputs(rng, B, T, U1, ldv)
        d_Nl, d_logq, d_Na = c(Nl), c(logq), c(Na)
        _raw("pk_rnnt_simple_tables_smooth", d_am.data_ptr(), d_lm.data_ptr(), ldv, d_amx.data_ptr(), d_lmx.data_ptr(), d_S.data_ptr(),
             U1p, d_y.data_ptr(), y.shape[1], d_T.data_ptr(), d_U.data_ptr(), B, T, U1, d_Nl.data_ptr(), d_logq.data_ptr(),
             d_Na.data_ptr(), lam_l, lam_a, lpb_b.data_ptr(), lpl_b.data_ptr())
    else:
        _raw("pk_rnnt_simple_tables", d_am.data_ptr(), d_lm.data_ptr(), ldv, d_amx.data_ptr(), d_lmx.data_ptr(), d_S.data_ptr(), U1p,
             d_y.data_ptr(), y.shape[1], d_T.data_ptr(), d_U.data_ptr(), B, T, U1, lpb_b.data_ptr(), lpl_b.data_ptr())
    _tail_ok(lpb_b, n, "lpb")
    _tail_ok(lpl_b, n, "lpl")
    lpb, lpl = lpb_b[:n].double().cpu().numpy(), lpl_b[:n].double().cpu().numpy()
    # float64 restatement, vectorised over the nodes (b, t, u)
    b, t, u = np.meshgrid(np.arange(B), np.arange(T), np.arange(U1), indexing="ij")
    valid = (t < Ts[b]) & (u <= Us[b])
    lab = valid & (u < Us[b])
    ar, lr = b * T + t, b * U1 + u
    yl = np.where(u < y.shape[1], y[b, np.minimum(u, y.shape[1] - 1)], 0)
    A, L = am.astype(np.float64), lm.astype(np.float64)
    Sv = S[ar, u].astype(np.float64)
    logS = np.log(np.maximum(Sv, float(FLOOR32)))
    N = logS + am_max[ar] + lm_max[lr]
    mag0 = np.abs(logS) + np.abs(am_max[ar]) + np.abs(lm_max[lr])
    if smooth:
        mu = float(np.float32(1) - np.float32(lam_l) - np.float32(lam_a))

        def lp(k):
            full = (A[ar, k] + L[lr, k]) - N
            return (mu * full + lam_l * (L[lr, k] - Nl[lr]) + lam_a * (A[ar, k] + logq[k] - Na[ar]),
                    np.abs(A[ar, k]) + np.abs(L[lr, k]) + mag0 + np.abs(Nl[lr]) + np.abs(Na[ar]) + np.abs(logq[k]))
        rtol = 2.0 ** -19
    else:
        def lp(k):
            return (A[ar, k] + L[lr, k]) - N, np.abs(A[ar, k]) + np.abs(L[lr, k]) + mag0
        rtol = 2.0 ** -20
    sk = (b * ND + t + u) * U1 + u
    for name, got, ok, k in (("lpb", lpb, valid, np.zeros_like(u)), ("lpl", lpl, lab, yl)):
        ref, mag = lp(k)
        err = np.abs(got[sk[ok]] - ref[ok])
        assert (err <= rtol * mag[ok] + 1e-30).all(), "%s: worst excess %g" % (name, (err - rtol * mag[ok]).max())
        untouched = np.ones(n, bool)
        untouched[sk[ok]] = False
        assert (got[untouched] == SENT).all(), "%s: %d skew entries of invalid nodes written" % (name, int((got[untouched] != SENT).sum()))


# ----------------------------------------------------------------------------------------------------------- pk_rnnt_lattice
def _lattice_check(lpb_t, lpl_t, Ts, Us, T, U1, scale, tables_mask=None):
    """lpb_t / lpl_t [B, T, U1] float32 (numpy, node layout) -> run pk_rnnt_lattice on the skewed tables and compare with float64"""
    from pika_b200 import kernels as K
    B = len(Ts)
    ND = T + U1 - 1
    lpb_s = np.full((B, ND, U1), np.nan, np.float32)     # cells no valid node maps to stay NaN: the kernel must not read them
    lpl_s = np.full((B, ND, U1), np.nan, np.float32)
    for b in range(B):
        tt, uu = np.meshgrid(np.arange(Ts[b]), np.arange(Us[b] + 1), indexing="ij")
        lpb_s[b, tt + uu, uu] = lpb_t[b, :Ts[b], :Us[b] + 1]
        lpl_s[b, tt + uu, uu] = lpl_t[b, :Ts[b], :Us[b] + 1]
    sc = torch.from_numpy(scale).cuda()
    costs, gb, gl = K.rnnt_lattice(torch.from_numpy(lpb_s).cuda(), torch.from_numpy(lpl_s).cuda(), _lens(Ts), _lens(Us), B, T, U1, sc)
    costs, gb, gl = costs.cpu().numpy(), gb.cpu().numpy(), gl.cpu().numpy()
    assert np.isfinite(gb).all() and np.isfinite(gl).all(), "NaN / inf in the gradient coefficients"
    for b in range(B):
        Tb, Ub = int(Ts[b]), int(Us[b])
        c, rb, rl = P.occupancy(lpb_t[b, :Tb, :Ub + 1].astype(np.float64), lpl_t[b, :Tb, :Ub].astype(np.float64), Tb, Ub, fast=True)
        if not np.isfinite(c):
            assert costs[b] == np.inf and not gb[b].any() and not gl[b].any(), b
            continue
        assert abs(costs[b] - c) <= 2e-7 * abs(c) + 1e-6, (b, costs[b], c)
        np.testing.assert_allclose(gb[b, :Tb, :Ub + 1], scale[b] * rb, rtol=2e-6, atol=1e-30)
        np.testing.assert_allclose(gl[b, :Tb, :Ub + 1], scale[b] * rl, rtol=2e-6, atol=1e-30)
        assert not gb[b, Tb:].any() and not gb[b, :, Ub + 1:].any() and not gl[b, Tb:].any() and not gl[b, :, Ub:].any()
        if tables_mask is not None:
            off = ~tables_mask[b, :Tb, :Ub + 1]
            assert not gb[b, :Tb, :Ub + 1][off].any() and not gl[b, :Tb, :Ub + 1][off].any(), "nonzero occupancy outside the windows"
    return costs


def test_lattice_on_windowed_tables_at_training_size():
    """B = 32, T = 240, U1 = 151 with tables -inf outside windows of R = 5, a grad_scale per utterance and one utterance whose
    tables are -inf everywhere (cost +inf, zero coefficients)"""
    rng = np.random.default_rng(240)
    B, T, U1, R = 32, 240, 151, 5
    Ts, Us = _ragged(rng, B, T, U1 - 1, t_min=40)
    lpb = (-np.abs(rng.standard_normal((B, T, U1))) * 2 - 0.3).astype(np.float32)
    lpl = (-np.abs(rng.standard_normal((B, T, U1))) * 2 - 0.3).astype(np.float32)
    mask = np.zeros((B, T, U1), bool)
    for b in range(B):
        s = P.prune_bounds_fast(rng.random((Ts[b], Us[b] + 1)).astype(np.float32), Ts[b], Us[b], R)
        mask[b, :Ts[b], :Us[b] + 1] = P.window_mask(s, Ts[b], Us[b], R)
    mask[2] = False
    lpb = np.where(mask, lpb, -np.inf).astype(np.float32)
    lpl = np.where(mask, lpl, -np.inf).astype(np.float32)
    scale = (0.5 + rng.random(B) * 1.5).astype(np.float32)
    costs = _lattice_check(lpb, lpl, Ts, Us, T, U1, scale, mask)
    assert costs[2] == np.inf and np.isfinite(np.delete(costs, 2)).all()


def test_lattice_at_u1_2048():
    rng = np.random.default_rng(2048)
    T, U1 = 5, 2048
    Ts, Us = np.array([5, 3, 4], np.int32), np.array([2047, 1000, 0], np.int32)
    lpb = (-np.abs(rng.standard_normal((3, T, U1))) - 0.1).astype(np.float32)
    lpl = (-np.abs(rng.standard_normal((3, T, U1))) * 0.1 - 0.01).astype(np.float32)
    _lattice_check(lpb, lpl, Ts, Us, T, U1, np.array([1.0, 0.25, 3.0], np.float32))


# ----------------------------------------------------------------------------------------------------------- pk_rnnt_simple_w
@pytest.mark.parametrize("size", ["small", "wrap"])
@pytest.mark.parametrize("with_lo", [False, True], ids=["hi", "hi_lo"])
def test_simple_w(size, with_lo):
    from pika_b200 import kernels as K
    rng = np.random.default_rng(3 if size == "small" else 4)
    if size == "small":
        B, T, U1, ld_w = 3, 6, 5, 16
    else:
        T, U1, ld_w = 240, 151, 160
        B = -(-_wrap_nodes() // (T * ld_w))
    Ts, Us = _ragged(rng, B, T, U1 - 1)
    gb = (-rng.random((B, T, U1))).astype(np.float32)
    gl = (-rng.random((B, T, U1))).astype(np.float32)
    gb[0, 0, 1] = gl[0, 0, 1] = 0.0                                         # a zero occupancy
    ld_s = U1 + 3
    S = np.exp(rng.standard_normal((B * T, ld_s)) * 3).astype(np.float32)
    S[0, 0], S[1, 1], S[2, 2] = FLOOR32, np.nextafter(FLOOR32, np.float32(0)), 0.0     # exactly the floor, and clamped nodes
    scale = (0.5 + rng.random(B)).astype(np.float32)
    n = B * T * ld_w
    hb = _guarded(n, torch.bfloat16)
    lb = _guarded(n, torch.bfloat16) if with_lo else None
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    K.rnnt_simple_w(c(gb), c(gl), c(S), _lens(Ts), _lens(Us), c(scale), hb[:n].view(B * T, ld_w),
                    lb[:n].view(B * T, ld_w) if with_lo else None)
    _tail_ok(hb, n, "w_hi")
    if with_lo:
        _tail_ok(lb, n, "w_lo")
    # the kernel's f32 arithmetic, restated on the CPU: w = (scale * g) / s at the valid unclamped nodes
    b, t, u = np.meshgrid(np.arange(B), np.arange(T), np.arange(ld_w), indexing="ij")
    uc = np.minimum(u, U1 - 1)
    s = S[b * T + t, uc]
    g = -(gb[b, t, uc] + gl[b, t, uc])
    ok = (u < U1) & (t < Ts[b]) & (u <= Us[b]) & (s >= FLOOR32) & (g != 0)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        w = np.where(ok, (scale[b] * g) / np.where(ok, s, np.float32(1)), np.float32(0)).astype(np.float32)
    wt = torch.from_numpy(w.reshape(B * T, ld_w))
    hi = wt.to(torch.bfloat16)
    assert torch.equal(hb[:n].view(B * T, ld_w).cpu(), hi)
    if with_lo:
        assert torch.equal(lb[:n].view(B * T, ld_w).cpu(), (wt - hi.float()).to(torch.bfloat16))


# ----------------------------------------------------------------------------------------------------- pk_rnnt_simple_grad[_smooth]
def _grad_inputs(rng, V, axis):
    B, T, U1 = 2, 5, 4
    Ts, Us = np.array([5, 2], np.int32), np.array([3, 0], np.int32)
    ldv = (V + 7) // 8 * 8
    y = np.array([[V - 1, 7 % V, 7 % V], [1 % V, 1 % V, 1 % V]], np.int32)          # V - 1 and a repeated label
    rows_b = T if axis == 0 else U1
    n_g = rows_b + 2 if axis == 0 else (U1 + 7) // 8 * 8                              # the U1p padding of the engine's WtE
    src = np.full((B * rows_b, ldv), 1e4, np.float32)                                 # columns [V, ldv) are never read
    src[:, :V] = rng.standard_normal((B * rows_b, V)) * 3
    rmax = src[:, :V].max(1).astype(np.float32)
    ld_g = ldv + 8
    G = (rng.standard_normal((B * n_g, ld_g)) * 0.1).astype(np.float32)
    gb = np.full((B, T, U1), 1e3, np.float32)                                         # invalid nodes: never read
    gl = np.full((B, T, U1), 1e3, np.float32)
    for b in range(B):
        gb[b, :Ts[b], :Us[b] + 1] = -rng.random((Ts[b], Us[b] + 1))
        gl[b, :Ts[b], :Us[b] + 1] = -rng.random((Ts[b], Us[b] + 1))
    scale = np.array([0.7, 1.3], np.float32)
    return B, T, U1, Ts, Us, y, src, rmax, G, n_g, gb, gl, scale


def _grad_ref(B, T, U1, Ts, Us, y, src, rmax, G, n_g, axis, gb, gl, scale, V, smooth=None):
    """float64 (value, sum of |terms|) [rows, ldv] of the simple gradient rows"""
    rows_b = T if axis == 0 else U1
    ldv = src.shape[1]
    ref = np.zeros((B * rows_b, ldv))
    mag = np.zeros((B * rows_b, ldv))
    for b in range(B):
        Tb, Ub = int(Ts[b]), int(Us[b])
        sc = float(scale[b])
        for i in range(rows_b):
            r = b * rows_b + i
            e = np.exp(src[r, :V].astype(np.float64) - float(rmax[r])) * G[b * n_g + i, :V]
            ref[r, :V] = e
            mag[r, :V] = np.abs(e)
            k = sc if smooth is None else sc * (smooth["mu"] + smooth["lam"])
            blank = lab = 0.0
            terms = []                                 # (column, occupancy)
            if axis == 0 and i < Tb:
                blank = float(gb[b, i, :Ub + 1].astype(np.float64).sum())
                terms.append((0, blank, np.abs(gb[b, i, :Ub + 1]).sum()))
                for u in range(Ub):
                    lab += float(gl[b, i, u])
                    terms.append((y[b, u], float(gl[b, i, u]), abs(float(gl[b, i, u]))))
            elif axis == 1 and i <= Ub:
                blank = float(gb[b, :Tb, i].astype(np.float64).sum())
                terms.append((0, blank, np.abs(gb[b, :Tb, i]).sum()))
                if i < Ub:
                    lab = float(gl[b, :Tb, i].astype(np.float64).sum())
                    terms.append((y[b, i], lab, np.abs(gl[b, :Tb, i]).sum()))
            for col, v, m in terms:
                ref[r, col] += k * v
                mag[r, col] += abs(k) * m
            if smooth is not None:
                w = -(blank + lab) * sc * smooth["lam"]
                if w != 0.0:
                    lq = smooth["logq"][:V] if axis == 0 else 0.0
                    extra = w * np.exp(src[r, :V].astype(np.float64) + lq - float(smooth["lse"][r]))
                    ref[r, :V] += extra
                    mag[r, :V] += 2 * np.abs(extra)            # its exponent's f32 rounding: a few 1e-6 relative
    return ref, mag


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("V,smooth", [(61, False), (61, True), (6000, False), (8192, False), (12289, False), (12289, True),
                                      (51200, False), (51200, True)])
def test_simple_grad(V, smooth, axis, dtype):
    from pika_b200 import kernels as K
    rng = np.random.default_rng(V + axis)
    B, T, U1, Ts, Us, y, src, rmax, G, n_g, gb, gl, scale = _grad_inputs(rng, V, axis)
    rows, ldv = src.shape
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    args = (c(src), V, c(rmax), c(G), n_g, axis, c(gb), c(gl), c(y), _lens(Ts), _lens(Us), c(scale))
    sm = None
    if smooth:
        lam_l, lam_a = 0.25, 0.125
        logq = (-rng.random(ldv) * 9).astype(np.float32)
        lse = (rng.standard_normal(rows) + 9).astype(np.float32)
        mu = float(np.float32(1) - np.float32(lam_l) - np.float32(lam_a))
        sm = dict(mu=mu, lam=lam_a if axis == 0 else lam_l, logq=logq, lse=lse)
    outs = []
    for _ in range(2):
        buf = _guarded(rows * ldv, dtype)
        out = buf[:rows * ldv].view(rows, ldv)
        if smooth:
            K.rnnt_simple_grad_smooth(*args, c(logq), c(lse), lam_l, lam_a, out)
        else:
            K.rnnt_simple_grad(*args, out)
        _tail_ok(buf, rows * ldv, "out")
        outs.append(out)
    assert torch.equal(outs[0], outs[1]), "not bit-identical on repeat"
    got = outs[0].double().cpu().numpy()
    ref, mag = _grad_ref(B, T, U1, Ts, Us, y, src, rmax, G, n_g, axis, gb, gl, scale, V, sm)
    tol = 4e-6 * mag + 1e-30                     # exp(x - m) of f32 x - m up to ~24: ~1.5e-6 relative from the argument's rounding
    if dtype == torch.bfloat16:
        tol = tol + _ulp_bf16(torch.from_numpy(ref)).numpy()
    err = np.abs(got - ref)
    assert (err <= tol).all(), "worst excess %g at %s" % ((err - tol).max(), np.unravel_index((err - tol).argmax(), err.shape))
    assert not got[:, V:].any()


# -------------------------------------------------------------------------------------------------- pk_rnnt_simple_smooth_stats
@pytest.mark.parametrize("B,U1", [(1, 64), (5, 13), (32, 151), (65535, 64)], ids=["rows64", "rows65", "rows4832", "rows4194240"])
def test_smooth_stats_row_chunks(B, U1):
    """the float64 check of tests/test_pruned_smoothed_gpu.py (test_smooth_stats_against_float64_...) at B * U1 = 64 (one chunk of
    the unigram's 64-row partials), 65 (a last chunk of one row), 4832 (the training batch: 76 chunks, boundaries inside utterances)
    and 4194240 (the limit: 65535 chunks), with every padded row holding large values that must not enter a sum"""
    from pika_b200 import kernels as K
    rng = np.random.default_rng(B * 1000 + U1)
    T = 1 if B > 1000 else 9
    V = 8 if B > 1000 else 500
    ldv = (V + 7) // 8 * 8
    assert B * U1 <= 4194240
    Ts, Us = _ragged(rng, B, T, U1 - 1)
    g = torch.Generator(device="cuda").manual_seed(B + U1)
    am = torch.randn(B, T, ldv, device="cuda", generator=g) * 3
    lm = torch.randn(B, U1, ldv, device="cuda", generator=g) * 3
    fl, ll = _lens(Ts), _lens(Us)
    tv = torch.arange(T, device="cuda")[None, :] < fl[:, None].long()                 # [B, T] valid frames
    uv = torch.arange(U1, device="cuda")[None, :] <= ll[:, None].long()              # [B, U1] valid label positions
    am[~tv] = 50.0 + am[~tv]
    lm[~uv] = 50.0 + lm[~uv]
    am[..., V:] = 1e4
    lm[..., V:] = 1e4
    a2, l2 = am.view(B * T, ldv), lm.view(B * U1, ldv)
    am_max = a2[:, :V].max(1).values.contiguous()
    lm_max = l2[:, :V].max(1).values.contiguous()
    Nl, logq, Na = K.rnnt_simple_smooth_stats(a2, l2, V, am_max, lm_max, fl, ll, B, T, U1)
    L = lm[..., :V].double()
    nl_ref = torch.logsumexp(L, -1)                                                   # [B, U1]
    sm = torch.exp(L - nl_ref[..., None]) * uv[..., None]
    ref_q = torch.log(sm.sum((0, 1)) / uv.sum() + 1e-10)
    na_ref = torch.logsumexp(am[..., :V].double() + ref_q, -1)
    q_tol = 2e-4 if B * U1 > 100000 else 2e-5
    torch.testing.assert_close(logq[:V].double(), ref_q, rtol=0, atol=q_tol)
    assert not logq[V:].any()
    Nl, Na = Nl.view(B, U1), Na.view(B, T)
    torch.testing.assert_close(Nl[uv].double(), nl_ref[uv], rtol=2e-6, atol=4e-6)
    torch.testing.assert_close(Na[tv].double(), na_ref[tv], rtol=2e-6, atol=1e-5)
    assert not Nl[~uv].any() and not Na[~tv].any()


# -------------------------------------------------------------------------------------------------------- pk_rnnt_prune_bounds
BOUNDS_CASES = {
    # T, U1, R, [(T_b, U_b)]: a tight U = T_b (R-1), feasible utterances, an infeasible U = T_b (R-1) + 1, T_b = 1
    "T257_R2": (257, 257, 2, [(256, 256), (257, 100), (200, 201), (1, 0)]),
    "T1000_R64": (1000, 301, 64, [(999, 300), (5, 300), (4, 253), (4, 252), (1000, 30)]),
    "T12288_R4": (12288, 40, 4, [(12287, 39), (12288, 0), (13, 39), (3, 10)]),
}


@pytest.mark.parametrize("case", list(BOUNDS_CASES))
def test_prune_bounds_long_utterances(case):
    T, U1, R, lens = BOUNDS_CASES[case]
    rng = np.random.default_rng(T + R)
    B = len(lens)
    Ts = np.array([t for t, _ in lens], np.int32)
    Us = np.array([u for _, u in lens], np.int32)
    gamma = rng.random((B, T, U1)).astype(np.float32)
    gamma[0, :, 3] = 0.75                                                  # ties between window starts
    gamma[0, :, 4] = 0.75
    n = B * T
    sb = _guarded(n, torch.int32)
    d_ga, d_T, d_U = torch.from_numpy(-gamma).cuda(), _lens(Ts), _lens(Us)
    for _ in range(2):
        _raw("pk_rnnt_prune_bounds", d_ga.data_ptr(), None, d_T.data_ptr(), d_U.data_ptr(), B, T, U1, R, sb.data_ptr())
        _tail_ok(sb, n, "bounds")
        s = sb[:n].view(B, T).cpu().numpy()
        for b, (Tb, Ub) in enumerate(lens):
            if Ub > Tb * (R - 1):
                assert (s[b] == -1).all(), "infeasible utterance %d not marked -1" % b
                continue
            ref = P.prune_bounds_fast(gamma[b], Tb, Ub, R)
            np.testing.assert_array_equal(s[b, :Tb], ref)
            assert (s[b, Tb:] == ref[-1]).all()
            P.check_bounds_properties(s[b], Tb, Ub, R)
            if Ub == Tb * (R - 1):
                np.testing.assert_array_equal(ref, np.arange(Tb) * (R - 1))          # every start forced


# -------------------------------------------------------------------------------------------------- pk_joint_gate_pruned_fwd/_bwd
def _gate_bounds(T, U1, R):
    """[3, T] bounds: utterance 0 holds s = 0 for 210 frames (u = 0 .. R-1 each summed over 210 frames), then jumps past label
    positions no window covers and ends clamped at U1 - 1 with padded frames copying it; utterance 1 steps through every u;
    utterance 2 is infeasible (-1)"""
    s0 = np.zeros(T, np.int64)
    s0[210:220] = 3
    s0[220:225] = min(3 + R + 2, U1 - 1)
    s0[225:] = U1 - 1
    s1 = np.minimum(np.arange(T) // 7, U1 - 1)
    return np.stack([s0, s1, np.full(T, -1)]).astype(np.int32), np.array([228, T, T], np.int32), np.array([U1 - 1, U1 - 1, U1 - 1])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("R", [1, 2, 8, 64])
@pytest.mark.parametrize("H", [1, 127, 129, 1024])
def test_joint_gate_pruned(H, R, dtype):
    from pika_b200 import kernels as K
    B, T, U1 = 3, 232, 40
    g = torch.Generator(device="cuda").manual_seed(H * 100 + R)
    ex = torch.randn(B * T, 2 * H, device="cuda", generator=g).to(dtype)
    py = torch.randn(B * U1, 2 * H, device="cuda", generator=g).to(dtype)
    sn, Tn, Un = _gate_bounds(T, U1, R)
    s = torch.from_numpy(sn).cuda()
    rows = B * T * R
    hb = _guarded(rows * H, dtype)
    K.joint_gate_pruned_fwd(ex, py, s, hb[:rows * H].view(rows, H), B, T, U1, R, H)
    _tail_ok(hb, rows * H, "h")
    h = hb[:rows * H].view(B, T, R, H)
    sl = s.long()
    u = (sl.clamp(min=0)[:, :, None] + torch.arange(R, device="cuda")).clamp(max=U1 - 1)          # [B, T, R]
    e2, p2 = ex.double().view(B, T, 2 * H), py.double().view(B, U1, 2 * H)
    pu = p2[torch.arange(B, device="cuda")[:, None, None], u]                                      # [B, T, R, 2H]
    a = torch.tanh(e2[:, :, None, :H] + pu[..., :H])
    gg = torch.sigmoid(e2[:, :, None, H:] + pu[..., H:])
    ref = a * gg
    if dtype == torch.float32:
        tol = torch.full_like(ref, 2e-6)
    else:
        tol = EPS_TANH * a.abs() * (gg + 0.5 * (2 * gg - 1).abs()) * (1 + 1e-3) + _ulp_bf16(ref)
    err = (h.double() - ref).abs()
    assert bool((err <= tol).all()), "forward: worst excess %g" % (err - tol).max().item()
    del pu
    # dh zero on the rows the loss masks (u > U_b, t >= T_b, bound -1), as pk_rnnt_pruned_loss writes it
    raw = sl[:, :, None] + torch.arange(R, device="cuda")
    live = (raw <= torch.from_numpy(Un).cuda()[:, None, None]) & (torch.arange(T, device="cuda")[None, :, None] <
                                                                   torch.from_numpy(Tn).cuda()[:, None, None]) & (sl[:, :, None] >= 0)
    dh = (torch.randn(B, T, R, H, device="cuda", generator=g) * live[..., None]).to(dtype)
    outs = []
    for _ in range(2):
        xb, yb = _guarded(B * T * 2 * H, dtype), _guarded(B * U1 * 2 * H, dtype)
        K.joint_gate_pruned_bwd(ex, py, s, dh.view(rows, H), xb[:B * T * 2 * H].view(B * T, 2 * H), yb[:B * U1 * 2 * H].view(B * U1, 2 * H),
                                B, T, U1, R, H)
        _tail_ok(xb, B * T * 2 * H, "dex")
        _tail_ok(yb, B * U1 * 2 * H, "dpy")
        outs.append((xb[:B * T * 2 * H].view(B, T, 2 * H), yb[:B * U1 * 2 * H].view(B, U1, 2 * H)))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "not bit-identical on repeat"
    dex, dpy = outs[0][0].double(), outs[0][1].double()
    d = dh.double()
    terms = torch.cat((d * gg * (1 - a * a), d * a * gg * (1 - gg)), -1)                         # [B, T, R, 2H]
    absd = torch.cat((d.abs(), d.abs()), -1)
    del a, gg
    idx = u.view(B, T * R, 1).expand(-1, -1, 2 * H)
    rpy, mpy, apy = (torch.zeros(B, U1, 2 * H, dtype=torch.float64, device="cuda").scatter_add_(1, idx, x.view(B, T * R, 2 * H))
                     for x in (terms, terms.abs(), absd))
    checks = (("dex", dex, terms.sum(2), terms.abs().sum(2), absd.sum(2)), ("dpy", dpy, rpy, mpy, apy))
    for name, got, r, m, ad in checks:
        if dtype == torch.float32:
            tol = 3e-5 * m + 5e-7 * ad + 1e-7
        else:               # each term off by <= 2^-9 |dh| (approximate tanh), then one rounding of the f32 sum to bf16
            tol = 2.0 ** -9 * ad + 3e-5 * m + _ulp_bf16(r) + 1e-30
        err = (got - r).abs()
        assert bool((err <= tol).all()), "%s: worst excess %g" % (name, (err - tol).max().item())
    covered = torch.zeros(B, U1, dtype=torch.int32, device="cuda").scatter_add_(1, u.view(B, -1), live.view(B, -1).int()) > 0
    assert not dpy[~covered].any(), "dpy of a label position no live row covers must be exactly 0"
    assert int((sn[0] == 0).sum()) >= 200


# -------------------------------------------------------------------------------------- pk_rnnt_pruned_tables / pk_rnnt_pruned_loss
def _pruned_case(rng, B, T, U1, R, V, Ts=None, Us=None):
    """lengths, labels and valid bounds (from random occupancies) for windows of R; R = 1 keeps only U_b = 0 feasible"""
    if Ts is None:
        Ts, Us = _ragged(rng, B, T, U1 - 1, t_min=max(1, -(-(U1 - 1) // max(R - 1, 1))))
    y = _labels(rng, B, U1 - 1, V)
    s = np.zeros((B, T), np.int32)
    for b in range(B):
        if R == 1:
            s[b] = 0
        elif Us[b] <= Ts[b] * (R - 1):
            s[b, :Ts[b]] = P.prune_bounds_fast(rng.random((Ts[b], Us[b] + 1)).astype(np.float32), Ts[b], Us[b], R)
            s[b, Ts[b]:] = s[b, Ts[b] - 1]
        else:
            s[b] = -1
    return np.asarray(Ts, np.int32), np.asarray(Us, np.int32), y, s


def _pruned_ref(z, Ts, Us, y, s, R, V, utts=None):
    """float64 pruned loss of logits z [B*T*R, ldv] (device, the rounded values) -> costs [B], dlogits [B*T*R, ldv] (device, f64; rows
    of the utterances in ``utts`` only), lpb, lpl [B, T, U1] tables (numpy)"""
    B, T = s.shape
    ldv = z.shape[1]
    zr = z.view(B, T, R, ldv)
    costs = np.full(B, np.nan)
    dl = torch.zeros(B, T, R, ldv, dtype=torch.float64, device=z.device)
    for b in (range(B) if utts is None else utts):
        Tb, Ub = int(Ts[b]), int(Us[b])
        lp = torch.log_softmax(zr[b, :Tb, :, :V].double(), -1)                    # [Tb, R, V]
        if s[b, 0] < 0:
            costs[b] = np.inf
            continue
        uu = s[b, :Tb, None].astype(np.int64) + np.arange(R)[None, :]             # [Tb, R]
        tt = np.broadcast_to(np.arange(Tb)[:, None], uu.shape)
        ok = uu <= Ub
        yl = y[b, np.minimum(uu, max(Ub - 1, 0))]
        lpb = np.full((Tb, Ub + 1), -np.inf)
        lpl = np.full((Tb, max(Ub, 1)), -np.inf)
        lpc = lp.cpu().numpy()
        rr = np.broadcast_to(np.arange(R)[None, :], uu.shape)
        lpb[tt[ok], uu[ok]] = lpc[tt[ok], rr[ok], 0]
        okl = uu < Ub
        lpl[tt[okl], uu[okl]] = lpc[tt[okl], rr[okl], yl[okl]]
        c, gb, gl = P.occupancy(lpb, lpl[:, :Ub], Tb, Ub, fast=True)
        costs[b] = c
        if not np.isfinite(c):
            continue
        gbr = np.where(ok, gb[tt, np.minimum(uu, Ub)], 0.0)
        glr = np.where(okl, gl[tt, np.minimum(uu, Ub)], 0.0)
        g = torch.zeros(Tb, R, V, dtype=torch.float64, device=z.device)
        g[..., 0] += torch.from_numpy(gbr).to(z.device)
        ti, ri = np.nonzero(okl)
        g[torch.from_numpy(ti).to(z.device), torch.from_numpy(ri).to(z.device), torch.from_numpy(yl[ti, ri].astype(np.int64)).to(z.device)] += \
            torch.from_numpy(glr[ti, ri]).to(z.device)
        dl[b, :Tb, :, :V] = g - torch.exp(lp) * g.sum(-1, keepdim=True)
    return costs, dl.view(B * T * R, ldv)


def _hand_parts(z, V, splits):
    """float64 per-row (max * log2(e), sum 2^(x log2(e) - max)) partials over column groups, as pk_gemm_desc.row_lse, with an empty
    (-inf, 0) partial first"""
    zz = z[:, :V].double() * LOG2E
    edges = np.linspace(0, V, splits + 1).astype(int)
    parts = [torch.stack((torch.full((z.shape[0],), -math.inf, device=z.device, dtype=torch.float64),
                          torch.zeros(z.shape[0], device=z.device, dtype=torch.float64)), -1)]
    for a, b in zip(edges[:-1], edges[1:]):
        m = zz[:, a:b].max(1).values
        parts.append(torch.stack((m, torch.exp2(zz[:, a:b] - m[:, None]).sum(1)), -1))
    return torch.stack(parts).float().contiguous()


def _gemm_logits(rows, V, dtype, seed, with_lse):
    """fc2-style logits [rows, ldv] from pk_gemm_bf16 (bf16 C: with its row_lse partials, block_n 256)"""
    from pika_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(seed)
    ldv = (V + 7) // 8 * 8
    Hd = 128
    h = (torch.randn(rows, Hd, device="cuda", generator=g)).to(torch.bfloat16)
    w = (torch.randn(V, Hd, device="cuda", generator=g) * 0.4).to(torch.bfloat16)
    bias = torch.randn(V, device="cuda", generator=g)
    z = torch.zeros(rows, ldv, dtype=dtype, device="cuda")
    parts = None
    if with_lse:
        parts = torch.empty(K.row_lse_parts(rows, V, 256), rows, 2, dtype=torch.float32, device="cuda")
        K.gemm(h, w, z[:, :V], bias=bias, row_lse=parts, block_n=256)
    else:
        K.gemm(h, w, z[:, :V], bias=bias)
    return z, parts


@pytest.mark.parametrize("V,n_parts", [(64, 1), (520, 3), (6000, 24)])
def test_pruned_tables_row_lse_merge(V, n_parts):
    """pk_rnnt_pruned_tables with the fc2 GEMM's row_lse partials, with hand-built float64 partials behind an empty (-inf, 0) one, and
    streamed: the same tables, within 1e-5 of each other and of float64"""
    from pika_b200 import kernels as K
    rng = np.random.default_rng(V)
    B, T, U1, R = 4, 37, 12, 4
    Ts, Us, y, s = _pruned_case(rng, B, T, U1, R, V)
    z, parts = _gemm_logits(B * T * R, V, torch.bfloat16, V, True)
    assert parts.shape[0] == n_parts
    args = (torch.from_numpy(y).cuda(), _lens(Ts), _lens(Us), torch.from_numpy(s).cuda(), U1, R, V)
    res = {k: K.rnnt_pruned_tables(z, *args, row_lse=p) for k, p in
           (("stream", None), ("gemm", parts), ("hand", _hand_parts(z, V, 3)))}
    ND = T + U1 - 1
    bb, tt, uu = np.meshgrid(np.arange(B), np.arange(T), np.arange(U1), indexing="ij")
    valid = (tt < Ts[bb]) & (uu <= Us[bb])
    sk = torch.from_numpy(((bb * ND + tt + uu) * U1 + uu)[valid]).cuda()
    lab = torch.from_numpy(((uu < Us[bb]) & valid)[valid]).cuda()
    # float64 tables: log-softmax of the bf16 logits at the window rows
    lp = torch.log_softmax(z[:, :V].double(), -1).view(B, T, R, V)
    r = torch.from_numpy(uu - s[bb, tt]).cuda()[torch.from_numpy(valid).cuda()]
    bv, tv = torch.from_numpy(bb[valid]).cuda(), torch.from_numpy(tt[valid]).cuda()
    inw = (r >= 0) & (r < R)
    rc = r.clamp(0, R - 1)
    yv = torch.from_numpy(y).cuda().long()[bv, torch.from_numpy(np.minimum(uu[valid], y.shape[1] - 1)).cuda()]
    ref_b = torch.where(inw, lp[bv, tv, rc, 0], -math.inf)
    ref_l = torch.where(inw, lp[bv, tv, rc, yv], -math.inf)
    for k, (lpb, lpl) in res.items():
        gb_, gl_ = lpb.view(-1)[sk].double(), lpl.view(-1)[sk].double()
        assert torch.equal(torch.isinf(gb_), ~inw) and torch.equal(torch.isinf(gl_[lab]), ~inw[lab]), k
        torch.testing.assert_close(gb_[inw], ref_b[inw], rtol=1e-5, atol=1e-5, msg=k)
        torch.testing.assert_close(gl_[lab & inw], ref_l[lab & inw], rtol=1e-5, atol=1e-5, msg=k)
    for k in ("gemm", "hand"):
        a, b2 = res[k][0].view(-1)[sk], res["stream"][0].view(-1)[sk]
        fin = torch.isfinite(b2)
        torch.testing.assert_close(a[fin], b2[fin], rtol=1e-5, atol=1e-5, msg=k)


PRUNED_LOSS_CASES = {
    # name: (B, T, U1, R, V, dtype, row_lse partials: None | "gemm" | "hand", grad)
    "V2_R1_f32": (4, 9, 5, 1, 2, torch.float32, None, True),
    "V2_R8_gt_U1_f32": (4, 9, 5, 8, 2, torch.float32, None, True),
    "V64_R8_bf16_gemm1": (5, 30, 12, 8, 64, torch.bfloat16, "gemm", True),
    "V6000_R8_bf16_gemm24": (3, 40, 15, 8, 6000, torch.bfloat16, "gemm", True),
    "V6000_R1_bf16_hand": (4, 12, 6, 1, 6000, torch.bfloat16, "hand", True),
    "V8192_R8_f32": (2, 21, 9, 8, 8192, torch.float32, None, True),
    "V8192_R8_bf16_gemm32": (2, 21, 9, 8, 8192, torch.bfloat16, "gemm", True),
    "V10000_R8_lossonly_f32": (2, 21, 9, 8, 10000, torch.float32, None, False),
    "V10000_R8_lossonly_bf16_hand": (2, 21, 9, 8, 10000, torch.bfloat16, "hand", False),
}


def _run_pruned(z, parts, Ts, Us, y, s, U1, R, V, grad, inplace=False, scale=None):
    from pika_b200 import kernels as K
    rows, ldv = z.shape
    args = (torch.from_numpy(y).cuda(), _lens(Ts), _lens(Us), torch.from_numpy(s).cuda(), U1, R, V)
    if not grad:
        return K.rnnt_pruned_loss(z, *args, grad_scale=scale, row_lse=parts), None, None
    cb = _guarded(ldv, torch.float32)
    if inplace:
        dl = z
    else:
        db = _guarded(rows * ldv, z.dtype)
        dl = db[:rows * ldv].view(rows, ldv)
    c = K.rnnt_pruned_loss(z, *args, grad_scale=scale, dlogits=dl, colsum=cb[:ldv], row_lse=parts)
    _tail_ok(cb, ldv, "colsum")
    if not inplace:
        _tail_ok(db, rows * ldv, "dlogits")
    return c, dl, cb[:ldv]


@pytest.mark.parametrize("case", list(PRUNED_LOSS_CASES))
def test_pruned_loss_against_float64(case):
    """costs and dlogits against the float64 pruned lattice; one utterance with bounds -1 gives +inf and zero rows and leaves the
    others bit for bit as they are with valid bounds; the colsum is the column sum of the stored rows, 0 past V, reproducible; and the
    in-place call (dlogits = logits) stores the same bits"""
    B, T, U1, R, V, dtype, lse_kind, grad = PRUNED_LOSS_CASES[case]
    rng = np.random.default_rng(sum(map(ord, case)))
    Ts, Us, y, s = _pruned_case(rng, B, T, U1, R, V)
    rows = B * T * R
    z, parts = _gemm_logits(rows, V, dtype, len(case), lse_kind == "gemm") if dtype == torch.bfloat16 else (None, None)
    if z is None:
        ldv = (V + 7) // 8 * 8
        g = torch.Generator(device="cuda").manual_seed(len(case))
        z = torch.zeros(rows, ldv, device="cuda")
        z[:, :V] = torch.randn(rows, V, device="cuda", generator=g) * 2
    if lse_kind == "hand":
        parts = _hand_parts(z, V, 3)
    ldv = z.shape[1]
    zb = _guarded(rows * ldv, dtype)                                    # the logits themselves in a guarded buffer (in-place call)
    zb[:rows * ldv].view(rows, ldv).copy_(z)
    z = zb[:rows * ldv].view(rows, ldv)
    # utterance B-1 infeasible: its bounds -1
    s_bad = s.copy()
    s_bad[B - 1] = -1
    c1, dl1, cs1 = _run_pruned(z, parts, Ts, Us, y, s_bad, U1, R, V, grad)
    c0, dl0, cs0 = _run_pruned(z, parts, Ts, Us, y, s, U1, R, V, grad)
    ref_c, ref_dl = _pruned_ref(z, Ts, Us, y, s, R, V)
    c0, c1 = c0.cpu().numpy(), c1.cpu().numpy()
    assert c1[B - 1] == np.inf
    assert np.array_equal(c1[:B - 1], c0[:B - 1]), "an infeasible utterance changed the others' costs"
    fin = np.isfinite(ref_c)
    assert np.array_equal(np.isfinite(c0), fin), (c0, ref_c)
    np.testing.assert_allclose(c0[fin], ref_c[fin], rtol=2e-5, atol=1e-4)
    if not grad:
        return
    per = T * R
    assert not dl1[(B - 1) * per:].any(), "rows of the infeasible utterance not zero"
    assert torch.equal(dl1[:(B - 1) * per], dl0[:(B - 1) * per]), "an infeasible utterance changed the others' rows"
    got = dl0.double()
    tol = 1e-5 + (_ulp_bf16(ref_dl) if dtype == torch.bfloat16 else 2e-6 * ref_dl.abs())
    err = (got - ref_dl).abs()
    assert bool((err <= tol).all()), "dlogits: worst excess %g" % (err - tol).max().item()
    assert not dl0[:, V:].any()
    col = got.sum(0)
    torch.testing.assert_close(cs0.double(), col, rtol=0, atol=1e-5 * float(got.abs().sum(0).max()) + 1e-6)
    assert not cs0[V:].any()
    c2, dl2, cs2 = _run_pruned(z, parts, Ts, Us, y, s, U1, R, V, grad)
    assert torch.equal(dl2, dl0) and torch.equal(cs2, cs0) and np.array_equal(c2.cpu().numpy(), c0)
    c3, dl3, cs3 = _run_pruned(z, parts, Ts, Us, y, s, U1, R, V, grad, inplace=True)
    _tail_ok(zb, rows * ldv, "in-place dlogits")
    assert torch.equal(dl3, dl0) and torch.equal(cs3, cs0) and np.array_equal(c3.cpu().numpy(), c0)


def test_pruned_loss_wraps_every_grid_stride_loop():
    """B = 32, T = 240, U1 = 151 (1.16 M nodes) and R >= 112: B*T*R rows wrap pruned_rows_kernel's and pruned_row_lse_kernel's grids
    several times and the nodes wrap pruned_tables_kernel's; f32 streamed and bf16 with hand-built partials"""
    rng = np.random.default_rng(112)
    B, T, U1, V = 32, 240, 151, 16
    R = max(112, -(-int(3.05 * _nsm() * 8 * 256) // (B * T)))
    rows = B * T * R
    assert rows >= 3 * _nsm() * 8 * 256 and B * T * U1 >= 3 * _nsm() * 8 * 256 and rows >= 3 * _nsm() * 32 * 8
    Ts, Us = _ragged(rng, B, T, U1 - 1, t_min=2)
    Ts, Us, y, s = _pruned_case(rng, B, T, U1, R, V, Ts, Us)
    g = torch.Generator(device="cuda").manual_seed(3)
    for dtype in (torch.float32, torch.bfloat16):
        z = (torch.randn(rows, V, device="cuda", generator=g) * 2).to(dtype)
        parts = _hand_parts(z, V, 3) if dtype == torch.bfloat16 else None
        c, dl, cs = _run_pruned(z, parts, Ts, Us, y, s, U1, R, V, True)
        ref_c, ref_dl = _pruned_ref(z, Ts, Us, y, s, R, V)
        np.testing.assert_allclose(c.cpu().numpy(), ref_c, rtol=2e-5, atol=1e-4)
        tol = 1e-5 + (_ulp_bf16(ref_dl) if dtype == torch.bfloat16 else 2e-6 * ref_dl.abs())
        err = (dl.double() - ref_dl).abs()
        assert bool((err <= tol).all()), "%s dlogits: worst excess %g" % (dtype, (err - tol).max().item())
        torch.testing.assert_close(cs.double(), dl.double().sum(0), rtol=0, atol=1e-5 * float(dl.double().abs().sum(0).max()) + 1e-6)


# ------------------------------------------------------------------------------------------------------------ host-side rejection
def _rejected(fn, match):
    from pika_b200 import _lib
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(_lib.PikaError, match=match):
        fn()
    assert _lib.launch_count() == n0, "a kernel ran before the argument was rejected"


def test_arguments_rejected_before_any_launch():
    from pika_b200 import kernels as K
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device="cuda")                    # noqa: E731
    one = _lens([1])
    # simple_grad: a row over the 200 KB shared-memory limit (ldv = 51208)
    ldv = 51208
    for fn in (lambda: K.rnnt_simple_grad(z(1, ldv), ldv, z(1), z(1, ldv), 1, 0, z(1, 1, 1), z(1, 1, 1), _lens([0]), one, _lens([0]),
                                          None, z(1, ldv)),
               lambda: K.rnnt_simple_grad_smooth(z(1, ldv), ldv, z(1), z(1, ldv), 1, 0, z(1, 1, 1), z(1, 1, 1), _lens([0]), one,
                                                 _lens([0]), None, z(ldv), z(1), 0.1, 0.1, z(1, ldv))):
        _rejected(fn, "ldv")
    # bounds: T = 12289 frames (dynamic shared memory over 48 KB) and R = 1
    _rejected(lambda: K.rnnt_prune_bounds(z(1, 12289, 1), None, _lens([12289]), _lens([0]), 4), "T too large")
    _rejected(lambda: K.rnnt_prune_bounds(z(1, 4, 2), None, _lens([4]), _lens([1]), 1), "R must be")
    # smooth stats: B * U1 = 4194241 rows, one more than 65535 chunks of 64
    B = 4194241
    _rejected(lambda: K.rnnt_simple_smooth_stats(z(B, 8), z(B, 8), 8, z(B), z(B), _lens([1] * 1).repeat(B), torch.zeros(B, dtype=torch.int32,
                                                                                                                         device="cuda"),
                                                 B, 1, 1), "4194240")
    # pruned loss: a gradient at ldv = 8200 (> 8192)
    zl = z(1 * 2 * 2, 8200)
    _rejected(lambda: K.rnnt_pruned_loss(zl, _lens([1]).view(1, 1), _lens([2]), _lens([1]), _lens([0, 0]).view(1, 2), 2, 2, 8200,
                                         dlogits=torch.empty_like(zl)), "8192")
    # smoothing scales out of range: negative, summing to 1, NaN
    am, lm, S = z(2, 8), z(2, 8), z(2, 8)
    for lam in ((-0.1, 0.2), (0.5, 0.5), (float("nan"), 0.1), (0.2, float("nan"))):
        _rejected(lambda: K.rnnt_simple_tables_smooth(am, lm, z(2), z(2), S, _lens([1]).view(1, 1), _lens([2]), _lens([1]), 1, 2, 2, z(2),
                                                      z(8), z(2), *lam), "lm_only_scale")
        _rejected(lambda: K.rnnt_simple_grad_smooth(z(2, 8), 8, z(2), z(2, 8), 2, 0, z(1, 2, 2), z(1, 2, 2), _lens([1]).view(1, 1),
                                                    _lens([2]), _lens([1]), None, z(8), z(2), *lam, z(2, 8)), "lm_only_scale")


# ------------------------------------------------------------------------------------------------ one training-size step end to end
def test_training_size_simple_bounds_and_fused_pruned_loss():
    """engine.simple_loss -> bounds -> an fc2 GEMM with its row log-sum-exp partials -> pk_rnnt_pruned_loss in place, bf16, at
    B = 32, T = 240, U = 150, V = 6000, R = 5: the simple costs and gradients of three utterances and the pruned costs and dlogits rows
    of three against float64, the bounds bit-equal to the oracle on the lattice's own occupancies, and every pruned cost within 1e-5
    of the streamed call"""
    from pika_b200 import engine, kernels as K
    old = engine.get_precision()
    engine.set_precision("bf16")
    try:
        rng = np.random.default_rng(150)
        B, T, U, V, R = 32, 240, 150, 6000, 5
        U1 = U + 1
        Ts, Us = _ragged(rng, B, T, U, t_min=60)
        y = _labels(rng, B, U, V)
        g = torch.Generator(device="cuda").manual_seed(150)
        am = torch.randn(B * T, V, device="cuda", generator=g)
        lm = torch.randn(B * U1, V, device="cuda", generator=g)
        yd, fl, ll = torch.from_numpy(y).cuda(), _lens(Ts), _lens(Us)
        costs, bounds, dam, dlm = engine.simple_loss(am, lm, V, B, T, U1, yd, fl, ll, R, 1.0)
        # the lattice's own occupancies, through the same kernels, for the bounds oracle
        E = torch.empty(B * T, V, dtype=torch.bfloat16, device="cuda")
        U1p = (U1 + 7) // 8 * 8
        Pm = torch.empty(B * U1p, V, dtype=torch.bfloat16, device="cuda")
        am_max = K.rnnt_simple_prep(am, V, B, T, T, E)
        lm_max = K.rnnt_simple_prep(lm, V, B, U1, U1p, Pm)
        S = torch.empty(B, T, U1p, dtype=torch.float32, device="cuda")
        engine.gemm_parts([[E.view(B, T, V)]], [[Pm.view(B, U1p, V)]], S)
        lpb, lpl = K.rnnt_simple_tables(am, lm, am_max, lm_max, S.view(B * T, U1p), yd, fl, ll, B, T, U1)
        c2, gb, gl = K.rnnt_lattice(lpb, lpl, fl, ll, B, T, U1)
        assert torch.equal(c2, costs)
        b2 = K.rnnt_prune_bounds(gb, gl, fl, ll, R)
        assert torch.equal(b2, bounds)
        gamma = (-(gb + gl)).cpu().numpy()
        sn = bounds.cpu().numpy()
        for b in range(B):
            np.testing.assert_array_equal(sn[b, :Ts[b]], P.prune_bounds_fast(gamma[b], Ts[b], Us[b], R))
            assert (sn[b, Ts[b]:] == sn[b, Ts[b] - 1]).all()
        picks = [0, 1, int(np.argmin(Ts[2:])) + 2]
        amn, lmn = am.view(B, T, V).cpu().numpy(), lm.view(B, U1, V).cpu().numpy()
        dam3, dlm3 = dam.float().view(B, T, V).cpu().numpy(), dlm.float().view(B, U1, V).cpu().numpy()
        for b in picks:
            Tb, Ub = int(Ts[b]), int(Us[b])
            c, da, dl, _, _ = P.simple_loss(amn[b, :Tb], lmn[b, :Ub + 1], y[b, :Ub], fast=True)
            assert abs(float(costs[b]) - c) <= 2e-2 * max(1.0, abs(c)), (b, float(costs[b]), c)
            np.testing.assert_allclose(dam3[b, :Tb], da, rtol=1e-2, atol=3e-2)          # dlm's blank column sums ~240 frames
            np.testing.assert_allclose(dlm3[b, :Ub + 1], dl, rtol=1e-2, atol=3e-2)
        # the pruned joint's fc2 with its row log-sum-exp partials (24 of them), then the loss in place over the logits
        rows = B * T * R
        z, parts = _gemm_logits(rows, V, torch.bfloat16, 5, True)
        assert parts.shape[0] == 24
        zq = z.clone()
        c_stream = K.rnnt_pruned_loss(z, yd, fl, ll, bounds, U1, R, V, row_lse=None)
        cs = torch.empty(V, device="cuda")
        c_fused = K.rnnt_pruned_loss(z, yd, fl, ll, bounds, U1, R, V, dlogits=z, colsum=cs, row_lse=parts)
        torch.testing.assert_close(c_fused, c_stream, rtol=1e-5, atol=0)
        ref_c, ref_dl = _pruned_ref(zq, Ts, Us, y, sn, R, V, utts=picks)
        for b in picks:
            assert abs(float(c_fused[b]) - ref_c[b]) <= 2e-5 * abs(ref_c[b]) + 1e-4, (b, float(c_fused[b]), ref_c[b])
            r0, r1 = b * T * R, (b + 1) * T * R
            err = (z[r0:r1].double() - ref_dl[r0:r1]).abs()
            tol = 1e-5 + _ulp_bf16(ref_dl[r0:r1])
            assert bool((err <= tol).all()), "utterance %d dlogits: worst excess %g" % (b, (err - tol).max().item())
    finally:
        engine.set_precision(old)
