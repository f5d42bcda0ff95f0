"""Gated joint kernels (pk_joint_gate_fwd / pk_joint_gate_bwd, csrc/elementwise.cu) called directly, against a float64
restatement on the same (for bf16: the same bf16-rounded) inputs:

    h[b,t,u]   = tanh(e1[b,t] + p1[b,u]) * sigmoid(eg[b,t] + pg[b,u])        ex = [e1 | eg] [B*T, 2H], py = [p1 | pg] [B*U1, 2H]
    dex[b,t]   = sum_u (dh*g*(1-a^2), dh*a*g*(1-g))                           a = tanh(e1+p1), g = sigmoid(eg+pg)
    dpy[b,u]   = sum_t (same terms)

The shapes reach every dispatch decision: the channel-sliced forward / fused backward (U+1 <= 160, H % 32 == 0, forward
only for T >= 8) with UI = ceil((U+1)/32) = 1..5 label blocks per lane, and the frame-major forward / two-pass backward
for U+1 > 160, H % 32 != 0 and (forward) T < 8."""
import pytest
import torch

pytestmark = pytest.mark.gpu

U1S = [1, 31, 32, 33, 64, 65, 128, 129, 151, 160, 161, 200, 300]
SHAPES = ([(2, T, U1, 128) for U1 in U1S for T in (1, 7, 8)]
          + [(2, 240, U1, 128) for U1 in (1, 33, 151, 160, 300)]
          + [(2, 8, 65, 1024), (3, 8, 160, 1024), (2, 7, 151, 1024), (2, 9, 200, 1024)]
          + [(2, 7, 33, 200), (3, 8, 65, 200), (2, 9, 161, 200), (2, 240, 151, 200)])
DTYPES = [torch.float32, torch.bfloat16]
SENTINEL = 77.0                       # exact in bf16; written nowhere by a correct kernel
# tanh.approx.f32 (the bf16 path's tanh, and its sigmoid through 0.5 * tanh(x / 2) + 0.5): the PTX ISA states a maximum
# relative error of 2^-11 over the full range
EPS_TANH = 2.0 ** -11


def _id(s):
    return "B%d-T%d-U1_%d-H%d" % s


def _inputs(shape, dtype, seed):
    B, T, U1, H = shape
    gen = torch.Generator(device="cuda").manual_seed(seed)
    ex = torch.randn(B * T, 2 * H, device="cuda", generator=gen).to(dtype)
    py = torch.randn(B * U1, 2 * H, device="cuda", generator=gen).to(dtype)
    return ex, py, gen


def _ref_act(ex, py, shape):
    """float64 (a, g) [B, T, U1, H] of the rounded inputs"""
    B, T, U1, H = shape
    s = ex.double().view(B, T, 1, 2 * H) + py.double().view(B, 1, U1, 2 * H)
    return torch.tanh(s[..., :H]), torch.sigmoid(s[..., H:])


def _ulp_bf16(x):
    """one bf16 ulp at |x| (0 at x == 0)"""
    m, e = torch.frexp(x.abs())
    return torch.where(m == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - 8))


def _fwd(ex, py, shape, pad):
    """h through pk_joint_gate_fwd with row pitch H + pad, into a buffer with one sentinel row after the last"""
    from pika_b200 import kernels
    B, T, U1, H = shape
    R = B * T * U1
    buf = torch.full((R + 1, H + pad), SENTINEL, dtype=ex.dtype, device="cuda")
    kernels.joint_gate_fwd(ex, py, buf[:R, :H], B, T, U1, H)
    torch.cuda.synchronize()
    assert torch.all(buf[R] == SENTINEL), "write past the last row"
    return buf[:R]


def _bwd(ex, py, dh, shape):
    from pika_b200 import kernels
    B, T, U1, H = shape
    dex = torch.full((B * T + 1, 2 * H), SENTINEL, dtype=ex.dtype, device="cuda")
    dpy = torch.full((B * U1 + 1, 2 * H), SENTINEL, dtype=ex.dtype, device="cuda")
    kernels.joint_gate_bwd(ex, py, dh, dex[:B * T], dpy[:B * U1], B, T, U1, H)
    torch.cuda.synchronize()
    assert torch.all(dex[B * T] == SENTINEL) and torch.all(dpy[B * U1] == SENTINEL), "write past the last row"
    return dex[:B * T].double(), dpy[:B * U1].double()


def _ref_bwd(a, g, dh, shape):
    """float64 (dex, dpy) and the matching sums of |terms| and of |dh|, all [rows, 2H]"""
    B, T, U1, H = shape
    d = dh.double().view(B, T, U1, H)
    dg = d * g
    terms = torch.cat((dg * (1 - a * a), dg * a * (1 - g)), -1)
    absd = torch.cat((d.abs(), d.abs()), -1)
    flat = lambda x, n: x.reshape(B * n, 2 * H)
    return ((flat(terms.sum(2), T), flat(terms.abs().sum(2), T), flat(absd.sum(2), T)),
            (flat(terms.sum(1), U1), flat(terms.abs().sum(1), U1), flat(absd.sum(1), U1)))


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_gate_fwd(shape, dtype):
    B, T, U1, H = shape
    ex, py, _ = _inputs(shape, dtype, seed=B * 100000 + T * 1000 + U1 + H)
    a, g = _ref_act(ex, py, shape)
    ref = (a * g).reshape(-1, H)
    if dtype == torch.float32:
        tol = torch.full_like(ref, 2e-6)
    else:
        # the approximate tanh's error in a and in g (|g' - g| <= 0.5 |tanh(x/2)| eps), then the output rounding
        tol = EPS_TANH * a.abs() * (g + 0.5 * (2 * g - 1).abs()) * (1 + 1e-3)
        tol = tol.reshape(-1, H) + _ulp_bf16(ref)
    outs = []
    for pad in (0, 8):                # pitch H (what the engine allocates) and H + 8 with the ones column of the fc2 bias gradient
        h = _fwd(ex, py, shape, pad)
        err = (h[:, :H].double() - ref).abs()
        assert torch.all(err <= tol), "pad %d: worst excess %g at row %d" % (pad, (err - tol).max().item(), int((err - tol).max(1).values.argmax()))
        if pad:
            one = torch.zeros(8, dtype=dtype, device="cuda")
            one[0] = 1
            assert torch.equal(h[:, H:], one.expand(h.shape[0], 8)), "pad columns must hold exactly (1, 0, ..., 0)"
        outs.append(h[:, :H])
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
def test_gate_bwd(shape, dtype):
    B, T, U1, H = shape
    ex, py, gen = _inputs(shape, dtype, seed=B * 100000 + T * 1000 + U1 + H + 7)
    dh = torch.randn(B * T * U1, H, device="cuda", generator=gen).to(dtype)
    a, g = _ref_act(ex, py, shape)
    (rex, mex, dex_abs), (rpy, mpy, dpy_abs) = _ref_bwd(a, g, dh, shape)
    dex, dpy = _bwd(ex, py, dh, shape)
    if dtype == torch.float32:
        # fp32 summation over at most 300 terms: 3e-5 of sum |terms| (one lost term out of ~150 is ~7e-3 of it).  Each term also
        # carries the absolute error of the fp32 tanh / sigmoid (a few 1e-8), which dominates where 1 - a^2 is tiny; 5e-7 |dh| covers it.
        for name, got, ref, mag, dabs in (("dex", dex, rex, mex, dex_abs), ("dpy", dpy, rpy, mpy, dpy_abs)):
            tol = 3e-5 * mag + 5e-7 * dabs + 1e-7
            err = (got - ref).abs()
            assert torch.all(err <= tol), "%s: worst excess %g" % (name, (err - tol).max().item())
    else:
        # the bf16 sums mix ~150 approximate terms; single missing terms are caught by test_gate_bwd_bf16_probes
        for name, got, ref in (("dex", dex, rex), ("dpy", dpy, rpy)):
            rel = ((got - ref).norm() / ref.norm()).item()
            assert rel < 1e-2, "%s: norm-relative error %g" % (name, rel)


PROBE_SHAPES = [(2, 8, 33, 128), (2, 9, 64, 128), (2, 8, 129, 128), (3, 7, 160, 128), (2, 8, 161, 128), (2, 12, 300, 128),
                (2, 1, 65, 128), (2, 24, 151, 1024), (2, 9, 151, 200)]


@pytest.mark.parametrize("shape", PROBE_SHAPES, ids=_id)
def test_gate_bwd_bf16_probes(shape):
    """bf16 backward with dh nonzero on a few rows only: (t, u) in {(0, 0), (T-1, 31), (0, 32), (T-1, U1-1)}, so that (for T > 1)
    every dex row has at most two terms and every dpy row at most two (u = 31 | 32 straddle both the lane halves of the fused
    kernel's butterfly and its first two label blocks; odd batch elements mirror t).  A missing, duplicated or misplaced term is
    then an O(1) error."""
    B, T, U1, H = shape
    ex, py, gen = _inputs(shape, torch.bfloat16, seed=B * 100000 + T * 1000 + U1 + H + 13)
    dh = torch.zeros(B, T, U1, H, device="cuda")
    for b in range(B):
        for t, u in ((0, 0), (T - 1, 31), (0, 32), (T - 1, U1 - 1)):
            if u < U1:
                tt = T - 1 - t if b % 2 else t
                dh[b, tt, u] = torch.randn(H, device="cuda", generator=gen)
    dh = dh.view(-1, H).to(torch.bfloat16)
    a, g = _ref_act(ex, py, shape)
    (rex, _, dex_abs), (rpy, _, dpy_abs) = _ref_bwd(a, g, dh, shape)
    dex, dpy = _bwd(ex, py, dh, shape)
    # per term: |d (1 - a'^2) g' - d (1 - a^2) g| <= 2.5 eps |d| and |d a' g' (1 - g') - d a g (1 - g)| <= 0.75 eps |d| for the
    # approximate tanh (eps = 2^-11), then one rounding of the fp32 sum to bf16 (<= 1 ulp)
    for name, got, ref, dabs in (("dex", dex, rex, dex_abs), ("dpy", dpy, rpy, dpy_abs)):
        tol = 3 * EPS_TANH * dabs + 2.0 ** -7 * ref.abs()
        err = (got - ref).abs()
        assert torch.all(err <= tol), "%s: worst excess %g at row %d" % (name, (err - tol).max().item(), int((err - tol).max(1).values.argmax()))
        assert torch.all(got[dabs == 0] == 0), "%s: nonzero output where no term exists" % name
    assert (rex != 0).any() and (rpy != 0).any()
