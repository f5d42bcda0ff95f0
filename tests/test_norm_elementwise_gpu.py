"""The memory-bound kernels of csrc/elementwise.cu called directly through the C ABI, f32 and bf16 on every path, against float64
restatements:

    pk_colsum                          every bias gradient (two-stage column sum: row slices, then a fixed-order reduce)
    pk_bn_fwd / pk_bn_bwd              every TDNN BatchNorm, with and without the ReLU mask
    pk_layernorm_fwd / _bwd            every transformer layer
    pk_cast_split                      the hi / lo bf16 operands of the fp32-class GEMMs and the scaled Q copy
    pk_dropout / pk_mask_nz / pk_add   Linear backward, MBR bias gradients, LSTM bias sums
    pk_log_softmax / pk_row_lse        decode
    pk_lstm_cell_fwd / _bwd            the fp32 prediction net and the beam step
    pk_embedding_fwd / _bwd, pk_gather_rows / pk_scatter_add_rows, pk_ce_grad      prediction net, ragged LSTM, MBR trainer

Every reference takes the kernel's own stored inputs: the BatchNorm / LayerNorm output and backward references use the mean / rstd
the forward wrote.  So each bound is the rounding of one step, not of a chain.  Sums are bounded by their summation order's worst
case (a sequential sum of k terms is off by at most k * 2^-24 * sum |term|), not by a norm-relative figure.  Errors are bounded
element by element, and a failure names the first offending (row, column).  Every output is filled with NaN before the call, with
one extra row or element past its end: each element must be written and nothing past the end.  The largest err / bound of each check
is printed when the module finishes; the figures beside the bounds were measured on an H100 80GB HBM3 (700 W)."""
import ctypes
import math

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}
CODE = {torch.float32: 0, torch.bfloat16: 1}         # PK_F32, PK_BF16
MANT = {torch.float32: 24, torch.bfloat16: 8}
U = 2.0 ** -24                                        # unit roundoff of f32
TINY = 1e-37
_WORST = {}
_SEEN = {}                                            # measured figures that are not ratios to a bound


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _WORST:
        print("\nlargest err / bound: " + ", ".join("%s %.3g" % kv for kv in sorted(_WORST.items())))
    if _SEEN:
        print("largest measured: " + ", ".join("%s %.3g" % kv for kv in sorted(_SEEN.items())))


def _k():
    from pika_b200 import kernels
    return kernels


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


L, I, F, U32 = ctypes.c_longlong, ctypes.c_int, ctypes.c_float, ctypes.c_uint32


def _abi(name, *args):
    """pk_<name>(args..., current stream): tensors pass as device pointers, None as NULL, everything else as the ctypes value given.
    Asserts a zero status and waits for the device."""
    from pika_b200 import _lib
    conv = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else ctypes.c_void_p(0) if a is None else a for a in args]
    rc = getattr(_lib.lib, name)(*conv, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, "%s: rc=%d %s" % (name, rc, _lib.lib.pk_last_error().decode())
    torch.cuda.synchronize()


def _ws_floats(C):
    from pika_b200 import _lib
    return int(_lib.lib.pk_colstats_ws_floats(C))


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, math.nan, dtype=dtype, device="cuda")


def _body(buf, n, what):
    """the first n rows (elements) of a NaN-filled buffer whose remainder the kernel must not touch"""
    assert bool(torch.isnan(buf[n:].float()).all()), "%s: write past the end" % what
    return buf[:n]


def half_ulp(x, dtype):
    m, e = torch.frexp(x.abs())
    return torch.where(m == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - 1 - MANT[dtype]))


def _check(what, got, ref, tol):
    """|got - ref| <= tol element by element (a NaN fails; tol 0 demands equality); records the largest err / tol"""
    err = (got.double() - ref).abs()
    ok = err <= tol
    if not bool(ok.all()):
        at = tuple((~ok).nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements outside the bound; first at %s: got %r, reference %r, bound %r"
                             % (what, int((~ok).sum()), ok.numel(), at, got[at].item(), ref[at].item(), tol[at].item()))
    ratio = torch.where(tol > 0, err / tol.clamp_min(1e-300), torch.zeros_like(err))
    _WORST[what] = max(_WORST.get(what, 0.0), float(ratio.max()) if ratio.numel() else 0.0)


def _equal(what, got, ref):
    if not torch.equal(got, ref):
        bad = (got != ref) & ~(torch.isnan(got.float()) & torch.isnan(ref.float()))
        at = tuple(bad.nonzero()[0].tolist()) if bool(bad.any()) else ()
        raise AssertionError("%s: not bit-equal; first at %s: got %r, expected %r" % (what, at, got[at].item(), ref[at].item()))


def _chunked_colsums(x, chunk=1 << 14):
    """float64 (sum x, sum |x|) over the rows of a large x without a float64 copy of all of it"""
    s = torch.zeros(x.shape[1], dtype=torch.float64, device="cuda")
    a = torch.zeros_like(s)
    for r in range(0, x.shape[0], chunk):
        xd = x[r:r + chunk].double()
        s += xd.sum(0)
        a += xd.abs().sum(0)
    return s, a


def colstats_depth(rows):
    """terms on the longest path of the column-statistics sum: a row slice of ceil(rows / gy) rows summed in one thread, then the
    slices strided over 8 threads, then those 8 (gy = min(296, ceil(rows / 64)) slices)"""
    gy = max(1, min(296, -(-rows // 64)))
    return -(-rows // gy) + -(-gy // 8) + 8


# ------------------------------------------------------------------------------------------------ 1. column sums
COLSUM_C = [8, 40, 1024, 1032, 6008]
COLSUM_ROWS = [1, 7, 63, 64, 65, 64 * 296, 64 * 296 + 1, 300_001]


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("rows", COLSUM_ROWS)
@pytest.mark.parametrize("C", COLSUM_C)
def test_colsum(C, rows, dtype):
    """bound: (depth + 1) 2^-24 sum |x|.  Measured: at most 0.16 of it (f32), 0.043 (bf16)."""
    dt = DTYPES[dtype]
    x = (torch.randn(rows, C, device="cuda", generator=_gen(rows * 7 + C)) + 0.5).to(dt)
    out = _nan(C + 1)
    ws = _nan(_ws_floats(C))
    _abi("pk_colsum", x, I(CODE[dt]), L(rows), I(C), out, ws)
    got = _body(out, C, "colsum").clone()
    ref, mag = _chunked_colsums(x)
    _check("colsum %s" % dtype, got, ref, (colstats_depth(rows) + 1) * U * mag + TINY)
    ws.fill_(math.nan)
    _abi("pk_colsum", x, I(CODE[dt]), L(rows), I(C), out, ws)
    _equal("colsum repeated call", out[:C], got)


# ------------------------------------------------------------------------------------------------ 2. BatchNorm
# channel c draws from kind c % 8: N(0,1); ReLU outputs (exact zeros, some of them -0.0); the constant 0.75 (rstd = 1/sqrt(eps));
# and channels whose mean is large against their spread -- an almost-always-on ReLU channel, bn_final after a residual stream.
BN_KINDS = ["normal", "relu", "const", "m5s.05", "m5s.01", "m20s.1", "off256", "s3"]
BN_LOC = [0.0, 0.0, 0.75, 5.0, 5.0, 20.0, 256.0, 0.0]
BN_SCALE = [1.0, 1.0, 0.0, 0.05, 0.01, 0.1, 1.0, 3.0]
BN_C = [8, 256, 1000, 1032, 2048]
BN_ROWS = [2, 15, 16, 17, 333, 9600, 64 * 296 + 1]
EPS_BN = 1e-5


def bn_input(rows, C, dt, gen):
    kind = torch.arange(C, device="cuda") % 8
    z = torch.randn(rows, C, device="cuda", generator=gen)
    loc = torch.tensor(BN_LOC, device="cuda")[kind]
    sc = torch.tensor(BN_SCALE, device="cuda")[kind]
    x = loc + sc * z
    flip = torch.rand(rows, C, device="cuda", generator=gen) < 0.5
    relu = torch.where((z <= 0) & flip, torch.full_like(z, -0.0), z.clamp_min(0.0))
    x = torch.where(kind == 1, relu, x)
    return x.to(dt)


def bn_stats_ref(x):
    """float64 (mean, biased var) per channel and the bounds of the kernel's shifted sums: the kernel sums d = x - x[0] and d^2, so
    mean = x[0] + s1/n is off by (depth + 2) 2^-24 sum |d| / n, and var = s2/n - (s1/n)^2 by 4 (depth + 4) 2^-24 sum d^2 / n
    (|s1/n| <= sum |d| / n <= sqrt(sum d^2 / n) bounds every other term)."""
    n = x.shape[0]
    xd = x.double()
    mean = xd.mean(0)
    var = ((xd - mean) ** 2).mean(0)
    d = xd - xd[0]
    g = (colstats_depth(n) + 2) * U
    a1, a2 = d.abs().sum(0) / n, (d * d).sum(0) / n
    return mean, var, g * a1 + 2 * U * (mean.abs() + a1) + TINY, 4 * (g + 2 * U) * a2 + TINY


def rstd_tol(var, tol_var, eps):
    """the interval of 1/sqrt(v + eps) over |v - var| <= tol_var, plus the f32 add and rsqrtf (2 ulp)"""
    r = 1.0 / torch.sqrt(var + eps)
    lo = 1.0 / torch.sqrt(var + eps + tol_var)
    hi = 1.0 / torch.sqrt((var + eps - tol_var).clamp_min(1e-300))
    return r, torch.maximum(r - lo, hi - r) + 6 * U * r


def _record_rstd(tag, got, ref, kinds):
    rel = ((got.double() - ref).abs() / ref)
    for k, name in enumerate(BN_KINDS):
        sel = kinds == k
        if bool(sel.any()):
            key = "bn rstd rel err %s %s" % (name, tag)
            _SEEN[key] = max(_SEEN.get(key, 0.0), float(rel[sel].max()))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("relu_mask", [0, 1])
@pytest.mark.parametrize("train", [1, 0], ids=["train", "eval"])
@pytest.mark.parametrize("rows", BN_ROWS)
@pytest.mark.parametrize("C", BN_C)
def test_batchnorm(C, rows, train, relu_mask, dtype):
    """forward (statistics, running statistics, y) and then backward on the forward's stored mean / rstd.
    Measured: mean at most 0.50 of its bound, rstd 0.26, running mean 0.62, running var 0.59, eval rstd 0.38, y 0.91 (f32) / 1 (bf16:
    the half ulp is attained), db 0.13, dw 0.18, dx 0.66 (f32) / 1 (bf16).  The largest relative rstd error of any channel kind is
    1.4e-5 (f32, a ReLU channel); the large-mean kinds stay below 1.9e-6.  Unshifted sums (sum x, sum x^2) failed the mean
    and rstd bounds on these channels, at relative rstd errors up to 26 (offset 256, f32)."""
    dt = DTYPES[dtype]
    gen = _gen(C * 100003 + rows * 17 + train * 3 + relu_mask)
    x = bn_input(rows, C, dt, gen)
    kinds = torch.arange(C, device="cuda") % 8
    w = torch.rand(C, device="cuda", generator=gen) * 1.5 + 0.25
    b = torch.randn(C, device="cuda", generator=gen) * 0.5
    rm0 = torch.randn(C, device="cuda", generator=gen) * 0.3
    rv0 = torch.rand(C, device="cuda", generator=gen) + 0.5
    rm, rv = torch.cat([rm0, _nan(1)]), torch.cat([rv0, _nan(1)])
    mom = 0.1
    y, mean, rstd = _nan(rows + 1, C, dtype=dt), _nan(C + 1), _nan(C + 1)
    ws = _nan(_ws_floats(C) + 2 * C)
    _abi("pk_bn_fwd", x, y, I(CODE[dt]), L(rows), I(C), w, b, F(EPS_BN), I(train), F(mom), rm, rv, mean, rstd, ws)
    y, mean, rstd = _body(y, rows, "bn y"), _body(mean, C, "bn mean"), _body(rstd, C, "bn rstd")
    rm, rv = _body(rm, C, "running mean"), _body(rv, C, "running var")
    if train:
        m_ref, v_ref, tol_m, tol_v = bn_stats_ref(x)
        _check("bn mean", mean, m_ref, tol_m)
        r_ref, tol_r = rstd_tol(v_ref, tol_v, EPS_BN)
        _record_rstd(dtype, rstd, r_ref, kinds)
        _check("bn rstd", rstd, r_ref, tol_r)
        # nn.BatchNorm1d: running_var takes the unbiased variance; momentum 0.1
        n = rows
        unb = v_ref * n / (n - 1) if n > 1 else v_ref
        rm_ref = (1 - mom) * rm0.double() + mom * m_ref
        rv_ref = (1 - mom) * rv0.double() + mom * unb
        _check("bn running mean", rm, rm_ref, mom * tol_m + 3 * U * ((1 - mom) * rm0.double().abs() + mom * m_ref.abs()) + TINY)
        _check("bn running var", rv, rv_ref, mom * tol_v * n / max(n - 1, 1) + 4 * U * ((1 - mom) * rv0.double() + mom * unb) + TINY)
    else:
        _equal("bn eval mean", mean, rm0)
        r_ref = 1.0 / torch.sqrt(rv0.double() + EPS_BN)
        _check("bn eval rstd", rstd, r_ref, 6 * U * r_ref)
        _equal("bn eval running mean", rm, rm0)
        _equal("bn eval running var", rv, rv0)
    # y = x * sc + sh, sc = rstd * w and sh = b - mean * sc rounded to f32
    xd, md, rd, wd, bd = x.double(), mean.double(), rstd.double(), w.double(), b.double()
    sc = rd * wd
    y_ref = (xd - md) * sc + bd
    inner = 2 * U * (xd.abs() * sc + (md * sc).abs() + bd.abs())
    _check("bn y %s" % dtype, y, y_ref, inner + half_ulp(y_ref.abs() + inner, dt) + TINY)

    dy = torch.randn(rows, C, device="cuda", generator=gen).to(dt)
    dx, dw, db = _nan(rows + 1, C, dtype=dt), _nan(C + 1), _nan(C + 1)
    ws2 = _nan(_ws_floats(C))
    _abi("pk_bn_bwd", dy, x, dx, I(CODE[dt]), L(rows), I(C), w, mean, rstd, I(train), I(relu_mask), dw, db, ws2)
    dx, dw, db = _body(dx, rows, "bn dx"), _body(dw, C, "bn dw"), _body(db, C, "bn db")
    dyd = dy.double()
    xhat = (xd - md) * rd
    g = colstats_depth(rows) * U
    db_ref, dw_ref = dyd.sum(0), (dyd * xhat).sum(0)
    tol_db = (g + U) * dyd.abs().sum(0) + TINY
    tol_dw = (g + 4 * U) * (dyd * xhat).abs().sum(0) + TINY
    _check("bn db", db, db_ref, tol_db)
    _check("bn dw", dw, dw_ref, tol_dw)
    a = wd * rd
    if train:
        n = rows
        k = rd * dw_ref / n
        dx_ref = a * (dyd - db_ref / n - xhat * dw_ref / n)
        inner = a * (tol_db + xhat.abs() * tol_dw) / n + 4 * U * ((a * dyd).abs() + (a * k).abs() * (xd.abs() + md.abs()) + (a * db_ref / n).abs())
    else:
        dx_ref = a * dyd
        inner = 2 * U * (a * dyd).abs()
    tol = inner + half_ulp(dx_ref.abs() + inner, dt) + TINY
    if relu_mask:
        off = ~(x.float() > 0)                         # x <= 0, -0.0 included: torch's ReLU backward gives exactly 0 there
        dx_ref = torch.where(off, torch.zeros_like(dx_ref), dx_ref)
        tol = torch.where(off, torch.zeros_like(tol), tol)
    _check("bn dx %s" % dtype, dx, dx_ref, tol)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("rows,loc,scale", [(9600, 5.0, 0.05), (9600, 5.0, 0.01), (40000, 20.0, 0.1), (9600, 256.0, 1.0),
                                             (40000, 256.0, 1.0)])
def test_batchnorm_large_mean_statistics(rows, loc, scale, dtype):
    """channels whose mean is large against their spread: forming the variance as sum(x^2)/n - mean^2 from f32 sums cancels.
    Relative rstd error measured with those unshifted sums (f32 / bf16): 5 +- 0.05 at 9600 rows 2.3e-3 / 1.1e-3, 5 +- 0.01 4.6e-2 /
    2.4e-2, 20 +- 0.1 at 40000 rows 8.1e-3 / 4.2e-3, 256 +- 1 at 9600 and 40000 rows 1.6e-2 / 6.2e-3.  With the shifted sums: at most
    1.6e-6, 0.016 of the rstd bound; the mean at most 0.43 of its bound."""
    dt = DTYPES[dtype]
    C = 1024
    x = (loc + scale * torch.randn(rows, C, device="cuda", generator=_gen(rows + int(loc)))).to(dt)
    w, b = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    y, mean, rstd = torch.empty_like(x), _nan(C), _nan(C)
    _abi("pk_bn_fwd", x, y, I(CODE[dt]), L(rows), I(C), w, b, F(EPS_BN), I(1), F(0.1), rm, rv, mean, rstd, _nan(_ws_floats(C) + 2 * C))
    m_ref, v_ref, tol_m, tol_v = bn_stats_ref(x)
    r_ref, tol_r = rstd_tol(v_ref, tol_v, EPS_BN)
    key = "bn rstd rel err rows%d loc%g s%g %s" % (rows, loc, scale, dtype)
    _SEEN[key] = float(((rstd.double() - r_ref).abs() / r_ref).max())
    _check("bn large-mean mean", mean, m_ref, tol_m)
    _check("bn large-mean rstd", rstd, r_ref, tol_r)


@pytest.mark.parametrize("momentum", [0.1, None])
def test_batchnorm_running_stats_match_torch(momentum):
    """BatchNormFn's running statistics over several steps against nn.BatchNorm1d in float64: momentum None is torch's cumulative
    average, factor 1 / num_batches_tracked after the increment.  The bound carries the batch statistics' bounds (bn_stats_ref) and
    the update's roundings from step to step.  Measured: at most 0.036 of it."""
    from pika_b200 import engine as E
    C, rows = 256, 700
    bn = nn.BatchNorm1d(C, momentum=momentum).cuda().train()
    ref = nn.BatchNorm1d(C, momentum=momentum).cuda().double().train()
    gen = _gen(5)
    tol_rm = tol_rv = 0.0
    for step in range(4):
        x = torch.randn(rows, C, device="cuda", generator=gen) * (1 + step) + step
        rm0, rv0 = ref.running_mean.clone(), ref.running_var.clone()
        E.BatchNormFn.apply(x, bn, True, bn.weight, bn.bias)
        with torch.no_grad():
            ref(x.double())
        torch.cuda.synchronize()
        assert int(bn.num_batches_tracked) == int(ref.num_batches_tracked) == step + 1
        m = momentum if momentum is not None else 1.0 / (step + 1)
        mean, var, tol_m, tol_v = bn_stats_ref(x)
        unb = var * rows / (rows - 1)
        tol_rm = (1 - m) * tol_rm + m * tol_m + 3 * U * ((1 - m) * rm0.abs() + m * mean.abs())
        tol_rv = (1 - m) * tol_rv + m * tol_v * rows / (rows - 1) + 4 * U * ((1 - m) * rv0 + m * unb)
        _check("running mean momentum=%s" % momentum, bn.running_mean, ref.running_mean, tol_rm)
        _check("running var momentum=%s" % momentum, bn.running_var, ref.running_var, tol_rv)


# ------------------------------------------------------------------------------------------------ 3. LayerNorm
LN_C = [8, 64, 256, 264, 512, 1000, 1024]


def ln_rows():
    return [1, 7, _sms() * 64 + 37]                  # the last: a second grid-stride pass with the next-row prefetch live


def ln_input(rows, C, dt, gen):
    """row r of kind r % 4: N(0,1); the constant 0.3; 100 + N(0,1); N(0, 0.01^2) (eps matters)"""
    z = torch.randn(rows, C, device="cuda", generator=gen)
    kind = (torch.arange(rows, device="cuda") % 4)[:, None]
    x = torch.where(kind == 1, torch.full_like(z, 0.3), z)
    x = torch.where(kind == 2, 100.0 + z, x)
    x = torch.where(kind == 3, 0.01 * z, x)
    return x.to(dt)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("eps", [1e-6, 1e-5])
@pytest.mark.parametrize("rows_i", [0, 1, 2], ids=["rows1", "rows7", "rows2pass"])
@pytest.mark.parametrize("C", LN_C)
def test_layernorm(C, rows_i, eps, dtype):
    """A row's sum runs over 8 * ceil(C / 256) terms per lane and a 5-level warp tree, then * (1/C): depth d = 8 ceil(C/256) + 6.
    mean: (d + 1) 2^-24 sum |x| / C.  The variance is a second pass over x - mean: an error e in the mean adds e^2, and the pass
    rounds (d + 4) 2^-24 of it.  dw / db: per-lane row sums, then 8 warps through shared atomics and one global atomic per CTA.
    Measured: mean at most 0.15 of its bound, rstd 0.21, y 0.56 (f32) / 1 (bf16), dx 0.33 / 1, dw 0.25, db 0.20."""
    dt = DTYPES[dtype]
    rows = ln_rows()[rows_i]
    gen = _gen(C * 31 + rows + int(eps * 1e7))
    x = ln_input(rows, C, dt, gen)
    w = torch.rand(C, device="cuda", generator=gen) * 1.5 + 0.25
    b = torch.randn(C, device="cuda", generator=gen) * 0.5
    y, mean, rstd = _nan(rows + 1, C, dtype=dt), _nan(rows + 1), _nan(rows + 1)
    _abi("pk_layernorm_fwd", x, y, I(CODE[dt]), L(rows), I(C), w, b, F(eps), mean, rstd)
    y, mean, rstd = _body(y, rows, "ln y"), _body(mean, rows, "ln mean"), _body(rstd, rows, "ln rstd")
    xd = x.double()
    d = 8 * -(-C // 256) + 6
    m_ref = xd.mean(1)
    v_ref = ((xd - m_ref[:, None]) ** 2).mean(1)
    tol_m = (d + 1) * U * xd.abs().mean(1) + 2 * U * m_ref.abs() + TINY
    _check("ln mean", mean, m_ref, tol_m)
    tol_v = tol_m ** 2 + (d + 4) * U * (v_ref + tol_m ** 2)
    r_ref, tol_r = rstd_tol(v_ref, tol_v, eps)
    _check("ln rstd", rstd, r_ref, tol_r)
    md, rd, wd, bd = mean.double()[:, None], rstd.double()[:, None], w.double(), b.double()
    xhat = (xd - md) * rd
    y_ref = xhat * wd + bd
    inner = 4 * U * ((xhat * wd).abs() + bd.abs())
    _check("ln y %s" % dtype, y, y_ref, inner + half_ulp(y_ref.abs() + inner, dt) + TINY)

    dy = torch.randn(rows, C, device="cuda", generator=gen).to(dt)
    dx, dw, db = _nan(rows + 1, C, dtype=dt), _nan(C + 1), _nan(C + 1)
    _abi("pk_layernorm_bwd", dy, x, dx, I(CODE[dt]), L(rows), I(C), w, mean, rstd, dw, db)
    dx, dw, db = _body(dx, rows, "ln dx"), _body(dw, C, "ln dw"), _body(db, C, "ln db")
    dyd = dy.double()
    gw = dyd * wd
    m_g = gw.mean(1, keepdim=True)
    m_gx = (gw * xhat).mean(1, keepdim=True)
    dx_ref = rd * (gw - m_g - xhat * m_gx)
    inner = rd * ((d + 1) * U * gw.abs().mean(1, keepdim=True) + xhat.abs() * (d + 4) * U * (gw * xhat).abs().mean(1, keepdim=True)
                  + 4 * U * (gw.abs() + m_g.abs() + (xhat * m_gx).abs()))
    _check("ln dx %s" % dtype, dx, dx_ref, inner + half_ulp(dx_ref.abs() + inner, dt) + TINY)
    grid = max(1, min(-(-rows // 8), _sms() * 2))
    depth = -(-rows // (8 * grid)) + 8 + grid + 1
    _check("ln dw", dw, (dyd * xhat).sum(0), (depth + 3) * U * (dyd * xhat).abs().sum(0) + TINY)
    _check("ln db", db, dyd.sum(0), (depth + 1) * U * dyd.abs().sum(0) + TINY)


# ------------------------------------------------------------------------------------------------ 4. cast / split
SENT = 77.0                                          # exact in bf16; written nowhere by a correct kernel


@pytest.mark.parametrize("with_lo", [True, False], ids=["hi-lo", "hi"])
@pytest.mark.parametrize("scale", [1.0, 0.125, 0.37])
@pytest.mark.parametrize("shape", [(37, 100, 120, 104, 112), (5000, 1000, 1000, 1000, 1000), (1, 8, 8, 16, 16)],
                         ids=["strided", "contiguous", "one-row"])
@pytest.mark.parametrize("src_dtype", list(DTYPES))
def test_cast_split(src_dtype, shape, scale, with_lo):
    """hi is bitwise (scale * x).to(bfloat16); lo bitwise (scale * x - hi).to(bfloat16), so hi + lo is within 2^-16 of scale * x
    relative (measured: at most 0.50 of that); pad columns [cols, cols_pad) are exactly 0; columns past cols_pad, and rows past
    the end, are not written"""
    rows, cols, ld_src, cols_pad, ld_dst = shape
    sdt = DTYPES[src_dtype]
    gen = _gen(rows + cols + int(scale * 100))
    src = torch.full((rows, ld_src), math.nan, device="cuda").to(sdt)
    src[:, :cols] = (torch.randn(rows, cols, device="cuda", generator=gen) * 10.0).to(sdt)
    src[0, :min(cols, 4)] = torch.tensor([0.0, -0.0, 1e-30, -3e5][:min(cols, 4)], device="cuda").to(sdt)
    hi = torch.full((rows + 1, ld_dst), SENT, dtype=torch.bfloat16, device="cuda")
    lo = torch.full_like(hi, SENT) if with_lo else None
    _abi("pk_cast_split", src, I(CODE[sdt]), L(ld_src), hi, lo, L(ld_dst), L(rows), I(cols), I(cols_pad), F(scale))
    v = src[:, :cols].float() * scale
    h_ref = v.to(torch.bfloat16)
    _equal("cast_split hi", hi[:rows, :cols], h_ref)
    outs = [("hi", hi)]
    if with_lo:
        l_ref = (v - h_ref.float()).to(torch.bfloat16)
        _equal("cast_split lo", lo[:rows, :cols], l_ref)
        recon = hi[:rows, :cols].double() + lo[:rows, :cols].double()
        _check("cast_split hi+lo", recon, v.double(), 2.0 ** -16 * v.double().abs())
        outs.append(("lo", lo))
    for name, o in outs:
        assert bool((o[:rows, cols:cols_pad] == 0).all()), "%s: pad columns must be 0" % name
        assert bool((o[:rows, cols_pad:] == SENT).all()) and bool((o[rows] == SENT).all()), "%s: written outside [rows, cols_pad)" % name


# ------------------------------------------------------------------------------------------------ 5. dropout / mask_nz / add
ELEM_N = [1, 7, 8, 9, 4095, (1 << 20) + 3]
_GEMM_MASK = {}


def gemm_keep_mask(p, seed):
    """the GEMM epilogue's dropout keep mask over flat indices [0, 2^20 + 100): an f32 C [M, 100] (N not a multiple of 8) of
    ones @ ones^T = 64 with drop_p, seed; its flat index is row * N + column, the convention pk_dropout shares"""
    key = (p, seed)
    if key not in _GEMM_MASK:
        N = 100
        M = -(-((1 << 20) + 3) // N)
        a = torch.ones(M, 64, dtype=torch.bfloat16, device="cuda")
        b = torch.ones(N, 64, dtype=torch.bfloat16, device="cuda")
        c = torch.empty(M, N, device="cuda")
        _k().gemm(a, b, c, drop_p=p, drop_seed=seed)
        torch.cuda.synchronize()
        scale = float(torch.tensor(1.0) / (torch.tensor(1.0) - torch.tensor(p, dtype=torch.float32)))
        assert bool(((c == 0) | (c == 64 * scale)).all())
        _GEMM_MASK[key] = c.view(-1) != 0
    return _GEMM_MASK[key]


def _nonzero_randn(n, gen, dt):
    x = torch.randn(n, device="cuda", generator=gen)
    return torch.where(x.abs() < 1e-3, torch.full_like(x, 0.5), x).to(dt)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("n", ELEM_N)
def test_dropout_matches_gemm_epilogue(n, p, dtype):
    """LinearFn.backward drops dy with pk_dropout where the forward's GEMM epilogue dropped: the keep masks are bitwise equal,
    and a kept element is exactly (x * (1/(1-p))) rounded to the element type"""
    dt = DTYPES[dtype]
    seed = 987654
    x = _nonzero_randn(n, _gen(n), dt)
    y = _nan(n + 8, dtype=dt)
    _abi("pk_dropout", x, y, I(CODE[dt]), L(n), F(p), U32(seed))
    y = _body(y, n, "dropout")
    keep = gemm_keep_mask(p, seed)[:n]
    _equal("dropout keep mask", y != 0, keep)
    scale = torch.tensor(1.0) / (torch.tensor(1.0) - torch.tensor(p, dtype=torch.float32))
    _equal("dropout values", y, torch.where(keep, (x.float() * scale.cuda()).to(dt), torch.zeros((), dtype=dt, device="cuda")))


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("scale", [1.0, 1.0 / 0.9])
@pytest.mark.parametrize("n", ELEM_N)
def test_mask_nz(n, scale, dtype):
    """dx = dy * scale where y != 0, else 0: y = 0 and y = -0.0 both mask"""
    dt = DTYPES[dtype]
    gen = _gen(n + 1)
    y = torch.randn(n, device="cuda", generator=gen)
    r = torch.rand(n, device="cuda", generator=gen)
    y = torch.where(r < 0.25, torch.zeros_like(y), torch.where(r < 0.5, torch.full_like(y, -0.0), y)).to(dt)
    dy = torch.randn(n, device="cuda", generator=gen).to(dt)
    dx = _nan(n + 8, dtype=dt)
    _abi("pk_mask_nz", dy, y, dx, I(CODE[dt]), L(n), F(scale))
    ref = torch.where(y != 0, (dy.float() * torch.tensor(scale, dtype=torch.float32, device="cuda")).to(dt),
                      torch.zeros((), dtype=dt, device="cuda"))
    _equal("mask_nz", _body(dx, n, "mask_nz"), ref)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("in_place", [False, True], ids=["out", "in-place"])
@pytest.mark.parametrize("n", ELEM_N)
def test_add(n, in_place, dtype):
    """o = a + b, one rounding of the f32 sum; o may be a"""
    dt = DTYPES[dtype]
    gen = _gen(n + 2)
    a = _nan(n + 8, dtype=dt)
    a[:n] = torch.randn(n, device="cuda", generator=gen).to(dt)
    b = torch.randn(n, device="cuda", generator=gen).to(dt)
    ref = (a[:n].float() + b.float()).to(dt)
    o = a if in_place else _nan(n + 8, dtype=dt)
    _abi("pk_add", a, b, o, I(CODE[dt]), L(n), )
    _equal("add", _body(o, n, "add"), ref)


# ------------------------------------------------------------------------------------------------ 6. log_softmax / row_lse
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("n", [1, 31, 33, 6000])
def test_log_softmax_and_row_lse(n, scale, dtype):
    """lse against float64: the exponents' argument error 2^-24 |x*scale - max|, expf's 2 ulp, the row sum (ceil(n/32) terms per
    lane and a 5-level warp tree), logf's ulp and the final add.  y == x * scale - lse bit for bit, with lse as pk_row_lse writes
    it.  Measured: lse at most 0.25 of its bound."""
    dt = DTYPES[dtype]
    rows = _sms() * 64 + 3 if n < 6000 else 2000
    ld = n + 5
    gen = _gen(n * 3 + int(scale * 2))
    x = _nan(rows, ld, dtype=dt)
    x[:, :n] = (torch.randn(rows, n, device="cuda", generator=gen) * 4.0).to(dt)
    y, lse = _nan(rows * n + 8), _nan(rows + 1)
    _abi("pk_log_softmax", x, I(CODE[dt]), L(ld), y, L(rows), I(n), F(scale))
    _abi("pk_row_lse", x, I(CODE[dt]), L(ld), lse, L(rows), I(n), F(scale))
    y, lse = _body(y, rows * n, "log_softmax").view(rows, n), _body(lse, rows, "row_lse")
    s = x[:, :n].float() * scale
    _equal("log_softmax y == x * scale - lse", y, s - lse[:, None])
    sd = s.double()
    m = sd.max(1).values
    arg = sd - m[:, None]
    logs = torch.log(torch.exp(arg).sum(1))
    ref = m + logs
    tol = U * (-(-n // 32) + 5 + 4 + arg.abs().max(1).values) + 2 * U * (logs.abs() + ref.abs()) + TINY
    _check("row_lse %s" % dtype, lse, ref, tol)


# ------------------------------------------------------------------------------------------------ 7. LSTM cell
LSTM_BH = [(1, 8), (3, 100), (7, 1000)]              # B * H = 8, 300, 7000: none a multiple of 256


def _sig_tol(z, s):
    # 1 / (1 + __expf(-z)): ex2.approx (2^-21 relative) after the argument's scaling by a rounded log2 e (1.5 2^-24 |z| in the
    # exponential), and z itself rounded once (the gx + gh add); then the add and the division
    return s * (1 - s) * (2.0 ** -21 + 3 * U * z.abs()) + 2 * U * s


def _tanh_tol(z, t):
    return 4 * U * t.abs() + (1 - t * t) * U * z.abs()   # tanhf: 2 ulp; z rounded once


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("step", ["first", "middle", "last"])
@pytest.mark.parametrize("B,H", LSTM_BH, ids=["B%d-H%d" % s for s in LSTM_BH])
def test_lstm_cell(B, H, step, dtype):
    """one step forward (first: no gh, no c_prev) and backward (last: no dh_rec, no dc_next; first: no c_prev), with strided
    gx / gh / h_out / dh_out.  The backward reference takes the stored gates, c and c_prev.
    Measured: gates at most 0.70 of their bounds, c 0.46, h 0.27 (f32) / 1 (bf16), dgates 0.51 / 1, dc_prev 0.59."""
    dt = DTYPES[dtype]
    gen = _gen(B * 1000 + H + len(step))
    G4 = 4 * H
    ld_gx, ld_gh, ld_h = G4 + 8, G4 + 16, H + 8
    gx = _nan(B, ld_gx)
    gx[:, :G4] = torch.randn(B, G4, device="cuda", generator=gen) * 2.0
    gh = None
    if step != "first":
        gh = _nan(B, ld_gh)
        gh[:, :G4] = torch.randn(B, G4, device="cuda", generator=gen)
    c_prev = None if step == "first" else torch.randn(B * H, device="cuda", generator=gen) * 2.0
    c_out, gates = _nan(B * H + 1), _nan(B + 1, G4)
    h_out = _nan(B + 1, ld_h, dtype=dt)
    _abi("pk_lstm_cell_fwd", gx, L(ld_gx), gh, L(ld_gh if gh is not None else 0), c_prev, c_out, h_out, I(CODE[dt]), L(ld_h), gates,
         I(B), I(H))
    c_out, gates = _body(c_out, B * H, "lstm c"), _body(gates, B, "lstm gates")
    assert bool(torch.isnan(h_out[:B, H:].float()).all()) and bool(torch.isnan(h_out[B].float()).all()), "h_out written outside [B, H]"
    z = gx[:, :G4].double() + (gh[:, :G4].double() if gh is not None else 0.0)
    zi, zf, zg, zo = z.split(H, 1)
    si, sf, tg, so = torch.sigmoid(zi), torch.sigmoid(zf), torch.tanh(zg), torch.sigmoid(zo)
    ti, tf, tgg, to = _sig_tol(zi, si), _sig_tol(zf, sf), _tanh_tol(zg, tg), _sig_tol(zo, so)
    for name, got, ref, tol in (("i", gates[:, :H], si, ti), ("f", gates[:, H:2 * H], sf, tf), ("g", gates[:, 2 * H:3 * H], tg, tgg),
                                ("o", gates[:, 3 * H:], so, to)):
        _check("lstm gate " + name, got, ref, tol + TINY)
    cp = c_prev.double().view(B, H) if c_prev is not None else torch.zeros_like(si)
    c_ref = sf * cp + si * tg
    tol_c = cp.abs() * tf + si * tgg + tg.abs() * ti + 3 * U * ((sf * cp).abs() + (si * tg).abs()) + TINY
    _check("lstm c", c_out.view(B, H), c_ref, tol_c)
    tc = torch.tanh(c_ref)
    h_ref = so * tc
    inner = tc.abs() * to + so * ((1 - tc * tc) * tol_c + 4 * U * tc.abs()) + 2 * U * h_ref.abs()
    _check("lstm h %s" % dtype, h_out[:B, :H], h_ref, inner + half_ulp(h_ref.abs() + inner, dt) + TINY)

    # backward from the stored gates / c
    dh_out = _nan(B, ld_h, dtype=dt)
    dh_out[:, :H] = torch.randn(B, H, device="cuda", generator=gen).to(dt)
    dh_rec = None if step == "last" else torch.randn(B * H, device="cuda", generator=gen)
    dc_next = None if step == "last" else torch.randn(B * H, device="cuda", generator=gen)
    dgates, dc_prev = _nan(B + 1, G4, dtype=dt), _nan(B * H + 1)
    _abi("pk_lstm_cell_bwd", dh_out, L(ld_h), dh_rec, dc_next, gates, c_out, c_prev, dgates, I(CODE[dt]), dc_prev, I(B), I(H))
    dgates, dc_prev = _body(dgates, B, "lstm dgates"), _body(dc_prev, B * H, "lstm dc_prev")
    gi, gf, gg, go = (t.double() for t in gates.split(H, 1))
    c = c_out.double().view(B, H)
    dh = dh_out[:, :H].double() + (dh_rec.double().view(B, H) if dh_rec is not None else 0.0)
    tcs = torch.tanh(c)
    tol_tc = 4 * U * tcs.abs()
    q = 1 - tcs * tcs
    dc = dh * go * q + (dc_next.double().view(B, H) if dc_next is not None else 0.0)
    tol_dc = (dh * go).abs() * (2 * tcs.abs() * tol_tc + U * tcs * tcs + 4 * U * q) + U * dh.abs() * go * q + 2 * U * dc.abs()
    refs = [dc * gg * gi * (1 - gi), dc * cp * gf * (1 - gf), dc * gi * (1 - gg * gg), dh * tcs * go * (1 - go)]
    inners = [(gg * gi * (1 - gi)).abs() * tol_dc + 5 * U * refs[0].abs(),
              (cp * gf * (1 - gf)).abs() * tol_dc + 5 * U * refs[1].abs(),
              (gi * (1 - gg * gg)).abs() * tol_dc + (dc * gi).abs() * U * gg * gg + 5 * U * refs[2].abs(),
              (dh * go * (1 - go)).abs() * tol_tc + 5 * U * refs[3].abs()]
    for k, name in enumerate("ifgo"):
        ref, inner = refs[k], inners[k]
        _check("lstm dgate %s %s" % (name, dtype), dgates[:, k * H:(k + 1) * H], ref, inner + half_ulp(ref.abs() + inner, dt) + TINY)
    _check("lstm dc_prev", dc_prev.view(B, H), dc * gf, gf * tol_dc + U * (dc * gf).abs() + TINY)


# ------------------------------------------------------------------------------------------------ 8. embedding, gather / scatter rows
def _acc_tol(init, counts_rows, src_abs):
    """a float32 entry that received k atomic adds on top of `init`: (k + 1) 2^-24 (|init| + sum |added|)"""
    return (counts_rows + 1) * U * (init.double().abs() + src_abs) + TINY


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("padding_idx", [None, 5], ids=["nopad", "pad5"])
@pytest.mark.parametrize("n,V,E,ld", [(300, 50, 100, 104), (7, 3, 1000, 1000), (64, 16, 8, 16)])
def test_embedding(n, V, E, ld, padding_idx, dtype):
    """forward: out[:, :E] == table[idx] rounded to the element type, out[:, E:ld] == 0.  backward: dtable accumulates (atomics),
    repeated indices add up, the padding row receives nothing.  Measured: dtable at most 0.50 of its bound."""
    dt = DTYPES[dtype]
    gen = _gen(n + V + E)
    idx = torch.randint(0, V, (n,), device="cuda", generator=gen)
    idx[:3] = torch.tensor([0, 0, V - 1], device="cuda")[:min(3, n)]
    if padding_idx is not None:
        padding_idx %= V
        idx[n // 2] = padding_idx
    table = torch.randn(V, E, device="cuda", generator=gen)
    out = _nan(n + 1, ld, dtype=dt)
    _abi("pk_embedding_fwd", idx, table, I(E), out, I(CODE[dt]), I(ld), L(n))
    out = _body(out, n, "embedding out")
    _equal("embedding fwd", out[:, :E], table[idx].to(dt))
    assert bool((out[:, E:] == 0).all()), "embedding pad columns must be 0"

    dout = _nan(n, ld, dtype=dt)
    dout[:, :E] = torch.randn(n, E, device="cuda", generator=gen).to(dt)
    init = torch.randn(V, E, device="cuda", generator=gen)
    dtable = init.clone()
    _abi("pk_embedding_bwd", idx, dout, I(CODE[dt]), I(ld), I(E), dtable, L(n), L(padding_idx if padding_idx is not None else -1))
    use = idx != padding_idx if padding_idx is not None else torch.ones_like(idx, dtype=torch.bool)
    d = dout[:, :E].double() * use[:, None]
    ref = init.double().index_add(0, idx, d)
    cnt = torch.zeros(V, device="cuda", dtype=torch.float64).index_add(0, idx, use.double())[:, None]
    _check("embedding dtable", dtable, ref, _acc_tol(init, cnt, torch.zeros_like(ref).index_add(0, idx, d.abs())))
    if padding_idx is not None:
        _equal("embedding padding row", dtable[padding_idx], init[padding_idx])


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("C", [8, 1032])
def test_gather_rows(C, dtype):
    dt = DTYPES[dtype]
    gen = _gen(C)
    src = torch.randn(50, C, device="cuda", generator=gen).to(dt)
    rows = 300
    idx = torch.randint(0, 50, (rows,), device="cuda", generator=gen, dtype=torch.int32)
    idx[:2] = 7                                     # duplicates
    dst = _nan(rows + 1, C, dtype=dt)
    _abi("pk_gather_rows", src, idx, dst, I(CODE[dt]), L(rows), I(C))
    _equal("gather_rows", _body(dst, rows, "gather_rows"), src[idx.long()])


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("C", [8, 13, 1030, 1032])
def test_scatter_add_rows(C, dtype):
    """dst[idx[r]] += src[r] in f32 atomics; duplicates add up; C need not be a multiple of 8.  Measured: at most 0.50 of the bound."""
    dt = DTYPES[dtype]
    gen = _gen(C + 1)
    rows, V = 300, 40
    src = torch.randn(rows, C, device="cuda", generator=gen).to(dt)
    idx = torch.randint(0, V, (rows,), device="cuda", generator=gen, dtype=torch.int32)
    idx[:5] = 3
    init = torch.randn(V, C, device="cuda", generator=gen)
    dst = torch.cat([init, _nan(1, C)])
    _abi("pk_scatter_add_rows", src, idx, dst, I(CODE[dt]), L(rows), I(C))
    dst = _body(dst, V, "scatter_add_rows")
    il = idx.long()
    ref = init.double().index_add(0, il, src.double())
    cnt = torch.zeros(V, device="cuda", dtype=torch.float64).index_add(0, il, torch.ones(rows, device="cuda", dtype=torch.float64))[:, None]
    _check("scatter_add_rows", dst, ref, _acc_tol(init, cnt, torch.zeros_like(ref).index_add(0, il, src.double().abs())))


# ------------------------------------------------------------------------------------------------ 9. ce_grad
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("in_place", [False, True], ids=["out", "in-place"])
@pytest.mark.parametrize("scale", [1.0, 0.7])
@pytest.mark.parametrize("n,ld", [(1, 8), (33, 40), (6000, 6008)])
def test_ce_grad(n, ld, scale, in_place, dtype):
    """against float64 autograd of sum_r coef[r] * log_softmax(scale * z[r])[tok[r]].  The softmax's relative error: the arguments
    (scale * z rounded, minus the max: 2^-24 (|scale z| + |arg|)), expf's 2 ulp, the row sum (ceil(n/32) + 5 deep) and 1/sum;
    the gradient adds three roundings.  Rows with coef == 0 come out entirely 0, pad included.  Measured: at most 0.54 of the bound
    (f32) / 1 (bf16)."""
    dt = DTYPES[dtype]
    rows = 300
    gen = _gen(n + int(scale * 10) + in_place)
    z = _nan(rows + 1, ld, dtype=dt)
    z[:rows, :n] = (torch.randn(rows, n, device="cuda", generator=gen) * 3.0).to(dt)
    zin = z[:rows, :n].clone()
    tok = torch.randint(0, n, (rows,), device="cuda", generator=gen, dtype=torch.int32)
    coef = torch.randn(rows, device="cuda", generator=gen)
    coef[::7] = 0.0
    zero = coef == 0
    z[:rows][zero, :n] = math.nan                    # a row that takes no part (coef 0) may hold anything: its gradient is still 0
    dz = z if in_place else _nan(rows + 1, ld, dtype=dt)
    _abi("pk_ce_grad", z, I(CODE[dt]), L(ld), tok, coef, F(scale), dz, L(rows), I(n))
    dz = _body(dz, rows, "ce_grad")
    assert bool((dz[zero] == 0).all()), "rows with coef == 0 must be entirely 0"
    assert bool((dz[:, n:] == 0).all()), "pad columns must be 0"
    zz = zin.double().requires_grad_(True)
    s32 = (zin.float() * scale).double()             # scale * z as the kernel rounds it
    lsm = torch.log_softmax(zz * scale, -1)
    loss = (coef.double() * lsm.gather(1, tok.long()[:, None])[:, 0]).sum()
    (ref,) = torch.autograd.grad(loss, zz)
    arg = s32 - s32.max(1, keepdim=True).values
    p = torch.exp(lsm.detach())
    e = U * (s32.abs() + arg.abs() + 6)
    rel = e + (U * (-(-n // 32) + 5 + 4) + e.max(1, keepdim=True).values)
    sc = (scale * coef.double()).abs()[:, None]
    inner = sc * p * rel + 3 * U * ref.abs() + U * sc * p
    _check("ce_grad %s" % dtype, dz[:, :n], ref, inner + half_ulp(ref.abs() + inner, dt) + TINY)
