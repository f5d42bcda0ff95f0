"""The persistent LSTM recurrence of csrc/lstm_seq.cu (pk_lstm_seq_fwd_ex / pk_lstm_seq_bwd_ex, the prediction net's and the LSTM
encoder's layers) called directly through the C ABI, on every launch path and at its limits, against float64 restatements.

Every reference takes the kernel's own stored values, so each bound is the rounding of one step, not of a chain:
  forward   h_{t-1} is the kernel's output of the row's previous step rounded to bf16 (what it exchanged through the workspace, also
            for an f32 ``out``); z = gx + W_hh h_{t-1} in float64 for all steps at once; the stored gates against sigma / tanh(z), the
            stored c against f c_prev + i g of the stored gates and the stored c_prev, out against o tanh(c).
  backward  dh = dout + W_hh^T dG_{next} from the kernel's own stored bf16 dG of the row's next step (what it multiplied); the dc
            recurrence runs in float64 beside a running bound on the drift of the kernel's f32 dc_state, which shrinks by f per step;
            dG within half a bf16 ulp of that.
Step s of sequence b is time t = s forward and t = L_b - 1 - s in a reverse direction.  The products run on mma.sync with f32
accumulators; bf16 products are exact in f32, and each mma.sync (16 products and the accumulator) is counted as 16 f32 additions of
at most one f32 ulp (2^-23, to allow a truncating accumulator) of the magnitude sum.

Every output is filled with NaN before the call, with a guard row past its end; inputs the kernel must not read (gx and dout at
t >= L_b, dout's columns past n_dir * H) are NaN too.  Padded out and dG must be exact zeros, padded gates_save / cs untouched (NaN);
the columns of out outside each direction's slice stay NaN; the zero row of the workspace stays zero after every call; a second run
on a scratch shared as kernels.py shares it, and a third with finite values in the unread inputs, must be bit-equal to the first.
Errors are bounded element by element, a failure names the first offending (sequence, time, column), and the largest err / bound
of each check is printed when the module finishes.  The figures beside the bounds were measured on an H100 80GB HBM3 (700 W)."""
import ctypes
import math

import pytest
import torch

from test_norm_elementwise_gpu import _sig_tol, _tanh_tol, half_ulp

pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}
CODE = {torch.float32: 0, torch.bfloat16: 1}          # PK_F32, PK_BF16
EPS = 2.0 ** -24                                      # unit roundoff of f32
ULP = 2.0 ** -23
TINY = 1e-37
LS_MB = 32                                            # sequences per cooperative launch
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _WORST:
        print("\nlargest err / bound: " + ", ".join("%s %.3g" % kv for kv in sorted(_WORST.items())))


def _lib():
    from pika_b200 import _lib
    return _lib


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def h_max(n_dir):
    """the largest H the device admits: a multiple of 64 with n_dir * H/8 <= #SMs (1024 / 512 on a 132-SM H100, 896 / 448 on 114)"""
    return (_sms() * 8 // n_dir) // 64 * 64


def _abi(name, *args):
    """pk_<name>(args..., current stream) -> return code: tensors pass as device pointers, None as NULL, ints as int"""
    conv = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else ctypes.c_void_p(0) if a is None else ctypes.c_int(a)
            for a in args]
    return getattr(_lib().lib, name)(*conv, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


def _ok(name, rc):
    assert rc == 0, "%s: rc=%d %s" % (name, rc, _lib().lib.pk_last_error().decode())
    torch.cuda.synchronize()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, math.nan, dtype=dtype, device="cuda")


def _bits(x):
    return x.view(torch.int32 if x.element_size() == 4 else torch.int16)


def _equal(what, got, ref):
    """bit equality, NaN patterns included"""
    bad = _bits(got) != _bits(ref)
    if bool(bad.any()):
        at = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d elements differ; first at %s: got %r, expected %r" % (what, int(bad.sum()), at, got[at].item(),
                                                                                            ref[at].item()))


def _check(what, got, ref, tol, where):
    """|got - ref| <= tol element by element (a NaN fails); rows of got are the (sequence, time) pairs in ``where``"""
    err = (got.double() - ref).abs()
    ok = err <= tol
    if not bool(ok.all()):
        n, col = (~ok).nonzero()[0].tolist()
        b, t = where[n].tolist()
        raise AssertionError("%s: %d of %d elements outside the bound; first at sequence %d, time %d, column %d: got %r, reference %r, "
                             "bound %r" % (what, int((~ok).sum()), ok.numel(), b, t, col, got[n, col].item(), ref[n, col].item(),
                                           tol[n, col].item()))
    ratio = torch.where(tol > 0, err / tol.clamp_min(1e-300), torch.zeros_like(err))
    _WORST[what] = max(_WORST.get(what, 0.0), float(ratio.max()) if ratio.numel() else 0.0)


def ws_bytes(nH):
    return int(_lib().lib.pk_lstm_seq_workspace_bytes(nH))


def _zero_row_intact(ws, nH, when):
    """ws = [barrier counters 256 B][hx bf16 2 x 32 x n_dir*H][4 n_dir*H zero bf16]: the last region is the recurrent input of a
    sequence's first backward step and is never written"""
    z = ws[256 + 2 * LS_MB * nH * 2:]
    assert z.numel() == 8 * nH and bool((z == 0).all()), "the zero row of the workspace was written (%s)" % when


_SHARED_WS = {}


def shared_ws(nH):
    """one scratch per n_dir * H for the whole module, as kernels.py keys it"""
    if nH not in _SHARED_WS:
        _SHARED_WS[nH] = torch.zeros(ws_bytes(nH), dtype=torch.uint8, device="cuda")
    return _SHARED_WS[nH]


def make_lens(kind, B, U):
    """None: every sequence runs U steps.  ragged: unsorted, ties, a length 1 and a length U.  zero1: ragged and one length 0.
    zero2nd: ragged, and every sequence of the second 32-sequence launch has length 0.  zero: every length 0."""
    if kind is None:
        return None
    g = torch.Generator().manual_seed(B * 1009 + U)
    L = torch.randint(1, U + 1, (B,), generator=g)
    L[0] = U
    L[B // 2] = 1
    if B > 2:
        L[-1] = L[1]
    if kind == "zero1":
        L[B // 3] = 0
    elif kind == "zero2nd":
        assert B > LS_MB
        L[LS_MB:2 * LS_MB] = 0
    elif kind == "zero":
        L.zero_()
    return L.tolist()


def step_map(Ls, B, U, rev):
    """step-major maps of one direction: S = max L_b, t [S, B] the time of step s of sequence b (0 where inactive), active [S, B]"""
    Lt = torch.tensor(Ls if Ls is not None else [U] * B, device="cuda")
    S = int(Lt.max()) if B else 0
    s = torch.arange(S, device="cuda")[:, None]
    active = s < Lt[None]
    t = (Lt[None] - 1 - s) if rev else s.expand(S, B)
    return S, torch.where(active, t, torch.zeros_like(t)), active


class Layer:
    """one call's inputs: gx [n_dir,B,U,4H] f32, w_hh bf16 [n_dir*4H,H], dout [B,U,ldo]; NaN where the kernel must not read"""

    def __init__(self, H, n_dir, reverse, dtype, B, U, lens, ldo_pad, saturate, seed):
        self.H, self.nd, self.reverse, self.dt, self.B, self.U = H, n_dir, reverse, DTYPES[dtype], B, U
        self.G4, self.nH, self.ldo = 4 * H, n_dir * H, n_dir * H + ldo_pad
        self.Ls = make_lens(lens, B, U)
        self.L = [min(max(v, 0), U) for v in self.Ls] if self.Ls is not None else [U] * B
        self.lens_t = torch.tensor(self.Ls, dtype=torch.int32, device="cuda") if self.Ls is not None else None
        gen = _gen(seed)
        G4 = self.G4
        gx = torch.randn(n_dir, B, U, G4, device="cuda", generator=gen) * 0.5
        if saturate:
            # forget gate held near 1 (sigma(6) = 0.9975), input gate on, g positive: c grows into the hundreds and tanh(c) saturates
            gx[..., :H] += 4.0
            gx[..., H:2 * H] = 6.0 + 0.2 * gx[..., H:2 * H]
            gx[..., 2 * H:3 * H] += 2.0
        self.w = ((torch.rand(n_dir * G4, H, device="cuda", generator=gen) * 2 - 1) / math.sqrt(H)).to(torch.bfloat16)
        dout = torch.randn(B, U, self.ldo, device="cuda", generator=gen).to(self.dt)
        pad = torch.arange(U, device="cuda")[None, :] >= torch.tensor(self.L, device="cuda")[:, None]        # [B, U]: t >= L_b
        self.pad = pad
        self.gx_fill = gx.clone()
        self.dout_fill = dout.clone()
        self.gx_fill[:, pad] = 1e30                                          # finite values where the kernel must not read
        self.dout_fill[pad] = 1e4
        gx[:, pad] = math.nan
        dout[pad] = math.nan
        dout[:, :, self.nH:] = math.nan
        self.gx, self.dout = gx, dout

    def dirs(self):
        """(buffer index, runs backwards in time) of each direction"""
        return [(d, d == 1 if self.nd == 2 else bool(self.reverse)) for d in range(self.nd)]

    def run(self, ws, fill=False):
        """forward then backward into fresh NaN-filled outputs (each with a guard row / element block past its end)"""
        B, U, H, G4, nd = self.B, self.U, self.H, self.G4, self.nd
        gx, dout = (self.gx_fill, self.dout_fill) if fill else (self.gx, self.dout)
        out = _nan(B + 1, U, self.ldo, dtype=self.dt)
        gates, cs = _nan(nd * U * B * G4 + G4), _nan(nd * U * B * H + H)
        dG = _nan(nd * U * B * G4 + G4, dtype=torch.bfloat16)
        _ok("pk_lstm_seq_fwd_ex", _abi("pk_lstm_seq_fwd_ex", gx, self.w, out, CODE[self.dt], self.ldo, gates, cs, self.lens_t, B, U, H,
                                       nd, self.reverse, ws))
        _zero_row_intact(ws, self.nH, "forward")
        _ok("pk_lstm_seq_bwd_ex", _abi("pk_lstm_seq_bwd_ex", dout, CODE[self.dt], self.ldo, gates, cs, self.w, dG, self.lens_t, B, U, H,
                                       nd, self.reverse, ws))
        _zero_row_intact(ws, self.nH, "backward")
        return out, gates, cs, dG


def check_layout(p, out, gates, cs, dG):
    """guards, padding and the columns outside each direction's slice"""
    B, U, H, G4, nd = p.B, p.U, p.H, p.G4, p.nd
    assert bool(torch.isnan(out[B].float()).all()), "out: write past the last sequence"
    assert bool(torch.isnan(out[:B, :, p.nH:].float()).all()), "out: columns outside the directions' slices were written"
    for name, buf, n in (("gates_save", gates, nd * U * B * G4), ("cs", cs, nd * U * B * H), ("dG", dG, nd * U * B * G4)):
        assert bool(torch.isnan(buf[n:].float()).all()), "%s: write past the end" % name
    o = out[:B, :, :p.nH]
    assert bool((o[p.pad] == 0).all()), "out at t >= L_b must be exact zeros"
    assert bool(torch.isfinite(o[~p.pad].float()).all()), "out at t < L_b must be finite"
    padT = p.pad.t()                                                          # [U, B] time-major
    for name, buf, w in (("gates_save", gates, G4), ("cs", cs, H)):
        v = buf[:nd * U * B * w].view(nd, U, B, w)
        assert bool(torch.isnan(v[:, padT]).all()), "%s at t >= L_b must be left untouched" % name
        assert bool(torch.isfinite(v[:, ~padT]).all()), "%s at t < L_b must be finite" % name
    g = dG[:nd * U * B * G4].view(nd, U, B, G4)
    assert bool((g[:, padT] == 0).all()), "dG at t >= L_b must be exact zeros"
    assert bool(torch.isfinite(g[:, ~padT].float()).all()), "dG at t < L_b must be finite"


def fwd_n_ops(H):
    return H // 64                                     # mma.sync per accumulator chain: 4 chains over K = H in steps of 64


def bwd_n_ops(H):
    kspan = H // 4                                     # per K-group and quarter; four-chain blocks of 64, then a tail of 16s on one chain
    return 4 * (kspan // 64 + (kspan % 64) // 16)


def check_forward(p, out, gates, cs, d, rev):
    B, U, H, G4 = p.B, p.U, p.H, p.G4
    S, t, active = step_map(p.L, B, U, rev)
    if S == 0:
        return
    bidx = torch.arange(B, device="cuda")[None].expand(S, B)
    hk = out[:B, :, d * H:(d + 1) * H].to(torch.bfloat16).double()          # what the kernel exchanged, for an f32 out as well
    hprev = torch.zeros(S, B, H, dtype=torch.float64, device="cuda")
    if S > 1:
        hprev[1:] = hk[bidx[1:], t[:-1]]
    hprev = torch.where(active[..., None], hprev, torch.zeros_like(hprev))
    Wd = p.w[d * G4:(d + 1) * G4].double()                                  # [4H, H]
    sel = active
    where = torch.stack([bidx[sel], t[sel]], 1)
    hp = hprev[sel]
    z = p.gx[d][bidx[sel], t[sel]].double() + hp @ Wd.t()
    acc_tol = (16 * fwd_n_ops(H) + 2) * ULP * (hp.abs() @ Wd.abs().t())
    gv = gates[:p.nd * U * B * G4].view(p.nd, U, B, G4)[d]
    gk = gv[t[sel], bidx[sel]]
    for k, name in enumerate("ifgo"):
        zk, ak = z[:, k * H:(k + 1) * H], acc_tol[:, k * H:(k + 1) * H]
        if name == "g":
            ref = torch.tanh(zk)
            tol = (1 - ref * ref) * ak + _tanh_tol(zk, ref)
        else:
            ref = torch.sigmoid(zk)
            tol = ref * (1 - ref) * ak + _sig_tol(zk, ref)
        _check("gate " + name, gk[:, k * H:(k + 1) * H], ref, tol + TINY, where)
    gi, gf, gg, go = (gk[:, k * H:(k + 1) * H].double() for k in range(4))
    cv = cs[:p.nd * U * B * H].view(p.nd, U, B, H)[d]
    c_all = cv[t, bidx].double()                                             # [S, B, H] (NaN where inactive)
    cprev = torch.zeros_like(c_all)
    if S > 1:
        cprev[1:] = c_all[:-1]
    cp = cprev[sel]
    c = c_all[sel]
    c_ref = gf * cp + gi * gg
    _check("c", c, c_ref, 3 * EPS * ((gf * cp).abs() + (gi * gg).abs()) + TINY, where)
    tc = torch.tanh(c)
    h_ref = go * tc
    inner = 4 * EPS * go * tc.abs() + 2 * EPS * h_ref.abs()
    h = out[:B, :, d * H:(d + 1) * H][bidx[sel], t[sel]]
    _check("h %s" % ("bf16" if p.dt == torch.bfloat16 else "f32"), h, h_ref, inner + half_ulp(h_ref.abs() + inner, p.dt) + TINY, where)


def check_backward(p, gates, cs, dG, d, rev):
    B, U, H, G4 = p.B, p.U, p.H, p.G4
    S, t, active = step_map(p.L, B, U, rev)
    if S == 0:
        return
    bidx = torch.arange(B, device="cuda")[None].expand(S, B)
    a3 = active[..., None]
    z = lambda x: torch.where(a3, x, torch.zeros_like(x))                    # noqa: E731
    Wd = p.w[d * G4:(d + 1) * G4].double()
    dGk = dG[:p.nd * U * B * G4].view(p.nd, U, B, G4)[d]
    dGnext = torch.zeros(S, B, G4, dtype=torch.float64, device="cuda")
    if S > 1:                                          # the row's next step; zero past its length (the kernel's zero row)
        dGnext[:-1] = torch.where(a3[1:], dGk[t[1:], bidx[1:]].double(), torch.zeros_like(dGnext[1:]))
    dGnext = z(dGnext)
    do = z(p.dout[:B, :, d * H:(d + 1) * H][bidx, t].double())
    dh = do + dGnext @ Wd
    tol_dh = (16 * bwd_n_ops(H) + 6) * ULP * (dGnext.abs() @ Wd.abs() + do.abs())
    g = z(gates[:p.nd * U * B * G4].view(p.nd, U, B, G4)[d][t, bidx].double())
    c_all = z(cs[:p.nd * U * B * H].view(p.nd, U, B, H)[d][t, bidx].double())
    cprev = torch.zeros_like(c_all)
    if S > 1:
        cprev[1:] = c_all[:-1]
    refs = torch.zeros(S, B, G4, dtype=torch.float64, device="cuda")
    tols = torch.zeros_like(refs)
    dcs = torch.zeros(B, H, dtype=torch.float64, device="cuda")               # dc_state in float64
    E = torch.zeros_like(dcs)                                                # bound on |kernel dc_state - dcs|
    for s in range(S - 1, -1, -1):
        a = active[s][:, None]
        gi, gf, gg, go = g[s].split(H, 1)
        c, cp, dhs, tdh = c_all[s], cprev[s], dh[s], tol_dh[s]
        tc = torch.tanh(c)
        tol_tc = 4 * EPS * tc.abs()
        q = 1 - tc * tc
        dc = dhs * go * q + dcs
        Edc = ((go * q).abs() * tdh + (dhs * go).abs() * (2 * tc.abs() * tol_tc + EPS * tc * tc + EPS * q) + 2 * EPS * (dhs * go * q).abs()
               + E + 2 * EPS * dc.abs())
        r = [dc * gg * gi * (1 - gi), dc * cp * gf * (1 - gf), dc * gi * (1 - gg * gg), dhs * tc * go * (1 - go)]
        inner = [(gg * gi * (1 - gi)).abs() * Edc + 5 * EPS * r[0].abs(),
                 (cp * gf * (1 - gf)).abs() * Edc + 5 * EPS * r[1].abs(),
                 (gi * (1 - gg * gg)).abs() * Edc + (dc * gi).abs() * EPS * gg * gg + 5 * EPS * r[2].abs(),
                 (tc * go * (1 - go)).abs() * tdh + (dhs * go * (1 - go)).abs() * tol_tc + 5 * EPS * r[3].abs()]
        refs[s] = torch.cat(r, 1)
        tols[s] = torch.cat(inner, 1)
        dcs = torch.where(a, dc * gf, torch.zeros_like(dc))
        E = torch.where(a, gf * Edc + EPS * (dc * gf).abs(), torch.zeros_like(E))
    sel = active
    where = torch.stack([bidx[sel], t[sel]], 1)
    got = dGk[t[sel], bidx[sel]]
    ref, inner = refs[sel], tols[sel]
    tol = inner + half_ulp(ref.abs() + inner, torch.bfloat16) + TINY
    for k, name in enumerate("ifgo"):
        cols = slice(k * H, (k + 1) * H)
        _check("dG " + name, got[:, cols], ref[:, cols], tol[:, cols], where)


# (H, n_dir, reverse, out / dout dtype, B, U, lengths, ldo - n_dir*H, forget gate held saturated).  H = 64 and 192 run only the
# backward's tail loop, 320 one four-chain block and a tail, 512 / 1024 only four-chain blocks; "max" is the largest H the device
# admits for that n_dir.  B = 33 and 65 leave a one-sequence launch.
CASES = [
    (64, 1, 0, "f32", 1, 1, None, 0, False),
    (64, 1, 1, "bf16", 33, 151, "ragged", 24, False),
    (64, 2, 0, "bf16", 65, 400, "zero2nd", 0, True),
    (64, 1, 0, "bf16", 5, 2, "zero", 24, False),
    (192, 1, 1, "f32", 31, 2, "ragged", 24, False),
    (192, 2, 0, "bf16", 64, 151, "zero1", 0, False),
    (192, 1, 0, "f32", 32, 1, "zero1", 0, False),
    (320, 2, 0, "f32", 33, 151, "ragged", 24, False),
    (320, 1, 1, "bf16", 64, 151, "zero2nd", 0, False),
    (320, 1, 0, "bf16", 31, 400, None, 24, True),
    (1024, 1, 0, "bf16", 32, 151, None, 0, False),            # the benchmark's prediction-net layer
    (1024, 1, 1, "f32", 33, 400, "ragged", 24, True),
    (1024, 1, 0, "bf16", 65, 2, "zero1", 24, False),
    (512, 2, 0, "bf16", 65, 151, "ragged", 24, False),
    (512, 2, 0, "f32", 1, 400, None, 0, True),
    (512, 2, 0, "bf16", 33, 151, "zero", 0, False),
    ("max", 1, 0, "f32", 64, 151, "ragged", 24, False),
    ("max", 2, 0, "bf16", 31, 151, "zero1", 0, False),
    ("max", 1, 1, "bf16", 1, 1, None, 24, False),
]


def _case_id(c):
    H, nd, rev, dt, B, U, lens, pad, sat = c
    return "H%s-%s-%s-B%d-U%d-%s-ldo+%d%s" % (H, "bi" if nd == 2 else "rev" if rev else "fwd", dt, B, U, lens or "full", pad,
                                               "-sat" if sat else "")


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_lstm_seq(case):
    """forward and backward against the float64 step references, layout and padding, bit-equal repeats.
    Measured: the gates at most 0.73 of their bounds (i 0.70, f 0.73, g 0.66, o 0.41), c 0.65, h 0.55 (f32) / 1 (bf16: the half ulp
    is attained), dG 0.998 (the half bf16 ulp is attained).  When the backward added the four K-group partials of dh_rec with
    shared-memory atomics, the repeated call gave different dG bits in 13 of these 19 cases."""
    H, nd, rev, dtype, B, U, lens, pad, sat = case
    if H == "max":
        H = h_max(nd)
    p = Layer(H, nd, rev, dtype, B, U, lens, pad, sat, seed=H * 7 + nd * 3 + rev + B * 11 + U)
    ws = torch.zeros(ws_bytes(p.nH), dtype=torch.uint8, device="cuda")
    first = p.run(ws)
    check_layout(p, *first)
    out, gates, cs, dG = first
    for d, r in p.dirs():
        check_forward(p, out, gates, cs, d, r)
        check_backward(p, gates, cs, dG, d, r)
    names = ("out", "gates_save", "cs", "dG")
    # the same inputs again, on a scratch that other layers of the same n_dir * H have used: the same bits
    for name, a, b in zip(names, first, p.run(shared_ws(p.nH))):
        _equal("repeated call on a shared scratch: " + name, b, a)
    # finite values where the kernel must not read (gx and dout at t >= L_b, dout's columns past n_dir * H): the same bits
    for name, a, b in zip(names, first, p.run(shared_ws(p.nH), fill=True)):
        _equal("unread inputs changed: " + name, b, a)


def test_lstm_seq_shared_scratch():
    """kernels.py keys the scratch by n_dir * H, so a bidirectional layer of H and a unidirectional layer of 2H share one (512 and
    1024 on an H100).  Alternating the two on one scratch gives the bits each gives on a fresh zeroed scratch."""
    h2 = h_max(2)
    layers = [Layer(h2, 2, 0, "bf16", 40, 60, "ragged", 0, False, seed=1), Layer(2 * h2, 1, 0, "bf16", 32, 60, None, 0, False, seed=2)]
    fresh = [p.run(torch.zeros(ws_bytes(p.nH), dtype=torch.uint8, device="cuda")) for p in layers]
    ws = torch.zeros(ws_bytes(2 * h2), dtype=torch.uint8, device="cuda")
    for rnd in range(2):
        for i, p in enumerate(layers):
            for name, a, b in zip(("out", "gates_save", "cs", "dG"), fresh[i], p.run(ws)):
                _equal("layer %d, round %d on the shared scratch: %s" % (i, rnd, name), b, a)


@pytest.mark.parametrize("n_dir", [1, 2])
def test_lstm_seq_rejects_h_past_the_sm_count(n_dir):
    """H = the largest admitted + 64: both entry points return < 0 with the #SMs message, launch nothing and write nothing"""
    H = h_max(n_dir) + 64
    B, U, G4 = 2, 3, 4 * H
    lib = _lib()
    gx = torch.zeros(n_dir, B, U, G4, device="cuda")
    w = torch.zeros(n_dir * G4, H, dtype=torch.bfloat16, device="cuda")
    out, dout = _nan(B, U, n_dir * H, dtype=torch.bfloat16), torch.zeros(B, U, n_dir * H, dtype=torch.bfloat16, device="cuda")
    gates, cs = _nan(n_dir, U, B, G4), _nan(n_dir, U, B, H)
    dG = _nan(n_dir, U, B, G4, dtype=torch.bfloat16)
    ws = torch.zeros(ws_bytes(n_dir * H), dtype=torch.uint8, device="cuda")
    before = lib.launch_count()
    rc = _abi("pk_lstm_seq_fwd_ex", gx, w, out, CODE[torch.bfloat16], n_dir * H, gates, cs, None, B, U, H, n_dir, 0, ws)
    err = lib.lib.pk_last_error().decode()
    assert rc < 0 and "#SMs" in err, (rc, err)
    rc = _abi("pk_lstm_seq_bwd_ex", dout, CODE[torch.bfloat16], n_dir * H, gates, cs, w, dG, None, B, U, H, n_dir, 0, ws)
    err = lib.lib.pk_last_error().decode()
    assert rc < 0 and "#SMs" in err, (rc, err)
    torch.cuda.synchronize()
    assert lib.launch_count() == before
    for name, buf in (("out", out), ("gates_save", gates), ("cs", cs), ("dG", dG)):
        assert bool(torch.isnan(buf.float()).all()), "%s written by a rejected call" % name
