"""Attention kernels called directly, each dispatch path chosen explicitly, against float64 restatements:

    pk_softmax_fwd / pk_softmax_masked_fwd / pk_softmax_bwd      csrc/elementwise.cu: <T, 4> for ld_p <= 1024, <T, 8> up to 2048
    pk_softmax_masked_relpos_fwd / pk_softmax_relpos_bwd         the relative-position band, bucket b(i, j) = clamp(j - i, -m, m) + m
    pk_attention_fwd / pk_attention_bwd                          csrc/attention_tc.cu: forward, dQ and dK/dV (on S^T) modes

Every reference takes the kernel's own stored inputs: the backward references use the P the forward wrote, rounded as stored, and
the bucket sums are formed from the stored Pd / dS.  So each bound is the rounding of one step, not of a chain.  Errors are bounded
element by element, which bounds every row separately; a failure names the first offending (row, column).  The largest err / bound
of each check is printed when the module finishes; the figures beside the bounds were measured on an H100 80GB HBM3.

Dropout masks are recovered explicitly: pk_softmax_fwd on S = 0 gives P = 1/n everywhere, so its Pd != 0 is exactly the keep mask M
of the counter-based generator every attention kernel shares (row r of the [rows, n] probability matrix; the fused attention's row of
(b, h, t) is (b * heads + h) * T + t)."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}
MANT = {torch.float32: 24, torch.bfloat16: 8}        # significand bits
TINY = 1e-37                                          # absorbs results the kernels flush to zero (ex2.approx.ftz)
ALPHA = 0.125                                         # 1 / sqrt(64)
_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _WORST:
        print("\nlargest err / bound: " + ", ".join("%s %.3g" % kv for kv in sorted(_WORST.items())))


def _k():
    from pika_b200 import kernels
    return kernels


def _r8(x):
    return (x + 7) // 8 * 8


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rows_two_passes(per):
    """a multiple of `per` above num_sms * 64: the softmax kernels run one warp per row on at most num_sms * 8 CTAs of 8 warps,
    so their grid-stride loop takes a second pass"""
    need = torch.cuda.get_device_properties(0).multi_processor_count * 64 + 1
    return per * max(2, -(-need // per))


# ------------------------------------------------------------------------------------------------ direct C-ABI calls
def _abi(name, *args):
    """calls pk_<name> with the current stream appended; tensors pass as device pointers, None as NULL, everything else must
    already be a ctypes value.  Returns the status code."""
    from pika_b200 import _lib
    conv = [ctypes.c_void_p(a.data_ptr()) if isinstance(a, torch.Tensor) else ctypes.c_void_p(0) if a is None else a for a in args]
    return getattr(_lib.lib, name)(*conv, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


L, I, F, U = ctypes.c_longlong, ctypes.c_int, ctypes.c_float, ctypes.c_uint32


def _ptr(t, elems=0):
    return ctypes.c_void_p(t.data_ptr() + elems * t.element_size())


# ------------------------------------------------------------------------------------------------ float64 references
def half_ulp(x, dtype):
    """half an ulp of dtype at |x| (the largest round-to-nearest error of a value of that magnitude)"""
    m, e = torch.frexp(x.abs())
    return torch.where(m == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - 1 - MANT[dtype]))


def drop_params(p):
    """(thresh16, keep-scale) of the kernels' 16-bit pair mask for drop probability p, in the kernels' f32 arithmetic"""
    if p <= 0:
        return 0, 1.0
    t = float(torch.tensor(p, dtype=torch.float32)) * 65536.0 + 0.5
    th = max(1, 65535 if t >= 65535.0 else int(t))
    one = torch.tensor(1.0, dtype=torch.float32)
    return th, float(one / (one - torch.tensor(th / 65536.0, dtype=torch.float32)))


def ref_softmax(x, keep):
    """float64 softmax over the last dim with the keys outside `keep` removed"""
    return torch.softmax(x.double().masked_fill(~keep, -math.inf), -1)


def tol_p(ref, dtype):
    # f32: __expf's error grows with |x - max| (the argument's rounding, |x| 2^-24, plus ex2.approx's 2 ulp), then 1 / sum: well
    # under 1e-5 relative for these scores (|x - max| < 60).  bf16: one rounding of that value on top.
    # Measured: f32 at most 0.30 of the bound (plain, masked, relative-position); bf16 0.998 (the half ulp is attained).
    inner = 1e-5 * ref
    return inner + (half_ulp(ref + inner, dtype) if dtype == torch.bfloat16 else 0) + TINY


def ref_softmax_bwd(P, d):
    """float64 dS = P (d - sum_c d P) from the stored P; d is the gradient of P (dropout mask and scale applied).  Also returns
    the magnitude the f32 evaluation's error is proportional to."""
    dot = (d * P).sum(-1, keepdim=True)
    return P * (d - dot), P * ((d * P).abs().sum(-1, keepdim=True) + d.abs() + dot.abs())


def tol_ds(ds, mag, dtype):
    # the f32 dot over <= 2048 terms (64 sequential per lane, then a 5-level warp tree: gamma_69 < 5e-6), d - dot and the product;
    # then the rounding of the stored value.  Measured: f32 at most 0.066 of the bound, bf16 0.999.
    inner = 5e-6 * mag
    return inner + half_ulp(ds.abs() + inner, dtype) + TINY


def ref_bucket(n, m, device="cuda"):
    """b(i, j) = clamp(j - i, -m, m) + m  as an [n (query i), n (key j)] index tensor"""
    i = torch.arange(n, device=device)[:, None]
    j = torch.arange(n, device=device)[None, :]
    return (j - i).clamp(-m, m) + m


def ref_relpos_gather(X, seqs, heads, n, m):
    """token-major X [seqs * n * heads, >= 2m+1] -> float64 X[(s, i, h), b(i, j)] as [seqs, heads, n, n]"""
    Xv = X[:, :2 * m + 1].double().reshape(seqs, n, heads, 2 * m + 1).permute(0, 2, 1, 3)
    return torch.gather(Xv, -1, ref_bucket(n, m, X.device).expand(seqs, heads, n, n))


def ref_relpos_sums(V, seqs, heads, n, m):
    """float64 V [seqs, heads, n, n] (stored Pd or dS) -> per-bucket sums and sums of |V|, token-major [seqs * n * heads, 2m+1]"""
    b = ref_bucket(n, m, V.device).expand(seqs, heads, n, n)
    z = V.new_zeros(seqs, heads, n, 2 * m + 1)
    tm = lambda x: x.permute(0, 2, 1, 3).reshape(seqs * n * heads, 2 * m + 1)
    return tm(z.scatter_add(-1, b, V)), tm(z.scatter_add(-1, b, V.abs()))


def tol_bucket(mag):
    # f32 sums of the stored values: 64 sequential per lane plus a 5-level warp tree (gamma_69 < 5e-6); singleton buckets are copies.
    # Measured: Pb at most 0.053 of the bound, dSb 0.046.
    return 5e-6 * mag + TINY


def ref_attention(q, k, v, alpha, M=None, scale=1.0):
    """float64 forward per (batch * head) of bf16 inputs [BH, T, 64]; M [BH, T, T] keep mask or None"""
    s = alpha * q @ k.transpose(1, 2)
    lse = torch.logsumexp(s, -1)
    P = torch.exp(s - lse[..., None])
    Pd = P if M is None else P * M * scale
    return P, Pd, Pd @ v, lse


def attention_tols(P, Pd, v, O, lse):
    # O: the kernel rounds the unnormalised probabilities to bf16 for the P V product (2^-8 relative each, so 2^-8 (Pd |V|) in O),
    #    plus the f32 score / row-sum / exponent errors (2e-4 relative: the 64-term f32 score sum, gamma_64 * alpha sum |q k|, is
    #    below 1e-4 for these inputs), then the bf16 rounding of O.
    # lse: the same score error plus the f32 row sum over T / 4 + 64 terms per lane (<= 4e-5 at T = 2048) and log2f.
    # Measured: O at most 0.76 of the bound (0.68 with dropout), lse 0.012.
    inner = (2.0 ** -8 + 2e-4) * (Pd @ v.abs())
    return inner + half_ulp(O.abs() + inner, torch.bfloat16) + TINY, 2e-4 + 2.0 ** -20 * lse.abs()


def ref_attention_bwd(q, k, v, P, Pd, dO, O, alpha, M=None, scale=1.0):
    """float64 (dQ, dK, dV) and their bounds.  D = sum_d dO O uses the stored O, as the kernel does."""
    D = (dO * O).sum(-1, keepdim=True)
    dP = dO @ v.transpose(1, 2)
    dPabs = dO.abs() @ v.abs().transpose(1, 2)
    if M is not None:
        dP, dPabs = dP * M * scale, dPabs * M * scale
    dS = P * (dP - D)
    dV = Pd.transpose(1, 2) @ dO
    dQ = alpha * dS @ k
    dK = alpha * dS.transpose(1, 2) @ q
    # dS is rounded to bf16 for the dQ / dK products (2^-8 relative); the probabilities recomputed from the stored lse carry the
    # score / lse error (2e-4 relative, as in the forward), and dP, D are f32 sums of exact products (gamma_64 of their |terms|).
    # dV: Pd rounded to bf16 for the Pd^T dO product.  Measured: dQ at most 0.74 of the bound, dK 0.72, dV 0.79.
    E = 2.0 ** -8 * dS.abs() + 2e-4 * P * (dPabs + (dO.abs() * O.abs()).sum(-1, keepdim=True))
    out = []
    for ref, inner in ((dQ, alpha * E @ k.abs()), (dK, alpha * E.transpose(1, 2) @ q.abs()),
                       (dV, (2.0 ** -8 + 2e-4) * (Pd.transpose(1, 2) @ dO.abs()))):
        out.append((ref, inner + half_ulp(ref.abs() + inner, torch.bfloat16) + TINY))
    return out


def _check(what, got, ref, tol):
    """|got - ref| <= tol element by element (a NaN fails); records the largest err / tol under `what`"""
    err = (got.double() - ref).abs()
    ok = err <= tol
    if not bool(ok.all()):
        at = tuple((~ok).nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements outside the bound; first at %s: got %r, reference %r, bound %r"
                             % (what, int((~ok).sum()), ok.numel(), at, got[at].item(), ref[at].item(), tol[at].item()))
    _WORST[what] = max(_WORST.get(what, 0.0), float((err / tol).max()))


# ------------------------------------------------------------------------------------------------ kernel drivers
def drop_mask(rows, n, p, seed):
    """keep mask M [rows, n] (bool) of the shared dropout generator: pk_softmax_fwd on S = 0 writes Pd = scale / n where kept"""
    ld = _r8(n)
    S = torch.zeros(rows, ld, device="cuda")
    P = torch.empty(rows, ld, device="cuda")
    Pd = torch.empty_like(P)
    _k().softmax_fwd(S, P, Pd, n, p, seed)
    return Pd[:, :n] != 0


def _scores(rows, ld_s, n, gen, scale=3.0):
    S = torch.randn(rows, ld_s, device="cuda", generator=gen) * scale
    S[:, n:] = math.nan                    # never read as a score: the engine leaves these columns uninitialised
    return S


def _outbuf(rows, ld, dtype):
    """[rows + 1, ld] NaN-filled: the extra row must survive, and every other entry must be written"""
    return torch.full((rows + 1, ld), math.nan, dtype=dtype, device="cuda")


def _tail_intact(buf, rows, what):
    assert bool(torch.isnan(buf[rows].float()).all()), "%s: write past the last row" % what
    return buf[:rows]


def _key_pad(seqs, n, gen):
    kp = (torch.rand(seqs, n, device="cuda", generator=gen) < 0.3).to(torch.uint8)
    kp[:, 0] = 0                           # key 0 survives every mask, so every row keeps a key
    return kp


def _keep(rows, n, q_len, heads, causal, key_pad):
    """[rows, n] keys that survive the mask of pk_softmax_masked_fwd (row = (sequence, head, query i))"""
    r = torch.arange(rows, device="cuda")
    keep = torch.ones(rows, n, dtype=torch.bool, device="cuda")
    if causal:
        keep &= torch.arange(n, device="cuda")[None, :] <= (r % q_len)[:, None]
    if key_pad is not None:
        keep &= key_pad[r // (heads * q_len)] == 0
    return keep


def _expect_pd(P, M, scale, dtype):
    """Pd as the kernels form it: the stored P times the keep-scale in f32, rounded to dtype, 0 where dropped"""
    return torch.where(M, (P.float() * scale).to(dtype), torch.zeros((), dtype=dtype, device=P.device))


# ------------------------------------------------------------------------------------------------ 1. plain and masked softmax
SOFTMAX_SHAPES = sorted({(ld, n) for ld in (8, 1024, 1032, 2048) for n in (1, ld - 7, ld)})


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("mask", ["none", "causal", "keypad", "both"])
@pytest.mark.parametrize("ld_p,n", SOFTMAX_SHAPES, ids=["ld%d-n%d" % s for s in SOFTMAX_SHAPES])
def test_softmax_fwd_bwd(ld_p, n, mask, dtype):
    K, dt = _k(), DTYPES[dtype]
    gen = _gen(ld_p * 7919 + n * 31 + len(mask))
    heads = 3
    if mask == "none":
        rows = _rows_two_passes(1)
        keep = torch.ones(rows, n, dtype=torch.bool, device="cuda")
    else:
        rows = _rows_two_passes(heads * n)                 # q_len = n, several sequences
        causal = mask in ("causal", "both")
        kp = _key_pad(rows // (heads * n), n, gen) if mask in ("keypad", "both") else None
        keep = _keep(rows, n, n, heads, causal, kp)
    S = _scores(rows, ld_p + 8, n, gen)
    Pb, Pdb = _outbuf(rows, ld_p, dt), _outbuf(rows, ld_p, dt)
    if mask == "none":
        K.softmax_fwd(S, Pb[:rows], Pdb[:rows], n, 0.0, 0)
    else:
        K.softmax_masked_fwd(S, Pb[:rows], Pdb[:rows], n, n, heads, causal, kp, 0.0, 0)
    torch.cuda.synchronize()
    P, Pd = _tail_intact(Pb, rows, "P"), _tail_intact(Pdb, rows, "Pd")
    assert bool((P[:, n:] == 0).all()) and bool((Pd[:, n:] == 0).all()), "row padding of P / Pd must be 0"
    ref = ref_softmax(S[:, :n], keep)
    _check("softmax P %s" % dtype, P[:, :n], ref, tol_p(ref, dt))
    assert torch.equal(P, Pd)

    dPd = _scores(rows, ld_p + 8, n, gen, 1.0)
    dSb = _outbuf(rows, ld_p, dt)
    K.softmax_bwd(dPd, P, dSb[:rows], n, 0.0, 0)
    torch.cuda.synchronize()
    dS = _tail_intact(dSb, rows, "dS")
    assert bool((dS[:, n:] == 0).all()), "row padding of dS must be 0"
    ds, mag = ref_softmax_bwd(P[:, :n].double(), dPd[:, :n].double())
    _check("softmax dS %s" % dtype, dS[:, :n], ds, tol_ds(ds, mag, dt))


# ------------------------------------------------------------------------------------------------ 2. dropout masks
@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("n", [151, 152, 1031, 2048])
def test_dropout_mask_shared_and_exact(n, dtype):
    K, dt = _k(), DTYPES[dtype]
    heads, seqs, m, p, seed = 3, 2, 5, 0.1, 4321
    rows, R = seqs * heads * n, seqs * n * heads
    ld_p = _r8(n)
    th, scale = drop_params(p)
    M = drop_mask(rows, n, p, seed)
    # keep fraction within 5 sigma of the binomial expectation
    q = 1.0 - th / 65536.0
    kept, N = int(M.sum()), M.numel()
    assert abs(kept - N * q) <= 5 * math.sqrt(N * q * (1 - q)), (kept, N * q)
    assert bool((M != drop_mask(rows, n, p, seed + 1)).any()), "another seed must give another mask"
    # the masked and relative-position forwards draw the same mask for the same (row, seed): S = 0 with nothing masked
    zeros = torch.zeros(rows, ld_p, device="cuda")
    P0, Pd0 = torch.empty(rows, ld_p, dtype=dt, device="cuda"), torch.empty(rows, ld_p, dtype=dt, device="cuda")
    K.softmax_masked_fwd(zeros, P0, Pd0, n, n, heads, False, torch.zeros(seqs, n, dtype=torch.uint8, device="cuda"), p, seed)
    assert torch.equal(Pd0[:, :n] != 0, M), "pk_softmax_masked_fwd draws another mask"
    QR0 = torch.zeros(R, _r8(2 * m + 1), device="cuda")
    Pb0 = torch.empty_like(QR0)
    K.softmax_masked_relpos_fwd(zeros, QR0, P0, Pd0, Pb0, n, heads, False, None, m, p, seed)
    assert torch.equal(Pd0[:, :n] != 0, M), "pk_softmax_masked_relpos_fwd draws another mask"

    # Pd == P * scale * M bit for bit, on real scores, through the plain and the relative-position forward
    gen = _gen(n * 13 + len(dtype))
    S = _scores(rows, ld_p + 8, n, gen)
    P, Pd = torch.empty(rows, ld_p, dtype=dt, device="cuda"), torch.empty(rows, ld_p, dtype=dt, device="cuda")
    K.softmax_fwd(S, P, Pd, n, p, seed)
    assert torch.equal(Pd[:, :n], _expect_pd(P[:, :n], M, scale, dt))
    ref = ref_softmax(S[:, :n], torch.ones_like(M))
    _check("dropout P %s" % dtype, P[:, :n], ref, tol_p(ref, dt))
    dPd = _scores(rows, ld_p + 8, n, gen, 1.0)
    dS = torch.empty(rows, ld_p, dtype=dt, device="cuda")
    K.softmax_bwd(dPd, P, dS, n, p, seed)
    ds, mag = ref_softmax_bwd(P[:, :n].double(), dPd[:, :n].double() * M * scale)
    _check("dropout softmax dS %s" % dtype, dS[:, :n], ds, tol_ds(ds, mag, dt))

    ld_r = _r8(2 * m + 1)
    QR = torch.randn(R, ld_r, device="cuda", generator=gen)
    Pr, Pdr, Pbr = torch.empty_like(P), torch.empty_like(Pd), torch.empty(R, ld_r, device="cuda")
    K.softmax_masked_relpos_fwd(S, QR, Pr, Pdr, Pbr, n, heads, True, None, m, p, seed)
    assert torch.equal(Pdr[:, :n], _expect_pd(Pr[:, :n], M, scale, dt))
    G = torch.randn(R, ld_r, device="cuda", generator=gen)
    dSb = torch.empty(R, ld_r, device="cuda")
    K.softmax_relpos_bwd(dPd, G, Pr, dS, dSb, n, heads, m, p, seed)
    d = (dPd[:, :n].double().view(seqs, heads, n, n) + ref_relpos_gather(G, seqs, heads, n, m)).view(rows, n) * M * scale
    ds, mag = ref_softmax_bwd(Pr[:, :n].double(), d)
    _check("dropout relpos dS %s" % dtype, dS[:, :n], ds, tol_ds(ds, mag, dt))


# ------------------------------------------------------------------------------------------------ 3. relative-position band
RELPOS_NM = [(1, 1), (1, 6), (8, 1), (8, 7), (8, 8), (8, 13), (151, 1), (151, 3), (151, 150), (151, 151), (151, 156),
             (1032, 1), (1032, 1024), (2048, 1), (2048, 1024)]
# (causal, key padding, heads, extra ld_r columns, drop_p): each of causal / key padding on and off, heads 1 and 3, ld_r at
# 2m+1 rounded up to 8 and 16 wider
RELPOS_FLAGS = [(False, False, 1, 0, 0.0), (True, False, 3, 16, 0.1), (False, True, 3, 0, 0.0), (True, True, 1, 16, 0.1)]


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("flags", RELPOS_FLAGS, ids=["causal%d-kp%d-h%d-ldr%d-p%g" % f for f in RELPOS_FLAGS])
@pytest.mark.parametrize("n,m", RELPOS_NM, ids=["n%d-m%d" % s for s in RELPOS_NM])
def test_relpos_fwd_bwd(n, m, flags, dtype):
    K, dt = _k(), DTYPES[dtype]
    causal, use_kp, heads, extra, p = flags
    seqs, seed = 2, 99
    rows = R = seqs * heads * n
    ld_p, ld_r = _r8(n), _r8(2 * m + 1) + extra
    gen = _gen(n * 1009 + m * 17 + heads + extra)
    S = _scores(rows, ld_p + 8, n, gen, 2.0)
    QR = torch.randn(R, ld_r, device="cuda", generator=gen)
    QR[:, 2 * m + 1:] = math.nan                        # no bucket reaches the padding of the table terms
    kp = _key_pad(seqs, n, gen) if use_kp else None
    keep = _keep(rows, n, n, heads, causal, kp)
    Pbuf, Pdbuf, Pbbuf = _outbuf(rows, ld_p, dt), _outbuf(rows, ld_p, dt), _outbuf(R, ld_r, torch.float32)
    K.softmax_masked_relpos_fwd(S, QR, Pbuf[:rows], Pdbuf[:rows], Pbbuf[:R], n, heads, causal, kp, m, p, seed)
    torch.cuda.synchronize()
    P, Pd, Pb = _tail_intact(Pbuf, rows, "P"), _tail_intact(Pdbuf, rows, "Pd"), _tail_intact(Pbbuf, R, "Pb")
    assert bool((P[:, n:] == 0).all()) and bool((Pd[:, n:] == 0).all())
    scores = S[:, :n].double().view(seqs, heads, n, n) + ref_relpos_gather(QR, seqs, heads, n, m)
    ref = ref_softmax(scores.view(rows, n), keep)
    _check("relpos P %s" % dtype, P[:, :n], ref, tol_p(ref, dt))
    scale = drop_params(p)[1]
    M = drop_mask(rows, n, p, seed) if p else torch.ones(rows, n, dtype=torch.bool, device="cuda")
    assert torch.equal(Pd[:, :n], _expect_pd(P[:, :n], M, scale, dt))
    sums, mag = ref_relpos_sums(Pd[:, :n].double().view(seqs, heads, n, n), seqs, heads, n, m)
    _check("relpos Pb", Pb[:, :2 * m + 1], sums, tol_bucket(mag))
    assert bool((Pb[:, 2 * m + 1:] == 0).all()), "padding of Pb must be 0"

    dPd = _scores(rows, ld_p + 8, n, gen, 1.0)
    G = torch.randn(R, ld_r, device="cuda", generator=gen)
    G[:, 2 * m + 1:] = math.nan
    dSbuf, dSbbuf = _outbuf(rows, ld_p, dt), _outbuf(R, ld_r, torch.float32)
    K.softmax_relpos_bwd(dPd, G, P, dSbuf[:rows], dSbbuf[:R], n, heads, m, p, seed)
    torch.cuda.synchronize()
    dS, dSb = _tail_intact(dSbuf, rows, "dS"), _tail_intact(dSbbuf, R, "dSb")
    assert bool((dS[:, n:] == 0).all())
    d = (dPd[:, :n].double().view(seqs, heads, n, n) + ref_relpos_gather(G, seqs, heads, n, m)).view(rows, n) * M * scale
    ds, mag = ref_softmax_bwd(P[:, :n].double(), d)
    _check("relpos dS %s" % dtype, dS[:, :n], ds, tol_ds(ds, mag, dt))
    sums, mag = ref_relpos_sums(dS[:, :n].double().view(seqs, heads, n, n), seqs, heads, n, m)
    _check("relpos dSb", dSb[:, :2 * m + 1], sums, tol_bucket(mag))
    assert bool((dSb[:, 2 * m + 1:] == 0).all()), "padding of dSb must be 0"


@pytest.mark.parametrize("dtype", list(DTYPES), ids=list(DTYPES))
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("n", [151, 1500])
def test_relpos_zero_table_is_the_plain_kernels(n, p, dtype):
    """QR = 0 (causal) gives pk_softmax_masked_fwd's P and Pd bit for bit, and G = 0 gives pk_softmax_bwd's dS"""
    K, dt = _k(), DTYPES[dtype]
    heads, seqs, m, seed = 3, 2, 16, 7
    rows = seqs * heads * n
    ld_p, ld_r = _r8(n), _r8(2 * m + 1)
    gen = _gen(n + int(p * 10))
    S = _scores(rows, ld_p + 8, n, gen)
    kp = _key_pad(seqs, n, gen)
    P1, Pd1, P2, Pd2 = (torch.empty(rows, ld_p, dtype=dt, device="cuda") for _ in range(4))
    K.softmax_masked_fwd(S, P1, Pd1, n, n, heads, True, kp, p, seed)
    zero = torch.zeros(rows, ld_r, device="cuda")
    K.softmax_masked_relpos_fwd(S, zero, P2, Pd2, torch.empty_like(zero), n, heads, True, kp, m, p, seed)
    assert torch.equal(P1, P2) and torch.equal(Pd1, Pd2)
    dPd = _scores(rows, ld_p + 8, n, gen, 1.0)
    dS1, dS2 = torch.empty_like(P1), torch.empty_like(P1)
    K.softmax_bwd(dPd, P1, dS1, n, p, seed)
    K.softmax_relpos_bwd(dPd, zero, P1, dS2, torch.empty_like(zero), n, heads, m, p, seed)
    assert torch.equal(dS1, dS2)


# ------------------------------------------------------------------------------------------------ 4. fused attention
def _bh(x, heads):
    """[B, T, >= heads*64] -> float64 [B * heads, T, 64]"""
    B, T = x.shape[:2]
    return x[..., :heads * 64].double().reshape(B, T, heads, 64).permute(0, 2, 1, 3).reshape(B * heads, T, 64)


def _attn_inputs(B, T, heads, seed):
    gen = _gen(seed)
    D = heads * 64
    qkv = (torch.randn(B, T, 3 * D, device="cuda", generator=gen) * 1.5).to(torch.bfloat16)
    dout = torch.randn(B, T, D, device="cuda", generator=gen).to(torch.bfloat16)
    return qkv, dout


def _attn_run(qkv, dout, heads, p, seed):
    """through kernels.attention_fwd / _bwd (fused [B, T, 3D] layout); lse padding zero as the engine allocates it"""
    K = _k()
    B, T, D3 = qkv.shape
    lse = torch.zeros(B * heads * K.attention_lse_stride(T), device="cuda")
    out = torch.empty(B, T, D3 // 3, dtype=torch.bfloat16, device="cuda")
    K.attention_fwd(qkv, out, lse, heads, ALPHA, p, seed)
    dqkv = torch.empty_like(qkv)
    K.attention_bwd(qkv, out, dout, lse, dqkv, heads, ALPHA, p, seed)
    torch.cuda.synchronize()
    return out, lse, dqkv


def _check_attention(tag, qkv, dout, heads, out, lse, dq, dk, dv, p=0.0, seed=0):
    B, T = qkv.shape[:2]
    D = heads * 64
    q, k, v = (_bh(qkv[..., i * D:(i + 1) * D], heads) for i in range(3))
    M, scale = None, 1.0
    if p:
        M = drop_mask(B * heads * T, T, p, seed).view(B * heads, T, T).double()
        scale = drop_params(p)[1]
    P, Pd, O, lse_ref = ref_attention(q, k, v, ALPHA, M, scale)
    O_k = _bh(out, heads)
    tol_o, tol_lse = attention_tols(P, Pd, v, O, lse_ref)
    _check("attention O" + tag, O_k, O, tol_o)
    _check("attention lse" + tag, lse.view(B * heads, -1)[:, :T], lse_ref, tol_lse)
    grads = ref_attention_bwd(q, k, v, P, Pd, _bh(dout, heads), O_k, ALPHA, M, scale)
    for name, got, (ref, tol) in zip(("dQ", "dK", "dV"), (dq, dk, dv), grads):
        _check("attention %s%s" % (name, tag), _bh(got, heads), ref, tol)


ATTN_T = [1, 2, 63, 64, 65, 127, 128, 129, 333, 1000, 2048]
ATTN_SHAPES = [(B, T, h) for T in ATTN_T for B, h in ((3, 1), (2, 5))] + [(48, 129, 5)]


@pytest.mark.parametrize("B,T,heads", ATTN_SHAPES, ids=["B%d-T%d-h%d" % s for s in ATTN_SHAPES])
def test_attention_fwd_bwd(B, T, heads):
    qkv, dout = _attn_inputs(B, T, heads, seed=B * 10007 + T * 31 + heads)
    out, lse, dqkv = _attn_run(qkv, dout, heads, 0.0, 0)
    D = heads * 64
    _check_attention("", qkv, dout, heads, out, lse, dqkv[..., :D], dqkv[..., D:2 * D], dqkv[..., 2 * D:])


@pytest.mark.parametrize("T", [65, 128, 333, 1000])
def test_attention_dropout_explicit_mask(T):
    """dropout in all three modes against the explicit mask; the dK/dV mode applies it transposed"""
    B, heads, p, seed = 2, 5, 0.1, 31337
    qkv, dout = _attn_inputs(B, T, heads, seed=T)
    out, lse, dqkv = _attn_run(qkv, dout, heads, p, seed)
    D = heads * 64
    _check_attention(" drop", qkv, dout, heads, out, lse, dqkv[..., :D], dqkv[..., D:2 * D], dqkv[..., 2 * D:], p, seed)


def test_attention_bit_reproducible():
    """every output element has one owner (no atomics): two identical calls agree bit for bit"""
    qkv, dout = _attn_inputs(2, 1000, 5, seed=5)
    a = _attn_run(qkv, dout, 5, 0.1, 77)
    b = _attn_run(qkv, dout, 5, 0.1, 77)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


SENT = 77.0                                            # exact in bf16; written nowhere by a correct kernel


def _strided(x, ld, fill):
    """x [B, T, C] copied into the first C columns of a [B*T + 1, ld] buffer filled with `fill`"""
    B, T, C = x.shape
    buf = torch.full((B * T + 1, ld), fill, dtype=x.dtype, device="cuda")
    buf[:B * T, :C] = x.reshape(B * T, C)
    return buf


def test_attention_strided_abi():
    """separate q / k / v with a padded row stride, padded ld_out / ld_dout, ld_dqkv != ld_qkv: the same bits as the fused
    layout, and nothing outside the [T, heads*64] views is written"""
    B, T, heads = 2, 129, 5
    D = heads * 64
    qkv, dout = _attn_inputs(B, T, heads, seed=3)
    out_ref, lse_ref, dqkv_ref = _attn_run(qkv, dout, heads, 0.1, 11)
    ld_qkv, ld_out, ld_dout, ld_dqkv = D + 24, D + 16, D + 8, D + 40
    q, k, v = (_strided(qkv[..., i * D:(i + 1) * D], ld_qkv, math.nan) for i in range(3))
    do = _strided(dout, ld_dout, math.nan)
    out = torch.full((B * T + 1, ld_out), SENT, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros_like(lse_ref)
    assert _abi("pk_attention_fwd", q, k, v, L(ld_qkv), out, L(ld_out), lse, I(B), I(T), I(heads), I(64), F(ALPHA), F(0.1), U(11)) == 0
    grads = [torch.full((B * T + 1, ld_dqkv), SENT, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
    ws = torch.zeros_like(lse)
    assert _abi("pk_attention_bwd", q, k, v, L(ld_qkv), out, L(ld_out), do, L(ld_dout), lse, ws, *grads, L(ld_dqkv), I(B), I(T), I(heads),
                I(64), F(ALPHA), F(0.1), U(11)) == 0
    torch.cuda.synchronize()
    assert torch.equal(out[:B * T, :D], out_ref.view(B * T, D)) and torch.equal(lse, lse_ref)
    assert bool((out[:B * T, D:] == SENT).all()) and bool((out[B * T] == SENT).all())
    for i, g in enumerate(grads):
        assert torch.equal(g[:B * T, :D], dqkv_ref.view(B * T, 3 * D)[:, i * D:(i + 1) * D])
        assert bool((g[:B * T, D:] == SENT).all()) and bool((g[B * T] == SENT).all())


@pytest.mark.parametrize("T", [65, 129, 1000])
def test_attention_bwd_ignores_lse_and_d_padding(T):
    """lse and the D scratch are [B*heads][pk_attention_lse_stride(T)], and a caller need not initialise either: the dK/dV mode
    streams whole 64-query tiles of both, so the kernels write the padding t >= T themselves.  NaN left there must not reach
    dK / dV."""
    K = _k()
    B, heads = 2, 5
    D = heads * 64
    qkv, dout = _attn_inputs(B, T, heads, seed=T + 1)
    out_ref, lse_ref, dqkv_ref = _attn_run(qkv, dout, heads, 0.0, 0)
    lse = torch.full_like(lse_ref, math.nan)
    out = torch.empty_like(out_ref)
    K.attention_fwd(qkv, out, lse, heads, ALPHA, 0.0, 0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(lse).all()), "the forward must write the lse padding"
    ws = torch.full_like(lse_ref, math.nan)
    dqkv = torch.empty_like(qkv)
    assert _abi("pk_attention_bwd", _ptr(qkv), _ptr(qkv, D), _ptr(qkv, 2 * D), L(3 * D), out, L(D), dout, L(D), lse, ws,
                _ptr(dqkv), _ptr(dqkv, D), _ptr(dqkv, 2 * D), L(3 * D), I(B), I(T), I(heads), I(64), F(ALPHA), F(0.0), U(0)) == 0
    torch.cuda.synchronize()
    assert bool(torch.isfinite(dqkv.float()).all()), "NaN padding of lse / D reached the gradients"
    assert torch.equal(out, out_ref) and torch.equal(dqkv, dqkv_ref)
    _check_attention(" nan-pad", qkv, dout, heads, out, lse, dqkv[..., :D], dqkv[..., D:2 * D], dqkv[..., 2 * D:])


# ------------------------------------------------------------------------------------------------ 5. argument rejection
REJECT_IDS = ["softmax-ld_p2056", "softmax-ld_p%8", "softmax-ld_s<ld_p", "masked-rows%(heads*q_len)", "masked-no-mask",
              "relpos-m0", "relpos-m1025", "relpos-ld_r<2m+1", "relpos-ld_r%8", "relpos-q_len!=n", "softmax_bwd-n>ld_p",
              "softmax_bwd-ld_d<ld_p", "attention-dh32", "attention-ld_qkv%8", "attention-drop_p1", "attention-B*heads65536",
              "attention_bwd-ld_dout%8", "attention_bwd-B*heads65536"]


def _rejections():
    """(expected message fragment, (entry point, arguments...)) in the order of REJECT_IDS"""
    buf = torch.zeros(1 << 22, device="cuda")                # 16 MB: more than any access these arguments could describe
    PF32, PBF16 = I(0), I(1)
    return [
        ("softmax rows", ("pk_softmax_fwd", buf, L(2056), buf, buf, PF32, L(2056), L(16), I(2048), F(0.0), U(0))),
        ("softmax rows", ("pk_softmax_fwd", buf, L(1024), buf, buf, PF32, L(1020), L(16), I(1000), F(0.0), U(0))),
        ("softmax rows", ("pk_softmax_fwd", buf, L(1024), buf, buf, PBF16, L(1032), L(16), I(1030), F(0.0), U(0))),
        ("sequences * heads * q_len", ("pk_softmax_masked_fwd", buf, L(64), buf, buf, PF32, L(64), L(30), I(64), I(4), I(2), I(1), None,
                                       F(0.0), U(0))),
        ("without a mask", ("pk_softmax_masked_fwd", buf, L(64), buf, buf, PF32, L(64), L(32), I(64), I(16), I(2), I(0), None, F(0.0), U(0))),
        ("max_rel", ("pk_softmax_masked_relpos_fwd", buf, L(64), buf, L(8), buf, buf, PF32, L(64), L(64), I(64), I(64), I(1), I(1), None,
                     I(0), buf, F(0.0), U(0))),
        ("max_rel", ("pk_softmax_masked_relpos_fwd", buf, L(64), buf, L(2056), buf, buf, PF32, L(64), L(64), I(64), I(64), I(1), I(1),
                     None, I(1025), buf, F(0.0), U(0))),
        ("max_rel", ("pk_softmax_relpos_bwd", buf, L(64), buf, L(16), buf, L(64), buf, PF32, L(64), I(64), I(64), I(1), I(8), buf,
                     F(0.0), U(0))),
        ("max_rel", ("pk_softmax_relpos_bwd", buf, L(64), buf, L(12), buf, L(64), buf, PF32, L(64), I(64), I(64), I(1), I(4), buf,
                     F(0.0), U(0))),
        ("self-attention", ("pk_softmax_masked_relpos_fwd", buf, L(64), buf, L(16), buf, buf, PF32, L(64), L(128), I(64), I(32), I(1), I(1),
                            None, I(4), buf, F(0.0), U(0))),
        ("softmax rows", ("pk_softmax_bwd", buf, L(64), buf, L(64), buf, PF32, L(16), I(72), F(0.0), U(0))),
        ("softmax rows", ("pk_softmax_bwd", buf, L(56), buf, L(64), buf, PF32, L(16), I(64), F(0.0), U(0))),
        ("head dim 64", ("pk_attention_fwd", buf, buf, buf, L(96), buf, L(32), buf, I(1), I(8), I(1), I(32), F(ALPHA), F(0.0), U(0))),
        ("multiples of 8", ("pk_attention_fwd", buf, buf, buf, L(196), buf, L(64), buf, I(1), I(8), I(1), I(64), F(ALPHA), F(0.0), U(0))),
        ("drop_p", ("pk_attention_fwd", buf, buf, buf, L(192), buf, L(64), buf, I(1), I(8), I(1), I(64), F(ALPHA), F(1.0), U(0))),
        ("B * heads", ("pk_attention_fwd", buf, buf, buf, L(192), buf, L(64), buf, I(65536), I(1), I(1), I(64), F(ALPHA), F(0.0), U(0))),
        ("multiples of 8", ("pk_attention_bwd", buf, buf, buf, L(192), buf, L(64), buf, L(68), buf, buf, buf, buf, buf, L(192), I(1), I(8),
                            I(1), I(64), F(ALPHA), F(0.0), U(0))),
        ("B * heads", ("pk_attention_bwd", buf, buf, buf, L(192), buf, L(64), buf, L(64), buf, buf, buf, buf, buf, L(192), I(16384), I(1),
                       I(4), I(64), F(ALPHA), F(0.0), U(0))),
    ]


@pytest.mark.parametrize("case", range(len(REJECT_IDS)), ids=REJECT_IDS)
def test_rejects_out_of_range_arguments(case):
    """a rejected call returns < 0 with a pk_last_error message and launches nothing"""
    from pika_b200 import _lib
    cases = _rejections()
    assert len(cases) == len(REJECT_IDS)
    msg, (name, *args) = cases[case]
    torch.cuda.synchronize()
    before = _lib.launch_count()
    rc = _abi(name, *args)
    assert rc < 0, "%s accepted bad arguments" % name
    assert msg in _lib.lib.pk_last_error().decode()
    assert _lib.launch_count() == before
