"""GPU parity of the fused log-softmax + RNN-T loss + gradient kernels against the oracle
(oracle/rnnt.py, oracle/rnnt_c.c) and the committed torchaudio goldens, through the C ABI.
Tolerance: costs 1e-4 relative (fp32 log-space DP vs float64 oracle), gradients 2e-5 absolute
(+5e-4 relative: fp32 log-space DP, well inside the 1e-3 the north star states)
for f32 logits; bf16 logits are compared after rounding the oracle's result to bf16."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def run_gpu(logits_np, labels, fl, ll, dtype, ldv=None, inplace=False, grad_scale=None):
    from pika_b200 import kernels
    B, T, U1, V = logits_np.shape
    ldv = ldv or V
    z = torch.zeros(B, T, U1, ldv, dtype=dtype, device="cuda")
    z[..., :V] = torch.from_numpy(logits_np).to("cuda").to(dtype)
    labels = np.ascontiguousarray(labels, np.int32)
    if labels.size == 0:          # U = 0 everywhere: no label is read, but the row pitch must be >= 1
        lab = torch.zeros(B, 1, dtype=torch.int32, device="cuda")
    else:
        lab = torch.from_numpy(labels).reshape(B, -1).cuda()
    gs = None if grad_scale is None else torch.tensor(grad_scale, dtype=torch.float32, device="cuda")
    costs, dz = kernels.rnnt_loss_fwd_bwd(z, lab, torch.from_numpy(np.asarray(fl, np.int32)).cuda(),
                                          torch.from_numpy(np.asarray(ll, np.int32)).cuda(), V=V,
                                          grad_scale=gs, dlogits=z if inplace else None)
    torch.cuda.synchronize()
    return costs.cpu().numpy(), dz.float().cpu().numpy(), z.float().cpu().numpy()


@pytest.mark.parametrize("i", [0, 1, 2, 3])
def test_golden_f32(golden_dir, i):
    from oracle import rnnt
    from make_inputs import rnnt_logits
    d = np.load(os.path.join(golden_dir, "rnnt_loss.npz"))
    logits, labels, fl, ll = rnnt_logits(d, i), d["labels_%d" % i], d["fl_%d" % i], d["ll_%d" % i]
    costs, dz, _ = run_gpu(logits, labels, fl, ll, torch.float32, ldv=((logits.shape[-1] + 3) // 4) * 4)
    np.testing.assert_allclose(costs, d["costs_%d" % i], rtol=1e-4, atol=1e-4)
    _, dz_ref = rnnt.rnnt_loss_from_logits(logits, labels, fl, ll)
    V = logits.shape[-1]
    np.testing.assert_allclose(dz[..., :V], dz_ref, atol=2e-5, rtol=5e-4)
    assert np.all(dz[..., V:] == 0)


def _ldv(V):
    return (V + 7) // 8 * 8       # a valid row pitch for both dtypes


@pytest.mark.parametrize("shape", [(3, 33, 12, 200), (2, 60, 40, 1000), (5, 17, 1, 64),
                                   # lattice width: 2 and 4 cells per thread, U+1 = 1534 (the first size whose two
                                   # diagonals per thread group need more than 48 KB of shared memory), T = 1, all U = 0
                                   (2, 6, 600, 16), (2, 5, 1533, 16), (2, 4, 2047, 16), (4, 1, 3, 8), (3, 9, 0, 8),
                                   # V at the gradient kernel's limit (ldv 8192), with and without row padding [V, ldv)
                                   (2, 5, 3, 8189), (2, 5, 3, 8191), (2, 5, 3, 8192)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ragged_vs_oracle(shape, dtype):
    from oracle import rnnt
    B, T, U, V = shape
    rng = np.random.default_rng(B * 1000 + T)
    logits = (3 * rng.standard_normal((B, T, U + 1, V))).astype(np.float32)
    labels = rng.integers(1, V, (B, U)).astype(np.int32)
    fl = rng.integers(max(1, T // 2), T + 1, B).astype(np.int32)
    ll = rng.integers(0, U + 1, B).astype(np.int32)
    fl[0], ll[0] = T, U
    if dtype == torch.bfloat16:
        logits = torch.from_numpy(logits).to(torch.bfloat16).float().numpy()    # same rounded inputs for both
    gs = rng.uniform(0.5, 2.0, B).astype(np.float32)
    costs, dz, _ = run_gpu(logits, labels, fl, ll, dtype, ldv=_ldv(V), grad_scale=gs)
    assert np.all(dz[..., V:] == 0)
    dz = dz[..., :V]
    c_ref, dz_ref = rnnt.rnnt_loss_from_logits(logits, labels, fl, ll)
    dz_ref = dz_ref * gs[:, None, None, None]
    np.testing.assert_allclose(costs, c_ref, rtol=1e-4, atol=1e-4)
    if dtype == torch.float32:
        np.testing.assert_allclose(dz, dz_ref, atol=3e-5, rtol=1e-3)   # fp32 log-space DP over T+U = 180 steps
    else:
        ref_b = torch.from_numpy(dz_ref).to(torch.bfloat16).float().numpy()
        np.testing.assert_allclose(dz, ref_b, atol=2e-5, rtol=1.6e-2)   # <= 2 bf16 ulps
    # padded nodes get exact zeros
    for n in range(B):
        assert np.all(dz[n, fl[n]:] == 0) and np.all(dz[n, :, ll[n] + 1:] == 0)


def test_inplace_aliasing_matches_out_of_place():
    rng = np.random.default_rng(9)
    logits = rng.standard_normal((2, 20, 9, 128)).astype(np.float32)
    labels = rng.integers(1, 128, (2, 8)).astype(np.int32)
    c1, dz1, _ = run_gpu(logits, labels, [20, 15], [8, 5], torch.bfloat16)
    c2, dz2, zbuf = run_gpu(logits, labels, [20, 15], [8, 5], torch.bfloat16, inplace=True)
    np.testing.assert_array_equal(c1, c2)
    np.testing.assert_array_equal(dz1, dz2)
    np.testing.assert_array_equal(zbuf, dz2)


def test_gradient_sums_to_zero_per_node_and_flow_conservation_large():
    """Size-independent properties at a larger shape: d/dlogits sums to ~0 over V at every node
    (softmax Jacobian), and sum_n costs equals the C oracle's."""
    B, T, U, V = 2, 120, 60, 2048
    rng = np.random.default_rng(1)
    logits = (2 * rng.standard_normal((B, T, U + 1, V))).astype(np.float32)
    labels = rng.integers(1, V, (B, U)).astype(np.int32)
    fl = np.array([T, T - 13], np.int32); ll = np.array([U, U - 7], np.int32)
    costs, dz, _ = run_gpu(logits, labels, fl, ll, torch.float32)
    assert np.abs(dz.sum(-1)).max() < 1e-4
    c_ref, dz_ref = c_oracle(logits, labels, fl, ll)
    np.testing.assert_allclose(costs, c_ref, rtol=1e-4)
    np.testing.assert_allclose(dz, dz_ref, atol=3e-5, rtol=1e-3)   # fp32 log-space DP over T+U = 180 steps


def c_oracle(logits, labels, fl, ll):
    """(costs f64, dlogits f32) from the C float64 oracle (oracle/rnnt_c.c) for sizes the numpy one is too slow for"""
    import ctypes, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = os.path.join(root, "oracle", "_build", "liboracle_rnnt.so")
    if not os.path.exists(so):
        subprocess.check_call(["make", "-C", os.path.join(root, "oracle")])
    lib = ctypes.CDLL(so)
    B, T, U1, V = logits.shape
    logits = np.ascontiguousarray(logits, np.float32)
    labels = np.ascontiguousarray(labels, np.int32)
    fl, ll = np.ascontiguousarray(fl, np.int32), np.ascontiguousarray(ll, np.int32)
    c_ref = np.zeros(B); dz_ref = np.zeros_like(logits)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert lib.oracle_rnnt_loss(p(logits), p(labels), p(fl), p(ll), B, T, U1, V, V, labels.shape[1], p(c_ref), p(dz_ref)) == 0
    return c_ref, dz_ref


def test_production_slice_bf16_in_place_vs_c_oracle():
    """A slice of the training shape: V = 6000, U+1 = 151, bf16 logits overwritten in place by their gradient."""
    B, T, U, V = 2, 24, 150, 6000
    rng = np.random.default_rng(6000)
    logits = torch.from_numpy((3 * rng.standard_normal((B, T, U + 1, V))).astype(np.float32)).to(torch.bfloat16).float().numpy()
    labels = rng.integers(1, V, (B, U)).astype(np.int32)
    fl = np.array([T, T - 5], np.int32); ll = np.array([U, U - 31], np.int32)
    costs, dz, _ = run_gpu(logits, labels, fl, ll, torch.bfloat16, inplace=True)
    c_ref, dz_ref = c_oracle(logits, labels, fl, ll)
    np.testing.assert_allclose(costs, c_ref, rtol=1e-4)
    ref_b = torch.from_numpy(dz_ref).to(torch.bfloat16).float().numpy()
    np.testing.assert_allclose(dz, ref_b, atol=2e-5, rtol=1.6e-2)   # <= 2 bf16 ulps


def _device_inputs(logits_np, labels, fl, ll, dtype, ldv):
    B, T, U1, V = logits_np.shape
    z = torch.zeros(B, T, U1, ldv, dtype=dtype, device="cuda")
    z[..., :V] = torch.from_numpy(logits_np).cuda().to(dtype)
    i32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()
    return z, i32(labels), i32(fl), i32(ll)


def _ragged_case(B, T, U, V, seed, dtype):
    """logits (rounded to dtype), labels and lengths of a ragged batch whose LAST utterance is full length, so the last
    gradient rows (the last column-sum partials) are live; utterance 1 has padded frames and labels"""
    rng = np.random.default_rng(seed)
    logits = (3 * rng.standard_normal((B, T, U + 1, V))).astype(np.float32)
    logits = torch.from_numpy(logits).to(dtype).float().numpy()
    labels = rng.integers(1, V, (B, U)).astype(np.int32)
    fl = np.full(B, T, np.int32); ll = np.full(B, U, np.int32)
    fl[1], ll[1] = T - 5, U - 3
    return logits, labels, fl, ll


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_colsum(dtype):
    """dlogits_colsum (the fc2 bias gradient): the column sums of the dlogits the same call returns, exactly zero over the row
    padding, bit-reproducible, and (f32) the column sums of the oracle's gradient."""
    from oracle import rnnt
    from pika_b200 import kernels
    B, T, U, V, ldv = 3, 20, 10, 997, 1008
    logits, labels, fl, ll = _ragged_case(B, T, U, V, 11, dtype)
    z, lab, flt, llt = _device_inputs(logits, labels, fl, ll, dtype, ldv)
    sums = []
    for _ in range(2):
        cs = torch.full((ldv,), 77.0, device="cuda")
        costs, dz = kernels.rnnt_loss_fwd_bwd(z, lab, flt, llt, V=V, colsum=cs)
        sums.append(cs)
    torch.cuda.synchronize()
    assert torch.equal(sums[0], sums[1]), "column sums are not bit-reproducible"
    cs = sums[0].double().cpu().numpy()
    dz = dz.double().cpu().numpy().reshape(-1, ldv)
    assert np.all(cs[V:] == 0) and np.all(dz[:, V:] == 0)
    mag = np.abs(dz[:, :V]).sum(0)
    assert np.all(np.abs(cs[:V] - dz[:, :V].sum(0)) <= 1e-5 * mag)
    assert mag.min() > 0
    c_ref, dz_ref = rnnt.rnnt_loss_from_logits(logits, labels, fl, ll)
    np.testing.assert_allclose(costs.cpu().numpy(), c_ref, rtol=1e-4)
    if dtype == torch.float32:
        dz_ref = dz_ref.reshape(-1, V)
        # the per-element gradient bound of test_ragged_vs_oracle, summed over the rows
        assert np.all(np.abs(cs[:V] - dz_ref.sum(0)) <= (3e-5 + 1e-3 * np.abs(dz_ref)).sum(0))


def _row_lse_parts(logits_np, layout):
    """[n_parts, rows, 2] f32 partials of every row, as the fc2 GEMM writes them: per column group (max * log2 e,
    sum 2^(x log2 e - max)), (-inf, 0) for a group with no column below V"""
    B, T, U1, V = logits_np.shape
    x = logits_np.reshape(-1, V).astype(np.float64) * np.log2(np.e)
    if layout == "one":
        groups = [(0, V)]
    else:
        n = {"groups3": 3, "groups24": 24, "empty_first": 3}[layout]
        groups = [(256 * i, min(256 * (i + 1), V)) for i in range(n)]
        if layout == "empty_first":
            groups = [(V, V)] + groups
    parts = np.zeros((len(groups), x.shape[0], 2), np.float32)
    for i, (c0, c1) in enumerate(groups):
        if c0 >= c1:
            parts[i, :, 0] = -np.inf
            continue
        m = x[:, c0:c1].max(1).astype(np.float32)
        parts[i, :, 0] = m
        parts[i, :, 1] = np.exp2(x[:, c0:c1] - m[:, None].astype(np.float64)).sum(1)
    return torch.from_numpy(parts).cuda()


@pytest.mark.parametrize("layout", ["one", "groups3", "groups24", "empty_first"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fused_lse_entry_matches_first_pass(dtype, layout):
    """pk_rnnt_loss_fwd_bwd_lse fed with row log-sum-exp partials built here (not by the GEMM) gives what pk_rnnt_loss_fwd_bwd
    gives on the same logits: only the fp32 summation order of the row log-sum-exp differs."""
    from pika_b200 import kernels
    B, T, U, V, ldv = 3, 9, 5, 700, 704
    logits, labels, fl, ll = _ragged_case(B, T, U, V, 21, dtype)
    z, lab, flt, llt = _device_inputs(logits, labels, fl, ll, dtype, ldv)
    parts = _row_lse_parts(logits, layout)
    cs1 = torch.empty(ldv, device="cuda")
    cs2 = torch.empty(ldv, device="cuda")
    c1, d1 = kernels.rnnt_loss_fwd_bwd(z, lab, flt, llt, V=V, colsum=cs1)
    c2, d2 = kernels.rnnt_loss_fwd_bwd(z, lab, flt, llt, V=V, colsum=cs2, row_lse=parts)
    c3, _ = kernels.rnnt_loss_fwd_bwd(z, lab, flt, llt, V=V, want_grad=False, row_lse=parts)
    torch.cuda.synchronize()
    c1, c2, c3 = c1.cpu().numpy(), c2.cpu().numpy(), c3.cpu().numpy()
    np.testing.assert_allclose(c2, c1, rtol=1e-5)
    np.testing.assert_array_equal(c3, c2)
    d1, d2 = d1.double().cpu().numpy(), d2.double().cpu().numpy()
    rows = d1.size // ldv
    mag = np.abs(d1).reshape(rows, ldv).sum(0)
    if dtype == torch.float32:
        np.testing.assert_allclose(d2, d1, rtol=1e-5, atol=1e-8)
        elem_tol = 1e-5 * mag + 1e-8 * rows
    else:
        assert np.all(np.abs(d2 - d1) <= 2.0 ** -7 * np.abs(d1)), "more than 1 bf16 ulp apart"
        elem_tol = 2.0 ** -7 * mag
    assert np.all(d2[..., V:] == 0)
    # column sums: the element bound summed over the rows, plus the fp32 summation of each side
    assert np.all(np.abs(cs2.double().cpu().numpy() - cs1.double().cpu().numpy()) <= elem_tol + 1e-5 * mag)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_limits_are_rejected(dtype):
    """U+1 > 2048 and (with a gradient) ldv > 8192 raise PikaError naming the limit, before anything out of range runs."""
    from pika_b200 import kernels
    from pika_b200._lib import PikaError
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device="cuda")
    z = torch.zeros(1, 1, 2049, 16, dtype=dtype, device="cuda")
    with pytest.raises(PikaError, match=r"U\+1 <= 2048"):
        kernels.rnnt_loss_fwd_bwd(z, torch.ones(1, 2048, dtype=torch.int32, device="cuda"), i32(1), i32(2048), want_grad=False)
    z = torch.zeros(1, 2, 2, 8200, dtype=dtype, device="cuda")
    with pytest.raises(PikaError, match=r"V <= 8192"):
        kernels.rnnt_loss_fwd_bwd(z, i32(3).view(1, 1), i32(2), i32(1))
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_loss_only_beyond_the_gradient_limit(dtype):
    """Without a gradient there is no V limit: the first pass and the lattice never hold a row."""
    from oracle import rnnt
    from pika_b200 import kernels
    B, T, U, V = 2, 6, 4, 10000
    logits, labels, fl, ll = _ragged_case(B, T, U, V, 31, dtype)
    z, lab, flt, llt = _device_inputs(logits, labels, fl, ll, dtype, V)
    costs, dz = kernels.rnnt_loss_fwd_bwd(z, lab, flt, llt, V=V, want_grad=False)
    assert dz is None
    np.testing.assert_allclose(costs.cpu().numpy(), rnnt.rnnt_loss_from_logits(logits, labels, fl, ll)[0], rtol=1e-4)
