"""The compacted joint backward (rnnt_loss_compact + the fc2 GEMMs over a device-side row count + the gate backward through the row
map) against the dense one on the same inputs.  Everything but the fc2 weight gradient must agree bit for bit, apart from the sign of
a zero; the fc2 weight gradient sums the same products in other k-blocks and split-K boundaries."""
import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu


def _pz(x):
    return x.detach().float() + 0.0          # -0 -> +0


def _model(H, V, w2_scale):
    class M(nn.Module):
        pass
    m = M()
    m.fc1, m.fc_gate, m.fc2 = nn.Linear(2 * H, H).cuda(), nn.Linear(2 * H, H).cuda(), nn.Linear(H, V).cuda()
    with torch.no_grad():
        m.fc2.weight.mul_(w2_scale)
    return m


def _run(E, m, enc0, pred0, labels, fl, ll, compact):
    E._COMPACT_GRAD = compact
    enc = enc0.clone().requires_grad_(True)
    pred = pred0.clone().requires_grad_(True)
    params = [enc, pred] + [p for l in (m.fc1, m.fc_gate, m.fc2) for p in l.parameters()]
    for p in params:
        p.grad = None
    costs = E.JointLossFn.apply(enc, pred, m, labels, fl, ll)
    costs.sum().backward()
    torch.cuda.synchronize()
    return costs.detach().clone(), [p.grad.detach().clone() for p in params]


CASES = {
    # name: (H, V, B, T, U, frame_lens, label_lens, fc2 weight scale)
    "bench_shape_B2": (1024, 6000, 2, 240, 150, [240, 240], [150, 150], 1.0),
    "ragged_U0_short_labels": (128, 520, 4, 37, 9, [37, 30, 12, 1], [9, 0, 4, 9], 1.0),
    "peaky_many_skipped": (256, 1000, 3, 96, 40, [96, 80, 50], [40, 33, 40], 12.0),
    "nothing_skipped": (128, 264, 2, 5, 3, [5, 4], [3, 2], 1.0),
    "all_skipped": (128, 264, 2, 9, 4, [0, 0], [4, 2], 1.0),
}


@pytest.mark.parametrize("case", list(CASES))
def test_compacted_joint_backward_matches_dense(case):
    from pika_b200 import engine as E
    H, V, B, T, U, fl, ll, w2s = CASES[case]
    prev, was = E.get_precision(), E._COMPACT_GRAD
    E.set_precision("bf16")
    torch.manual_seed(0)
    try:
        m = _model(H, V, w2s)
        labels = torch.randint(1, V, (B, U), device="cuda").int()
        fl_t = torch.tensor(fl, dtype=torch.int32, device="cuda")
        ll_t = torch.tensor(ll, dtype=torch.int32, device="cuda")
        gen = torch.Generator(device="cuda").manual_seed(1)
        enc0 = torch.randn(B, T, H, device="cuda", generator=gen).bfloat16()
        pred0 = torch.randn(B, U + 1, H, device="cuda", generator=gen).bfloat16()
        c_d, g_d = _run(E, m, enc0, pred0, labels, fl_t, ll_t, False)
        c_c, g_c = _run(E, m, enc0, pred0, labels, fl_t, ll_t, True)
        assert torch.equal(c_d, c_c)
        names = ["enc", "pred", "fc1.w", "fc1.b", "gate.w", "gate.b", "fc2.w", "fc2.b"]
        for name, a, b in zip(names, g_d, g_c):
            if name == "fc2.w":
                # fp32 sums of the same bf16 products over other k-block groupings: a few ulps of the largest partial sums
                scale = float(a.abs().max()) + 1e-30
                assert float((a - b).abs().max()) <= 1e-5 * scale, (name, float((a - b).abs().max()), scale)
            else:
                assert torch.equal(_pz(a), _pz(b)), (name, float((_pz(a) - _pz(b)).abs().max()))
        if case == "all_skipped":
            assert float(g_c[6].abs().max()) == 0.0
    finally:
        E._COMPACT_GRAD = was
        E.set_precision(prev)


@pytest.mark.parametrize("case", ["ragged_U0_short_labels", "peaky_many_skipped", "all_skipped"])
def test_compacted_gradient_rebuilds_the_dense_one(case):
    """dlogits rebuilt from dz_c and row_map equals the dense gradient (every skipped row is all zeros there, and the map keeps
    row order); h_c holds the kept rows of h and the 64-row tail after them is zero"""
    from pika_b200 import kernels as K
    H, V, B, T, U, fl, ll, w2s = CASES[case]
    ldv = (V + 7) // 8 * 8
    gen = torch.Generator(device="cuda").manual_seed(2)
    logits = torch.zeros(B, T, U + 1, ldv, device="cuda", dtype=torch.bfloat16)
    logits[..., :V] = (torch.randn(B, T, U + 1, V, device="cuda", generator=gen) * (4.0 * w2s)).bfloat16()
    labels = torch.randint(1, V, (B, U), device="cuda", generator=gen).int()
    fl_t = torch.tensor(fl, dtype=torch.int32, device="cuda")
    ll_t = torch.tensor(ll, dtype=torch.int32, device="cuda")
    R = B * T * (U + 1)
    h = torch.randn(R, H, device="cuda", generator=gen).bfloat16()
    cs_d = torch.empty(ldv, device="cuda")
    cs_c = torch.empty(ldv, device="cuda")
    costs_d, dl = K.rnnt_loss_fwd_bwd(logits, labels, fl_t, ll_t, V=V, colsum=cs_d)
    costs_c, dz_c, h_c, row_map, rows = K.rnnt_loss_compact(logits, labels, fl_t, ll_t, h, V=V, colsum=cs_c)
    torch.cuda.synchronize()
    assert torch.equal(costs_d, costs_c)
    assert torch.equal(_pz(cs_d), _pz(cs_c))
    n = int(rows.item())
    mp = row_map.long()
    kept = mp >= 0
    assert n == int(kept.sum())
    assert torch.equal(mp[kept], torch.arange(n, device="cuda"))
    dense = dl.view(R, ldv)
    assert bool((dense[~kept] == 0).all())
    assert torch.equal(_pz(dz_c[:n]), _pz(dense[kept]))
    assert torch.equal(h_c[:n], h[kept])
    tail = min(R, (n + 63) // 64 * 64)
    assert bool((dz_c[n:tail] == 0).all()) and bool((h_c[n:tail] == 0).all())
    if case == "all_skipped":
        assert n == 0
    if case == "peaky_many_skipped":
        assert 0 < n < R


@pytest.mark.parametrize("rows,a_mn", [(0, True), (1, True), (100, True), (4097, True), (0, False), (1, False), (200, False),
                                       (1000, False)])
def test_gemm_device_row_count(rows, a_mn):
    """a_rows_dev: MN-major A (the wgrad) reduces over the first rows only, every split-K split included (an empty split adds
    zeros); K-major A (the dgrad) writes the first rows of C"""
    from pika_b200 import kernels as K
    gen = torch.Generator(device="cuda").manual_seed(3)
    Rmax = 4160
    cnt = torch.tensor([rows], dtype=torch.int32, device="cuda")
    if a_mn:
        M, N = 520, 256
        a = torch.randn(Rmax, M, device="cuda", generator=gen).bfloat16()
        b = torch.randn(Rmax, N, device="cuda", generator=gen).bfloat16()
        tail = min(Rmax, (rows + 63) // 64 * 64)
        a[rows:tail] = 0
        b[rows:tail] = 0
        c = torch.full((M, N), float("nan"), device="cuda")
        K.gemm(a, b, c, a_mn=True, b_mn=True, a_rows_dev=cnt)
        ref = a[:rows].float().t() @ b[:rows].float()
        assert bool(torch.isfinite(c).all())
        assert float((c - ref).abs().max()) <= 1e-3 * (float(ref.abs().max()) + 1.0)
    else:
        Kd, N = 264, 256
        a = torch.randn(Rmax, Kd, device="cuda", generator=gen).bfloat16()
        w = torch.randn(Kd, N, device="cuda", generator=gen).bfloat16()
        c = torch.zeros(Rmax, N, device="cuda", dtype=torch.bfloat16)
        K.gemm(a, w, c, b_mn=True, a_rows_dev=cnt)
        ref = a[:rows].float() @ w.float()
        if rows:
            assert float((c[:rows].float() - ref).abs().max()) <= 2e-2 * (float(ref.abs().max()) + 1.0)
        tiles_end = min(Rmax, (rows + 127) // 128 * 128)
        assert bool((c[tiles_end:] == 0).all())          # tiles past the count are not written
