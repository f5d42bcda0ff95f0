"""GPU parity tests of the wgmma GEMM (pika_b200/csrc/gemm.cu) through the C ABI.
Reference = torch fp32 matmul on the same bf16-rounded operands (fp32 accumulation order differs,
so f32 outputs are compared at 2e-5 norm-relative, bf16 outputs at bf16 rounding 4e-3)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def K():
    from pika_b200 import kernels
    return kernels


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("cdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mnk", [(300, 200, 136), (128, 256, 64), (1000, 520, 1024), (77, 40, 240)])
def test_gemm_kmajor(bn, cdt, mnk):
    M, N, Kd = mnk
    a, b = rnd(M, Kd, seed=1), rnd(N, Kd, seed=2)
    c = torch.full((M, N), float("nan"), device="cuda", dtype=cdt)
    K().gemm(a, b, c, block_n=bn)
    ref = a.float() @ b.float().t()
    assert rel(c, ref) < (2e-5 if cdt == torch.float32 else 4e-3)


@pytest.mark.parametrize("a_mn,b_mn", [(False, True), (True, False), (True, True)])
@pytest.mark.parametrize("bn", [64, 256])
def test_gemm_mn_major(a_mn, b_mn, bn):
    M, N, Kd = 328, 264, 200
    a = rnd(Kd, M, seed=3) if a_mn else rnd(M, Kd, seed=3)
    b = rnd(Kd, N, seed=4) if b_mn else rnd(N, Kd, seed=4)
    c = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float32)
    K().gemm(a, b, c, a_mn=a_mn, b_mn=b_mn, block_n=bn)
    af = a.float().t() if a_mn else a.float()
    bf = b.float().t() if b_mn else b.float()
    assert rel(c, af @ bf.t()) < 2e-5


def test_gemm_epilogue_bias_relu_residual_alpha():
    M, N, Kd = 260, 384, 128
    a, b = rnd(M, Kd, seed=5), rnd(N, Kd, seed=6)
    bias = torch.randn(N, device="cuda")
    res = rnd(M, N, seed=7)
    c = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    k = K()
    k.gemm(a, b, c, alpha=0.5, bias=bias, act=k.ACT_RELU, aux=res, aux_mode=k.AUX_ADD)
    ref = torch.relu(0.5 * (a.float() @ b.float().t()) + bias) + res.float()
    assert rel(c, ref) < 4e-3
    # mask-by-nonzero (ReLU/dropout backward form), f32 aux
    saved = torch.relu(torch.randn(M, N, device="cuda"))
    c2 = torch.empty(M, N, device="cuda", dtype=torch.float32)
    k.gemm(a, b, c2, aux=saved, aux_mode=k.AUX_MASK_NZ, aux_scale=1.25)
    ref2 = (a.float() @ b.float().t()) * (saved != 0).float() * 1.25
    assert rel(c2, ref2) < 2e-5


def test_gemm_dropout_is_deterministic_and_unbiased():
    M, N, Kd = 512, 512, 64
    a, b = rnd(M, Kd, seed=8), rnd(N, Kd, seed=9)
    k = K()
    c1 = torch.empty(M, N, device="cuda", dtype=torch.float32)
    c2 = torch.empty_like(c1)
    k.gemm(a, b, c1, drop_p=0.2, drop_seed=123)
    k.gemm(a, b, c2, drop_p=0.2, drop_seed=123)
    assert torch.equal(c1, c2)
    ref = a.float() @ b.float().t()
    kept = c1 != 0
    frac = kept.float().mean().item()
    assert abs(frac - 0.8) < 0.01
    assert rel(c1[kept], ref[kept] * 1.25) < 2e-5
    c3 = torch.empty_like(c1)
    k.gemm(a, b, c3, drop_p=0.2, drop_seed=124)
    assert not torch.equal(c1 != 0, c3 != 0)


@pytest.mark.parametrize("dil,stride", [(1, 1), (3, 1), (3, 4)])
def test_gemm_tdnn_taps_batched(dil, stride):
    """3-tap TDNN as three accumulated (A_k, W_k) pairs over strided views -- no im2col."""
    B, T, C, Nout = 3, 150, 256, 320
    x = rnd(B, T, C, seed=10)
    w = rnd(Nout, 1, 3, C, scale=0.05, seed=11)
    bias = torch.randn(Nout, device="cuda")
    t_out = (T - 2 * dil - 1) // stride + 1
    a = [x[:, k * dil: k * dil + (t_out - 1) * stride + 1: stride, :] for k in range(3)]
    bw = [w[:, 0, k, :] for k in range(3)]
    y = torch.full((B, t_out, Nout), float("nan"), device="cuda", dtype=torch.float32)
    k_ = K()
    k_.gemm(a, bw, y, a_sel=(k_.SEL_ZB0, k_.SEL_ZERO), b_sel=(k_.SEL_ZERO, k_.SEL_ZERO), bias=bias, act=k_.ACT_RELU)
    ref = torch.nn.functional.conv2d(x.float().unsqueeze(1), w.float(), bias, dilation=(dil, 1), stride=(stride, 1))
    ref = torch.relu(ref).squeeze(-1).transpose(1, 2)
    assert y.shape == ref.shape
    assert rel(y, ref) < 2e-5


def test_gemm_negative_row_offset_dgrad_form():
    """dX[b,tau] = sum_k dY[b, tau - k*d] @ W_k : negative row coordinates are zero-filled by TMA."""
    B, T, C, Nout, dil = 2, 140, 192, 128, 3
    t_out = T - 2 * dil
    dy = rnd(B, t_out, Nout, seed=12)
    w = rnd(Nout, 1, 3, C, scale=0.05, seed=13)
    dx = torch.full((B, T, C), float("nan"), device="cuda", dtype=torch.float32)
    k_ = K()
    k_.gemm([dy] * 3, [w[:, 0, k, :] for k in range(3)], dx, b_mn=True,
            a_sel=(k_.SEL_ZB0, k_.SEL_ZERO), b_sel=(k_.SEL_ZERO, k_.SEL_ZERO),
            a_row_off=[0, -dil, -2 * dil])
    xr = torch.zeros(B, T, C, device="cuda", requires_grad=True)
    yr = torch.nn.functional.conv2d(xr.unsqueeze(1), w.float(), None, dilation=(dil, 1)).squeeze(-1).transpose(1, 2)
    yr.backward(dy.float())
    assert rel(dx, xr.grad) < 2e-5


def test_gemm_batched_reduction_wgrad_form():
    """dW_k[n,c] = sum_b sum_t dY[b,t,n] * X[b, t+k*d, c]: both operands MN-major, reduction over (b,t)."""
    B, T, C, Nout, dil = 3, 100, 192, 256, 3
    t_out = T - 2 * dil
    dy = rnd(B, t_out, Nout, seed=14)
    x = rnd(B, T, C, seed=15)
    dw = torch.full((Nout, 1, 3, C), float("nan"), device="cuda", dtype=torch.float32)
    k_ = K()
    for k in range(3):
        k_.gemm(dy, x[:, k * dil: k * dil + t_out, :], dw[:, 0, k, :], a_mn=True, b_mn=True,
                a_sel=(k_.SEL_KZ, k_.SEL_ZERO), b_sel=(k_.SEL_KZ, k_.SEL_ZERO), kz_count=B)
    wr = torch.zeros(Nout, 1, 3, C, device="cuda", requires_grad=True)
    yr = torch.nn.functional.conv2d(x.float().unsqueeze(1), wr, None, dilation=(dil, 1)).squeeze(-1).transpose(1, 2)
    yr.backward(dy.float())
    assert rel(dw, wr.grad) < 2e-5


def test_gemm_attention_shapes_4d():
    """S = Q K^T / sqrt(d) and O = P V over (batch, head) without materialising transposes."""
    B, T, H, D = 2, 100, 4, 64
    qkv = rnd(B, T, 3 * H * D, seed=16)
    q = qkv[:, :, 0:H * D].view(B, T, H, D).permute(0, 2, 1, 3)          # (B,H,T,D) strided view
    kk = qkv[:, :, H * D:2 * H * D].view(B, T, H, D).permute(0, 2, 1, 3)
    v = qkv[:, :, 2 * H * D:].view(B, T, H, D).permute(0, 2, 1, 3)
    Tp = 104
    s = torch.zeros(B, H, T, Tp, device="cuda", dtype=torch.float32)
    k_ = K()
    k_.gemm(q, kk, s[:, :, :, :T], alpha=0.125)
    ref = torch.matmul(q.float(), kk.float().transpose(2, 3)) * 0.125
    assert rel(s[:, :, :, :T], ref) < 2e-5
    p = torch.softmax(ref, -1).to(torch.bfloat16)
    pp = torch.zeros(B, H, T, Tp, device="cuda", dtype=torch.bfloat16)
    pp[:, :, :, :T] = p
    o = torch.empty(B, T, H * D, device="cuda", dtype=torch.bfloat16)
    ov = o.view(B, T, H, D).permute(0, 2, 1, 3)
    k_.gemm(pp[:, :, :, :T], v, ov, b_mn=True)
    oref = torch.matmul(p.float(), v.float())
    assert rel(ov, oref) < 4e-3


def test_gemm_accumulate_and_multi_tile_persistence():
    M, N, Kd = 128 * 40, 256 * 9, 192          # 360 tiles > 132 SMs: exercises the persistent loop
    a, b = rnd(M, Kd, seed=17), rnd(N, Kd, seed=18)
    c = torch.ones(M, N, device="cuda", dtype=torch.float32)
    K().gemm(a, b, c, accumulate=True)
    assert rel(c, a.float() @ b.float().t() + 1.0) < 2e-5


def test_gemm_split_bf16_fp32_class():
    """hi/lo split operands, 3 pairs: fp32-class accuracy from bf16 tensor cores."""
    M, N, Kd = 256, 256, 512
    g = torch.Generator(device="cuda").manual_seed(19)
    af = torch.randn(M, Kd, device="cuda", generator=g)
    bf = torch.randn(N, Kd, device="cuda", generator=g)
    ah = af.to(torch.bfloat16); al = (af - ah.float()).to(torch.bfloat16)
    bh = bf.to(torch.bfloat16); bl = (bf - bh.float()).to(torch.bfloat16)
    c = torch.empty(M, N, device="cuda", dtype=torch.float32)
    K().gemm([ah, ah, al], [bh, bl, bh], c)
    ref = (af.double() @ bf.double().t()).float()
    assert rel(c, ref) < 3e-5


@pytest.mark.parametrize("mnk", [(300, 6000, 256), (128, 256, 64), (1000, 520, 192), (2049, 6000, 128)])
def test_gemm_row_lse_partials(mnk):
    """pk_gemm_desc.row_lse: per-row, per-column-group (max*log2e, sum 2^(x*log2e-max)) of the ROUNDED bf16 outputs: one group per
    256-wide N tile."""
    import math
    M, N, Kd = mnk
    a, b = rnd(M, Kd, seed=11, scale=0.5), rnd(N, Kd, seed=12, scale=0.5)
    bias = torch.randn(N, device="cuda")
    c = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    nt = K().row_lse_parts(M, N, 256)
    gw = 256 * ((N + 255) // 256) // nt                 # columns per group
    assert nt == (N + 255) // 256
    parts = torch.full((nt, M, 2), float("nan"), device="cuda")
    K().gemm(a, b, c, bias=bias, block_n=256, row_lse=parts)
    ref = a.float() @ b.float().t() + bias
    assert rel(c, ref) < 4e-3
    m = parts[:, :, 0].max(0).values
    s = (parts[:, :, 1] * torch.exp2(parts[:, :, 0] - m)).sum(0)
    lse = (m + torch.log2(s)) * math.log(2.0)
    want = torch.logsumexp(c.float(), -1)               # of the rounded outputs, as the loss kernels read them
    assert (lse - want).abs().max().item() < 2e-5 * max(1.0, want.abs().max().item())
    # every tile's partial alone equals the log-sum-exp of its own column block
    for i in range(nt):
        blk = c[:, i * gw:(i + 1) * gw].float()
        if blk.shape[1] == 0:                              # a group entirely beyond N: the empty partial (max = -inf, sum = 0)
            assert bool((parts[i, :, 1] == 0).all())
            continue
        got = (parts[i, :, 0] + torch.log2(parts[i, :, 1])) * math.log(2.0)
        assert (got - torch.logsumexp(blk, -1)).abs().max().item() < 1e-4


@pytest.mark.parametrize("mnk,a_mn,b_mn,ks", [((300, 520, 4096), 0, 0, 0), ((304, 520, 4096), 1, 1, 0), ((1664, 3072, 1024), 0, 0, 0),
                                               ((1664, 3072, 1024), 1, 1, 0), ((128 * 37, 1024, 2048), 0, 1, 2), ((6000, 1024, 9000), 1, 1, 0),
                                               ((4096, 1024, 4832), 1, 1, 0), ((200, 136, 1000), 0, 0, 7)])
def test_gemm_split_k(mnk, a_mn, b_mn, ks):
    """split-K over the flattened reduction (auto heuristic or forced): partial tiles meet in C via TMA reduce-add;
    the result must equal the plain product, also when accumulating into a pre-filled C."""
    M, N, Kd = mnk
    a = rnd(Kd, M, seed=31) if a_mn else rnd(M, Kd, seed=31)
    b = rnd(Kd, N, seed=32) if b_mn else rnd(N, Kd, seed=32)
    ref = (a.float().t() if a_mn else a.float()) @ (b.float() if b_mn else b.float().t())
    c = torch.full((M, N), float("nan"), device="cuda")
    K().gemm(a, b, c, a_mn=bool(a_mn), b_mn=bool(b_mn), k_splits=ks)
    assert rel(c, ref) < 2e-5
    c0 = torch.randn(M, N, device="cuda")
    c = c0.clone()
    K().gemm(a, b, c, a_mn=bool(a_mn), b_mn=bool(b_mn), k_splits=ks, accumulate=True)
    assert rel(c, ref + c0) < 2e-5
    c = torch.full((M, N), float("nan"), device="cuda")
    K().gemm(a, b, c, a_mn=bool(a_mn), b_mn=bool(b_mn), k_splits=1)          # forced off: same answer
    assert rel(c, ref) < 2e-5


@pytest.mark.parametrize("cdt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("mnk", [(304, 520, 136), (2048, 1024, 1024), (136, 256, 64), (1000, 264, 200)])
def test_gemm_bn256_every_layout_ragged(mnk, a_mn, b_mn, cdt):
    """256-wide tiles with bias on every operand layout and both C types, incl. ragged M / N (a last row tile with few valid rows,
    a last N tile with few valid columns)"""
    M, N, Kd = mnk
    a = rnd(Kd, M, seed=21) if a_mn else rnd(M, Kd, seed=21)
    b = rnd(Kd, N, seed=22) if b_mn else rnd(N, Kd, seed=22)
    c = torch.full((M, N), float("nan"), device="cuda", dtype=cdt)
    bias = torch.randn(N, device="cuda")
    K().gemm(a, b, c, a_mn=a_mn, b_mn=b_mn, bias=bias, block_n=256)
    af = a.float().t() if a_mn else a.float()
    bf = b.float().t() if b_mn else b.float()
    assert rel(c, af @ bf.t() + bias) < (2e-5 if cdt == torch.float32 else 4e-3)


def test_gemm_bn256_split_k_taps_and_full_epilogue():
    """256-wide tiles: split-K with reduce-add, three accumulated taps with row offsets, ReLU + dropout + residual epilogue"""
    M, N, Kd = 6000, 1024, 4000
    a, b = rnd(Kd, M, seed=31, scale=0.3), rnd(Kd, N, seed=32, scale=0.3)
    c = torch.full((M, N), float("nan"), device="cuda")
    K().gemm(a, b, c, a_mn=True, b_mn=True, block_n=256, k_splits=3)
    assert rel(c, a.float().t() @ b.float()) < 2e-5
    # taps: y[t] = sum_k x[t + k] W_k^T
    T, C, Nn = 700, 128, 512
    x = rnd(T + 2, C, seed=33)
    w = [rnd(Nn, C, seed=40 + k) for k in range(3)]
    y = torch.empty(T, Nn, device="cuda")
    K().gemm([x[k:k + T] for k in range(3)], w, y, block_n=256)
    ref = sum(x[k:k + T].float() @ w[k].float().t() for k in range(3))
    assert rel(y, ref) < 2e-5
    res = rnd(T, Nn, seed=50)
    y = torch.empty(T, Nn, device="cuda", dtype=torch.bfloat16)
    K().gemm(x[:T], w[0], y, block_n=256, drop_p=0.2, drop_seed=99, aux=res, aux_mode=K().AUX_ADD, act=K().ACT_RELU)
    # the same counter-based mask without the residual: a dropped element is exactly 0 there (and where the ReLU gives 0, dropped
    # or kept make no difference)
    m = torch.empty_like(y)
    K().gemm(x[:T], w[0], m, block_n=256, drop_p=0.2, drop_seed=99, act=K().ACT_RELU)
    kept = m != 0
    ref = torch.where(kept, torch.relu(x[:T].float() @ w[0].float().t()) / 0.8, 0.0) + res.float()
    assert rel(y, ref) < 4e-3
