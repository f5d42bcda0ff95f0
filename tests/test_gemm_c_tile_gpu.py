"""The bf16 GEMM's C tile in shared memory is handed from the consumer warpgroups to the epilogue warps and back once per
output tile.  These cases give every persistent CTA several tiles, with M and N ragged and N not a multiple of the
256-wide tile, so the tile, its bias and its barriers are reused across units and the LSE partials see partial tiles."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-20)).item()


@pytest.mark.parametrize("lse", [False, True])
def test_gemm_bf16_c_tile_reused_across_units(lse):
    from pika_b200 import kernels as K
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    # ~6 tiles per worker; N = 5 * 256 + 136 leaves a last tile with one full 64-column chunk, one of 64 and one of 8 columns;
    # K = 200 is 4 k-blocks, the last one zero-filled, so the 3-stage ring wraps inside a tile
    M, N, Kd = 128 * n_sm + 77, 5 * 256 + 136, 200
    a, b = rnd(M, Kd, seed=11), rnd(N, Kd, seed=12, scale=0.5)
    bias = torch.randn(N, device="cuda")
    c = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    act = K.ACT_NONE if lse else K.ACT_RELU
    parts = None
    if lse:
        parts = torch.full((K.row_lse_parts(M, N, 256), M, 2), float("nan"), device="cuda")
    K.gemm(a, b, c, alpha=0.5, bias=bias, act=act, block_n=256, row_lse=parts)
    ref = 0.5 * (a.float() @ b.float().t()) + bias
    if act == K.ACT_RELU:
        ref = torch.relu(ref)
    assert rel(c, ref) < 4e-3
    if not lse:
        return
    # the partials are taken over the rounded bf16 output the kernel wrote, one per 256-wide N tile
    l2e = 1.4426950408889634
    assert parts.shape[0] == math.ceil(N / 256)
    for nb in range(parts.shape[0]):
        x = c[:, nb * 256:(nb + 1) * 256].float()
        m_ref = x.max(dim=1).values * l2e
        s_ref = torch.exp2(x.double() * l2e - m_ref.double()[:, None]).sum(dim=1)
        m, s = parts[nb, :, 0], parts[nb, :, 1]
        assert torch.allclose(m, m_ref, rtol=1e-6, atol=0), nb
        assert torch.allclose(s.double(), s_ref, rtol=2e-5, atol=0), nb
