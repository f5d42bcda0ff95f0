"""The bf16 GEMM's row log-sum-exp partials: the consumer warps take each row's max in registers while they round the tile, and the
exp-sum of that tile while the next tile's main loop runs, one slice per k-block, with the slices left over after it (short K) and
the whole sum of a worker's last tile after its unit loop.  These cases reach every part of that schedule: a single k-block and
fewer k-blocks than slices, one tile per persistent worker and about six, ragged M, a last N tile with 8 valid columns and one whose
second 128-column half is empty, and rows shifted far below zero."""
import pytest
import torch

pytestmark = pytest.mark.gpu

L2E = 1.4426950408889634


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def shape(case, n_sm):
    if case == "one_tile_per_worker":      # n_sm // 2 row tiles x 2 N tiles; the last N tile has 8 valid columns
        return 128 * (n_sm // 2) - 40, 256 + 8
    return 256 * n_sm + 77, 2 * 256 + 128  # ~6 tiles per worker; the last N tile's second 128-column half is empty


@pytest.mark.parametrize("Kd", [64, 200])
@pytest.mark.parametrize("case", ["one_tile_per_worker", "six_tiles_per_worker"])
def test_gemm_row_lse_partials(Kd, case):
    from pika_b200 import kernels as K
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    M, N = shape(case, n_sm)
    a, b = rnd(M, Kd, seed=21), rnd(N, Kd, seed=22, scale=0.5)
    # the last k column adds -200 to every fifth row: those rows lie far below zero, where 2^(x * log2e) alone underflows
    a[:, -1] = 0
    a[::5, -1] = -400
    b[:, -1] = 1
    bias = torch.randn(N, device="cuda") * 3
    c = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    parts = torch.full((K.row_lse_parts(M, N, 256), M, 2), float("nan"), device="cuda")
    K.gemm(a, b, c, alpha=0.5, bias=bias, block_n=256, row_lse=parts)
    ref = 0.5 * (a.float() @ b.float().t()) + bias
    assert ((c.float() - ref).norm() / ref.norm()).item() < 4e-3
    assert parts.shape[0] == (N + 255) // 256
    # the partials are taken over the rounded bf16 output the kernel wrote, one per 256-wide N tile
    for nb in range(parts.shape[0]):
        x = c[:, nb * 256:(nb + 1) * 256].float()
        m_ref = x.max(dim=1).values * L2E
        s_ref = torch.exp2(x.double() * L2E - m_ref.double()[:, None]).sum(dim=1)
        m, s = parts[nb, :, 0], parts[nb, :, 1]
        assert torch.equal(m, m_ref), nb
        assert torch.allclose(s.double(), s_ref, rtol=2e-5, atol=0), nb
