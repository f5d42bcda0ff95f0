"""The row-skip test of the compacted RNN-T gradient (grad_row_kept in csrc/rnnt_loss.cu), restated in numpy: a row is skipped when
the magnitude bits of its f32 occupancy terms gb, gl sum to less than 0x2000 (|gb| + |gl| < 2^-136), and then every entry of its
gradient row rounds to bf16 +-0.  The row map is the order-keeping compaction of the kept rows."""
import numpy as np


def kept(gb, gl):
    bits = lambda x: x.astype(np.float32).view(np.uint32).astype(np.uint64) & 0x7FFFFFFF
    return bits(gb) + bits(gl) >= 0x2000


def bf16_is_zero(x):
    """round-to-nearest-even of f32 to bf16 gives +-0"""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return (r & 0x7FFF) == 0


def row_map(keep):
    m = np.full(keep.shape, -1, np.int64)
    m[keep] = np.arange(int(keep.sum()))
    return m


def test_skipped_rows_store_only_zeros():
    rng = np.random.default_rng(0)
    n = 20000
    # occupancies around the threshold, both signs (gb and gl share the sign of the upstream gradient)
    e = rng.uniform(-150.0, -125.0, (n, 2))
    sign = np.where(rng.random(n) < 0.5, -1.0, 1.0)[:, None]
    g = (sign * np.exp2(e)).astype(np.float32)
    gb, gl = g[:, 0], g[:, 1]
    keep = kept(gb, gl)
    assert 0 < keep.sum() < n
    # |gb| + |gl| < 2^-136 exactly when skipped (both are subnormals there, so the f64 sum is exact)
    s = np.abs(gb.astype(np.float64)) + np.abs(gl.astype(np.float64))
    assert np.array_equal(~keep, s < 2.0 ** -136)
    # the entries the gradient kernel forms, in f32: p * -(gb + gl) (+ gb in the blank column, + gl in the label column), p in [0, 1]
    p = rng.random((n, 16)).astype(np.float32)
    p[:, 0] = 1.0
    gsum = -(gb + gl)
    ent = p * gsum[:, None]
    ent[:, 1] += gb
    ent[:, 2] += gl
    ent[:, 3] = np.float32(1.0) * gsum + gb
    assert bf16_is_zero(ent[~keep]).all()


def test_row_map_keeps_order():
    keep = np.array([0, 1, 1, 0, 0, 1, 0, 1], bool)
    assert row_map(keep).tolist() == [-1, 0, 1, -1, -1, 2, -1, 3]
    assert row_map(np.zeros(5, bool)).tolist() == [-1] * 5
