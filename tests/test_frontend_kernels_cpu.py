"""The front-end kernel oracle (tests/frontend_kernels_oracle.py) pinned to the existing oracles: on Kaldi's own tables its fbank and
MFCC are tests/fbank_opts_oracle.kaldi_fbank and tests/mfcc_oracle.kaldi_mfcc, and its splice / CMN / CMVN / SpecAugment is
oracle/frontend.py's batch assembly within float32 rounding."""
import numpy as np
import pytest

import fbank_opts_oracle as fo
import frontend_kernels_oracle as fko
import mfcc_oracle as mo
from oracle import frontend as ofe

WINDOWS = ("hamming", "hanning", "povey", "rectangular", "blackman")


def _signal(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = 4000 * np.sin(2 * np.pi * 440 * t / 16000) + rng.normal(0, 1500, n) + 300
    return np.clip(np.round(x), -32768, 32767).astype(np.float32)


@pytest.mark.parametrize("window_type", WINDOWS)
@pytest.mark.parametrize("snip_edges", [True, False])
def test_fbank_from_tables_is_kaldi_fbank(window_type, snip_edges):
    from pika_b200.frontend import FbankOptions, fbank_tables
    kw = dict(num_mel_bins=40, sample_frequency=16000.0, frame_length=25.0, frame_shift=10.0, window_type=window_type,
              snip_edges=snip_edges, low_freq=40.0, high_freq=-200.0)
    o = FbankOptions(dither=0.0, **kw)
    win, _, w, lo, hi = fbank_tables(o)
    wave = _signal(5123, 1)
    ref = fo.kaldi_fbank(wave, **kw)
    got, mel, _ = fko.fbank_from_tables(wave, ref.shape[0], win, w, lo, hi, o.n_fft, o.frame_shift_samples, snip_edges)
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, atol=2e-4)            # float32 power spectrum and mel product on the Kaldi side


@pytest.mark.parametrize("window_type", WINDOWS)
@pytest.mark.parametrize("snip_edges", [True, False])
@pytest.mark.parametrize("use_energy,raw_energy,htk_compat,energy_floor", [(1, 1, 0, 0.0), (1, 0, 1, 0.0), (0, 1, 1, 0.0),
                                                                            (1, 1, 0, 1e12)])
def test_mfcc_from_tables_is_kaldi_mfcc(window_type, snip_edges, use_energy, raw_energy, htk_compat, energy_floor):
    from pika_b200.frontend import MfccOptions, fbank_tables, mfcc_tables
    kw = dict(num_ceps=13, num_mel_bins=23, use_energy=bool(use_energy), raw_energy=bool(raw_energy), htk_compat=bool(htk_compat),
              energy_floor=energy_floor, cepstral_lifter=22.0, window_type=window_type, snip_edges=snip_edges)
    o = MfccOptions(dither=0.0, **kw)
    win, _, w, lo, hi = fbank_tables(o)
    wave = _signal(4711, 2)
    ref = mo.kaldi_mfcc(wave, **kw)
    got, _ = fko.mfcc_from_tables(wave, ref.shape[0], win, w, lo, hi, o.n_fft, o.frame_shift_samples, mfcc_tables(o),
                                  use_energy, raw_energy, energy_floor, htk_compat, snip_edges)
    assert got.shape == ref.shape
    if energy_floor > 0.0:
        assert (ref[:, 0] == np.float32(np.log(energy_floor))).any()       # the floor binds on some frames
    np.testing.assert_allclose(got, ref, atol=2e-4, rtol=1e-5)              # the DCT table is float32 with the lifter folded in


def test_reflect_matches_kaldi_frame_indices():
    for n, fl, fs in [(1, 400, 160), (7, 400, 160), (250, 512, 100), (5000, 400, 160)]:
        T = fo.num_frames(n, fl, fs, False)
        ref = fo.frame_indices(n, fl, fs, False)
        idx = fko.reflect(fko.frame_starts(T, fl, fs, False)[:, None] + np.arange(fl)[None, :], n)
        np.testing.assert_array_equal(idx, ref)


@pytest.mark.parametrize("stride", [1, 3])
def test_splice_cmn_f32_matches_oracle_chain(stride):
    rng = np.random.default_rng(5 + stride)
    lens = [150, 37, 2, 1]
    feats = [(rng.standard_normal((n, 20)) * 3 + 7).astype(np.float32) for n in lens]
    lctx, rctx = 2, 1
    data, _, out_lens, _ = ofe.assemble_batch(feats, [[1]] * len(feats), lctx, rctx, stride, tu_limit=10 ** 9)
    t_max = data.shape[1]
    assert list(out_lens) == [(n + stride - 1) // stride for n in lens]
    off, sc = rng.standard_normal(data.shape[2]), np.abs(rng.standard_normal(data.shape[2])) + 0.5
    sa = (data.shape[2] - 5, 9, t_max - 3, 40)                    # both masks run past the end
    ref = ofe.spec_augment(ofe.apply_cmvn(data, off, sc, cmn=True), *sa)
    got = fko.splice_cmn_f32(feats, t_max, lctx, rctx, stride, True, off, sc, sa)
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=2e-5 * float(np.abs(ref).max()))
    assert (got[:, :, -5:] == 0).all() and (got[:, t_max - 3:] == 0).all()
    plain = fko.splice_cmn_f32(feats, t_max, lctx, rctx, stride, False)
    np.testing.assert_array_equal(plain, data)                   # the splice itself is a gather: exact
    b16 = fko.splice_cmn_f32(feats, t_max, lctx, rctx, stride, True, off, sc, sa, bf16=True)
    import torch
    np.testing.assert_array_equal(b16, torch.from_numpy(got).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16))


def test_cmn_sums_order_is_blockwise():
    """column sums whose float32 rounding tells block order from a flat row-order sum: 2^24 + 1 + 1 rounds to 2^24 row by row,
    while block 1's partial 1 + 1 = 2 added to 2^24 is exact"""
    x = np.zeros((129, 1), np.float32)
    x[0], x[64], x[65], x[128] = 2.0 ** 24, 1.0, 1.0, -(2.0 ** 24)
    flat = np.float32(0.0)
    for v in x[:, 0]:
        flat = np.float32(flat + v)
    assert flat == 0.0
    assert fko.cmn_sums(x)[0] == np.float32(2.0)
