"""Kaldi fbank options of the GPU front end, host side: option parsing and Kaldi's validation, the frame arithmetic against
torchaudio's, the numpy oracle against the torchaudio fixture (tests/golden/fbank_opts.npz), the host tables against the oracle's,
and the loader's ``--stride`` lengths and TU filter against the oracle's batch assembly."""
import json
import os
import random

import numpy as np
import pytest

import fbank_opts_oracle as fo


def fixture_configs(golden_dir):
    d = np.load(os.path.join(golden_dir, "fbank_opts.npz"))
    return d, json.loads(str(d["configs"]))


def oracle_kwargs(o):
    return dict(num_mel_bins=o.num_mel_bins, sample_frequency=o.sample_frequency, frame_length=o.frame_length,
                frame_shift=o.frame_shift, window_type=o.window_type, snip_edges=o.snip_edges, remove_dc_offset=o.remove_dc_offset,
                preemphasis_coefficient=o.preemphasis_coefficient, low_freq=o.low_freq, high_freq=o.high_freq,
                blackman_coeff=o.blackman_coeff)


def test_from_config_parses_every_option(tmp_path):
    from pika_b200.frontend import FbankOptions
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--sample-frequency=8000\n--frame-length=30\n--frame-shift=12.5\n--window-type=blackman\n--blackman-coeff=0.4\n"
                   "--snip-edges=false\n--remove-dc-offset=false\n--round-to-power-of-two=true\n--preemphasis-coefficient=0.9\n"
                   "--dither=0\n--low-freq=60\n--high-freq=3500\n--num-mel-bins=30\n")
    o = FbankOptions.from_config(str(cfg))
    assert (o.sample_frequency, o.frame_length, o.frame_shift, o.window_type, o.blackman_coeff) == (8000.0, 30.0, 12.5, "blackman", 0.4)
    assert (o.snip_edges, o.remove_dc_offset, o.preemphasis_coefficient, o.dither) == (False, False, 0.9, 0.0)
    assert (o.low_freq, o.high_freq, o.num_mel_bins) == (60.0, 3500.0, 30)
    assert (o.frame_len, o.frame_shift_samples, o.n_fft, o.log2_nfft) == (240, 100, 256, 8)
    assert o.geometry() == dict(frame_len=240, frame_shift=100, snip_edges=False)
    # Kaldi's defaults without a config file; the recipe's keywords keep their meaning
    d = FbankOptions()
    assert (d.window_type, d.num_mel_bins, d.low_freq, d.high_freq, d.frame_len, d.frame_shift_samples, d.n_fft) == \
        ("povey", 23, 20.0, 0.0, 400, 160, 512)
    assert d.snip_edges and d.remove_dc_offset and d.round_to_power_of_two
    r = FbankOptions(num_mel_bins=80, low_freq=40.0, high_freq=-200.0, dither=0.0, window_type="hamming")
    assert r.geometry() == dict(frame_len=400, frame_shift=160, snip_edges=True) and r.log2_nfft == 9


@pytest.mark.parametrize("line", ["--use-energy=false", "--raw-energy=true", "--energy-floor=1", "--htk-compat=false",
                                  "--use-log-fbank=true", "--use-power=true", "--vtln-warp=1.0", "--vtln-low=100", "--vtln-high=-500",
                                  "--allow-downsample=true", "--allow-upsample=true", "--round-to-power-of-two=false",
                                  "--window-type=sine", "--snip-edges=maybe", "--sample-frequency=0", "--frame-length=0.01",
                                  "--sample-frequency=2000", "--sample-frequency=96000", "--frame-length=50\n--sample-frequency=44100",
                                  "--no-such-option=1", "--snip-edges"])
def test_from_config_rejects(tmp_path, line):
    from pika_b200.frontend import FbankOptions
    cfg = tmp_path / "bad.conf"
    cfg.write_text(line + "\n")
    with pytest.raises(ValueError):
        FbankOptions.from_config(str(cfg))


@pytest.mark.parametrize("kw", [dict(sample_frequency=8000.0, num_mel_bins=100),           # low mel bins without an FFT bin
                                dict(sample_frequency=8000.0, num_mel_bins=128, low_freq=40.0, high_freq=-200.0),
                                dict(low_freq=8000.0), dict(low_freq=4000.0, high_freq=3000.0), dict(high_freq=8001.0),
                                dict(high_freq=-8000.0), dict(low_freq=-1.0), dict(num_mel_bins=257), dict(num_mel_bins=2)])
def test_mel_bank_validation_raises_where_kaldi_does(kw):
    from pika_b200.frontend import FbankOptions, fbank_tables
    with pytest.raises(ValueError):
        fbank_tables(FbankOptions(**kw))


def test_frame_counts_match_torchaudio():
    tk = pytest.importorskip("torchaudio.compliance.kaldi")
    import torch
    from pika_b200.frontend import FbankOptions, Frontend
    for sr, ms, snip in [(8000.0, 25.0, True), (8000.0, 25.0, False), (16000.0, 50.0, False), (44100.0, 25.0, True),
                         (44100.0, 25.0, False), (22050.0, 30.0, False)]:
        o = FbankOptions(sample_frequency=sr, frame_length=ms, snip_edges=snip, num_mel_bins=23)
        L, S = o.frame_len, o.frame_shift_samples
        ns = [L, L + 1, L + S - 1, L + S, L + S // 2, L + S // 2 + 1, 3 * L + 7, 5000]
        _, frames = Frontend.lengths(ns, [1.0] * len(ns), **o.geometry())
        for n, t in zip(ns, frames):
            f = tk.fbank(torch.ones(1, n), sample_frequency=sr, frame_length=ms, snip_edges=snip, dither=0.0, num_mel_bins=23)
            assert f.shape[0] == t == fo.num_frames(n, L, S, snip), (sr, ms, snip, n)
    # the recipe's arithmetic is kept as the default
    assert Frontend.lengths([160240, 399], [1.0, 1.0]) == ([160240, 399], [1000, 0])


def test_oracle_matches_torchaudio_fixture(golden_dir):
    from pika_b200.frontend import FbankOptions
    d, cfgs = fixture_configs(golden_dir)
    assert len(cfgs) == 7
    for c, cfg in enumerate(cfgs):
        o = FbankOptions(**dict(cfg, dither=0.0))
        for k in range(3):
            ref = d["fbank_%d_%d" % (c, k)]
            got = fo.kaldi_fbank(d["pcm_%d_%d" % (c, k)].astype(np.float32), **oracle_kwargs(o))
            assert got.shape == ref.shape, (c, k)
            np.testing.assert_allclose(got, ref, atol=1e-3)
            assert np.abs(got - ref).mean() < 2e-5, (c, k)


def test_host_tables_match_the_oracle(golden_dir):
    from oracle import frontend as ofe
    from pika_b200.frontend import FbankOptions, fbank_tables
    _, cfgs = fixture_configs(golden_dir)
    for cfg in cfgs + [dict(window_type="blackman", blackman_coeff=0.38)]:
        o = FbankOptions(**cfg)
        win, tw, w, lo, hi = fbank_tables(o)
        assert win.shape == (o.frame_len,) and tw.shape == (o.n_fft // 2, 2) and w.shape == (o.num_mel_bins, o.n_fft // 2)
        np.testing.assert_allclose(win, fo.window(o.frame_len, o.window_type, o.blackman_coeff), atol=1e-6)
        np.testing.assert_allclose(w, ofe.mel_banks(o.num_mel_bins, o.sample_frequency, o.low_freq, o.high_freq, o.n_fft), atol=1e-6)
        for j in range(o.num_mel_bins):
            nz = np.nonzero(w[j])[0]
            assert lo[j] == nz[0] and hi[j] == nz[-1] + 1
    # the recipe's tables are the ones the 16 kHz front end always used
    o = FbankOptions(num_mel_bins=80, low_freq=40.0, high_freq=-200.0, dither=0.0, window_type="hamming")
    win, _, w, _, _ = fbank_tables(o)
    np.testing.assert_array_equal(win, ofe.hamming_window(400))
    np.testing.assert_array_equal(w, ofe.mel_banks(80, n_fft=512))


def test_oracle_reflects_a_signal_shorter_than_one_frame():
    """snip_edges=false on 120 samples at 8 kHz (200-sample frames, shift 80): two frames, every window sample reflected about the
    signal's edges as many times as needed (Kaldi's ExtractWindow loop) -- a case torchaudio's single reflection cannot produce"""
    n, L, S = 120, 200, 80
    idx = fo.frame_indices(n, L, S, snip_edges=False)
    assert idx.shape == (2, L)
    for t in range(2):
        for i in range(L):
            s = t * S + S // 2 - L // 2 + i
            while s < 0 or s >= n:
                s = -s - 1 if s < 0 else 2 * n - 1 - s
            assert idx[t, i] == s
    rng = np.random.default_rng(0)
    wave = rng.normal(0, 1000, n).astype(np.float32)
    f = fo.kaldi_fbank(wave, num_mel_bins=40, sample_frequency=8000.0, window_type="hamming", snip_edges=False, low_freq=20.0,
                       high_freq=0.0)
    assert f.shape == (2, 40) and np.isfinite(f).all()


@pytest.mark.parametrize("stride,config", [(2, None), (3, "--sample-frequency=8000\n--num-mel-bins=40\n--snip-edges=false\n")])
def test_loader_stride_lengths_and_tu_filter(tmp_path, stride, config):
    """--stride: lens / t_max are the strided row counts (ceil(n_frames / stride)), the TU filter and --max_len apply to them, and the
    raw batch keeps the fbank frame counts for the front end -- against oracle/frontend.py:assemble_batch on the same draws"""
    from oracle import frontend as ofe
    from test_loader_cpu import loader_args, make_dataset
    from pika_b200.frontend import FbankOptions, Frontend
    from pika_b200.loader import otf_utt_loader as L
    lst, utts = make_dataset(tmp_path, n_utts=8, shards=1)
    kw = dict(stride=stride, TU_limit=40, max_len=18)
    opts = FbankOptions(num_mel_bins=80)
    if config:
        cfg = tmp_path / "fbank.conf"
        cfg.write_text(config)
        kw.update(feat_config=str(cfg), sample_rate=8000)
        opts = FbankOptions.from_config(str(cfg))
    a = loader_args(**kw)
    random.seed(7); np.random.seed(7)
    batches = list(L.dataloader(lst, [], [], a))
    assert len(batches) == 2
    random.seed(7); np.random.seed(7)
    k = 0
    for raw, target, lens, ali_lens in batches:
        feats, labels, frames_kept = [], [], []
        for _ in range(a.batch_size):
            pcm, lab = utts[k]
            spr = [0.9, 1.0, 1.1][random.randint(0, 2)]
            np.random.uniform(-50.0, -10.0)
            _, frames = Frontend.lengths([len(pcm)], [spr], **opts.geometry())
            rows = -(-frames[0] // stride)
            if 0 < rows <= a.max_len:
                feats.append(np.zeros((frames[0], 1), np.float32))
                labels.append(lab)
                frames_kept.append(frames[0])
            k += 1
        data, tgt, ref_lens, ref_ali = ofe.assemble_batch(feats, labels, 0, 0, stride=stride, tu_limit=a.TU_limit, padding_tgt=99)
        if data is None:
            assert raw is None and lens.tolist() == [0]
            continue
        assert lens.tolist() == ref_lens.tolist() and ali_lens.tolist() == ref_ali.tolist()
        assert target.numpy().tolist() == tgt.tolist()
        assert raw["t_max"] == data.shape[1] == max(lens.tolist())
        kept = [f for f, lab in zip(frames_kept, labels) if len(lab) * (-(-f // stride)) // 3 <= a.TU_limit]
        assert raw["n_frames"].tolist() == kept
    assert k == 8


def test_loader_refuses_a_sample_rate_other_than_the_configs(tmp_path):
    from test_loader_cpu import loader_args, make_dataset
    from pika_b200.loader import otf_utt_loader as L
    lst, _ = make_dataset(tmp_path, n_utts=4, shards=1)
    with pytest.raises(ValueError):
        next(L.dataloader(lst, [], [], loader_args(sample_rate=8000)))
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--sample-frequency=8000\n--num-mel-bins=40\n")
    with pytest.raises(ValueError):
        next(L.dataloader(lst, [], [], loader_args(feat_config=str(cfg))))
