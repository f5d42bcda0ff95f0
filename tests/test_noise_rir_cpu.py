"""On-the-fly noise and reverberation without a GPU: the numpy restatement against the reference fixture
(tests/golden/frontend_noise_rir.npz), the loader's draw order, --snr_range, the audio banks and the workspace query."""
import os
import random

import numpy as np
import pytest
import torch

import noise_rir_oracle as nro
from test_loader_cpu import loader_args, make_dataset


def fixture_cases(golden_dir):
    d = np.load(os.path.join(golden_dir, "frontend_noise_rir.npz"))
    for key in d["cases"]:
        key = str(key)
        rate, db, snr, off = d["meta_" + key]
        rir = str(d["rirname_" + key])
        yield d, key, float(rate), float(db), (None if np.isnan(snr) else float(snr)), int(off), (d["rir_" + rir] if rir else None)


def test_oracle_matches_reference_fixture(golden_dir):
    from oracle import frontend as ofe
    n = 0
    for d, key, rate, db, snr, off, rir in fixture_cases(golden_dir):
        aug = nro.augment(d["pcm"], rate, db, noise=d["noise"] if snr is not None else None, off=off, snr=snr, rir=rir)
        np.testing.assert_array_equal(aug, d["aug_" + key], err_msg=key)
        fb = ofe.kaldi_fbank(aug.astype(np.float32))
        np.testing.assert_allclose(fb, d["fbank_" + key], rtol=0, atol=2e-3, err_msg=key)
        n += 1
    assert n == 11


def exact_conv_augment(pcm, rate, db, noise, off, snr, rir):
    """the oracle chain with the convolution in float64 (what the GPU computes), rounded to float32 on the rate == 1.0 branch"""
    from oracle import frontend as ofe
    s = nro.normalize_inplace(ofe.change_speed(ofe.to_float32(pcm), rate), db)
    if noise is not None:
        s = nro.add_noise(s, noise, off, np.float64(snr))
    if rir is not None:
        from scipy import signal
        t = ofe.rms_db(s)
        y = signal.fftconvolve(s.astype(np.float64), ofe.to_float32(rir).astype(np.float64), "same").astype(s.dtype)
        s = nro.normalize_inplace(y, t)
    return ofe.to_int16(s)


def test_float64_convolution_stays_within_the_gpu_bounds(golden_dir):
    """the GPU test's bounds, set here: a float64 convolution moves no int16 sample on the float64 branches, and at most 1 LSB on
    a small share of the samples on the rate == 1.0 branch, where the reference's fftconvolve runs in float32"""
    for d, key, rate, db, snr, off, rir in fixture_cases(golden_dir):
        if rir is None:
            continue
        got = exact_conv_augment(d["pcm"], rate, db, d["noise"] if snr is not None else None, off, snr, rir)
        diff = np.abs(got.astype(np.int32) - d["aug_" + key].astype(np.int32))
        assert diff.max() <= 1, key
        assert (diff != 0).mean() < (0.05 if rate == 1.0 else 1e-3), (key, (diff != 0).mean())


def test_snr_range_parsing():
    from pika_b200.loader.otf_utt_loader import snr_params
    assert snr_params("") == (10.0, 10.0)
    assert snr_params("5,15") == (10.0, 5.0)
    assert snr_params("-5,25") == (10.0, 15.0)
    for bad in ("5", "10,10", "20,0", "1,2,3"):
        with pytest.raises(ValueError):
            snr_params(bad)


def write_bank(tmp_path, name, lengths, seed):
    rng = np.random.default_rng(seed)
    mrk, seq = tmp_path / (name + ".mrk"), tmp_path / (name + ".seq")
    segs, off = [], 0
    with open(mrk, "w") as fm, open(seq, "wb") as fs:
        for i, n in enumerate(lengths):
            s = rng.integers(-2000, 2000, n).astype(np.int16)
            segs.append(s)
            fm.write("%s_%d %d %d\n" % (name, i, off, 2 * n))
            fs.write(s.tobytes())
            off += 2 * n
    lst = tmp_path / (name + ".lst")
    lst.write_text("%s %s\n\n" % (mrk, seq))
    return str(lst), segs


def test_noise_bank_rms_and_short_segment_filter(tmp_path):
    from pika_b200.loader.audio_bank import AudioBank, max_new_len
    from oracle import frontend as ofe
    assert max_new_len(100) == 16399
    lst, segs = write_bank(tmp_path, "nz", [16399, 16398, 20000, 500], 1)
    bank = AudioBank.noise(lst, 100)
    assert len(bank) == 2 and bank.ids == ["nz_0", "nz_2"]
    assert bank.lengths.tolist() == [16399, 20000] and bank.offsets.tolist() == [0, 16399]
    np.testing.assert_array_equal(bank.samples, np.concatenate([segs[0], segs[2]]))
    for i, s in zip(range(2), (segs[0], segs[2])):
        assert bank.rms_db[i] == float(ofe.rms_db(ofe.to_float32(s)))
    with pytest.raises(ValueError, match="20399"):
        AudioBank.noise(lst, 125)


def test_rir_bank_length_limit(tmp_path):
    from pika_b200.loader.audio_bank import AudioBank
    lst, segs = write_bank(tmp_path, "rir", [1, 777, 65536], 2)
    bank = AudioBank.rir(lst)
    assert bank.lengths.tolist() == [1, 777, 65536] and bank.rms_db is None
    lst2, _ = write_bank(tmp_path, "long", [100, 65537], 3)
    with pytest.raises(ValueError, match="long_1"):
        AudioBank.rir(lst2)


def test_workspace_query_rejects_rir_lengths_without_a_device():
    from pika_b200._lib import lib
    assert lib.pk_frontend_noise_rir_workspace_bytes(4, 20000, 120, 80, 240, 0) < 0
    assert lib.pk_frontend_noise_rir_workspace_bytes(4, 20000, 120, 80, 240, 65537) < 0
    base = lib.pk_frontend_workspace_bytes(4, 20000, 120, 80, 240)
    for m in (1, 777, 16000, 65536):
        assert lib.pk_frontend_noise_rir_workspace_bytes(4, 20000, 120, 80, 240, m) > base
    assert lib.pk_conv_same_f64_workspace_bytes(2, 1000, 0) < 0 and lib.pk_conv_same_f64_workspace_bytes(2, 1000, 65537) < 0


def test_raw_batch_keys_unchanged_without_banks(tmp_path):
    from pika_b200.loader import otf_utt_loader as L
    lst, _ = make_dataset(tmp_path, n_utts=4, shards=1)
    random.seed(1); np.random.seed(1)
    (raw, _, _, _), = list(L.dataloader(lst, [], [], loader_args()))
    assert sorted(raw) == ["n_frames", "n_samples", "new_len", "pcm", "rate", "t_max", "target_db"]


def test_loader_draw_order_with_noise_and_rir(tmp_path):
    """per utterance read (the TU filter's drops included): randint (speed), uniform (gain), truncnorm (snr), randint (noise
    segment), randint (noise offset), randint (RIR)"""
    from scipy.stats import truncnorm
    from pika_b200.frontend import Frontend
    from pika_b200.loader import otf_utt_loader as L
    from pika_b200.loader.audio_bank import AudioBank
    lst, utts = make_dataset(tmp_path, n_utts=8, shards=1)
    nlst, _ = write_bank(tmp_path, "nz", [16399, 30000, 17000], 4)
    rlst, _ = write_bank(tmp_path, "rir", [1, 800, 4000], 5)
    noise, rir = AudioBank.noise(nlst, 100), AudioBank.rir(rlst)
    a = loader_args(max_len=100, snr_range="-5,25", TU_limit=60)        # some utterances fail the TU filter
    random.seed(7); np.random.seed(7)
    batches = list(L.dataloader(lst, rir, noise, a))
    random.seed(7); np.random.seed(7)
    kept = []
    for pcm, lab in utts:
        spr = [0.9, 1.0, 1.1][random.randint(0, 2)]
        db = np.random.uniform(-50.0, -10.0)
        new_len, frames = Frontend.lengths([len(pcm)], [spr])
        snr = truncnorm.rvs(-1.0, 1.0, loc=10.0, scale=15.0)
        k = random.randint(0, len(noise) - 1)
        off = random.randint(0, max(0, int(noise.lengths[k]) - new_len[0]))
        r = random.randint(0, len(rir) - 1)
        if 0 < frames[0] <= 100 and len(lab) * frames[0] // 3 <= 60:
            kept.append((spr, db, snr, k, off, r))
    assert 0 < len(kept) < len(utts)
    got = []
    for raw, _, _, _ in batches:
        if raw is None:
            continue
        assert raw["noise_idx"].dtype == torch.int32 and raw["noise_off"].dtype == torch.int64 and raw["snr"].dtype == torch.float64
        assert raw["rir_max_len"] == int(rir.lengths[raw["rir_idx"].numpy()].max())
        for i in range(raw["pcm"].shape[0]):
            got.append((float(raw["rate"][i]), float(raw["target_db"][i]), float(raw["snr"][i]), int(raw["noise_idx"][i]),
                        int(raw["noise_off"][i]), int(raw["rir_idx"][i])))
            assert int(raw["noise_off"][i]) + int(raw["new_len"][i]) <= noise.lengths[int(raw["noise_idx"][i])]
    assert len(got) == len(kept)
    for g, k in zip(got, kept):
        assert g[0] == pytest.approx(k[0]) and g[1] == pytest.approx(float(np.float32(k[1])))
        assert g[2] == k[2] and g[3:] == k[3:]
