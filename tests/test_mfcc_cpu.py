"""Kaldi MFCC options and host tables of the front end, the numpy MFCC oracle against the torchaudio fixture
(tests/golden/mfcc.npz), the MFCC entry points' argument checks, and ``--feat_type`` / ``--feats_dim`` in the loader and the CMVN
tool.  No GPU needed."""
import argparse
import json
import os

import numpy as np
import pytest

import mfcc_oracle as mo


def test_defaults_are_kaldis():
    from pika_b200.frontend import FbankOptions, MfccOptions
    o = MfccOptions()
    assert (o.num_ceps, o.use_energy, o.energy_floor, o.raw_energy, o.cepstral_lifter, o.htk_compat) == (13, True, 0.0, True, 22.0, False)
    f = FbankOptions()
    for k in ("num_mel_bins", "sample_frequency", "low_freq", "high_freq", "dither", "window_type", "preemphasis_coefficient",
              "frame_length", "frame_shift", "snip_edges", "remove_dc_offset", "blackman_coeff", "round_to_power_of_two", "frame_len",
              "frame_shift_samples", "n_fft"):
        assert getattr(o, k) == getattr(f, k), k
    assert (o.num_mel_bins, o.dither) == (23, 1.0)


def test_from_config_parses_every_option(tmp_path):
    from pika_b200.frontend import MfccOptions
    cfg = tmp_path / "mfcc_hires.conf"
    cfg.write_text("--use-energy=false   # only non-default options\n--num-mel-bins=40\n--num-ceps=40\n--low-freq=20\n--high-freq=-400\n"
                   "--energy-floor=0.5\n--raw-energy=false\n--cepstral-lifter=0\n--htk-compat=true\n--sample-frequency=8000\n"
                   "--frame-length=20\n--frame-shift=8\n--window-type=hamming\n--snip-edges=false\n--remove-dc-offset=false\n"
                   "--preemphasis-coefficient=0.9\n--dither=0\n--blackman-coeff=0.4\n--round-to-power-of-two=true\n")
    o = MfccOptions.from_config(str(cfg))
    assert (o.use_energy, o.num_mel_bins, o.num_ceps, o.low_freq, o.high_freq) == (False, 40, 40, 20.0, -400.0)
    assert (o.energy_floor, o.raw_energy, o.cepstral_lifter, o.htk_compat) == (0.5, False, 0.0, True)
    assert (o.sample_frequency, o.frame_len, o.frame_shift_samples, o.n_fft, o.window_type) == (8000.0, 160, 64, 256, "hamming")
    assert (o.snip_edges, o.remove_dc_offset, o.preemphasis_coefficient, o.dither, o.blackman_coeff) == (False, False, 0.9, 0.0, 0.4)


@pytest.mark.parametrize("line", ["--num-ceps=0", "--num-ceps=24", "--num-mel-bins=12", "--use-log-fbank=true", "--use-power=false",
                                  "--vtln-warp=1.1", "--vtln-low=100", "--vtln-high=-500", "--allow-downsample=true",
                                  "--allow-upsample=true", "--no-such-option=1", "--round-to-power-of-two=false"])
def test_from_config_rejects(tmp_path, line):
    """num-ceps outside [1, num-mel-bins] (23 by default), fbank-only, VTLN, resampling and unknown options"""
    from pika_b200.frontend import MfccOptions
    cfg = tmp_path / "mfcc.conf"
    cfg.write_text(line + "\n")
    with pytest.raises(ValueError):
        MfccOptions.from_config(str(cfg))


def test_num_ceps_above_num_mel_bins_is_refused_with_kaldis_message():
    from pika_b200.frontend import MfccOptions
    with pytest.raises(ValueError, match="num-ceps cannot be larger than num-mel-bins"):
        MfccOptions(num_ceps=41, num_mel_bins=40)
    assert MfccOptions(num_ceps=40, num_mel_bins=40).num_ceps == 40


@pytest.mark.parametrize("num_ceps,n", [(13, 23), (40, 40), (20, 80), (1, 3)])
def test_dct_table_is_the_orthonormal_dct_ii(num_ceps, n):
    from scipy.fft import dct
    from pika_b200.frontend import dct_matrix
    ref = dct(np.eye(n), type=2, norm="ortho", axis=0)[:num_ceps]
    np.testing.assert_allclose(dct_matrix(num_ceps, n), ref, rtol=0, atol=1e-14)
    np.testing.assert_allclose(dct_matrix(num_ceps, n), mo.dct_matrix(num_ceps, n), rtol=0, atol=1e-14)


def test_lifter_table_and_its_fold_into_the_dct():
    from pika_b200.frontend import MfccOptions, dct_matrix, lifter_coeffs, mfcc_tables
    lift = lifter_coeffs(13, 22.0)
    assert lift[0] == 1.0
    np.testing.assert_allclose(lift, [1.0 + 11.0 * np.sin(np.pi * i / 22.0) for i in range(13)], rtol=1e-15)
    assert np.array_equal(lifter_coeffs(40, 0.0), np.ones(40))
    assert lift.max() == pytest.approx(12.0, rel=1e-3)                       # the peak 1 + Q/2 near i = Q/2
    t = mfcc_tables(MfccOptions(num_ceps=13, num_mel_bins=23))
    assert t.shape == (23, 13) and t.dtype == np.float32 and t.flags.c_contiguous
    np.testing.assert_array_equal(t, (dct_matrix(13, 23) * lift[:, None]).T.astype(np.float32))
    t0 = mfcc_tables(MfccOptions(num_ceps=40, num_mel_bins=40, cepstral_lifter=0.0))
    np.testing.assert_array_equal(t0, dct_matrix(40, 40).T.astype(np.float32))


def coefficient_scale(kw):
    """|lifter_k| * sum_j |dct[k, j]| per output column (1 for the energy column): the factor by which an error bound on every log
    mel energy bounds the error of each coefficient"""
    s = np.abs(mo.lifter(kw["num_ceps"], kw["cepstral_lifter"])) * np.abs(mo.dct_matrix(kw["num_ceps"], kw["num_mel_bins"])).sum(1)
    if kw["use_energy"]:
        s[0] = 1.0
    if kw["htk_compat"]:
        s = np.concatenate([s[1:], [s[0] * (1.0 if kw["use_energy"] else np.sqrt(2.0))]])
    return s


def fixture(golden_dir):
    import make_golden_mfcc as mg
    d = np.load(os.path.join(golden_dir, "mfcc.npz"))
    return d, [dict(mg.KALDI, **c) for c in json.loads(str(d["configs"]))]


def test_fixture_covers_the_grid(golden_dir):
    d, cfgs = fixture(golden_dir)
    assert {c["sample_frequency"] for c in cfgs} >= {8000.0, 16000.0, 22050.0, 48000.0}
    assert {(c["num_ceps"], c["num_mel_bins"]) for c in cfgs} >= {(13, 23), (40, 40), (20, 80)}
    for key in ("use_energy", "raw_energy", "htk_compat", "snip_edges"):
        assert {c[key] for c in cfgs} == {True, False}, key
    assert {c["htk_compat"] and c["use_energy"] for c in cfgs} == {True, False}
    assert {c["htk_compat"] and not c["use_energy"] for c in cfgs} == {True, False}
    assert {c["energy_floor"] > 0 for c in cfgs if c["use_energy"]} == {True, False}
    assert {c["cepstral_lifter"] for c in cfgs} == {0.0, 22.0}
    assert len({c["window_type"] for c in cfgs}) == 5
    eps_hit = floor_hit = False
    for c, kw in enumerate(cfgs):
        if not kw["use_energy"]:
            continue
        col = kw["num_ceps"] - 1 if kw["htk_compat"] else 0
        e = np.concatenate([d["mfcc_%d_%d" % (c, k)][:, col] for k in range(3)])
        if kw["energy_floor"] > 0:
            floor_hit |= bool((e == np.float32(np.log(kw["energy_floor"]))).any())
        else:
            eps_hit |= bool((np.abs(e - np.log(np.finfo(np.float32).eps)) < 1e-5).any())
    assert eps_hit and floor_hit


def test_oracle_matches_torchaudio_fixture(golden_dir):
    d, cfgs = fixture(golden_dir)
    for c, kw in enumerate(cfgs):
        s = coefficient_scale(kw)
        for k in range(3):
            got = mo.kaldi_mfcc(d["pcm_%d_%d" % (c, k)].astype(np.float32), **kw)
            ref = d["mfcc_%d_%d" % (c, k)]
            assert got.shape == ref.shape, (c, k)
            assert (np.abs(got - ref) / s).max() < 1e-4, (c, k)


def _null_mfcc_call(num_ceps, n_mel=23, dct=True):
    import ctypes
    from pika_b200 import _lib
    buf = ctypes.c_float(0.0)
    dct_ptr = ctypes.addressof(buf) if dct else None
    rc = _lib.lib.pk_mfcc(None, 400, None, None, 1, 1, n_mel, None, None, None, None, None, 400, 160, 9, 1, 1, 0.97, None, 0.0, 0, None,
                          dct_ptr, num_ceps, 1, 1, 0.0, 0)
    return rc, _lib.lib.pk_last_error()


@pytest.mark.parametrize("num_ceps,n_mel,dct", [(0, 23, True), (24, 23, True), (13, 23, False)])
def test_mfcc_entry_rejects_bad_arguments_before_touching_the_device(num_ceps, n_mel, dct):
    rc, msg = _null_mfcc_call(num_ceps, n_mel, dct)
    assert rc != 0 and b"MFCC" in msg


def loader_args(tmp_path, feat_type, feats_dim, conf=None):
    from pika_b200.loader import otf_utt_loader as L
    p = argparse.ArgumentParser()
    L.register(p)
    argv = ["--feat_type", feat_type, "--feats_dim", str(feats_dim)]
    if conf is not None:
        cfg = tmp_path / "feat.conf"
        cfg.write_text(conf)
        argv += ["--feat_config", str(cfg)]
    return p.parse_args(argv)


def test_loader_feat_type_and_feats_dim(tmp_path):
    from pika_b200.frontend import FbankOptions, MfccOptions
    from pika_b200.loader import otf_utt_loader as L
    assert loader_args(tmp_path, "fbank", 40).feat_type == "fbank"
    p = argparse.ArgumentParser()
    L.register(p)
    assert p.parse_args([]).feat_type == "fbank"
    with pytest.raises(SystemExit):
        p.parse_args(["--feat_type", "plp"])
    o = L.feature_options(loader_args(tmp_path, "mfcc", 40, "--num-mel-bins=40\n--num-ceps=40\n--use-energy=false\n"))
    assert type(o) is MfccOptions and (o.num_ceps, o.num_mel_bins, o.use_energy) == (40, 40, False)
    assert type(L.feature_options(loader_args(tmp_path, "fbank", 40, "--num-mel-bins=40\n"))) is FbankOptions
    o = L.feature_options(loader_args(tmp_path, "mfcc", 13))
    assert type(o) is MfccOptions and (o.num_ceps, o.num_mel_bins) == (13, 23)
    with pytest.raises(ValueError, match="feats_dim"):
        L.feature_options(loader_args(tmp_path, "mfcc", 40, "--num-ceps=13\n"))
    with pytest.raises(ValueError):                                            # an MFCC option in an fbank config
        L.feature_options(loader_args(tmp_path, "fbank", 13, "--num-ceps=13\n"))
    with pytest.raises(ValueError):                                            # 40 cepstra from Kaldi's default 23 mel bins
        L.feature_options(loader_args(tmp_path, "mfcc", 40))


def test_loader_frontend_cache_is_keyed_by_feat_type(tmp_path, monkeypatch):
    from pika_b200.loader import otf_utt_loader as L
    monkeypatch.setattr(L, "_frontends", {})
    monkeypatch.setattr(L, "Frontend", lambda opts, lctx, rctx, device, stride=1: opts)
    a = loader_args(tmp_path, "fbank", 13, "--num-mel-bins=40\n")            # the same config file read as either feature type
    fb = L._frontend_for(a, "cpu")
    a.feat_type = "mfcc"
    a.feats_dim = 13
    mf = L._frontend_for(a, "cpu")
    assert type(fb).__name__ == "FbankOptions" and type(mf).__name__ == "MfccOptions" and len(L._frontends) == 2


def cmvn_args(tmp_path, feat_type, feat_dim, conf=None):
    a = argparse.Namespace(feat_type=feat_type, feat_dim=feat_dim, sample_rate=16000, feat_config=None)
    if conf is not None:
        cfg = tmp_path / "cmvn_feat.conf"
        cfg.write_text(conf)
        a.feat_config = str(cfg)
    return a


def test_cmvn_tool_feat_type_and_feat_dim(tmp_path):
    from pika_b200.frontend import FbankOptions, MfccOptions
    from pika_b200.utils import compute_global_cmvn as C
    o = C.feature_options(cmvn_args(tmp_path, "mfcc", 40, "--num-mel-bins=40\n--num-ceps=40\n"))
    assert type(o) is MfccOptions and o.num_ceps == 40
    assert type(C.feature_options(cmvn_args(tmp_path, "fbank", 80, "--num-mel-bins=80\n"))) is FbankOptions
    assert C.feature_options(cmvn_args(tmp_path, "mfcc", 13)).num_ceps == 13
    with pytest.raises(ValueError, match="num-ceps"):
        C.feature_options(cmvn_args(tmp_path, "mfcc", 40, "--num-mel-bins=40\n--num-ceps=20\n"))
    with pytest.raises(ValueError, match="num-mel-bins"):
        C.feature_options(cmvn_args(tmp_path, "fbank", 40, "--num-mel-bins=80\n"))
    cfg = tmp_path / "m.conf"
    cfg.write_text("--num-ceps=13\n")
    with pytest.raises(ValueError, match="num-ceps"):                            # before any data or device is touched
        C.main(["no.lst", str(tmp_path / "stats"), "--feat_type", "mfcc", "--feat_config", str(cfg), "--feat_dim", "40"])


@pytest.mark.parametrize("num_ceps,n_mel,dct", [(0, 23, True), (24, 23, True), (13, 23, False)])
def test_full_chain_mfcc_entry_rejects_bad_arguments_before_touching_the_device(num_ceps, n_mel, dct):
    import ctypes
    from pika_b200 import _lib
    buf = ctypes.c_float(0.0)
    head = (None, 400, None, None, None, None, None, 1, 400, 1, n_mel, 1, 1, 1, None, None, None, None, None, 400, 160, 9, 1, 1, 0.97, 0,
            None, None, 0, 0, 0, 0, None, 0, None, None, 0, None, 0.0, 0, None)
    rc = _lib.lib.pk_frontend_fwd_mfcc(*head, *(None,) * 9, 1, ctypes.addressof(buf) if dct else None, num_ceps, 1, 1, 0.0, 0)
    assert rc != 0 and b"MFCC" in _lib.lib.pk_last_error()
