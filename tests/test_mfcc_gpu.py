"""The GPU front end's Kaldi MFCC: ``Frontend.mfcc`` over the torchaudio fixture's grid (tests/golden/mfcc.npz) on ragged batches; the
whole chain with MFCC (speed / gain, splice, stride, CMN, CMVN, SpecAugment) against the oracle composition; the noise / RIR path
against its own stages; the loader's ``--feat_type mfcc``; and a short trainer run on an MFCC config."""
import argparse
import os
import types

import numpy as np
import pytest
import torch

import mfcc_oracle as mo
from test_fbank_opts_gpu import f32, i32, run
from test_mfcc_cpu import coefficient_scale, fixture

pytestmark = pytest.mark.gpu

# The fbank features are held to 5e-3 per log mel energy (max) and 2e-4 (mean) against torchaudio (tests/test_fbank_opts_gpu.py).
# A cepstral coefficient is c_k = lifter_k * sum_j dct[k, j] * logmel_j, so those bounds carry to |lifter_k| * sum_j |dct[k, j]| times
# themselves (coefficient_scale); the energy column is a log like a mel energy and keeps them as they are.
ATOL, MEAN = 5e-3, 2e-4


def options(kw):
    from pika_b200.frontend import MfccOptions
    return MfccOptions(**dict(kw, dither=0.0))


def kaldi_kw(o):
    return {k: getattr(o, k) for k in ("num_ceps", "num_mel_bins", "use_energy", "energy_floor", "raw_energy", "cepstral_lifter",
                                       "htk_compat", "sample_frequency", "frame_length", "frame_shift", "window_type", "snip_edges",
                                       "remove_dc_offset", "preemphasis_coefficient", "low_freq", "high_freq", "blackman_coeff")}


def check_mfcc(got, ref, kw, what):
    s = coefficient_scale(kw)
    err = np.abs(got - ref) / s
    assert err.max() < ATOL, (what, err.max(), np.unravel_index(err.argmax(), err.shape))
    assert err.mean() < MEAN, (what, err.mean())


def test_mfcc_matches_torchaudio_fixture(golden_dir):
    from pika_b200.frontend import Frontend
    d, cfgs = fixture(golden_dir)
    for c, kw in enumerate(cfgs):
        fe = Frontend(options(kw), 1, 1, "cuda")
        assert fe.n_feat == kw["num_ceps"] and fe.n_mel == kw["num_mel_bins"] and fe.D == 3 * kw["num_ceps"]
        order = [2, 0, 1]                                                   # longest first: the others are ragged inside the batch
        pcms = [d["pcm_%d_%d" % (c, k)] for k in order]
        refs = [d["mfcc_%d_%d" % (c, k)] for k in order]
        n = [len(p) for p in pcms]
        wave = torch.zeros(3, max(n) + 37, dtype=torch.float32)              # padded past the longest signal
        for k, p in enumerate(pcms):
            wave[k, :n[k]] = torch.from_numpy(p.astype(np.float32))
        frames = [r.shape[0] for r in refs]
        assert Frontend.lengths(n, [1.0] * 3, **fe.opts.geometry())[1] == frames, c
        got = fe.mfcc(wave.cuda(), i32(frames), max(frames), dither=0.0, n_samples=i32(n)).cpu().numpy()
        assert got.shape == (3, max(frames), kw["num_ceps"])
        for k in range(3):
            check_mfcc(got[k, :frames[k]], refs[k], kw, "config %d signal %d" % (c, order[k]))


CHAIN = [(dict(), 2, 1),                                                                          # Kaldi's defaults, 13 / 23
         (dict(sample_frequency=8000.0, num_ceps=40, num_mel_bins=40, use_energy=False, htk_compat=True, snip_edges=False), 1, 3),
         (dict(sample_frequency=48000.0, num_ceps=20, num_mel_bins=80, raw_energy=False, energy_floor=1.0, window_type="hamming"), 3, 2)]


@pytest.mark.parametrize("kw,ctx,stride", CHAIN)
def test_full_chain_with_mfcc_vs_oracle(kw, ctx, stride):
    """speed / gain augmentation -> MFCC -> splice +-ctx -> [::stride] -> CMN over the padded rows -> CMVN -> SpecAugment: the GPU's
    MFCC frames against the numpy oracle on the augmented samples, then through oracle/frontend.py's assemble_batch, apply_cmvn and
    spec_augment"""
    from oracle import frontend as ofe
    from pika_b200.frontend import Frontend
    o = options(kw)
    nc, sr = o.num_ceps, int(o.sample_frequency)
    fe0 = Frontend(o, 0, 0, "cuda")
    fe = Frontend(o, ctx, ctx, "cuda", stride=stride)
    rng = np.random.default_rng(ctx * 10 + stride)
    pcms = [np.clip(np.round(rng.normal(0, 2500, n)), -32768, 32767).astype(np.int16) for n in (sr // 4, sr // 2 + 173, sr // 3, sr)]
    pcms[1][sr // 10:sr // 5] = 0                                              # whole frames of zeros
    rates, dbs = [1.0, 0.9, 1.1, 1.0], [-20.0, -30.0, -25.0, -35.0]
    raw, wave, new_len, frames = run(fe0, pcms, rates, dbs, cmn=False)
    for i in range(len(pcms)):
        check_mfcc(raw[i, :frames[i]], mo.kaldi_mfcc(wave[i, :new_len[i]].astype(np.float32), **kaldi_kw(o)), kaldi_kw(o), i)
    feats = [raw[i, :frames[i]] for i in range(len(pcms))]
    data, _, lens, _ = ofe.assemble_batch(feats, [[1]] * len(pcms), ctx, ctx, stride=stride)
    assert lens.tolist() == fe.out_lens(frames)
    D = nc * (2 * ctx + 1)
    assert fe.D == D
    stats = np.zeros((2, nc + 1))
    mean, var, n = rng.standard_normal(nc) * 3, np.abs(rng.standard_normal(nc)) * 20 + 1.0, 1000.0
    stats[0, :nc], stats[0, nc], stats[1, :nc] = mean * n, n, (var + mean * mean) * n
    off, sc = ofe.cmvn_from_stats(stats, 2 * ctx + 1)
    sa = (D // 3, 5, 2, 3)
    out, _, _, _ = run(fe, pcms, rates, dbs, cmn=True, offset=f32(off), scale=f32(sc), specaug=sa)
    assert out.shape == data.shape
    ref = ofe.spec_augment(ofe.apply_cmvn(data, off, sc, cmn=True), *sa)
    np.testing.assert_allclose(out, ref, rtol=1e-5, atol=2e-4)


def test_noise_rir_path_with_mfcc_is_its_stages():
    """noise + reverberation, then MFCC and splice: the features are the MFCC of the augmented samples the same call returns, spliced,
    bit for bit; without banks the MFCC entry point gives the plain path's output"""
    from oracle import frontend as ofe
    from pika_b200.frontend import Frontend
    from pika_b200.loader.audio_bank import AudioBank
    o = options(dict(num_ceps=20, num_mel_bins=40, htk_compat=True, energy_floor=1.0))
    fe = Frontend(o, 1, 1, "cuda", stride=2)
    rng = np.random.default_rng(11)
    pcms = [np.clip(np.round(rng.normal(0, 2500, n)), -32768, 32767).astype(np.int16) for n in (9000, 16000, 5003)]
    noise = AudioBank(["n0", "n1"], [np.clip(np.round(rng.normal(0, 4000, n)), -32768, 32767).astype(np.int16) for n in (40000, 30000)],
                      with_rms=True)
    h = [np.round(rng.normal(0, 3000, m) * np.exp(-np.arange(m) / (m / 4.0))).astype(np.int16) for m in (1, 700, 4000)]
    for x in h:
        x[0] = 20000                                                           # a direct path: no RIR is all zeros
    rir = AudioBank(["h1", "h700", "h4000"], h)
    rates, dbs = [1.0, 0.9, 1.1], [-20.0, -30.0, -25.0]
    kw = dict(noise=noise, noise_idx=[0, 1, 0], noise_off=[100, 0, 20000], snr=[5.0, 15.0, 10.0], rir=rir, rir_idx=[2, 1, 0])
    out, wave, new_len, frames = run(fe, pcms, rates, dbs, cmn=False, **kw)
    assert int(fe.err.item()) == 0
    B = len(pcms)
    w = torch.zeros(B, wave.shape[1], dtype=torch.float32)
    w[:] = torch.from_numpy(wave.astype(np.float32))
    t_fb = max(frames)
    cep = fe.mfcc(w.cuda(), i32(frames), t_fb, dither=0.0, n_samples=i32(new_len)).cpu().numpy()
    feats = [cep[i, :frames[i]] for i in range(B)]
    data, _, lens, _ = ofe.assemble_batch(feats, [[1]] * B, 1, 1, stride=2)
    assert out.shape == data.shape and np.array_equal(out, data)
    plain, pw, _, _ = run(fe, pcms, rates, dbs, cmn=False)
    assert not np.array_equal(pw, wave)
    w[:] = torch.from_numpy(pw.astype(np.float32))
    cep = fe.mfcc(w.cuda(), i32(frames), t_fb, dither=0.0, n_samples=i32(new_len)).cpu().numpy()
    data, _, _, _ = ofe.assemble_batch([cep[i, :frames[i]] for i in range(B)], [[1]] * B, 1, 1, stride=2)
    assert np.array_equal(plain, data)


def test_raw_to_features_with_feat_type_mfcc(tmp_path):
    from test_loader_cpu import make_dataset
    from pika_b200.loader import kaldi_io, otf_utt_loader as L
    lst, _ = make_dataset(tmp_path, n_utts=5, shards=1)
    cfg = tmp_path / "mfcc.conf"
    cfg.write_text("--num-ceps=13\n--dither=0\n")
    p = argparse.ArgumentParser()
    L.register(p)
    args = p.parse_args(["--feat_type", "mfcc", "--feat_config", str(cfg), "--feats_dim", "13", "--lctx", "2", "--rctx", "3",
                         "--stride", "2", "--batch_size", "5", "--num_workers", "1", "--padding_tgt", "99"])
    assert L.get_inputdim(args) == 13 * 6
    raw, target, lens, _ = next(L.otf_utt_generator(kaldi_io.read_lst(lst), [], [], args))
    x = L.raw_to_features(raw, args)
    assert x.shape == (len(lens), raw["t_max"], 13 * 6) and torch.isfinite(x).all()
    fe = L._frontend_for(args, "cuda")
    assert fe.is_mfcc and fe.n_feat == 13 and fe.D == 78


def test_train_cli_on_an_mfcc_config(tmp_path):
    """the RNN-T trainer with --feat_type mfcc and mfcc_hires.conf's 40 cepstra: the same batch each epoch (no speed perturbation, a
    fixed gain, no dither), so the epoch loss must fall.  40 x 3 = 120 inputs: the LSTM encoder's GEMMs need a spliced width that is a
    multiple of 8 (13 x 3 = 39 is refused there, as 23 x 3 fbank bins are)"""
    from test_loader_cpu import make_dataset
    from pika_b200.model.transducer import Net
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    lst, _ = make_dataset(tmp_path, n_utts=4, shards=1, n_lo=9000, n_hi=14000)
    cfg = tmp_path / "mfcc.conf"
    cfg.write_text("--use-energy=false\n--num-mel-bins=40\n--num-ceps=40\n--low-freq=20\n--high-freq=-400\n--dither=0\n")
    out = tmp_path / "out"
    out.mkdir()
    margs = types.SimpleNamespace(rnn_size=256, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="rnn", embd_dim=64,
                                  padding_idx=60, dropout=0.0, dec_layers=1, enc_layers=2)
    torch.manual_seed(777)
    m0 = Net(margs, 120, 60)
    init = tmp_path / "init.model"
    torch.save(m0, str(init))
    log = tmp_path / "log.WORKER-ID"
    argv = ["transducer", lst, str(log), str(out), "--cuda", "--local_rank", "0", "--init_model", str(init), "--encoder_type", "rnn",
            "--brnn", "--enc_layers", "2", "--decoder_type", "rnn", "--rnn_size", "256", "--embd_dim", "64", "--output_dim", "60",
            "--padding_idx", "60", "--padding_tgt", "60", "--dec_layers", "1", "--dropout", "0.0", "--model_lctx", "0", "--model_rctx", "0",
            "--model_stride", "1", "--lctx", "1", "--rctx", "1", "--stride", "2", "--feat_type", "mfcc", "--feats_dim", "40",
            "--feat_config", str(cfg), "--batch_size", "4", "--num_workers", "1", "--batch_first", "--max_len", "1600",
            "--TU_limit", "50000", "--gain_range", "25,25", "--speed_rate", "1.0", "--grad_clip", "3.0", "--initial_lr", "0.002",
            "--final_lr", "0.002", "--momentum", "0.9", "--num_epochs", "4", "--num_batches_per_epoch", "1", "--sync_period", "1",
            "--block_momentum", "0.9", "--block_lr", "1.0", "--seed", "777"]
    os.environ.setdefault("WORLD_SIZE", "1")
    T.main(argv)
    text = open(str(log).replace("WORKER-ID", "0")).read()
    losses = [float(l.split("Loss:")[1].split()[0]) for l in text.splitlines() if "Overall Avg Loss" in l]
    assert "Training Finished" in text and len(losses) == 4 and np.isfinite(losses).all() and losses[0] > 0, losses
    assert all(b < a for a, b in zip(losses, losses[1:])), losses
    m = torch.load(str(out / "model.epoch.3.0"), weights_only=False)
    assert m.input_dim == 120
