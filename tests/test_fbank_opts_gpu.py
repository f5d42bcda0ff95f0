"""The GPU front end at every fbank configuration of the torchaudio fixture (tests/golden/fbank_opts.npz): sample rates 8 to 48 kHz,
FFT sizes 256 to 2048, every window type, snip_edges=false and remove_dc_offset=false; the reflected edges of a signal shorter than
one frame; ``stride`` through splice + CMN + CMVN + SpecAugment against the numpy oracle; the noise / RIR entry point without banks;
and the trainer at 8 kHz with ``--stride 3``."""
import json
import os
import types

import numpy as np
import pytest
import torch

import fbank_opts_oracle as fo

pytestmark = pytest.mark.gpu


def i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def f32(v):
    return torch.tensor(v, dtype=torch.float32, device="cuda")


def oracle_fbank(wave, o):
    return fo.kaldi_fbank(wave, num_mel_bins=o.num_mel_bins, sample_frequency=o.sample_frequency, frame_length=o.frame_length,
                          frame_shift=o.frame_shift, window_type=o.window_type, snip_edges=o.snip_edges,
                          remove_dc_offset=o.remove_dc_offset, preemphasis_coefficient=o.preemphasis_coefficient, low_freq=o.low_freq,
                          high_freq=o.high_freq, blackman_coeff=o.blackman_coeff)


def run(fe, pcms, rates, dbs, **kw):
    """one padded batch through Frontend.__call__ -> (features [B, t_max, D], augmented int16 waves, new_len, fbank frames)"""
    from pika_b200.frontend import Frontend
    B = len(pcms)
    n = [len(p) for p in pcms]
    new_len, frames = Frontend.lengths(n, rates, **fe.opts.geometry())
    n_max = max(max(n), max(new_len))
    pcm = torch.zeros(B, n_max, dtype=torch.int16)
    for i, p in enumerate(pcms):
        pcm[i, :len(p)] = torch.from_numpy(p)
    t_max = max(fe.out_lens(frames))
    out, wave = fe(pcm.cuda(), i32(n), f32(rates), f32(dbs), i32(new_len), i32(frames), t_max, want_wave=True, **kw)
    torch.cuda.synchronize()
    return out.float().cpu().numpy(), wave.cpu().numpy(), new_len, frames


def test_fbank_matches_torchaudio_fixture(golden_dir):
    from pika_b200.frontend import FbankOptions, Frontend
    d = np.load(os.path.join(golden_dir, "fbank_opts.npz"))
    cfgs = json.loads(str(d["configs"]))
    for c, cfg in enumerate(cfgs):
        fe = Frontend(FbankOptions(**dict(cfg, dither=0.0)), 1, 1, "cuda")
        pcms = [d["pcm_%d_%d" % (c, k)] for k in range(3)]
        refs = [d["fbank_%d_%d" % (c, k)] for k in range(3)]
        n = [len(p) for p in pcms]
        wave = torch.zeros(3, max(n), dtype=torch.float32)
        for k, p in enumerate(pcms):
            wave[k, :n[k]] = torch.from_numpy(p.astype(np.float32))
        frames = [r.shape[0] for r in refs]
        assert Frontend.lengths(n, [1.0] * 3, **fe.opts.geometry())[1] == frames, c
        got = fe.fbank(wave.cuda(), i32(frames), max(frames), dither=0.0, n_samples=i32(n)).cpu().numpy()
        for k in range(3):
            g = got[k, :frames[k]]
            np.testing.assert_allclose(g, refs[k], atol=5e-3, err_msg="config %d signal %d" % (c, k))
            assert np.abs(g - refs[k]).mean() < 2e-4, (c, k, np.abs(g - refs[k]).mean())


@pytest.mark.parametrize("cfg", [dict(sample_frequency=8000.0, num_mel_bins=40, window_type="hamming", snip_edges=False),
                                 dict(sample_frequency=48000.0, num_mel_bins=80, window_type="povey", snip_edges=False, low_freq=40.0,
                                      high_freq=-200.0)])
def test_full_path_with_reflected_edges_and_a_signal_shorter_than_one_frame(cfg):
    """augmentation + fbank + splice at snip_edges=false, against the oracle on the augmented samples; the batch holds a signal shorter
    than one frame (120 samples at 8 kHz, 700 at 48 kHz), whose windows reflect about both edges more than once"""
    from pika_b200.frontend import FbankOptions, Frontend
    o = FbankOptions(**dict(cfg, dither=0.0))
    fe = Frontend(o, 1, 1, "cuda")
    rng = np.random.default_rng(5)
    short = 120 if o.sample_frequency == 8000.0 else 700
    assert short < o.frame_len
    pcms = [np.clip(np.round(rng.normal(0, 2500, n)), -32768, 32767).astype(np.int16) for n in (short, 3 * o.frame_len + 17, 9000)]
    rates, dbs = [1.0, 0.9, 1.1], [-20.0, -30.0, -25.0]
    out, wave, new_len, frames = run(fe, pcms, rates, dbs, cmn=False)
    assert frames[0] == (short + o.frame_shift_samples // 2) // o.frame_shift_samples > 0
    from oracle import frontend as ofe
    for i in range(3):
        ref = ofe.splice(oracle_fbank(wave[i, :new_len[i]].astype(np.float32), o), 1, 1)
        got = out[i, :frames[i]]
        np.testing.assert_allclose(got, ref, atol=5e-3, err_msg=str(i))
        assert np.abs(got - ref).mean() < 2e-4


@pytest.mark.parametrize("stride", [2, 3])
@pytest.mark.parametrize("ctx", [1, 3])
def test_stride_through_cmn_cmvn_specaug_vs_oracle(stride, ctx):
    """splice(feats)[::stride] with last-row padding, CMN over the padded rows, CMVN and SpecAugment: the GPU's own unstrided fbank
    frames through oracle/frontend.py's assemble_batch + apply_cmvn + spec_augment"""
    from oracle import frontend as ofe
    from pika_b200.frontend import FbankOptions, Frontend
    o = FbankOptions(sample_frequency=8000.0, num_mel_bins=40, dither=0.0)
    fe0 = Frontend(o, 0, 0, "cuda")
    fe = Frontend(o, ctx, ctx, "cuda", stride=stride)
    rng = np.random.default_rng(stride * 10 + ctx)
    pcms = [np.clip(np.round(rng.normal(0, 2500, n)), -32768, 32767).astype(np.int16) for n in (2000, 4173, 3371, 8000)]
    rates, dbs = [1.0, 0.9, 1.1, 1.0], [-20.0, -30.0, -25.0, -35.0]
    fb, wave, new_len, frames = run(fe0, pcms, rates, dbs, cmn=False)
    for i in range(len(pcms)):
        np.testing.assert_allclose(fb[i, :frames[i]], oracle_fbank(wave[i, :new_len[i]].astype(np.float32), o), atol=5e-3)
    feats = [fb[i, :frames[i]] for i in range(len(pcms))]
    data, _, lens, _ = ofe.assemble_batch(feats, [[1]] * len(pcms), ctx, ctx, stride=stride)
    assert lens.tolist() == fe.out_lens(frames)
    D = 40 * (2 * ctx + 1)
    stats = np.zeros((2, 41))
    mean, var, n = rng.standard_normal(40) * 3 + 8, np.abs(rng.standard_normal(40)) + 1.0, 1000.0
    stats[0, :40], stats[0, 40], stats[1, :40] = mean * n, n, (var + mean * mean) * n
    off, sc = ofe.cmvn_from_stats(stats, 2 * ctx + 1)
    sa = (D // 3, 7, 2, 3)
    out, _, _, _ = run(fe, pcms, rates, dbs, cmn=True, offset=f32(off), scale=f32(sc), specaug=sa)
    assert out.shape == data.shape
    ref = ofe.spec_augment(ofe.apply_cmvn(data, off, sc, cmn=True), *sa)
    np.testing.assert_allclose(out, ref, atol=2e-4)


def test_noise_rir_entry_without_banks_is_the_plain_entry_at_8khz():
    from pika_b200 import kernels as K
    from pika_b200._lib import check, lib
    from pika_b200.frontend import FbankOptions, Frontend
    o = FbankOptions(sample_frequency=8000.0, num_mel_bins=40, window_type="hamming", snip_edges=False, dither=0.0)
    fe = Frontend(o, 1, 1, "cuda", stride=2)
    rng = np.random.default_rng(8)
    pcms = [np.clip(np.round(rng.normal(0, 2500, n)), -32768, 32767).astype(np.int16) for n in (5000, 7777, 150)]
    rates, dbs = [1.0, 0.9, 1.1], [-20.0, -30.0, -25.0]
    plain, wave, new_len, frames = run(fe, pcms, rates, dbs, cmn=True)
    B, n_max = len(pcms), max(max(len(p) for p in pcms), max(new_len))
    pcm = torch.zeros(B, n_max, dtype=torch.int16)
    for i, p in enumerate(pcms):
        pcm[i, :len(p)] = torch.from_numpy(p)
    pcm = pcm.cuda()
    t_max = max(fe.out_lens(frames))
    need = int(lib.pk_frontend_noise_rir_workspace_bytes(B, n_max, t_max * fe.stride, fe.n_mel, fe.D, 1))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    out = torch.empty(B, t_max, fe.D, dtype=torch.float32, device="cuda")
    w2 = torch.zeros(B, n_max, dtype=torch.int16, device="cuda")
    P = K._P
    ns, nl, nf, rt, db = i32([len(p) for p in pcms]), i32(new_len), i32(frames), f32(rates), f32(dbs)
    check(lib.pk_frontend_fwd_noise_rir(P(pcm), pcm.stride(0), P(ns), P(rt), P(nl), P(db), P(nf), B, n_max, t_max, fe.n_mel, 1, 1,
                                        fe.stride, P(fe.window), P(fe.twiddle), P(fe.mel_w), P(fe.mel_lo), P(fe.mel_hi),
                                        *fe._geometry_args(), 1, None, None, 0, 0, 0, 0, P(out), K._dt(out), P(w2), P(ws), need,
                                        P(fe.err), 0.0, 1, K._stream(), None, None, None, None, None, None, None, None, None, 1),
          "pk_frontend_fwd_noise_rir")
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), plain) and np.array_equal(w2.cpu().numpy(), wave)


def test_train_cli_8khz_rnn_encoder_stride_3(tmp_path):
    """the RNN-T trainer on 8 kHz .seq data with a --sample-frequency=8000 feature config, the LSTM encoder and --stride 3"""
    from test_loader_cpu import make_dataset
    from pika_b200.model.transducer import Net
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    lst, _ = make_dataset(tmp_path, n_utts=6, shards=1, n_lo=7000, n_hi=12000)
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--sample-frequency=8000\n--num-mel-bins=40\n--dither=1\n")
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
            "--model_stride", "1", "--lctx", "1", "--rctx", "1", "--stride", "3", "--sample_rate", "8000", "--feats_dim", "40",
            "--feat_config", str(cfg), "--batch_size", "3", "--num_workers", "1", "--batch_first", "--max_len", "1600", "--TU_limit", "50000",
            "--gain_range", "25,25", "--speed_rate", "0.9,1.0,1.1", "--grad_clip", "3.0", "--initial_lr", "0.002", "--final_lr", "0.001",
            "--momentum", "0.9", "--num_epochs", "1", "--num_batches_per_epoch", "2", "--sync_period", "1", "--block_momentum", "0.9",
            "--block_lr", "1.0", "--seed", "777"]
    os.environ.setdefault("WORLD_SIZE", "1")
    T.main(argv)
    text = open(str(log).replace("WORKER-ID", "0")).read()
    losses = [float(l.split("Loss:")[1].split()[0]) for l in text.splitlines() if "Overall Avg Loss" in l]
    assert "Training Finished" in text and losses and np.isfinite(losses).all() and losses[0] > 0
    m = torch.load(str(out / "model.epoch.0.0"), weights_only=False)
    assert m.input_dim == 120
    moved = [not torch.equal(p.detach().cpu(), q.detach()) for p, q in zip(m.parameters(), m0.parameters())]
    assert all(bool(torch.isfinite(p).all()) for p in m.parameters()) and sum(moved) >= len(moved) // 2
