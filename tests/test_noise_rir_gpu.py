"""On-the-fly noise and reverberation on the GPU: the float64 same-mode convolution against scipy, the front end against the
reference fixture (tests/golden/frontend_noise_rir.npz), determinism, the unchanged path without banks, and one training run
with --noise_lst / --rir_lst / --snr_range."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows", [
    [(5000, 1), (3000, 777), (10000, 1024), (2500, 1025), (1000, 4000)],          # Lb 1024: M = 1, Lb, Lb + 1, M > N
    [(50000, 16000), (4097, 4096), (9000, 4097), (7000, 12000)],                   # Lb 4096
    [(70001, 65536), (30000, 65536), (100000, 33333)],                             # the longest RIR, M > N
])
def test_conv_same_f64_matches_scipy(rows):
    from scipy import signal
    from pika_b200 import kernels as K
    rng = np.random.default_rng(len(rows))
    B, n, m = len(rows), max(r[0] for r in rows), max(r[1] for r in rows)
    x = np.zeros((B, n)); h = np.zeros((B, m))
    for b, (N, M) in enumerate(rows):
        x[b, :N] = rng.standard_normal(N)
        h[b, :M] = rng.standard_normal(M) * np.exp(-np.arange(M) / max(M / 5.0, 1.0))
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
    y = K.conv_same_f64(torch.from_numpy(x).cuda(), i32([r[0] for r in rows]), torch.from_numpy(h).cuda(), i32([r[1] for r in rows]))
    y = y.cpu().numpy()
    for b, (N, M) in enumerate(rows):
        ref = signal.fftconvolve(x[b, :N], h[b, :M], "same")
        err = np.abs(y[b, :N] - ref).max() / np.abs(ref).max()
        assert err < 1e-11, (N, M, err)


def make_frontend():
    from pika_b200.frontend import FbankOptions, Frontend
    return Frontend(FbankOptions(num_mel_bins=80, low_freq=40.0, high_freq=-200.0, dither=0.0, window_type="hamming"), 1, 1, "cuda")


def run_cases(fe, d, cases, noise_bank, rir_bank, rir_names):
    """one batch of fixture cases sharing a mode (noise, RIR or both)"""
    from pika_b200.frontend import Frontend
    B = len(cases)
    pcm = d["pcm"]
    rates = [float(d["meta_" + k][0]) for k in cases]
    dbs = [float(d["meta_" + k][1]) for k in cases]
    new_len, frames = Frontend.lengths([len(pcm)] * B, rates)
    n_max = max(len(pcm), max(new_len))
    x = torch.zeros(B, n_max, dtype=torch.int16)
    x[:, :len(pcm)] = torch.from_numpy(pcm)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device="cuda")
    kw = {}
    if noise_bank is not None:
        kw.update(noise=noise_bank, noise_idx=[0] * B, noise_off=[int(d["meta_" + k][3]) for k in cases],
                  snr=[float(d["meta_" + k][2]) for k in cases])
    if rir_bank is not None:
        kw.update(rir=rir_bank, rir_idx=[rir_names.index(str(d["rirname_" + k])) for k in cases])
    out, wave = fe(x.cuda(), i32([len(pcm)] * B), f32(rates), f32(dbs), i32(new_len), i32(frames), max(frames), cmn=False,
                   want_wave=True, **kw)
    torch.cuda.synchronize()
    return out.cpu().numpy(), wave.cpu().numpy(), rates, new_len, frames


def banks(d):
    from pika_b200.loader.audio_bank import AudioBank
    names = ["h1", "h777", "h16000", "hlong"]
    return AudioBank(["noise"], [d["noise"]], with_rms=True), AudioBank(names, [d["rir_" + n] for n in names]), names


def test_frontend_noise_rir_vs_reference_golden(golden_dir):
    d = np.load(os.path.join(golden_dir, "frontend_noise_rir.npz"))
    fe = make_frontend()
    noise, rir, names = banks(d)
    keys = [str(k) for k in d["cases"]]
    groups = [([k for k in keys if k.endswith("_n")], noise, None),
              ([k for k in keys if "_h" in k], None, rir),
              ([k for k in keys if "_nh" in k], noise, rir)]
    assert sum(len(g[0]) for g in groups) == len(keys)
    for cases, nb, rb in groups:
        out, wave, rates, new_len, frames = run_cases(fe, d, cases, nb, rb, names)
        for i, k in enumerate(cases):
            aug = d["aug_" + k]
            assert new_len[i] == len(aug) and frames[i] == d["fbank_" + k].shape[0]
            diff = np.abs(wave[i, :len(aug)].astype(np.int32) - aug.astype(np.int32))
            assert diff.max() <= 1, k
            # the rate == 1.0 branch: the reference's samples and its fftconvolve are float32; float64 elsewhere
            assert (diff != 0).mean() < (0.05 if rates[i] == 1.0 else 1e-3), (k, (diff != 0).mean())
            # features: the front-end tolerance on every spliced block whose source frame has the reference's samples exactly.  A
            # 1-LSB flip inside a frame is not held to it: a long RIR leaves spectral nulls where a mel bin's energy is ~1 (int16
            # units), and there the flip moves the log energy by up to ~0.2
            nf, got, ref = frames[i], out[i, :frames[i]][::5], d["splice_" + k]
            same = np.array([np.array_equal(wave[i, t * 160:t * 160 + 400], aug[t * 160:t * 160 + 400]) for t in range(nf)])
            rows = np.arange(0, nf, 5)
            for blk, dt in enumerate((-1, 0, 1)):
                m = same[np.clip(rows + dt, 0, nf - 1)]
                if rates[i] != 1.0:
                    assert m.mean() > 0.5, k
                np.testing.assert_allclose(got[m, blk * 80:(blk + 1) * 80], ref[m, blk * 80:(blk + 1) * 80], atol=5e-3, err_msg=k)
            assert np.abs(got - ref).mean() < 2e-3, (k, np.abs(got - ref).mean())
    assert int(fe.err.item()) == 0


def test_deterministic_and_unchanged_without_banks(golden_dir):
    from pika_b200._lib import launch_count
    d = np.load(os.path.join(golden_dir, "frontend_noise_rir.npz"))
    fe = make_frontend()
    noise, rir, names = banks(d)
    cases = ["r09_nh16000", "r10_nh777", "r11_nhlong", "r09_nh1"]
    o1, w1, *_ = run_cases(fe, d, cases, noise, rir, names)
    o2, w2, *_ = run_cases(fe, d, cases, noise, rir, names)
    assert np.array_equal(o1, o2) and np.array_equal(w1, w2)
    # without banks: pk_frontend_fwd's launches (resample, gain + quantise, fbank, splice) and its output, bit for bit
    c0 = launch_count()
    p1, v1, *_ = run_cases(fe, d, cases, None, None, names)
    assert launch_count() - c0 == 4
    from pika_b200.frontend import Frontend
    plain = Frontend(fe.opts, 1, 1, "cuda")
    p2, v2, *_ = run_cases(plain, d, cases, None, None, names)
    assert np.array_equal(p1, p2) and np.array_equal(v1, v2)
    assert not np.array_equal(v1, w1)


def test_train_cli_with_noise_and_rir(tmp_path):
    from test_loader_cpu import make_dataset
    from test_noise_rir_cpu import write_bank
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    lst, _ = make_dataset(tmp_path, n_utts=8, shards=1, n_lo=14000, n_hi=22000)
    nlst, _ = write_bank(tmp_path, "noise", [40000, 33000, 1000], 11)           # the 1000-sample segment is dropped
    rlst, _ = write_bank(tmp_path, "rir", [800, 8000], 12)
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--window-type=hamming\n--sample-frequency=16000\n--dither=1\n--low-freq=40\n--high-freq=-200\n--num-mel-bins=80\n")
    out = tmp_path / "out"
    out.mkdir()
    log = tmp_path / "log.WORKER-ID"
    argv = ["transducer", lst, str(log), str(out), "--cuda", "--local_rank", "0", "--encoder_type", "transformer",
            "--rnn_size", "1024", "--embd_dim", "100", "--output_dim", "60", "--padding_idx", "60", "--padding_tgt", "60",
            "--dec_layers", "2", "--dropout", "0.0", "--brnn", "--model_lctx", "21", "--model_rctx", "21", "--model_stride", "4",
            "--lctx", "1", "--rctx", "1", "--feats_dim", "80", "--feat_config", str(cfg), "--batch_size", "4",
            "--num_workers", "1", "--batch_first", "--max_len", "200", "--TU_limit", "50000", "--gain_range", "25,25",
            "--grad_clip", "3.0", "--initial_lr", "0.002", "--final_lr", "0.001", "--momentum", "0.9", "--num_epochs", "2",
            "--num_batches_per_epoch", "2", "--sync_period", "1", "--seed", "777",
            "--noise_lst", nlst, "--rir_lst", rlst, "--snr_range", "0,15"]
    os.environ.setdefault("WORLD_SIZE", "1")
    T.main(argv)
    text = open(str(log).replace("WORKER-ID", "0")).read()
    assert "Training Finished" in text
    losses = [float(l.split("Loss:")[1].split()[0]) for l in text.splitlines() if "Overall Avg Loss" in l]
    assert len(losses) == 2 and np.isfinite(losses).all()
