"""The front-end kernels (pika_b200/csrc/frontend.cu) through their C entry points, on every FFT size, convolution block length and
splice shape, and at their limits, against the numpy restatements of tests/frontend_kernels_oracle.py, oracle/frontend.py and
tests/noise_rir_oracle.py.

Every output the caller allocates goes into the head of a larger buffer whose tail holds sentinel values that a correct kernel never
writes; rows and samples past each utterance's length must keep their initial values too.  Dither stays at 0 (bit-reproducible)."""
import math

import numpy as np
import pytest
import torch

import frontend_kernels_oracle as fko
import noise_rir_oracle as nro
from oracle import frontend as ofe

pytestmark = pytest.mark.gpu

GUARD = 257
SENT = 77.0                 # exact in bf16
SENT_I16 = -7777
SENT_U8 = 0xA5
LOG_ATOL, LOG_MEAN = 5e-3, 2e-4        # the front end's log-mel bar (tests/test_frontend_gpu.py)
LIN_REL = 1e-5                          # mel energies below 1e-3 of the frame's largest: error relative to its total energy


def _lib():
    from pika_b200 import _lib
    return _lib


def _dev(a, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dt is None else t.to(dt)).cuda()


def _i32(v):
    return torch.tensor(list(v), dtype=torch.int32, device="cuda")


def _P(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(n, dtype, fill):
    return torch.full((n + GUARD,), fill, dtype=dtype, device="cuda")


def _tail_ok(buf, n, fill, what):
    assert bool((buf[n:] == fill).all()), "%s: write past the end" % what


# ------------------------------------------------------------------------------------------------------------ tables
def _twiddle(n_fft):
    k = np.arange(n_fft // 2, dtype=np.float64)
    return np.stack([np.cos(2 * np.pi * k / n_fft), -np.sin(2 * np.pi * k / n_fft)], 1).astype(np.float32)


def random_tables(n_fft, frame_len, n_mel, rng, min_width=1):
    """window, mel weights and [lo, hi) ranges that no Kaldi option produces: filters over the whole spectrum (lo = 0, hi = N/2),
    from bin 0, up to N/2, single-bin (min_width = 1) and random overlapping ones; non-zero weights outside [lo, hi) that the kernel
    must not read"""
    nb = n_fft // 2
    win = rng.uniform(0.2, 1.0, frame_len).astype(np.float32)
    win[0] = 1.0                                           # sample 0 counts fully (its pre-emphasis uses itself)
    lo, hi = np.zeros(n_mel, np.int32), np.zeros(n_mel, np.int32)
    for j in range(n_mel):
        kind = j % 5
        if kind == 0:
            lo[j], hi[j] = 0, nb
        elif kind == 1:
            lo[j], hi[j] = 0, rng.integers(max(min_width, 4), nb // 2 + 1)
        elif kind == 2:
            lo[j], hi[j] = rng.integers(nb // 2, nb - max(min_width, 2) + 1), nb
        elif kind == 3:
            lo[j] = rng.integers(2, nb - min_width)
            hi[j] = lo[j] + min_width
        else:
            lo[j] = rng.integers(1, nb - max(min_width, 2))
            hi[j] = min(nb, lo[j] + rng.integers(max(min_width, 2), 41))
    w = rng.uniform(0.05, 1.0, (n_mel, nb)).astype(np.float32)
    return win, _twiddle(n_fft), w, lo, hi


def kaldi_tables(num_mel_bins=80):
    from pika_b200.frontend import FbankOptions, fbank_tables
    o = FbankOptions(num_mel_bins=num_mel_bins, low_freq=40.0, high_freq=-200.0, dither=0.0, window_type="hamming")
    return fbank_tables(o), (o.frame_len, o.frame_shift_samples, o.log2_nfft, 1, 1, o.preemphasis_coefficient)


def dct_table(num_ceps, n_mel, lifter=22.0):
    from pika_b200.frontend import dct_matrix, lifter_coeffs
    d = dct_matrix(num_ceps, n_mel) * lifter_coeffs(num_ceps, lifter)[:, None]
    return np.ascontiguousarray(d.T).astype(np.float32)


def _signal(n, rng, amp=2000.0):
    t = np.arange(n)
    x = amp * np.sin(2 * np.pi * t * rng.uniform(0.01, 0.2)) + rng.normal(0, amp, n) + rng.uniform(-300, 300)
    return np.clip(np.round(x), -32768, 32767)


# ------------------------------------------------------------------------------------------------------------ fbank / MFCC
def _num_frames(n, frame_len, shift, snip):
    if snip:
        return 0 if n < frame_len else 1 + (n - frame_len) // shift
    return (n + shift // 2) // shift


def _fbank_batch(n_fft, frame_len, shift, snip, rng):
    """four signals: a long one, one without frames, one shorter than half a frame (snip_edges = 0) or exactly one frame, a
    medium one; rows padded with garbage past each signal (ld_wave wider than the longest)"""
    short = max(1, frame_len // 2 - 1) if not snip else frame_len
    n = [frame_len + 11 * shift + 3, 0, short, frame_len + 3 * shift + shift // 2]
    ld = max(n) + 37
    wave = rng.uniform(-1e4, 1e4, (len(n), ld)).astype(np.float32)
    amps = [2000.0, 1.0, 3.0, 500.0]
    for b, m in enumerate(n):
        wave[b, :m] = _signal(m, rng, amps[b])
    frames = [_num_frames(m, frame_len, shift, snip) for m in n]
    return wave, n, frames


def _run_fbank(wave, n, frames, tables, geom, mfcc=None):
    """pk_fbank (mfcc None) or pk_mfcc into sentinel-filled [B, t_max, n_out]; -> (feats numpy, t_max)"""
    win, tw, w, lo, hi = tables
    frame_len, shift, log2n, snip, dc, preemph = geom
    B, n_mel = wave.shape[0], w.shape[0]
    t_max = max(frames) + 5
    n_out = mfcc[1] if mfcc is not None else n_mel
    size = B * t_max * n_out
    feats = _guarded(size, torch.float32, SENT)
    T = [_dev(a) for a in (wave, win, tw, w, lo, hi)]
    lens = [_i32(n), _i32(frames)]                     # held until the kernel has run
    args = (T[0].data_ptr(), wave.shape[1], lens[0].data_ptr(), lens[1].data_ptr(), B, t_max, n_mel, *[t.data_ptr() for t in T[1:]],
            frame_len, shift, log2n, snip, dc, preemph, feats.data_ptr(), 0.0, 0, _stream())
    L = _lib()
    if mfcc is None:
        L.check(L.lib.pk_fbank(*args), "pk_fbank")
    else:
        dct = _dev(mfcc[0])
        L.check(L.lib.pk_mfcc(*args, dct.data_ptr(), *mfcc[1:]), "pk_mfcc")
    torch.cuda.synchronize()
    _tail_ok(feats, size, SENT, "feats")
    out = feats[:size].view(B, t_max, n_out).cpu().numpy()
    for b in range(B):
        assert (out[b, frames[b]:] == SENT).all(), "rows past n_frames[%d] = %d written" % (b, frames[b])
    return out, t_max


def check_fbank(got, ref_log, mel, power, what):
    """log domain where the mel energy is at least 1e-3 of the frame's largest; the rest in the linear domain, relative to the
    frame's total energy"""
    big = mel >= 1e-3 * mel.max(axis=1, keepdims=True)
    err = np.abs(got.astype(np.float64) - ref_log)
    assert big.any(axis=1).all()
    assert err[big].max() < LOG_ATOL, (what, err[big].max(), np.argwhere(err * big == (err * big).max())[0])
    assert err[big].mean() < LOG_MEAN, (what, err[big].mean())
    lin = np.abs(np.exp(got.astype(np.float64)) - np.maximum(mel, fko.EPS))
    tol = LIN_REL * power.sum(axis=1, keepdims=True) + 1e-6
    assert (lin <= tol)[~big].all(), (what, (lin / tol)[~big].max())


FRAME_LENS = {"half+1": lambda n: n // 2 + 1, "3/4": lambda n: 3 * n // 4, "full": lambda n: n}


@pytest.mark.parametrize("log2n", [7, 8, 9, 10, 11])
@pytest.mark.parametrize("fl", list(FRAME_LENS))
def test_fbank_every_fft_size_and_geometry(log2n, fl):
    n_fft = 1 << log2n
    frame_len = FRAME_LENS[fl](n_fft)
    rng = np.random.default_rng(100 * log2n + len(fl))
    case = 0
    for snip in (1, 0):
        for dc in (1, 0):
            for n_mel in (1, 23, 256):
                shift = frame_len // 3 + 1 if case % 2 == 0 else frame_len + 7         # frames overlap / leave gaps
                case += 1
                tables = random_tables(n_fft, frame_len, n_mel, rng)
                wave, n, frames = _fbank_batch(n_fft, frame_len, shift, snip, rng)
                assert frames[1] == 0 and max(frames) >= 10
                geom = (frame_len, shift, log2n, snip, dc, 0.97)
                got, _ = _run_fbank(wave, n, frames, tables, geom)
                win, _, w, lo, hi = tables
                for b in range(len(n)):
                    if frames[b] == 0:
                        continue
                    ref, mel, power = fko.fbank_from_tables(wave[b, :n[b]], frames[b], win, w, lo, hi, n_fft, shift, snip, dc,
                                                            0.97)
                    check_fbank(got[b, :frames[b]], ref, mel, power,
                                "N %d frame_len %d shift %d snip %d dc %d n_mel %d signal %d" % (n_fft, frame_len, shift, snip, dc,
                                                                                               n_mel, b))


ENERGY = [(ue, re, htk) for ue in (1, 0) for re in (1, 0) for htk in (0, 1)]


@pytest.mark.parametrize("log2n", [7, 8, 9, 10, 11])
def test_mfcc_every_fft_size_and_energy_option(log2n):
    n_fft = 1 << log2n
    rng = np.random.default_rng(700 + log2n)
    for i, (use_energy, raw_energy, htk) in enumerate(ENERGY):
        frame_len = [n_fft, 3 * n_fft // 4, n_fft // 2 + 1][i % 3]
        snip, dc = i % 2, (i // 2) % 2
        shift = frame_len // 3 + 1 if i % 4 < 2 else frame_len + 7
        for n_mel, num_ceps in ((23, 1), (23, 13), (256, 256), (40, 40)):
            tables = random_tables(n_fft, frame_len, n_mel, rng, min_width=8)
            win, _, w, lo, hi = tables
            dct = dct_table(num_ceps, n_mel)
            wave, n, frames = _fbank_batch(n_fft, frame_len, shift, snip, rng)
            floor = 0.0
            if (i + num_ceps) % 2 == 0:
                floor = 1e5                                        # without use_energy the floor must change nothing
                if use_energy:                                     # the median frame energy: binds on half of the frames
                    e = np.concatenate([fko.mfcc_from_tables(wave[b, :n[b]], frames[b], win, w, lo, hi, n_fft, shift, dct, 1,
                                                             raw_energy, 0.0, 0, snip, dc, 0.97)[0][:, 0]
                                        for b in range(len(n)) if frames[b] > 0])
                    floor = float(np.float32(np.exp(np.median(e))))
            geom = (frame_len, shift, log2n, snip, dc, 0.97)
            got, _ = _run_fbank(wave, n, frames, tables, geom, (dct, num_ceps, use_energy, raw_energy, floor, htk))
            floored = above = 0
            s = np.abs(dct).sum(0).astype(np.float64)             # the factor by which a log-mel bound bounds each coefficient
            if use_energy:
                s[0] = 1.0
            elif htk:
                s[0] *= math.sqrt(2.0)
            if htk:
                s = np.concatenate([s[1:], s[:1]])
            what = "N %d frame_len %d snip %d dc %d n_mel %d num_ceps %d energy %d raw %d htk %d floor %g" % (
                n_fft, frame_len, snip, dc, n_mel, num_ceps, use_energy, raw_energy, htk, floor)
            for b in range(len(n)):
                if frames[b] == 0:
                    continue
                ref, mel = fko.mfcc_from_tables(wave[b, :n[b]], frames[b], win, w, lo, hi, n_fft, shift, dct, use_energy, raw_energy,
                                                floor, htk, snip, dc, 0.97)
                err = np.abs(got[b, :frames[b]] - ref) / s[None, :]
                assert err.max() < LOG_ATOL, (what, b, err.max(), np.unravel_index(err.argmax(), err.shape))
                assert err.mean() < LOG_MEAN, (what, b, err.mean())
                if use_energy and floor > 0.0:
                    energy = ref[:, -1 if htk else 0]
                    floored += int((energy == math.log(np.float32(floor))).sum())
                    above += int((energy > math.log(np.float32(floor))).sum())
            if use_energy and floor > 0.0:
                assert floored > 0 and above > 0, (what, floored, above)          # the floor binds on some frames, not on all


# ------------------------------------------------------------------------------------------------------------ whole entry points
def _frontend(pcms, rates, dbs, tables, geom, lctx=1, rctx=1, stride=1, cmn=0, offset=None, scale=None, specaug=(0, 0, 0, 0),
              bf16=False, mfcc=None, noise=None, rir=None, t_max=None, entry=None):
    """one call of pk_frontend_fwd / pk_frontend_fwd_noise_rir / pk_frontend_fwd_mfcc with sentinel-guarded outputs and workspace.
    noise = (AudioBank, idx, off in segment, snr dB), rir = (AudioBank, idx).  -> (out numpy [B, t_max, D] (bf16 as uint16 bits),
    augmented int16 wave [B, n_max], new_len, n_frames)"""
    from pika_b200.frontend import Frontend
    L = _lib()
    win, tw, w, lo, hi = tables
    frame_len, shift, log2n, snip, dc, preemph = geom
    B, n_mel = len(pcms), w.shape[0]
    n = [len(p) for p in pcms]
    new_len, frames = Frontend.lengths(n, rates, frame_len, shift, bool(snip))
    n_max = max(max(n), max(new_len), frame_len)
    n_feat = mfcc[1] if mfcc is not None else n_mel
    D = n_feat * (lctx + 1 + rctx)
    if t_max is None:
        t_max = max(1, max((f + stride - 1) // stride for f in frames))
    pcm = np.zeros((B, n_max), np.int16)
    for b, p in enumerate(pcms):
        pcm[b, :len(p)] = p
    banks = noise is not None or rir is not None
    rir_max_len = 1
    if rir is not None:
        rir_max_len = int(rir[0].lengths[np.asarray(rir[1])].max())
    if banks:
        need = int(L.lib.pk_frontend_noise_rir_workspace_bytes(B, n_max, t_max * stride, n_feat, D, rir_max_len))
    else:
        need = int(L.lib.pk_frontend_workspace_bytes(B, n_max, t_max * stride, n_feat, D))
    ws = _guarded(need, torch.uint8, SENT_U8)
    dt = torch.bfloat16 if bf16 else torch.float32
    size = B * t_max * D
    out = _guarded(size, dt, SENT)
    wave = _guarded(B * n_max, torch.int16, SENT_I16)
    err = _guarded(1, torch.int32, 0)
    T = [_dev(a) for a in (pcm, win, tw, w, lo, hi)]
    off_t = None if offset is None else _dev(np.asarray(offset, np.float32))
    sc_t = None if scale is None else _dev(np.asarray(scale, np.float32))
    keep = [_i32(n), _dev(np.asarray(rates, np.float32)), _i32(new_len), _dev(np.asarray(dbs, np.float32)), _i32(frames)]
    args = (T[0].data_ptr(), n_max, *[t.data_ptr() for t in keep[:5]], B, n_max, t_max, n_mel, lctx, rctx, stride,
            *[t.data_ptr() for t in T[1:]], frame_len, shift, log2n, snip, dc, preemph, int(cmn), _P(off_t), _P(sc_t), *specaug,
            out.data_ptr(), L.PK_BF16 if bf16 else L.PK_F32, wave.data_ptr(), ws.data_ptr(), need, err.data_ptr(), 0.0, 0, _stream())
    nz, rr = (None,) * 5, (None,) * 4
    if noise is not None:
        bank, idx, off, snr = noise
        samples, offs, _, rms = bank.device("cuda")
        start = offs[torch.as_tensor(idx).cuda().long()] + torch.as_tensor(off, dtype=torch.int64).cuda()
        keep += [_i32(idx), start, torch.as_tensor(snr, dtype=torch.float64).cuda()]
        nz = (samples.data_ptr(), keep[-3].data_ptr(), start.data_ptr(), keep[-1].data_ptr(), rms.data_ptr())
    if rir is not None:
        samples, offs, lens, _ = rir[0].device("cuda")
        keep.append(_i32(rir[1]))
        rr = (samples.data_ptr(), offs.data_ptr(), lens.data_ptr(), keep[-1].data_ptr())
    if mfcc is not None:
        dct = _dev(mfcc[0])
        L.check(L.lib.pk_frontend_fwd_mfcc(*args, *nz, *rr, rir_max_len, dct.data_ptr(), *mfcc[1:]), "pk_frontend_fwd_mfcc")
    elif banks or entry == "noise_rir":
        L.check(L.lib.pk_frontend_fwd_noise_rir(*args, *nz, *rr, rir_max_len), "pk_frontend_fwd_noise_rir")
    else:
        L.check(L.lib.pk_frontend_fwd(*args), "pk_frontend_fwd")
    torch.cuda.synchronize()
    _tail_ok(out, size, SENT, "out")
    _tail_ok(wave, B * n_max, SENT_I16, "wave_i16_out")
    _tail_ok(ws, need, SENT_U8, "workspace")
    _tail_ok(err, 1, 0, "err_flag")
    assert int(err[0]) == 0, "err_flag set"
    wv = wave[:B * n_max].view(B, n_max).cpu().numpy()
    for b in range(B):
        assert (wv[b, new_len[b]:] == SENT_I16).all(), "wave_i16_out written past new_len[%d]" % b
    o = out[:size].view(B, t_max, D)
    o = o.view(torch.int16).cpu().numpy().view(np.uint16) if bf16 else o.cpu().numpy()
    return o, wv, new_len, frames


def check_wave(got, ref, rate, what):
    """<= 1 LSB; on at most 1e-3 of the samples after speed perturbation (float64, the mean square's summation order is the only
    freedom), at most 5 % on the rate == 1.0 branch (float32 like numpy, mean square in float64 here)"""
    assert got.shape == ref.shape, what
    diff = np.abs(got.astype(np.int32) - ref.astype(np.int32))
    if diff.size == 0:
        return
    assert diff.max() <= 1, (what, diff.max())
    assert (diff != 0).mean() <= (0.05 if rate == 1.0 else 1e-3), (what, (diff != 0).mean())


def _pcm(n, rng):
    return _signal(n, rng, 3000.0).astype(np.int16)


AUG_BATCHES = [
    # (n_samples, rate, target_db): the grid-stride wrap at 64 x 256 = 16384 samples, 480 000-sample utterances (30 passes),
    # L = int(n / rate) of 1 and 2 samples, and targets that clip at both rails
    [(1, 1.0, 6.0), (16383, 0.9, -20.0), (16384, 1.0, -25.0), (16385, 1.1, -18.0), (480000, 0.9, -23.0), (3, 2.9, 6.0),
     (5, 2.5, 6.0), (480000, 1.0, 4.0)],
    [(480000, 1.1, -30.0), (1, 0.9, 6.0), (16384, 1.1, 3.0), (16385, 0.9, -21.0), (16383, 1.0, -26.0), (2, 1.9, 6.0),
     (7, 3.4, 6.0), (300001, 1.0, -15.0)],
]


@pytest.mark.parametrize("batch", range(len(AUG_BATCHES)))
def test_augmentation_at_training_lengths(batch):
    rows = AUG_BATCHES[batch]
    rng = np.random.default_rng(40 + batch)
    pcms = [_pcm(n, rng) for n, _, _ in rows]
    for p in pcms:
        if 2 <= len(p) <= 7:
            p[0], p[-1] = 1200, -3000          # L = 1 takes the first sample (numpy.linspace(0, n, 1) = [0]), not the last
    rates, dbs = [r[1] for r in rows], [r[2] for r in rows]
    tables, geom = kaldi_tables()
    _, wave, new_len, _ = _frontend(pcms, rates, dbs, tables, geom)
    clipped = 0
    for b, (n, rate, db) in enumerate(rows):
        ref = ofe.augment(pcms[b], rate, db)
        assert len(ref) == new_len[b]
        check_wave(wave[b, :new_len[b]], ref, rate, "signal %d: n %d rate %g" % (b, n, rate))
        clipped += int((ref == 32767).any() and (ref == -32768).any())
    assert clipped >= 2


def _conv_geom(m_max):
    lb = 1024
    while lb < 4096 and 4 * lb < m_max:
        lb <<= 1
    return lb


def _conv_ws_bytes(B, n_max, m_max):
    a = lambda v: (v + 255) & ~255                                         # noqa: E731
    lb = _conv_geom(m_max)
    p_max, j_max = -(-m_max // lb), -(-n_max // lb)
    return a(lb * 16) + a(B * p_max * (lb + 1) * 16) + a(B * (j_max + p_max - 1) * (lb + 1) * 16)


def _rir(m, rng):
    h = rng.normal(0, 8000, m) * np.exp(-np.arange(m) / max(m / 6.0, 1.0))
    h[0] = 20000
    return np.clip(np.round(h), -32768, 32767).astype(np.int16)


NOISE_RIR = [
    # rows (n, rate, target_db, rir length or None, noise offset: "end" = the slice ends at its segment's end), the block length
    ([(200000, 0.9, -20.0, 4096, 17), (150000, 1.0, -25.0, 1, "end"), (16385, 1.1, -30.0, 777, 0), (90001, 1.0, -18.0, 4000, 5)], 1024),
    ([(240000, 1.1, -22.0, 4097, "end"), (100000, 0.9, -26.0, 3000, 3), (50000, 1.0, -20.0, 4097, 11), (16384, 1.0, -24.0, 1, 0)], 2048),
    ([(180000, 1.0, -21.0, 8192, 0), (120000, 0.9, -19.0, 6000, "end"), (70000, 1.1, -27.0, 8192, 9)], 2048),
    ([(160000, 0.9, -23.0, 8193, 1), (100000, 1.0, -20.0, 16384, "end"), (40000, 1.1, -17.0, 2, 4)], 4096),
    ([(210000, 1.0, -22.0, 16385, 2), (130000, 1.1, -25.0, 16384, 0), (16383, 0.9, -28.0, 5000, "end")], 4096),
    ([(300000, 0.9, -21.0, None, "end"), (220000, 1.0, -20.0, None, 0), (16385, 1.1, -24.0, None, 6)], None),   # noise alone
]


@pytest.mark.parametrize("case,with_noise", [(c, wn) for c in range(len(NOISE_RIR)) for wn in (True, False)
                                             if wn or NOISE_RIR[c][1] is not None])
def test_noise_and_reverberation_every_block_length(case, with_noise):
    from pika_b200.loader.audio_bank import AudioBank
    rows, lb = NOISE_RIR[case]
    rng = np.random.default_rng(60 + case)
    pcms = [_pcm(r[0], rng) for r in rows]
    rates, dbs = [r[1] for r in rows], [r[2] for r in rows]
    new_len = [int(n) if r == 1.0 else int(int(n) / float(r)) for n, r, *_ in rows]
    segs = [_pcm(max(new_len) + 5000, rng), _pcm(max(new_len) + 77, rng)]
    nbank = AudioBank(["n0", "n1"], segs, with_rms=True)
    idx = [b % 2 for b in range(len(rows))]
    offs = [len(segs[idx[b]]) - new_len[b] if r[4] == "end" else r[4] for b, r in enumerate(rows)]
    snr = [float(rng.uniform(0, 15)) for _ in rows]
    noise = (nbank, idx, offs, snr) if with_noise else None
    rir, hs = None, None
    if lb is not None:
        hs = [_rir(r[3], rng) for r in rows]
        rir = (AudioBank(["h%d" % b for b in range(len(rows))], hs), list(range(len(rows))))
        m_max = max(r[3] for r in rows)
        assert _conv_geom(m_max) == lb
        assert int(_lib().lib.pk_conv_same_f64_workspace_bytes(len(rows), max(new_len), m_max)) == \
            _conv_ws_bytes(len(rows), max(new_len), m_max)
    tables, geom = kaldi_tables()
    _, wave, got_len, _ = _frontend(pcms, rates, dbs, tables, geom, noise=noise, rir=rir, entry="noise_rir")
    assert got_len == new_len
    for b, r in enumerate(rows):
        kw = {}
        if with_noise:
            kw.update(noise=segs[idx[b]], off=offs[b], snr=snr[b])
        if hs is not None:
            kw.update(rir=hs[b])
        ref = nro.augment(pcms[b], r[1], np.float32(r[2]), **kw)
        check_wave(wave[b, :new_len[b]], ref, r[1], "case %d signal %d (%s)" % (case, b, r))


@pytest.mark.parametrize("rows", [
    [(1500, 5000), (1, 4100), (30000, 1), (3000, 8192), (20000, 6000), (4097, 4097)],     # Lb 2048: N < Lb, N = 1, M = 1, M > N
    [(1, 4097), (2048, 1), (2049, 8000), (100, 8192)],
])
def test_conv_same_f64_block_length_2048(rows):
    from scipy import signal
    L = _lib()
    rng = np.random.default_rng(len(rows) + 90)
    B, n, m = len(rows), max(r[0] for r in rows), max(r[1] for r in rows)
    assert _conv_geom(m) == 2048
    x, h = np.zeros((B, n)), np.zeros((B, m))
    for b, (N, M) in enumerate(rows):
        x[b, :N] = rng.standard_normal(N)
        h[b, :M] = rng.standard_normal(M) * np.exp(-np.arange(M) / max(M / 5.0, 1.0))
    need = int(L.lib.pk_conv_same_f64_workspace_bytes(B, n, m))
    assert need == _conv_ws_bytes(B, n, m)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    y = _guarded(B * n, torch.float64, SENT)
    xd, hd = _dev(x), _dev(h)
    n_len, m_len = _i32([r[0] for r in rows]), _i32([r[1] for r in rows])
    L.check(L.lib.pk_conv_same_f64(xd.data_ptr(), n, n_len.data_ptr(), hd.data_ptr(), m, m_len.data_ptr(), B, n, m, y.data_ptr(), n,
                                   ws.data_ptr(), need, _stream()),
            "pk_conv_same_f64")
    torch.cuda.synchronize()
    _tail_ok(y, B * n, SENT, "y")
    yv = y[:B * n].view(B, n).cpu().numpy()
    for b, (N, M) in enumerate(rows):
        ref = signal.fftconvolve(x[b, :N], h[b, :M], "same")
        assert np.abs(yv[b, :N] - ref).max() / np.abs(ref).max() < 1e-11, (N, M)
        assert (yv[b, N:] == SENT).all(), "y written past n_len"


# ------------------------------------------------------------------------------------------------------------ splice / CMN / masks
SPLICE = [
    # (kind, n_mel, n_feat, lctx, rctx, stride, t_max, bf16, cmn, cmvn, masks): masks "past" start inside and run past D and t_max,
    # "inside" end inside both
    ("fbank", 1, 1, 0, 0, 1, 1, False, True, True, "past"),              # D = 1, t_max = 1
    ("fbank", 1, 1, 0, 0, 3, 1, True, False, False, "inside"),           # D = 1, t_max = 1: the spliced value itself
    ("fbank", 40, 40, 1, 1, 3, 1, False, False, True, "past"),           # t_max = 1, D = 120
    ("fbank", 1, 1, 0, 0, 3, 65, True, True, False, "inside"),
    ("fbank", 40, 40, 1, 1, 1, 64, False, True, True, "past"),           # D = 120, one CMN block
    ("fbank", 40, 40, 1, 1, 3, 129, True, True, True, "inside"),         # three CMN blocks
    ("fbank", 40, 40, 1, 1, 1, 1000, False, False, True, "past"),
    ("fbank", 256, 256, 1, 2, 1, 1000, False, True, True, "inside"),     # D = 1024
    ("fbank", 256, 256, 1, 2, 3, 129, True, True, True, "past"),
    ("mfcc", 128, 128, 3, 4, 1, 129, False, True, True, "inside"),       # D = 1024 of cepstra
    ("mfcc", 128, 128, 3, 4, 3, 65, True, True, False, "past"),
    ("mfcc", 23, 1, 0, 0, 1, 1000, False, True, True, "past"),           # D = 1
    ("mfcc", 64, 40, 1, 1, 3, 1000, True, True, True, "inside"),         # D = 120
]


def _splice_lengths(t_max, stride, frame_len, shift):
    """samples of four utterances: the longest fills t_max rows, one has fewer frames than the stride, one none"""
    nf = [t_max * stride, max(1, stride - 1), (t_max * stride) // 2 + 1, 0]
    return [frame_len + (f - 1) * shift if f > 0 else frame_len // 2 for f in nf]


@pytest.mark.parametrize("case", SPLICE, ids=lambda c: "%s-m%d-f%d-l%d-r%d-s%d-t%d-%s-cmn%d-cmvn%d-%s" % (
    c[0], c[1], c[2], c[3], c[4], c[5], c[6], "bf16" if c[7] else "f32", c[8], c[9], c[10]))
def test_splice_cmn_cmvn_specaugment_bit_exact(case):
    kind, n_mel, n_feat, lctx, rctx, stride, t_max, bf16, cmn, cmvn, masks = case
    rng = np.random.default_rng(sum(case[1:7]))
    n_fft, frame_len, shift = 512, 400, 160
    tables = random_tables(n_fft, frame_len, n_mel, rng, min_width=8)
    geom = (frame_len, shift, 9, 1, 1, 0.97)
    mfcc = (dct_table(n_feat, n_mel), n_feat, 1, 1, 0.0, 0) if kind == "mfcc" else None
    pcms = [_pcm(m, rng) for m in _splice_lengths(t_max, stride, frame_len, shift)]
    rates, dbs = [1.0] * len(pcms), [-20.0, -25.0, -30.0, -22.0]
    # the same call's fbank frames: no context, stride 1, no CMN
    raw, _, _, frames = _frontend(pcms, rates, dbs, tables, geom, 0, 0, 1, mfcc=mfcc)
    assert frames[3] == 0 and (stride == 1 or frames[1] < stride)
    feats = [raw[b, :frames[b]] for b in range(len(pcms))]
    D = n_feat * (lctx + 1 + rctx)
    off = sc = None
    if cmvn:
        off, sc = rng.standard_normal(D).astype(np.float32), (np.abs(rng.standard_normal(D)) + 0.5).astype(np.float32)
    if masks == "past":
        f0, fs, t0, ts = max(0, D - 3), 7, max(0, t_max - 2), 50
    else:
        f0, fs, t0, ts = D // 3, max(1, D // 4), t_max // 3, max(1, t_max // 4)
    # a mask from column 0 or row 0 would cover the whole output at D = 1 or t_max = 1: there it is off
    specaug = (f0, fs if f0 > 0 else 0, t0, ts if t0 > 0 else 0)
    got, _, _, _ = _frontend(pcms, rates, dbs, tables, geom, lctx, rctx, stride, cmn, off, sc, specaug, bf16, mfcc, t_max=t_max)
    ref = fko.splice_cmn_f32(feats, t_max, lctx, rctx, stride, cmn, off, sc, specaug, bf16)
    assert got.shape == ref.shape
    kept = ref[:, :t0 if specaug[3] else t_max, :f0 if specaug[1] else D]          # outside both masks
    for b in range(len(pcms)):
        if frames[b] > 0:
            assert (kept[b] != 0).any(), "utterance %d: the compared values are all zero" % b
    bad = got != ref
    assert not bad.any(), "%d of %d values differ, first at %s: %r vs %r" % (bad.sum(), bad.size, np.argwhere(bad)[0],
                                                                           got[bad][0], ref[bad][0])
    # and the chain of the padded-batch oracle, within float32 rounding
    if not bf16 and all(len(f) for f in feats[:3]):
        data, _, _, _ = ofe.assemble_batch(feats[:3], [[1]] * 3, lctx, rctx, stride, tu_limit=10 ** 9)
        if data.shape[1] == t_max:
            chain = ofe.apply_cmvn(data, off if cmvn else np.zeros(D), sc if cmvn else np.ones(D), cmn=cmn)
            chain = ofe.spec_augment(chain, *specaug)
            np.testing.assert_allclose(got[:3], chain, rtol=1e-5, atol=1e-4 * max(1.0, float(np.abs(chain).max())))


# ------------------------------------------------------------------------------------------------------------ determinism
def _training_batch(rng, B=32):
    from pika_b200.loader.audio_bank import AudioBank
    n = [int(rng.integers(8 * 16000, 15 * 16000 + 1)) for _ in range(B)]
    pcms = [_pcm(m, rng) for m in n]
    rates = [float(rng.choice([0.9, 1.0, 1.1])) for _ in range(B)]
    dbs = [float(rng.uniform(-45, -15)) for _ in range(B)]
    new_len = [int(m) if r == 1.0 else int(int(m) / r) for m, r in zip(n, rates)]
    seg = _pcm(max(new_len) + 20000, rng)
    nbank = AudioBank(["n"], [seg], with_rms=True)
    noise = (nbank, [0] * B, [int(rng.integers(0, len(seg) - L + 1)) for L in new_len], [float(rng.uniform(0, 15)) for _ in range(B)])
    lens = [800, 4000, 8000, 12000]
    rbank = AudioBank(["h%d" % i for i in range(4)], [_rir(m, rng) for m in lens])
    rir = (rbank, [int(rng.integers(0, 4)) for _ in range(B)])
    return pcms, rates, dbs, noise, rir


@pytest.mark.parametrize("entry", ["fwd", "noise_rir", "mfcc"])
def test_training_batch_is_bit_reproducible(entry):
    """B = 32 utterances of 8-15 s at 16 kHz with CMN and CMVN (about 1500 rows: 24 CMN blocks), noise and reverberation, twice"""
    rng = np.random.default_rng(123)
    pcms, rates, dbs, noise, rir = _training_batch(rng)
    tables, geom = kaldi_tables()
    mfcc = (dct_table(13, 80), 13, 1, 1, 0.0, 0) if entry == "mfcc" else None
    D = (13 if mfcc else 80) * 3
    off, sc = rng.standard_normal(D).astype(np.float32), (np.abs(rng.standard_normal(D)) + 0.5).astype(np.float32)
    kw = dict(cmn=1, offset=off, scale=sc, specaug=(10, 5, 100, 20), mfcc=mfcc)
    if entry != "fwd":
        kw.update(noise=noise, rir=rir)
    o1, w1, _, frames = _frontend(pcms, rates, dbs, tables, geom, **kw)
    o2, w2, _, _ = _frontend(pcms, rates, dbs, tables, geom, **kw)
    assert o1.shape[1] > 128 * 8
    assert np.array_equal(w1, w2)
    assert np.array_equal(o1.view(np.uint32), o2.view(np.uint32)), "%d of %d features differ between two runs" % (
        (o1.view(np.uint32) != o2.view(np.uint32)).sum(), o1.size)


# ------------------------------------------------------------------------------------------------------------ host-side rejection
def _rejected(fn, match):
    L = _lib()
    torch.cuda.synchronize()
    n0 = L.launch_count()
    with pytest.raises(L.PikaError, match=match):
        fn()
    assert L.launch_count() == n0, "a kernel ran before the argument was rejected"


def _fbank_call(entry="fbank", log2n=9, frame_len=400, shift=160, n_mel=23, num_ceps=13, dct=True, snip=1, n_samples=True):
    L = _lib()
    rng = np.random.default_rng(0)
    tables = random_tables(512, 400, 256, rng)
    T = [_dev(a) for a in tables]
    wave = torch.zeros(2, 4000, device="cuda")
    feats = torch.zeros(2 * 30 * 256, device="cuda")
    d = _dev(dct_table(13, 23))
    n, nf = _i32([4000, 4000]), _i32([20, 20])
    args = (wave.data_ptr(), 4000, n.data_ptr() if n_samples else None, nf.data_ptr(), 2, 30, n_mel,
            *[t.data_ptr() for t in T], frame_len, shift, log2n, snip, 1, 0.97, feats.data_ptr(), 0.0, 0, _stream())
    if entry == "fbank":
        return L.check(L.lib.pk_fbank(*args), "pk_fbank")
    return L.check(L.lib.pk_mfcc(*args, d.data_ptr() if dct else None, num_ceps, 1, 1, 0.0, 0), "pk_mfcc")


def _fe_call(entry="fwd", n_mel=23, lctx=1, rctx=1, stride=1, t_max=30, log2n=9, frame_len=400, shift=160, ws_delta=0,
             rir_max_len=4000, noise_draws=True, num_ceps=13, dct=True, with_banks=True):
    """a valid call of a front-end entry point but for the one argument changed"""
    from pika_b200.loader.audio_bank import AudioBank
    L = _lib()
    rng = np.random.default_rng(1)
    B, n_max = 2, 8000
    tables = [_dev(a) for a in random_tables(512, 400, 256, rng)]
    mf = entry == "mfcc"
    n_feat = num_ceps if mf else n_mel
    D = n_feat * (lctx + 1 + rctx)
    banks = entry == "noise_rir" or (mf and with_banks)
    if t_max * stride > 0x7FFFFFFF:
        need = 1 << 20                  # the entry point refuses t_max * stride past int before it reads the workspace
    elif banks:
        need = int(L.lib.pk_frontend_noise_rir_workspace_bytes(B, n_max, t_max * stride, n_feat, D, rir_max_len))
    else:
        need = int(L.lib.pk_frontend_workspace_bytes(B, n_max, t_max * stride, n_feat, D))
    if need < 0:
        need = int(L.lib.pk_frontend_noise_rir_workspace_bytes(B, n_max, t_max * stride, n_feat, D, 4000))
    ws = torch.zeros(need + 64, dtype=torch.uint8, device="cuda")
    out = torch.zeros(B * min(t_max, 1 << 16) * max(D, 1) + 64, device="cuda")
    pcm = torch.zeros(B, n_max, dtype=torch.int16, device="cuda")
    i = _i32([n_max, n_max])
    f = torch.ones(B, device="cuda")
    nf = _i32([t_max // 2, t_max // 2])
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    args = (pcm.data_ptr(), n_max, i.data_ptr(), f.data_ptr(), i.data_ptr(), f.data_ptr(), nf.data_ptr(), B, n_max, t_max, n_mel,
            lctx, rctx, stride, *[t.data_ptr() for t in tables], frame_len, shift, log2n, 1, 1, 0.97, 1, None, None, 0, 0, 0, 0,
            out.data_ptr(), L.PK_F32, None, ws.data_ptr(), need + ws_delta, err.data_ptr(), 0.0, 0, _stream())
    if entry == "fwd":
        return L.check(L.lib.pk_frontend_fwd(*args), "pk_frontend_fwd")
    nb = AudioBank(["n"], [np.ones(20000, np.int16)], with_rms=True)
    rb = AudioBank(["h"], [np.ones(4000, np.int16)])
    ns, no, _, nr = nb.device("cuda")
    rs, ro, rl, _ = rb.device("cuda")
    z32, z64, snr = _i32([0, 0]), torch.zeros(B, dtype=torch.int64, device="cuda"), torch.zeros(B, dtype=torch.float64, device="cuda")
    nz = (ns.data_ptr(), z32.data_ptr(), z64.data_ptr(), snr.data_ptr(), nr.data_ptr()) if noise_draws else \
        (ns.data_ptr(), None, None, None, None)
    rr = (rs.data_ptr(), ro.data_ptr(), rl.data_ptr(), z32.data_ptr())
    if not banks:
        nz, rr = (None,) * 5, (None,) * 4
    if entry == "noise_rir":
        return L.check(L.lib.pk_frontend_fwd_noise_rir(*args, *nz, *rr, rir_max_len), "pk_frontend_fwd_noise_rir")
    d = _dev(dct_table(num_ceps if 1 <= num_ceps <= 23 else 13, 23))
    return L.check(L.lib.pk_frontend_fwd_mfcc(*args, *nz, *rr, rir_max_len, d.data_ptr() if dct else None, num_ceps, 1, 1, 0.0, 0),
                   "pk_frontend_fwd_mfcc")


def test_valid_calls_of_the_rejection_cases_run():
    """the baseline the rejection cases change one argument of is itself accepted, and launches"""
    L = _lib()
    for fn in (lambda: _fbank_call("fbank"), lambda: _fbank_call("mfcc"), lambda: _fe_call("fwd"), lambda: _fe_call("noise_rir"),
               lambda: _fe_call("mfcc"), lambda: _fe_call("mfcc", with_banks=False)):
        n0 = L.launch_count()
        fn()
        torch.cuda.synchronize()
        assert L.launch_count() > n0


@pytest.mark.parametrize("entry", ["fbank", "mfcc"])
def test_fbank_arguments_rejected_before_any_launch(entry):
    geom = "bad fbank geometry"
    _rejected(lambda: _fbank_call(entry, log2n=6, frame_len=64), geom)
    _rejected(lambda: _fbank_call(entry, log2n=12), geom)
    _rejected(lambda: _fbank_call(entry, frame_len=0), geom)
    _rejected(lambda: _fbank_call(entry, frame_len=513), geom)
    _rejected(lambda: _fbank_call(entry, shift=0), geom)
    _rejected(lambda: _fbank_call(entry, n_mel=0), "bad fbank dims")
    _rejected(lambda: _fbank_call(entry, n_mel=257), "bad fbank dims")
    _rejected(lambda: _fbank_call(entry, snip=0, n_samples=False), "needs the sample counts")
    if entry == "mfcc":
        _rejected(lambda: _fbank_call(entry, num_ceps=0), "bad MFCC arguments")
        _rejected(lambda: _fbank_call(entry, num_ceps=24), "bad MFCC arguments")
        _rejected(lambda: _fbank_call(entry, dct=False), "bad MFCC arguments")


@pytest.mark.parametrize("entry", ["fwd", "noise_rir", "mfcc"])
def test_frontend_arguments_rejected_before_any_launch(entry):
    geom = "bad fbank geometry"
    _rejected(lambda: _fe_call(entry, log2n=6, frame_len=64), geom)
    _rejected(lambda: _fe_call(entry, log2n=12), geom)
    _rejected(lambda: _fe_call(entry, frame_len=0), geom)
    _rejected(lambda: _fe_call(entry, frame_len=513), geom)
    _rejected(lambda: _fe_call(entry, shift=0), geom)
    _rejected(lambda: _fe_call(entry, n_mel=0), "bad")
    _rejected(lambda: _fe_call(entry, n_mel=257), "bad")
    _rejected(lambda: _fe_call(entry, stride=0), "bad splice stride")
    _rejected(lambda: _fe_call(entry, t_max=1 << 16, stride=1 << 15), "bad splice stride")
    _rejected(lambda: _fe_call(entry, ws_delta=-1), "workspace too small")
    if entry == "mfcc":
        _rejected(lambda: _fe_call(entry, num_ceps=0), "bad MFCC arguments")
        _rejected(lambda: _fe_call(entry, num_ceps=24), "bad MFCC arguments")
        _rejected(lambda: _fe_call(entry, dct=False), "bad MFCC arguments")
        _rejected(lambda: _fe_call(entry, num_ceps=23, lctx=20, rctx=24), "bad frontend dims")      # D = 23 * 45 = 1035
        _rejected(lambda: _fe_call(entry, with_banks=False, ws_delta=-1), "workspace too small")
    else:
        _rejected(lambda: _fe_call(entry, n_mel=205, lctx=2, rctx=2), "bad frontend dims")          # D = 1025
    if entry != "fwd":
        _rejected(lambda: _fe_call(entry, rir_max_len=0), "rir_max_len")
        _rejected(lambda: _fe_call(entry, rir_max_len=65537), "rir_max_len")
        _rejected(lambda: _fe_call(entry, noise_draws=False), "noise bank without")


@pytest.mark.parametrize("B,n_max,m_max,short,match", [(0, 100, 10, 0, "bad conv dims"), (1, 100, 0, 0, "bad conv dims"),
                                                       (1, 100, 65537, 0, "bad conv dims"), (2, 5000, 4097, 1, "workspace too small"),
                                                       (1, 0, 10, 0, "bad conv dims")])
def test_conv_same_f64_arguments_rejected_before_any_launch(B, n_max, m_max, short, match):
    L = _lib()
    x = torch.zeros(4, 5000, dtype=torch.float64, device="cuda")
    n = _i32([10] * 4)
    need = _conv_ws_bytes(max(B, 1), max(n_max, 1), min(max(m_max, 1), 65536))
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    _rejected(lambda: L.check(L.lib.pk_conv_same_f64(x.data_ptr(), 5000, n.data_ptr(), x.data_ptr(), 5000, n.data_ptr(), B, n_max,
                                                     m_max, x.data_ptr(), 5000, ws.data_ptr(), need - short, _stream()),
                              "pk_conv_same_f64"), match)
