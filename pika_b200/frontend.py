"""GPU front end: host-side tables + the call into pk_frontend_fwd (include/pika_b200.h).

Replaces the CPU chain of loader/otf_utt_loader.py:218-250 (AudioSegment augmentation -> PyKaldi
Fbank -> splice) plus trainer/train_transducer_bmuf_otfaug.py:86-93 (CMN/CMVN, SpecAugment).
Feature options are Kaldi's, read from a Kaldi-style config file such as egs/fbank.conf.
"""
import math

import numpy as np
import torch

from . import kernels as K
from ._lib import check, lib

FRAME_LEN, FRAME_SHIFT, NFFT = 400, 160, 512


class FbankOptions:
    """The subset of Kaldi FbankOptions the reference recipes set (egs/fbank.conf) + defaults."""

    def __init__(self, num_mel_bins=23, sample_frequency=16000.0, low_freq=20.0, high_freq=0.0, dither=1.0,
                 window_type="povey", preemphasis_coefficient=0.97):
        self.num_mel_bins, self.sample_frequency = int(num_mel_bins), float(sample_frequency)
        self.low_freq, self.high_freq, self.dither = float(low_freq), float(high_freq), float(dither)
        self.window_type, self.preemphasis_coefficient = window_type, float(preemphasis_coefficient)

    @classmethod
    def from_config(cls, path):
        """Kaldi option file: one ``--name=value`` per line, ``#`` comments (ParseOptions.read_config_file,
        loader/otf_utt_loader.py:195-200)."""
        kw = {}
        names = {"window-type": "window_type", "sample-frequency": "sample_frequency", "dither": "dither",
                 "low-freq": "low_freq", "high-freq": "high_freq", "num-mel-bins": "num_mel_bins",
                 "preemphasis-coefficient": "preemphasis_coefficient"}
        with open(path) as f:
            for line in f:
                line = line.split("#")[0].strip()
                if not line:
                    continue
                if not line.startswith("--") or "=" not in line:
                    raise ValueError("bad config line: %r" % line)
                k, v = line[2:].split("=", 1)
                if k.strip() not in names:
                    raise ValueError("unsupported fbank option --%s" % k)
                kw[names[k.strip()]] = v.strip()
        return cls(**kw)


def noise_rir_kwargs(raw):
    """the Frontend keyword arguments for the noise / reverberation draws of a raw batch (empty without them)"""
    return {k: raw[k] for k in ("noise_idx", "noise_off", "snr", "rir_idx", "rir_max_len") if k in raw}


def _mel(f):
    return 1127.0 * math.log(1.0 + f / 700.0)


class Frontend:
    """Device-resident tables + workspace; ``__call__`` runs one padded batch."""

    def __init__(self, opts, lctx=1, rctx=1, device="cuda"):
        if opts.window_type != "hamming":
            raise NotImplementedError("only the recipe's hamming window is implemented")
        if opts.sample_frequency != 16000.0:
            raise NotImplementedError("16 kHz only (25 ms / 10 ms frames = 400 / 160 samples)")
        self.opts, self.lctx, self.rctx, self.device = opts, lctx, rctx, device
        self.n_mel = opts.num_mel_bins
        self.D = self.n_mel * (lctx + 1 + rctx)
        i = np.arange(FRAME_LEN, dtype=np.float64)
        win = (0.54 - 0.46 * np.cos(2.0 * np.pi * i / (FRAME_LEN - 1))).astype(np.float32)
        k = np.arange(NFFT // 2, dtype=np.float64)
        tw = np.stack([np.cos(2 * np.pi * k / NFFT), -np.sin(2 * np.pi * k / NFFT)], 1).astype(np.float32)
        nyq = 0.5 * opts.sample_frequency
        hi = opts.high_freq + nyq if opts.high_freq <= 0 else opts.high_freq
        m_lo, m_hi = _mel(opts.low_freq), _mel(hi)
        delta = (m_hi - m_lo) / (self.n_mel + 1)
        nb = NFFT // 2
        melf = np.array([_mel(opts.sample_frequency / NFFT * b) for b in range(nb)])
        w = np.zeros((self.n_mel, nb), np.float64)
        lo = np.zeros(self.n_mel, np.int32)
        hi_i = np.zeros(self.n_mel, np.int32)
        for j in range(self.n_mel):
            left, center, right = m_lo + j * delta, m_lo + (j + 1) * delta, m_lo + (j + 2) * delta
            inside = (melf > left) & (melf < right)
            w[j] = np.where(inside, np.where(melf <= center, (melf - left) / (center - left), (right - melf) / (right - center)), 0.0)
            nz = np.nonzero(inside)[0]
            lo[j], hi_i[j] = (nz[0], nz[-1] + 1) if len(nz) else (0, 0)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
        self.window, self.twiddle, self.mel_w, self.mel_lo, self.mel_hi = t(win), t(tw), t(w.astype(np.float32)), t(lo), t(hi_i)
        self.err = torch.zeros(1, dtype=torch.int32, device=device)
        self._ws = None
        self.noise = self.rir = None           # AudioBank defaults for on-the-fly noise / reverberation (loader/audio_bank.py)
        self.dither_seed = 0x243F6A88          # advanced once per batch: every batch draws fresh dither noise

    @staticmethod
    def lengths(n_samples, rate):
        """host arithmetic: new_len = int(N / rate) (loader/audio.py:233), snip-edges frame count."""
        new_len = [int(n) if r == 1.0 else int(int(n) / float(r)) for n, r in zip(n_samples, rate)]
        frames = [0 if n < FRAME_LEN else 1 + (n - FRAME_LEN) // FRAME_SHIFT for n in new_len]
        return new_len, frames

    def __call__(self, pcm, n_samples, rate, target_db, new_len, n_frames, t_max, out_dtype=torch.float32, cmn=True,
                 offset=None, scale=None, specaug=(0, 0, 0, 0), want_wave=False, noise=None, noise_idx=None, noise_off=None,
                 snr=None, rir=None, rir_idx=None, rir_max_len=None):
        """pcm int16 [B, n_max] (device); n_samples/new_len/n_frames int32 [B], rate/target_db f32 [B] (device);
        -> feats [B, t_max, D] (out_dtype) [, augmented int16 wave].

        On-the-fly noise (loader/audio.py:467-513 add_noise) runs when ``noise_idx`` is given: noise_idx int32 [B] segment of
        ``noise`` (an ``AudioBank``, default ``self.noise``), noise_off int64 [B] offset inside that segment, snr f64 [B] dB.
        Reverberation (convolve_and_normalize, :450-465) runs when ``rir_idx`` int32 [B] is given, with ``rir`` (default
        ``self.rir``); rir_max_len: host int >= the longest drawn RIR (computed from the bank when omitted)."""
        B, n_max = pcm.shape
        aug = noise_idx is not None or rir_idx is not None
        if aug:
            rir_max_len = self._rir_max_len(rir, rir_idx, rir_max_len)
            need = int(lib.pk_frontend_noise_rir_workspace_bytes(B, n_max, t_max, self.n_mel, self.D, rir_max_len))
            if need < 0:
                raise ValueError("rir_max_len %d outside [1, 65536]" % rir_max_len)
        else:
            need = int(lib.pk_frontend_workspace_bytes(B, n_max, t_max, self.n_mel, self.D))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        out = torch.empty(B, t_max, self.D, dtype=out_dtype, device=self.device)
        wave = torch.zeros(B, n_max, dtype=torch.int16, device=self.device) if want_wave else None
        P = K._P
        f0, fs, t0, ts = specaug
        args = (P(pcm), pcm.stride(0), P(n_samples), P(rate), P(new_len), P(target_db),
                P(n_frames), B, n_max, t_max, self.n_mel, self.lctx, self.rctx, P(self.window), P(self.twiddle),
                P(self.mel_w), P(self.mel_lo), P(self.mel_hi), self.opts.preemphasis_coefficient,
                int(cmn), P(offset), P(scale), int(f0), int(fs), int(t0), int(ts), P(out), K._dt(out), P(wave),
                P(self._ws), need, P(self.err), self.opts.dither, self._next_dither_seed(), K._stream())
        if not aug:
            check(lib.pk_frontend_fwd(*args), "pk_frontend_fwd")
            return (out, wave) if want_wave else out
        dev = lambda t, dt: torch.as_tensor(t).to(device=self.device, dtype=dt, non_blocking=True)  # noqa: E731
        nz = (None,) * 5
        if noise_idx is not None:
            bank = noise if noise is not None else self.noise
            if bank is None:
                raise ValueError("noise draws given without a noise bank")
            samples, offs, _, rms = bank.device(self.device)
            idx = dev(noise_idx, torch.int32)
            start = offs[idx.long()] + dev(noise_off, torch.int64)                 # absolute bank offset of the first sample
            nz = (samples, idx, start, dev(snr, torch.float64), rms)
        rr = (None,) * 4
        if rir_idx is not None:
            bank = rir if rir is not None else self.rir
            samples, offs, lens, _ = bank.device(self.device)
            rr = (samples, offs, lens, dev(rir_idx, torch.int32))
        check(lib.pk_frontend_fwd_noise_rir(*args, *[P(t) for t in nz], *[P(t) for t in rr], int(rir_max_len)),
              "pk_frontend_fwd_noise_rir")
        return (out, wave) if want_wave else out

    def _rir_max_len(self, rir, rir_idx, rir_max_len):
        if rir_idx is None:
            return 1
        bank = rir if rir is not None else self.rir
        if bank is None:
            raise ValueError("RIR draws given without an RIR bank")
        if rir_max_len is None:
            rir_max_len = int(bank.lengths[torch.as_tensor(rir_idx).cpu().numpy()].max())
        return int(rir_max_len)

    def _next_dither_seed(self):
        self.dither_seed = (self.dither_seed * 1664525 + 1013904223) & 0xFFFFFFFF
        return self.dither_seed

    def fbank(self, wave_f32, n_frames, t_max, dither=None, seed=None):
        """wave f32 [B, n] of int16-scaled samples -> [B, t_max, n_mel] log-mel (rows >= n_frames[b] undefined)."""
        B = wave_f32.shape[0]
        feats = torch.zeros(B, t_max, self.n_mel, dtype=torch.float32, device=self.device)
        P = K._P
        check(lib.pk_fbank(P(wave_f32), wave_f32.stride(0), P(n_frames), B, t_max, self.n_mel, P(self.window),
                           P(self.twiddle), P(self.mel_w), P(self.mel_lo), P(self.mel_hi), self.opts.preemphasis_coefficient, P(feats),
                           self.opts.dither if dither is None else dither,
                           (self._next_dither_seed() if seed is None else seed) & 0xFFFFFFFF, K._stream()), "pk_fbank")
        return feats
