"""GPU front end: host-side tables + the call into pk_frontend_fwd (include/pika_b200.h).

Replaces the CPU chain of loader/otf_utt_loader.py:218-250 (AudioSegment augmentation -> PyKaldi
Fbank -> splice) plus trainer/train_transducer_bmuf_otfaug.py:86-93 (CMN/CMVN, SpecAugment).
Feature options are Kaldi's fbank or MFCC options, read from a Kaldi-style config file such as egs/fbank.conf.
"""
import math

import numpy as np
import torch

from . import kernels as K
from ._lib import check, lib

FRAME_LEN, FRAME_SHIFT = 400, 160                     # egs/fbank.conf at 16 kHz: 25 / 10 ms frames
LOG2_NFFT_MIN, LOG2_NFFT_MAX = 7, 11                   # FFT sizes of the fbank kernel: 128 .. 2048
WINDOW_TYPES = ("hamming", "hanning", "povey", "rectangular", "blackman")
# Kaldi fbank / frame-extraction options the front end does not implement; a config that sets one is refused
UNSUPPORTED = ("use-energy", "raw-energy", "energy-floor", "htk-compat", "use-log-fbank", "use-power", "vtln-warp", "vtln-low",
               "vtln-high", "allow-downsample", "allow-upsample")


def _bool(v):
    if isinstance(v, bool):
        return v
    if v in ("true", "True", "1"):
        return True
    if v in ("false", "False", "0"):
        return False
    raise ValueError("expected true or false, got %r" % v)


class FbankOptions:
    """Kaldi FbankOptions (feat/feature-fbank.h, feature-window.h, mel-computations.h): names, defaults and meaning of the
    options the front end implements.  Frame length and shift are in ms; frame_len / frame_shift_samples / n_fft are the sample
    counts Kaldi derives from them (FrameExtractionOptions::WindowSize, WindowShift, PaddedWindowSize)."""

    def __init__(self, num_mel_bins=23, sample_frequency=16000.0, low_freq=20.0, high_freq=0.0, dither=1.0,
                 window_type="povey", preemphasis_coefficient=0.97, frame_length=25.0, frame_shift=10.0, snip_edges=True,
                 remove_dc_offset=True, blackman_coeff=0.42, round_to_power_of_two=True):
        self.num_mel_bins, self.sample_frequency = int(num_mel_bins), float(sample_frequency)
        self.low_freq, self.high_freq, self.dither = float(low_freq), float(high_freq), float(dither)
        self.window_type, self.preemphasis_coefficient = window_type, float(preemphasis_coefficient)
        self.frame_length, self.frame_shift = float(frame_length), float(frame_shift)
        self.snip_edges, self.remove_dc_offset = _bool(snip_edges), _bool(remove_dc_offset)
        self.blackman_coeff, self.round_to_power_of_two = float(blackman_coeff), _bool(round_to_power_of_two)
        if not self.round_to_power_of_two:
            raise ValueError("--round-to-power-of-two=false is not supported: the fbank FFT sizes are powers of two")
        if self.window_type not in WINDOW_TYPES:
            raise ValueError("--window-type=%s: expected one of %s" % (self.window_type, ", ".join(WINDOW_TYPES)))
        if not self.sample_frequency > 0:
            raise ValueError("--sample-frequency must be positive, got %g" % self.sample_frequency)
        self.frame_len = int(self.sample_frequency * 0.001 * self.frame_length)
        self.frame_shift_samples = int(self.sample_frequency * 0.001 * self.frame_shift)
        if self.frame_len < 1 or self.frame_shift_samples < 1:
            raise ValueError("frame length %g ms / shift %g ms is under one sample at %g Hz"
                             % (self.frame_length, self.frame_shift, self.sample_frequency))
        self.log2_nfft = max(0, (self.frame_len - 1).bit_length())
        self.n_fft = 1 << self.log2_nfft
        if not LOG2_NFFT_MIN <= self.log2_nfft <= LOG2_NFFT_MAX:
            raise ValueError("%d-sample frames need a %d-point FFT; the fbank kernel supports %d to %d"
                             % (self.frame_len, self.n_fft, 1 << LOG2_NFFT_MIN, 1 << LOG2_NFFT_MAX))

    def geometry(self):
        """keyword arguments of ``Frontend.lengths`` for these options"""
        return dict(frame_len=self.frame_len, frame_shift=self.frame_shift_samples, snip_edges=self.snip_edges)

    # Kaldi option names of the options above, and the Kaldi options refused (ValueError) rather than ignored
    NAMES = {"window-type": "window_type", "sample-frequency": "sample_frequency", "dither": "dither",
             "low-freq": "low_freq", "high-freq": "high_freq", "num-mel-bins": "num_mel_bins",
             "preemphasis-coefficient": "preemphasis_coefficient", "frame-length": "frame_length",
             "frame-shift": "frame_shift", "snip-edges": "snip_edges", "remove-dc-offset": "remove_dc_offset",
             "blackman-coeff": "blackman_coeff", "round-to-power-of-two": "round_to_power_of_two"}
    REFUSED = UNSUPPORTED
    KIND = "fbank"

    @classmethod
    def from_config(cls, path):
        """Kaldi option file: one ``--name=value`` per line, ``#`` comments (ParseOptions.read_config_file,
        loader/otf_utt_loader.py:195-200)."""
        kw = {}
        with open(path) as f:
            for line in f:
                line = line.split("#")[0].strip()
                if not line:
                    continue
                if not line.startswith("--") or "=" not in line:
                    raise ValueError("bad config line: %r" % line)
                k, v = line[2:].split("=", 1)
                k = k.strip()
                if k in cls.REFUSED:
                    raise ValueError("%s option --%s is not supported by the GPU front end" % (cls.KIND, k))
                if k not in cls.NAMES:
                    raise ValueError("unsupported %s option --%s" % (cls.KIND, k))
                kw[cls.NAMES[k]] = v.strip()
        return cls(**kw)


class MfccOptions(FbankOptions):
    """Kaldi MfccOptions (feat/feature-mfcc.h): FbankOptions' frame and mel options with their defaults (23 mel bins, dither 1), plus
    num-ceps 13, use-energy true, energy-floor 0, raw-energy true, cepstral-lifter 22 and htk-compat false.  Kaldi's MFCC has no
    --use-log-fbank or --use-power (it always takes the log of the power spectrum's mel energies); a config that sets one is refused."""

    NAMES = dict(FbankOptions.NAMES, **{"num-ceps": "num_ceps", "use-energy": "use_energy", "energy-floor": "energy_floor",
                                        "raw-energy": "raw_energy", "cepstral-lifter": "cepstral_lifter", "htk-compat": "htk_compat"})
    REFUSED = ("use-log-fbank", "use-power", "vtln-warp", "vtln-low", "vtln-high", "allow-downsample", "allow-upsample")
    KIND = "MFCC"

    def __init__(self, num_ceps=13, use_energy=True, energy_floor=0.0, raw_energy=True, cepstral_lifter=22.0, htk_compat=False, **fbank):
        super().__init__(**fbank)
        self.num_ceps, self.use_energy, self.energy_floor = int(num_ceps), _bool(use_energy), float(energy_floor)
        self.raw_energy, self.cepstral_lifter, self.htk_compat = _bool(raw_energy), float(cepstral_lifter), _bool(htk_compat)
        if not 1 <= self.num_ceps <= self.num_mel_bins:
            raise ValueError("--num-ceps=%d: num-ceps cannot be larger than num-mel-bins (%d) and must be at least 1"
                             % (self.num_ceps, self.num_mel_bins))


def noise_rir_kwargs(raw):
    """the Frontend keyword arguments for the noise / reverberation draws of a raw batch (empty without them)"""
    return {k: raw[k] for k in ("noise_idx", "noise_off", "snr", "rir_idx", "rir_max_len") if k in raw}


def _mel(f):
    return 1127.0 * math.log(1.0 + f / 700.0)


def window_function(opts):
    """Kaldi FeatureWindowFunction: [frame_len] float32"""
    n = opts.frame_len
    i = np.arange(n, dtype=np.float64)
    c = np.cos(2.0 * np.pi * i / (n - 1)) if n > 1 else np.ones(n)
    if opts.window_type == "hamming":
        w = 0.54 - 0.46 * c
    elif opts.window_type == "hanning":
        w = 0.5 - 0.5 * c
    elif opts.window_type == "povey":
        w = (0.5 - 0.5 * c) ** 0.85
    elif opts.window_type == "rectangular":
        w = np.ones(n)
    else:
        c2 = np.cos(4.0 * np.pi * i / (n - 1)) if n > 1 else np.ones(n)
        w = opts.blackman_coeff - 0.5 * c + (0.5 - opts.blackman_coeff) * c2
    return w.astype(np.float32)


def fbank_tables(opts):
    """host tables of the fbank kernel: window [frame_len], twiddle [N/2, 2], mel weights [n_mel, N/2] (float32) and each mel bin's
    first / one-past-last FFT bin [n_mel] (int32).  Raises ValueError where Kaldi's MelBanks does."""
    n_mel, nfft = opts.num_mel_bins, opts.n_fft
    if not 3 <= n_mel <= 256:
        raise ValueError("--num-mel-bins=%d: the front end supports 3 to 256" % n_mel)
    nyq = 0.5 * opts.sample_frequency
    hi = opts.high_freq + nyq if opts.high_freq <= 0 else opts.high_freq
    if opts.low_freq < 0.0 or opts.low_freq >= nyq or hi <= 0.0 or hi > nyq or hi <= opts.low_freq:
        raise ValueError("Bad values in options: low-freq %g and high-freq %g vs. nyquist %g" % (opts.low_freq, opts.high_freq, nyq))
    k = np.arange(nfft // 2, dtype=np.float64)
    tw = np.stack([np.cos(2 * np.pi * k / nfft), -np.sin(2 * np.pi * k / nfft)], 1).astype(np.float32)
    m_lo, m_hi = _mel(opts.low_freq), _mel(hi)
    delta = (m_hi - m_lo) / (n_mel + 1)
    nb = nfft // 2
    melf = np.array([_mel(opts.sample_frequency / nfft * b) for b in range(nb)])
    w = np.zeros((n_mel, nb), np.float64)
    lo = np.zeros(n_mel, np.int32)
    hi_i = np.zeros(n_mel, np.int32)
    for j in range(n_mel):
        left, center, right = m_lo + j * delta, m_lo + (j + 1) * delta, m_lo + (j + 2) * delta
        inside = (melf > left) & (melf < right)
        w[j] = np.where(inside, np.where(melf <= center, (melf - left) / (center - left), (right - melf) / (right - center)), 0.0)
        nz = np.nonzero(inside)[0]
        if not len(nz):
            raise ValueError("mel bin %d of %d has no FFT bin of the %d-point FFT: you may have set --num-mel-bins too large"
                             % (j, n_mel, nfft))
        lo[j], hi_i[j] = nz[0], nz[-1] + 1
    return window_function(opts), tw, w.astype(np.float32), lo, hi_i


def dct_matrix(num_ceps, n):
    """Kaldi ComputeDctMatrix (matrix/matrix-functions.cc): the orthonormal DCT-II of size n, row 0 scaled by sqrt(1/n) and the others
    by sqrt(2/n), first num_ceps rows: [num_ceps, n] float64"""
    k = np.arange(num_ceps, dtype=np.float64)[:, None]
    m = np.sqrt(2.0 / n) * np.cos(np.pi / n * (np.arange(n, dtype=np.float64)[None, :] + 0.5) * k)
    m[0] = np.sqrt(1.0 / n)
    return m


def lifter_coeffs(num_ceps, q):
    """Kaldi ComputeLifterCoeffs: 1 + 0.5 Q sin(pi i / Q), all ones when Q = 0 (no liftering): [num_ceps] float64"""
    if q == 0.0:
        return np.ones(num_ceps)
    return 1.0 + 0.5 * q * np.sin(np.pi * np.arange(num_ceps, dtype=np.float64) / q)


def mfcc_tables(opts):
    """host table of the MFCC epilogue: [n_mel, num_ceps] float32, the DCT rows times the lifter, transposed.  Folding the lifter into
    the DCT (in float64, one rounding to float32) changes only the rounding against Kaldi's separate multiply by the lifter."""
    d = dct_matrix(opts.num_ceps, opts.num_mel_bins) * lifter_coeffs(opts.num_ceps, opts.cepstral_lifter)[:, None]
    return np.ascontiguousarray(d.T).astype(np.float32)


class Frontend:
    """Device-resident tables + workspace; ``__call__`` runs one padded batch.  ``stride`` keeps every stride-th spliced frame
    (loader/otf_utt_loader.py:243-250): an utterance of n fbank frames yields ceil(n / stride) rows.  ``opts`` is an FbankOptions
    (log mel energies, n_feat = num_mel_bins per frame) or an MfccOptions (cepstra, n_feat = num_ceps per frame); n_mel is the
    number of mel bins either way."""

    def __init__(self, opts, lctx=1, rctx=1, device="cuda", stride=1):
        if int(stride) < 1:
            raise ValueError("stride must be >= 1, got %r" % stride)
        self.opts, self.lctx, self.rctx, self.device, self.stride = opts, lctx, rctx, device, int(stride)
        self.n_mel = opts.num_mel_bins
        self.is_mfcc = isinstance(opts, MfccOptions)
        self.n_feat = opts.num_ceps if self.is_mfcc else self.n_mel
        self.D = self.n_feat * (lctx + 1 + rctx)
        if self.D > 1024:
            raise ValueError("spliced dimension %d above 1024" % self.D)
        win, tw, w, lo, hi_i = fbank_tables(opts)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
        self.window, self.twiddle, self.mel_w, self.mel_lo, self.mel_hi = t(win), t(tw), t(w), t(lo), t(hi_i)
        self.dct = t(mfcc_tables(opts)) if self.is_mfcc else None
        self.err = torch.zeros(1, dtype=torch.int32, device=device)
        self._ws = None
        self.noise = self.rir = None           # AudioBank defaults for on-the-fly noise / reverberation (loader/audio_bank.py)
        self.dither_seed = 0x243F6A88          # advanced once per batch: every batch draws fresh dither noise

    def _geometry_args(self):
        o = self.opts
        return (o.frame_len, o.frame_shift_samples, o.log2_nfft, int(o.snip_edges), int(o.remove_dc_offset), o.preemphasis_coefficient)

    def _mfcc_args(self):
        o = self.opts
        return (K._P(self.dct), o.num_ceps, int(o.use_energy), int(o.raw_energy), o.energy_floor, int(o.htk_compat))

    def out_lens(self, n_frames):
        """rows per utterance after the stride: ceil(n_frames / stride), for an int, a list or a tensor"""
        s = self.stride
        if s == 1:
            return n_frames
        if isinstance(n_frames, (list, tuple)):
            return [(int(n) + s - 1) // s for n in n_frames]
        return (n_frames + s - 1) // s

    @staticmethod
    def lengths(n_samples, rate, frame_len=FRAME_LEN, frame_shift=FRAME_SHIFT, snip_edges=True):
        """host arithmetic: new_len = int(N / rate) (loader/audio.py:233) and Kaldi's NumFrames of new_len samples (fbank frames,
        before any stride); the defaults are the 16 kHz recipe's 25 / 10 ms frames, ``FbankOptions.geometry()`` gives the rest."""
        new_len = [int(n) if r == 1.0 else int(int(n) / float(r)) for n, r in zip(n_samples, rate)]
        if snip_edges:
            frames = [0 if n < frame_len else 1 + (n - frame_len) // frame_shift for n in new_len]
        else:
            frames = [(n + frame_shift // 2) // frame_shift for n in new_len]
        return new_len, frames

    def __call__(self, pcm, n_samples, rate, target_db, new_len, n_frames, t_max, out_dtype=torch.float32, cmn=True,
                 offset=None, scale=None, specaug=(0, 0, 0, 0), want_wave=False, noise=None, noise_idx=None, noise_off=None,
                 snr=None, rir=None, rir_idx=None, rir_max_len=None):
        """pcm int16 [B, n_max] (device); n_samples/new_len/n_frames int32 [B], rate/target_db f32 [B] (device);
        -> feats [B, t_max, D] (out_dtype) [, augmented int16 wave], D = n_feat * (lctx + 1 + rctx).  n_frames counts fbank frames (``lengths``), t_max output
        rows: at least the longest ``out_lens(n_frames)``.

        On-the-fly noise (loader/audio.py:467-513 add_noise) runs when ``noise_idx`` is given: noise_idx int32 [B] segment of
        ``noise`` (an ``AudioBank``, default ``self.noise``), noise_off int64 [B] offset inside that segment, snr f64 [B] dB.
        Reverberation (convolve_and_normalize, :450-465) runs when ``rir_idx`` int32 [B] is given, with ``rir`` (default
        ``self.rir``); rir_max_len: host int >= the longest drawn RIR (computed from the bank when omitted)."""
        B, n_max = pcm.shape
        aug = noise_idx is not None or rir_idx is not None
        if aug:
            rir_max_len = self._rir_max_len(rir, rir_idx, rir_max_len)
            need = int(lib.pk_frontend_noise_rir_workspace_bytes(B, n_max, t_max * self.stride, self.n_feat, self.D, rir_max_len))
            if need < 0:
                raise ValueError("rir_max_len %d outside [1, 65536]" % rir_max_len)
        else:
            need = int(lib.pk_frontend_workspace_bytes(B, n_max, t_max * self.stride, self.n_feat, self.D))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        out = torch.empty(B, t_max, self.D, dtype=out_dtype, device=self.device)
        wave = torch.zeros(B, n_max, dtype=torch.int16, device=self.device) if want_wave else None
        P = K._P
        f0, fs, t0, ts = specaug
        args = (P(pcm), pcm.stride(0), P(n_samples), P(rate), P(new_len), P(target_db),
                P(n_frames), B, n_max, t_max, self.n_mel, self.lctx, self.rctx, self.stride, P(self.window), P(self.twiddle),
                P(self.mel_w), P(self.mel_lo), P(self.mel_hi), *self._geometry_args(),
                int(cmn), P(offset), P(scale), int(f0), int(fs), int(t0), int(ts), P(out), K._dt(out), P(wave),
                P(self._ws), need, P(self.err), self.opts.dither, self._next_dither_seed(), K._stream())
        if not aug:
            if self.is_mfcc:
                check(lib.pk_frontend_fwd_mfcc(*args, *(None,) * 9, 1, *self._mfcc_args()), "pk_frontend_fwd_mfcc")
            else:
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
        banks = (*[P(t) for t in nz], *[P(t) for t in rr], int(rir_max_len))
        if self.is_mfcc:
            check(lib.pk_frontend_fwd_mfcc(*args, *banks, *self._mfcc_args()), "pk_frontend_fwd_mfcc")
        else:
            check(lib.pk_frontend_fwd_noise_rir(*args, *banks), "pk_frontend_fwd_noise_rir")
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

    def fbank(self, wave_f32, n_frames, t_max, dither=None, seed=None, n_samples=None):
        """wave f32 [B, n] of int16-scaled samples -> [B, t_max, n_mel] log-mel (rows >= n_frames[b] undefined).  n_samples int32
        [B] (device): each signal's length, which the reflected edges need when snip_edges is false."""
        if not self.opts.snip_edges and n_samples is None:
            raise ValueError("Frontend.fbank: snip_edges=false needs n_samples")
        B = wave_f32.shape[0]
        feats = torch.zeros(B, t_max, self.n_mel, dtype=torch.float32, device=self.device)
        P = K._P
        check(lib.pk_fbank(P(wave_f32), wave_f32.stride(0), P(n_samples), P(n_frames), B, t_max, self.n_mel, P(self.window),
                           P(self.twiddle), P(self.mel_w), P(self.mel_lo), P(self.mel_hi), *self._geometry_args(), P(feats),
                           self.opts.dither if dither is None else dither,
                           (self._next_dither_seed() if seed is None else seed) & 0xFFFFFFFF, K._stream()), "pk_fbank")
        return feats

    def mfcc(self, wave_f32, n_frames, t_max, dither=None, seed=None, n_samples=None):
        """the MFCC counterpart of ``fbank`` (MfccOptions only): wave f32 [B, n] of int16-scaled samples -> [B, t_max, num_ceps]
        cepstra (rows >= n_frames[b] undefined)"""
        if not self.is_mfcc:
            raise ValueError("Frontend.mfcc needs MfccOptions")
        if not self.opts.snip_edges and n_samples is None:
            raise ValueError("Frontend.mfcc: snip_edges=false needs n_samples")
        B = wave_f32.shape[0]
        feats = torch.zeros(B, t_max, self.n_feat, dtype=torch.float32, device=self.device)
        P = K._P
        check(lib.pk_mfcc(P(wave_f32), wave_f32.stride(0), P(n_samples), P(n_frames), B, t_max, self.n_mel, P(self.window),
                          P(self.twiddle), P(self.mel_w), P(self.mel_lo), P(self.mel_hi), *self._geometry_args(), P(feats),
                          self.opts.dither if dither is None else dither,
                          (self._next_dither_seed() if seed is None else seed) & 0xFFFFFFFF, K._stream(), *self._mfcc_args()), "pk_mfcc")
        return feats
