"""Numpy restatement of Kaldi's fbank at any sample rate, frame geometry and window (feat/feature-window.cc ExtractWindow,
ProcessWindow, FeatureWindowFunction; feat/feature-fbank.cc Compute; feat/mel-computations.cc MelBanks), for the tests of the
GPU front end's fbank options.  Test infrastructure only.  With its defaults it is oracle/frontend.py's kaldi_fbank (egs/fbank.conf);
it is pinned against torchaudio.compliance.kaldi.fbank through tests/golden/fbank_opts.npz.  dither = 0."""
import numpy as np

from oracle import frontend as ofe


def frame_samples(sample_frequency=16000.0, frame_length=25.0, frame_shift=10.0):
    """FrameExtractionOptions::WindowSize / WindowShift / PaddedWindowSize (round-to-power-of-two)"""
    n = int(sample_frequency * 0.001 * frame_length)
    return n, int(sample_frequency * 0.001 * frame_shift), 1 << (n - 1).bit_length()


def num_frames(n_samples, frame_len=400, frame_shift=160, snip_edges=True):
    """feature-window.cc NumFrames"""
    if snip_edges:
        return 0 if n_samples < frame_len else 1 + (n_samples - frame_len) // frame_shift
    return (n_samples + frame_shift // 2) // frame_shift


def window(frame_len, window_type="hamming", blackman_coeff=0.42):
    """FeatureWindowFunction, a = 2 pi / (frame_len - 1)"""
    i = np.arange(frame_len, dtype=np.float64)
    a = 2.0 * np.pi / (frame_len - 1)
    if window_type == "hanning":
        w = 0.5 - 0.5 * np.cos(a * i)
    elif window_type == "hamming":
        w = 0.54 - 0.46 * np.cos(a * i)
    elif window_type == "povey":
        w = np.power(0.5 - 0.5 * np.cos(a * i), 0.85)
    elif window_type == "rectangular":
        w = np.ones(frame_len)
    elif window_type == "blackman":
        w = blackman_coeff - 0.5 * np.cos(a * i) + (0.5 - blackman_coeff) * np.cos(2 * a * i)
    else:
        raise ValueError(window_type)
    return w.astype(np.float32)


def frame_indices(n_samples, frame_len, frame_shift, snip_edges):
    """[T, frame_len] sample index of every window sample; snip_edges=False reflects indices outside [0, n) (ExtractWindow)"""
    T = num_frames(n_samples, frame_len, frame_shift, snip_edges)
    start = np.arange(T) * frame_shift
    if not snip_edges:
        start = start + frame_shift // 2 - frame_len // 2
    idx = start[:, None] + np.arange(frame_len)[None, :]
    if not snip_edges:
        while ((idx < 0) | (idx >= n_samples)).any():
            idx = np.where(idx < 0, -idx - 1, idx)
            idx = np.where(idx >= n_samples, 2 * n_samples - 1 - idx, idx)
    return idx


def kaldi_fbank(wave, num_mel_bins=80, sample_frequency=16000.0, frame_length=25.0, frame_shift=10.0, window_type="hamming",
                snip_edges=True, remove_dc_offset=True, preemphasis_coefficient=0.97, low_freq=40.0, high_freq=-200.0,
                blackman_coeff=0.42):
    """wave: 1-D int16-scaled samples -> [T, num_mel_bins] float32 log-mel energies"""
    wave = np.asarray(wave, dtype=np.float32)
    frame_len, shift, n_fft = frame_samples(sample_frequency, frame_length, frame_shift)
    idx = frame_indices(wave.shape[0], frame_len, shift, snip_edges)
    if idx.shape[0] == 0:
        return np.zeros((0, num_mel_bins), np.float32)
    fr = wave[idx].astype(np.float32)
    if remove_dc_offset:
        fr = fr - fr.mean(axis=1, keepdims=True, dtype=np.float32)
    pre = np.empty_like(fr)
    c = np.float32(preemphasis_coefficient)
    pre[:, 1:] = fr[:, 1:] - c * fr[:, :-1]
    pre[:, 0] = fr[:, 0] - c * fr[:, 0]
    pre = pre * window(frame_len, window_type, blackman_coeff)[None, :]
    spec = np.fft.rfft(pre.astype(np.float64), n=n_fft, axis=1)
    power = (spec.real ** 2 + spec.imag ** 2).astype(np.float32)[:, : n_fft // 2]
    mel = power @ ofe.mel_banks(num_mel_bins, sample_frequency, low_freq, high_freq, n_fft=n_fft).T
    return np.log(np.maximum(mel, np.finfo(np.float32).eps)).astype(np.float32)
