"""Numpy restatement of Kaldi's MFCC (feat/feature-mfcc.cc MfccComputer::Compute, feat/feature-window.cc ProcessWindow,
matrix/matrix-functions.cc ComputeDctMatrix, feat/feature-functions.cc ComputeLifterCoeffs) at any sample rate, frame geometry and
window, for the tests of the GPU front end's MFCC.  Test infrastructure only: framing, window and mel banks come from
tests/fbank_opts_oracle.py and oracle/frontend.py; it is pinned against torchaudio.compliance.kaldi.mfcc through
tests/golden/mfcc.npz.  dither = 0."""
import math

import numpy as np

import fbank_opts_oracle as fo
from oracle import frontend as ofe

EPS = np.finfo(np.float32).eps


def dct_matrix(num_ceps, n):
    """ComputeDctMatrix: M[0, j] = sqrt(1/n), M[k, j] = sqrt(2/n) cos(pi/n (j + 1/2) k); the first num_ceps rows"""
    m = np.empty((num_ceps, n))
    for k in range(num_ceps):
        for j in range(n):
            m[k, j] = math.sqrt(1.0 / n) if k == 0 else math.sqrt(2.0 / n) * math.cos(math.pi / n * (j + 0.5) * k)
    return m


def lifter(num_ceps, q):
    """ComputeLifterCoeffs: 1 + 0.5 Q sin(pi i / Q); none (ones) when Q = 0"""
    return np.array([1.0 + 0.5 * q * math.sin(math.pi * i / q) if q != 0.0 else 1.0 for i in range(num_ceps)])


def kaldi_mfcc(wave, num_ceps=13, num_mel_bins=23, use_energy=True, energy_floor=0.0, raw_energy=True, cepstral_lifter=22.0,
               htk_compat=False, sample_frequency=16000.0, frame_length=25.0, frame_shift=10.0, window_type="povey", snip_edges=True,
               remove_dc_offset=True, preemphasis_coefficient=0.97, low_freq=20.0, high_freq=0.0, blackman_coeff=0.42, **_):
    """wave: 1-D int16-scaled samples -> [T, num_ceps] float32 cepstra (Kaldi's defaults)"""
    wave = np.asarray(wave, dtype=np.float32)
    frame_len, shift, n_fft = fo.frame_samples(sample_frequency, frame_length, frame_shift)
    idx = fo.frame_indices(wave.shape[0], frame_len, shift, snip_edges)
    if idx.shape[0] == 0:
        return np.zeros((0, num_ceps), np.float32)
    fr = wave[idx].astype(np.float64)
    if remove_dc_offset:
        fr = fr - fr.mean(axis=1, keepdims=True)
    raw_e = (fr * fr).sum(axis=1)
    pre = np.empty_like(fr)
    c = float(np.float32(preemphasis_coefficient))
    pre[:, 1:] = fr[:, 1:] - c * fr[:, :-1]
    pre[:, 0] = fr[:, 0] - c * fr[:, 0]
    pre = pre * fo.window(frame_len, window_type, blackman_coeff).astype(np.float64)[None, :]
    energy = np.log(np.maximum(raw_e if raw_energy else (pre * pre).sum(axis=1), EPS))
    if energy_floor > 0.0:
        energy = np.maximum(energy, math.log(energy_floor))
    spec = np.fft.rfft(pre, n=n_fft, axis=1)
    power = (spec.real ** 2 + spec.imag ** 2)[:, : n_fft // 2]
    mel = power @ ofe.mel_banks(num_mel_bins, sample_frequency, low_freq, high_freq, n_fft=n_fft).T.astype(np.float64)
    logmel = np.log(np.maximum(mel, EPS))
    ceps = logmel @ dct_matrix(num_ceps, num_mel_bins).T * lifter(num_ceps, cepstral_lifter)[None, :]
    if use_energy:
        ceps[:, 0] = energy
    if htk_compat:
        c0 = ceps[:, 0] * (1.0 if use_energy else math.sqrt(2.0))
        ceps = np.concatenate([ceps[:, 1:], c0[:, None]], axis=1)
    return ceps.astype(np.float32)
