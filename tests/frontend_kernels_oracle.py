"""Numpy restatements of the front-end kernels (pika_b200/csrc/frontend.cu) over the kernels' own tables, for the kernel tests in
tests/test_frontend_kernels_gpu.py.  Test infrastructure only.

``fbank_from_tables`` / ``mfcc_from_tables`` restate ``fbank_kernel`` in float64 from its inputs: window, mel weights with their
[lo, hi) bin ranges, MFCC DCT table.  They accept tables that Kaldi's MelBanks would refuse (random weights, 256 bins at a 128-point
FFT), so the kernel can be driven to its limits; on Kaldi's tables they are Kaldi's fbank and MFCC (pinned in
tests/test_frontend_kernels_cpu.py against tests/fbank_opts_oracle.py and tests/mfcc_oracle.py).

``splice_cmn_f32`` restates ``splice_colsum`` + ``splice_colmerge`` + ``splice_finalize`` bit for bit in float32: the CMN column sums
run in row order within blocks of 64 output rows, then in block order, which is the order the kernels use."""
import math

import numpy as np

EPS = np.float32(np.finfo(np.float32).eps)
CMN_BLOCK = 64


def frame_starts(n_frames, frame_len, frame_shift, snip_edges):
    """first sample of every frame (Kaldi's ExtractWindow; negative when snip_edges is off)"""
    start = np.arange(n_frames, dtype=np.int64) * frame_shift
    return start if snip_edges else start + frame_shift // 2 - frame_len // 2


def reflect(idx, n):
    """samples outside [0, n) reflected about the signal's edges until inside (n >= 1)"""
    idx = np.array(idx, dtype=np.int64)
    while ((idx < 0) | (idx >= n)).any():
        idx = np.where(idx < 0, -idx - 1, idx)
        idx = np.where(idx >= n, 2 * n - 1 - idx, idx)
    return idx


def frames(wave, n_frames, frame_len, frame_shift, snip_edges, n_len=None):
    """[n_frames, frame_len] float64 windows of wave (int16-scaled samples); n_len: the signal's length (reflection bound)"""
    wave = np.asarray(wave, dtype=np.float32).astype(np.float64)
    idx = frame_starts(n_frames, frame_len, frame_shift, snip_edges)[:, None] + np.arange(frame_len)[None, :]
    if not snip_edges:
        idx = reflect(idx, len(wave) if n_len is None else n_len)
    return wave[idx]


def _process(fr, window, remove_dc, preemph):
    """DC removal, pre-emphasis x[i] -= c x[i-1] with x[0] -= c x[0], window: -> (raw frames after DC removal, windowed frames)"""
    if remove_dc:
        fr = fr - fr.mean(axis=1, keepdims=True)
    c = float(np.float32(preemph))
    pre = np.empty_like(fr)
    pre[:, 1:] = fr[:, 1:] - c * fr[:, :-1]
    pre[:, 0] = fr[:, 0] - c * fr[:, 0]
    return fr, pre * np.asarray(window, np.float32).astype(np.float64)[None, :]


def power_spectrum(windowed, n_fft):
    """|rfft|^2 of the zero-padded frames, bins 0 .. N/2 - 1 (the Nyquist bin is never used)"""
    spec = np.fft.rfft(windowed, n=n_fft, axis=1)[:, : n_fft // 2]
    return spec.real ** 2 + spec.imag ** 2


def mel_energies(power, mel_w, mel_lo, mel_hi):
    """linear mel energies [T, n_mel]: mel bin j sums w[j, k] power[k] over k in [lo[j], hi[j]) only"""
    k = np.arange(power.shape[1])[None, :]
    w = np.where((k >= np.asarray(mel_lo)[:, None]) & (k < np.asarray(mel_hi)[:, None]), np.asarray(mel_w, np.float32), 0.0)
    return power @ w.T.astype(np.float64)


def fbank_from_tables(wave, n_frames, window, mel_w, mel_lo, mel_hi, n_fft, frame_shift, snip_edges=True, remove_dc=True,
                      preemph=0.97, n_len=None):
    """-> (log mel energies [T, n_mel] float64 floored at FLT_EPSILON, linear mel energies [T, n_mel], power spectra [T, N/2])"""
    fr = frames(wave, n_frames, len(window), frame_shift, snip_edges, n_len)
    _, win = _process(fr, window, remove_dc, preemph)
    power = power_spectrum(win, n_fft)
    mel = mel_energies(power, mel_w, mel_lo, mel_hi)
    return np.log(np.maximum(mel, EPS)), mel, power


def mfcc_from_tables(wave, n_frames, window, mel_w, mel_lo, mel_hi, n_fft, frame_shift, dct, use_energy=True, raw_energy=True,
                     energy_floor=0.0, htk_compat=False, snip_edges=True, remove_dc=True, preemph=0.97, n_len=None):
    """MFCC epilogue over ``fbank_from_tables``: dct [n_mel, num_ceps] (the kernel's transposed table, lifter folded in).
    -> (cepstra [T, num_ceps] float64 in output column order, linear mel energies [T, n_mel])"""
    fr = frames(wave, n_frames, len(window), frame_shift, snip_edges, n_len)
    raw, win = _process(fr, window, remove_dc, preemph)
    mel = mel_energies(power_spectrum(win, n_fft), mel_w, mel_lo, mel_hi)
    ceps = np.log(np.maximum(mel, EPS)) @ np.asarray(dct, np.float32).astype(np.float64)
    if use_energy:
        e = ((raw * raw) if raw_energy else (win * win)).sum(axis=1)
        e = np.log(np.maximum(e, EPS))
        if energy_floor > 0.0:
            e = np.maximum(e, math.log(np.float32(energy_floor)))
        ceps[:, 0] = e
    elif htk_compat:
        ceps[:, 0] *= math.sqrt(2.0)
    if htk_compat:
        ceps = np.concatenate([ceps[:, 1:], ceps[:, :1]], axis=1)
    return ceps, mel


def bf16_bits(x):
    """float32 -> bfloat16 bit patterns (uint16), round to nearest even (finite inputs)"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
    return u.astype(np.uint16)


def splice_rows(feats, t_max, lctx, rctx, stride):
    """padded, strided splice of one utterance's frames [n_frames, n_feat] -> [t_max, D] float32 (zeros without frames)"""
    feats = np.asarray(feats, np.float32)
    nf, n_feat = feats.shape
    K = lctx + 1 + rctx
    if nf == 0:
        return np.zeros((t_max, n_feat * K), np.float32)
    n_out = (nf + stride - 1) // stride
    tt = np.minimum(np.arange(t_max), n_out - 1) * stride
    src = np.clip(tt[:, None] + np.arange(K)[None, :] - lctx, 0, nf - 1)
    return feats[src].reshape(t_max, n_feat * K)


def cmn_sums(x):
    """column sums of [t_max, D] float32 in the kernels' order: row order within each 64-row block, then block order"""
    tot = np.zeros(x.shape[1], np.float32)
    for t0 in range(0, x.shape[0], CMN_BLOCK):
        s = np.zeros(x.shape[1], np.float32)
        for t in range(t0, min(t0 + CMN_BLOCK, x.shape[0])):
            s += x[t]
        tot += s
    return tot


def splice_cmn_f32(feats_list, t_max, lctx=1, rctx=1, stride=1, cmn=True, offset=None, scale=None, specaug=(0, 0, 0, 0),
                   bf16=False):
    """splice -> stride -> last-row padding -> CMN over the padded rows -> (v + offset) * scale -> freq / time masks, in float32.
    -> [B, t_max, D] float32, or its bfloat16 bit patterns (uint16) when bf16"""
    f0, fs, t0, ts = specaug
    out = []
    for f in feats_list:
        x = splice_rows(f, t_max, lctx, rctx, stride)
        if cmn:
            mean = cmn_sums(x) / np.float32(t_max) if len(f) else np.zeros(x.shape[1], np.float32)
            x = x - mean[None, :]
        if offset is not None:
            x = (x + np.asarray(offset, np.float32)[None, :]) * np.asarray(scale, np.float32)[None, :]
        if fs > 0:
            x[:, f0:f0 + fs] = 0.0
        if ts > 0:
            x[t0:t0 + ts, :] = 0.0
        out.append(x.astype(np.float32))
    out = np.stack(out)
    return bf16_bits(out) if bf16 else out
