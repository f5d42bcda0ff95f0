#!/usr/bin/env python
"""Generate tests/golden/fbank_opts.npz: Kaldi fbank features of a few seeded int16 signals for each fbank configuration of the
grid below, computed by ``torchaudio.compliance.kaldi.fbank`` (independent of this project's code) with dither = 0.

Keys: ``configs`` (JSON list of the FbankOptions keyword arguments of each configuration, Kaldi's defaults where absent),
``pcm_<c>_<k>`` int16 signal k of configuration c, ``fbank_<c>_<k>`` float32 [T, num_mel_bins].

    python tests/golden/make_golden_fbank_opts.py
"""
import json
import os

import numpy as np
import torch
import torchaudio.compliance.kaldi as tk

HERE = os.path.dirname(os.path.abspath(__file__))

CONFIGS = [
    dict(sample_frequency=8000.0, window_type="povey", num_mel_bins=40),
    dict(sample_frequency=8000.0, window_type="hamming", num_mel_bins=40, snip_edges=False),
    dict(),                                                                  # Kaldi's defaults: 16 kHz, povey, 23 bins, 20 Hz..Nyquist
    dict(frame_length=50.0, frame_shift=12.5, window_type="hanning"),
    dict(sample_frequency=22050.0, window_type="blackman"),
    dict(sample_frequency=44100.0, window_type="rectangular", snip_edges=False),
    dict(sample_frequency=48000.0, window_type="hamming", remove_dc_offset=False),
]
DURATIONS = (0.2, 0.35, 0.6)                                                # seconds, every one above a frame


def signal(rng, n, sr):
    """a few tones under noise, scaled like int16 speech"""
    t = np.arange(n) / sr
    x = rng.normal(0.0, 600.0, n)
    for f in rng.uniform(80.0, 0.45 * sr, 4):
        x += rng.uniform(500.0, 3000.0) * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi))
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


def main():
    rng = np.random.default_rng(20261017)
    out = {"configs": np.array(json.dumps(CONFIGS))}
    for c, cfg in enumerate(CONFIGS):
        kw = dict(cfg, dither=0.0)
        sr = kw.get("sample_frequency", 16000.0)
        for k, d in enumerate(DURATIONS):
            pcm = signal(rng, int(d * sr), sr)
            f = tk.fbank(torch.from_numpy(pcm.astype(np.float32))[None], **kw).numpy().astype(np.float32)
            assert np.isfinite(f).all()
            out["pcm_%d_%d" % (c, k)] = pcm
            out["fbank_%d_%d" % (c, k)] = f
    path = os.path.join(HERE, "fbank_opts.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
