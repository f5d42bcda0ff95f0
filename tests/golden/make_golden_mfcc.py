#!/usr/bin/env python
"""Generate tests/golden/mfcc.npz: Kaldi MFCC features of a few seeded int16 signals for each MFCC configuration of the grid below,
computed by ``torchaudio.compliance.kaldi.mfcc`` (independent of this project's code) with dither = 0.

torchaudio's MFCC defaults are not Kaldi's (use_energy=False, energy_floor=1.0, dither=0.0 there; Kaldi's MfccOptions has
use-energy=true, energy-floor=0, dither=1).  Every argument is therefore passed explicitly: each configuration's MfccOptions
keyword arguments over Kaldi's defaults, with dither 0.

The signals are tones under noise with exact-zero stretches, several frames long: a frame inside one has zero energy, so both the
log(FLT_EPSILON) floor of the energy and of the mel energies, and --energy-floor where it is set, are hit.

Keys: ``configs`` (JSON list of the MfccOptions keyword arguments of each configuration, Kaldi's defaults where absent),
``pcm_<c>_<k>`` int16 signal k of configuration c, ``mfcc_<c>_<k>`` float32 [T, num_ceps].

    python tests/golden/make_golden_mfcc.py
"""
import json
import os

import numpy as np
import torch
import torchaudio.compliance.kaldi as tk

HERE = os.path.dirname(os.path.abspath(__file__))

CONFIGS = [
    dict(sample_frequency=8000.0, window_type="povey"),                                        # 13 / 23, Kaldi's defaults at 8 kHz
    dict(sample_frequency=8000.0, window_type="hamming", snip_edges=False, num_ceps=20, num_mel_bins=80, use_energy=False,
         htk_compat=True),
    dict(),                                                                                    # Kaldi's defaults: 16 kHz, povey, 13 / 23
    dict(num_ceps=40, num_mel_bins=40, use_energy=False, low_freq=20.0, high_freq=-400.0),     # mfcc_hires.conf
    dict(frame_length=50.0, frame_shift=12.5, window_type="hanning", raw_energy=False, energy_floor=1.0, htk_compat=True),
    dict(sample_frequency=22050.0, window_type="blackman", energy_floor=1.0, cepstral_lifter=0.0),
    dict(sample_frequency=44100.0, window_type="rectangular", snip_edges=False, num_ceps=40, num_mel_bins=40, raw_energy=False,
         cepstral_lifter=0.0, htk_compat=True),
    dict(sample_frequency=48000.0, window_type="hamming", remove_dc_offset=False, num_ceps=20, num_mel_bins=80, energy_floor=2.0),
]
KALDI = dict(num_ceps=13, num_mel_bins=23, use_energy=True, energy_floor=0.0, raw_energy=True, cepstral_lifter=22.0, htk_compat=False,
             sample_frequency=16000.0, frame_length=25.0, frame_shift=10.0, window_type="povey", snip_edges=True, remove_dc_offset=True,
             low_freq=20.0, high_freq=0.0, preemphasis_coefficient=0.97, blackman_coeff=0.42)
# (seconds, zero stretches as (start, end) in seconds)
SIGNALS = ((0.2, ()), (0.35, ((0.0, 0.08),)), (0.6, ((0.2, 0.32), (0.5, 0.6))))


def signal(rng, n, sr, zeros):
    """a few tones under noise, scaled like int16 speech, with exact-zero stretches"""
    t = np.arange(n) / sr
    x = rng.normal(0.0, 600.0, n)
    for f in rng.uniform(80.0, 0.45 * sr, 4):
        x += rng.uniform(500.0, 3000.0) * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi))
    for a, b in zeros:
        x[int(a * sr):int(b * sr)] = 0.0
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


def main():
    rng = np.random.default_rng(20261018)
    out = {"configs": np.array(json.dumps(CONFIGS))}
    for c, cfg in enumerate(CONFIGS):
        kw = dict(KALDI, **cfg)
        sr = kw["sample_frequency"]
        for k, (d, zeros) in enumerate(SIGNALS):
            pcm = signal(rng, int(d * sr), sr, zeros)
            f = tk.mfcc(torch.from_numpy(pcm.astype(np.float32))[None], dither=0.0, **kw).numpy().astype(np.float32)
            assert np.isfinite(f).all() and f.shape[1] == kw["num_ceps"]
            out["pcm_%d_%d" % (c, k)] = pcm
            out["mfcc_%d_%d" % (c, k)] = f
    path = os.path.join(HERE, "mfcc.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
