#!/usr/bin/env python
"""Generate tests/golden/frontend_noise_rir.npz by EXECUTING THE REFERENCE's own AudioSegment (loader/audio.py:
change_speed, normalize, add_noise, convolve_and_normalize, _convert_samples_from_float32), imported from /root/reference
through tests/golden/ref_shim.py, with torchaudio's Kaldi fbank as the PyKaldi stand-in (as make_golden.py:golden_frontend).

The reference draws the noise start time from ``rng.uniform``; the generator passes an ``rng`` whose ``uniform`` returns
``off / 16000`` and checks that the slice the reference superimposed is exactly samples [off, off + new_len) of the noise.

Run in the build container only:   python tests/golden/make_golden_noise_rir.py
The GPU box never runs this script.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

ref_shim.install()

# (key, rate, target_db, snr or None, offset "0" | "max" | None, rir name or None)
CASES = [
    ("r09_n", 0.9, -23.5, -5.0, "0", None),
    ("r10_n", 1.0, -41.0, 7.3, "max", None),
    ("r11_n", 1.1, -12.25, 20.0, "0", None),
    ("r09_h777", 0.9, -30.0, None, None, "h777"),
    ("r10_h16000", 1.0, -25.0, None, None, "h16000"),
    ("r11_h1", 1.1, -20.0, None, None, "h1"),
    ("r10_hlong", 1.0, -35.0, None, None, "hlong"),
    ("r09_nh16000", 0.9, -28.0, 7.3, "max", "h16000"),
    ("r10_nh777", 1.0, -22.0, -5.0, "0", "h777"),
    ("r11_nhlong", 1.1, -33.0, 20.0, "max", "hlong"),
    ("r09_nh1", 0.9, -18.0, 20.0, "0", "h1"),
]


class FixedStart:
    """stands in for random.Random in AudioSegment.random_subsegment: the start time of sample ``off``"""

    def __init__(self, off):
        self.off = off

    def uniform(self, a, b):
        assert 0.0 <= self.off / 16000.0 <= b + 1e-12
        return self.off / 16000.0


def make_inputs():
    rng = np.random.default_rng(21)
    n = 400 + 124 * 160 + 37                       # 1.27 s
    t = np.arange(n) / 16000.0
    wav = 3000 * np.sin(2 * np.pi * 220 * t) + 1500 * np.sin(2 * np.pi * 1330 * t + 1.0) + 800 * rng.standard_normal(n)
    pcm = np.clip(np.round(wav), -32768, 32767).astype(np.int16)
    n_noise = 24000                                 # covers the 0.9x speed-perturbed utterance (22530 samples)
    white = rng.standard_normal(n_noise + 64)
    noise = np.convolve(white, np.ones(64) / 8.0, "valid")[:n_noise] * 2000 + 300 * rng.standard_normal(n_noise)
    noise = np.clip(np.round(noise), -32768, 32767).astype(np.int16)
    rirs = {}
    for name, m in (("h1", 1), ("h777", 777), ("h16000", 16000), ("hlong", 24001)):
        k = np.arange(m)
        h = rng.standard_normal(m) * np.exp(-k / (0.15 * 16000 / 6.9)) * 6000
        h[0] = 24000
        rirs[name] = np.clip(np.round(h), -32768, 32767).astype(np.int16)
    return pcm, noise, rirs


def main():
    import torchaudio
    from loader.audio import AudioSegment
    from loader.otf_utt_loader import splice
    pcm, noise, rirs = make_inputs()
    out = dict(pcm=pcm, noise=noise, cases=np.array([c[0] for c in CASES]))
    out.update({"rir_" + k: v for k, v in rirs.items()})
    orig_subsegment = AudioSegment.subsegment
    for key, rate, db, snr, off_kind, rir in CASES:
        seg = AudioSegment(pcm, 16000)
        seg.change_speed(rate)
        seg.normalize(db)
        new_len = seg.num_samples
        off = -1
        if snr is not None:
            off = 0 if off_kind == "0" else len(noise) - new_len
            picked = []

            def recording_subsegment(self, start_sec=None, end_sec=None):
                orig_subsegment(self, start_sec, end_sec)
                picked.append(self._samples.copy())
            AudioSegment.subsegment = recording_subsegment
            try:
                seg.add_noise(AudioSegment(noise, 16000), np.float64(snr), rng=FixedStart(off))
            finally:
                AudioSegment.subsegment = orig_subsegment
            want = noise[off:off + new_len].astype(np.float32) * np.float32(1.0 / 2 ** 15)
            # the samples random_subsegment kept, before the noise gain is applied in place
            assert len(picked) == 1 and np.array_equal(picked[0], want), key
        if rir is not None:
            seg.convolve_and_normalize(AudioSegment(rirs[rir], 16000))
        aug = seg._convert_samples_from_float32(seg._samples, "int16")
        out["aug_" + key] = aug
        out["meta_" + key] = np.array([rate, db, np.nan if snr is None else snr, off])
        out["rirname_" + key] = np.array("" if rir is None else rir)
        fb = torchaudio.compliance.kaldi.fbank(torch.from_numpy(aug.astype(np.float32)).unsqueeze(0), num_mel_bins=80,
                                               sample_frequency=16000.0, dither=0.0, low_freq=40.0, high_freq=-200.0,
                                               window_type="hamming", energy_floor=0.0)
        out["fbank_" + key] = fb.numpy()
        out["splice_" + key] = splice(fb.numpy(), 1, 1)[::5]
        print(key, "new_len", new_len, "off", off, "rms", float(np.sqrt(np.mean((aug.astype(np.float64) / 32768) ** 2))))
    np.savez_compressed(os.path.join(HERE, "frontend_noise_rir.npz"), **out)


if __name__ == "__main__":
    main()
