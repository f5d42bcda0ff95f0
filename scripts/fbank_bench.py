#!/usr/bin/env python
"""The GPU front end alone (augmentation + fbank + splice, dither = 0, no CMN) at B = 32 ten-second utterances, timed with CUDA
events after warm-up, at three fbank geometries:

    16k   16 kHz, egs/fbank.conf (hamming, 80 bins, 40 Hz .. Nyquist - 200 Hz): 400 / 160-sample frames, 512-point FFT
    8k    8 kHz, same options: 200 / 80-sample frames, 256-point FFT
    48k   48 kHz, same options: 1200 / 480-sample frames, 2048-point FFT
    mfcc13  16 kHz Kaldi MFCC defaults (povey, 13 cepstra from 23 mel bins, log energy, lifter 22), 512-point FFT
    mfcc40  16 kHz mfcc_hires.conf (40 cepstra from 40 mel bins, 20 Hz .. Nyquist - 400 Hz, no energy), 512-point FFT

Each run prints one JSON line per geometry (median and spread of the per-call times over --repeats windows of --iters calls) with the
card's name and power limit.  ``--dump DIR`` writes the 16k features to DIR/fbank_16k.npy, so that two builds can be compared bit
for bit.  Only the 16k geometry uses what every version of the front end has, so ``--configs 16k`` also runs on older trees.

    python scripts/fbank_bench.py [--configs 16k,8k,48k,mfcc13,mfcc40] [--iters 50] [--warmup 10] [--repeats 5] [--dump DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pika_b200.frontend import FbankOptions, Frontend  # noqa: E402

RATES = {"16k": 16000.0, "8k": 8000.0, "48k": 48000.0, "mfcc13": 16000.0, "mfcc40": 16000.0}
MFCC = {"mfcc13": dict(dither=0.0),
        "mfcc40": dict(num_ceps=40, num_mel_bins=40, use_energy=False, low_freq=20.0, high_freq=-400.0, dither=0.0)}
B, SECONDS = 32, 10


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def batch(sr, dev):
    rng = np.random.default_rng(int(sr))
    n = int(SECONDS * sr)
    pcm = torch.from_numpy(np.clip(np.round(rng.normal(0, 3000, (B, n))), -32768, 32767).astype(np.int16)).to(dev)
    return pcm, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="16k,8k,48k,mfcc13,mfcc40")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--dump", metavar="DIR", default=None)
    ap.add_argument("--label", default="", help="free-form tag copied into the JSON lines")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "fbank_bench measures the GPU front end"
    dev = torch.device("cuda", 0)
    name, pl = card()
    for key in a.configs.split(","):
        sr = RATES[key]
        if key in MFCC:
            from pika_b200.frontend import MfccOptions
            opts = MfccOptions(**MFCC[key])
        else:
            kw = dict(num_mel_bins=80, low_freq=40.0, high_freq=-200.0, dither=0.0, window_type="hamming")
            if sr != 16000.0:
                kw["sample_frequency"] = sr
            opts = FbankOptions(**kw)
        fe = Frontend(opts, 1, 1, dev)
        pcm, n = batch(sr, dev)
        frame_len, shift = int(sr * 0.025), int(sr * 0.010)
        new_len, frames = Frontend.lengths([n] * B, [1.0] * B, *(() if sr == 16000.0 else (frame_len, shift)))
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)          # noqa: E731
        args = (pcm, i32([n] * B), torch.ones(B, device=dev), torch.full((B,), -25.0, device=dev), i32(new_len), i32(frames),
                max(frames))
        call = lambda: fe(*args, out_dtype=torch.float32, cmn=False)              # noqa: E731
        for _ in range(a.warmup):
            out = call()
        torch.cuda.synchronize()
        per_call = []
        for _ in range(a.repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            per_call.append(e0.elapsed_time(e1) / a.iters)
        if a.dump and key == "16k":
            os.makedirs(a.dump, exist_ok=True)
            np.save(os.path.join(a.dump, "fbank_16k.npy"), out.cpu().numpy())
        print(json.dumps(dict(label=a.label, config=key, B=B, seconds=SECONDS, frames=int(max(frames)), n_fft=fe.mel_w.shape[1] * 2,
                              D=int(out.shape[2]),
                              ms_median=round(float(np.median(per_call)), 4), ms_min=round(min(per_call), 4),
                              ms_max=round(max(per_call), 4), card=name, power_limit=pl)), flush=True)


if __name__ == "__main__":
    main()
