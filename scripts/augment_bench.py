#!/usr/bin/env python
"""Front end with and without on-the-fly noise + reverberation, timed with CUDA events after warm-up.

Shapes: B = 32 utterances of 10 s (the config-2 shape, T = 1000) and of 16 s (the recipe's --max_len 1600), RIRs of 0.25 s,
1 s and 4 s.  Also times pk_conv_same_f64 alone, with the bytes and FLOPs of its three stages computed from the shapes.
Prints the card name and its power limit, which belong beside every number.

    python scripts/augment_bench.py [--iters 20] [--warmup 5]
"""
import argparse
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pika_b200 import kernels as K  # noqa: E402
from pika_b200.frontend import FbankOptions, Frontend  # noqa: E402
from pika_b200.loader.audio_bank import AudioBank  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters + 1)]
    ev[0].record()
    for i in range(iters):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    t = [ev[i].elapsed_time(ev[i + 1]) for i in range(iters)]
    return float(np.median(t))


def conv_cost(B, N, M):
    """(bytes, flops) of the overlap-save convolution, block length as in frontend.cu (conv_block_len)"""
    lb = 1024
    while lb < 4096 and 4 * lb < M:
        lb *= 2
    n = 2 * lb
    P, J = math.ceil(M / lb), math.ceil(N / lb)
    fft = 5.0 * n * math.log2(n)
    flops = B * ((P + J + P - 1) * fft + J * fft + J * P * (lb + 1) * 8)
    spec = (lb + 1) * 16
    bytes_ = B * ((P + J + P - 1) * spec + J * P * 2 * spec + (J + P) * n * 8 + N * 8 + M * 8)
    return lb, bytes_, flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    name, pl = card()
    print("card: %s, power limit: %s" % (name, pl))
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0)
    fe = Frontend(FbankOptions(num_mel_bins=80, low_freq=40.0, high_freq=-200.0, dither=1.0, window_type="hamming"), 1, 1, dev)
    B = 32
    for secs in (10, 16):
        N = secs * 16000 + 240
        pcm = torch.from_numpy(rng.integers(-3000, 3000, (B, N)).astype(np.int16)).to(dev)
        rate = [(0.9, 1.0, 1.1)[i % 3] for i in range(B)]
        new_len, frames = Frontend.lengths([N] * B, rate)
        n_max = max(new_len)
        x = torch.zeros(B, n_max, dtype=torch.int16, device=dev)
        x[:, :N] = pcm
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)  # noqa: E731
        f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)  # noqa: E731
        args = (x, i32([N] * B), f32(rate), f32([-25.0] * B), i32(new_len), i32(frames), max(frames))
        base = timed(lambda: fe(*args, out_dtype=torch.bfloat16), a.iters, a.warmup)
        noise = AudioBank(["n"], [rng.integers(-2000, 2000, n_max + 16000).astype(np.int16)], with_rms=True)
        print("B=%d x %d s: front end alone %.3f ms" % (B, secs, base))
        for rir_s in (0.25, 1.0, 4.0):
            M = int(rir_s * 16000)
            h = (rng.standard_normal(M) * np.exp(-np.arange(M) / (M / 6.9)) * 8000).astype(np.int16)
            rir = AudioBank(["h"], [h])
            kw = dict(noise=noise, noise_idx=[0] * B, noise_off=[int(v) for v in rng.integers(0, 16000, B)], snr=[10.0] * B,
                      rir=rir, rir_idx=[0] * B, rir_max_len=M)
            t = timed(lambda: fe(*args, out_dtype=torch.bfloat16, **kw), a.iters, a.warmup)
            kwn = dict(noise=noise, noise_idx=kw["noise_idx"], noise_off=kw["noise_off"], snr=kw["snr"])
            tn = timed(lambda: fe(*args, out_dtype=torch.bfloat16, **kwn), a.iters, a.warmup)
            xs = torch.randn(B, n_max, dtype=torch.float64, device=dev)
            hs = torch.from_numpy(np.tile(h.astype(np.float64) / 32768.0, (B, 1))).to(dev)
            y = torch.empty_like(xs)
            nl, ml = i32(new_len), i32([M] * B)
            tc = timed(lambda: K.conv_same_f64(xs, nl, hs, ml, y), a.iters, a.warmup)
            lb, by, fl = conv_cost(B, int(np.mean(new_len)), M)
            print("  RIR %.2f s: + noise %.3f ms | + noise + RIR %.3f ms (+%.3f over the front end) | conv alone %.3f ms "
                  "(Lb %d, %.2f GB, %.1f GB/s, %.1f GFLOP, %.0f GFLOP/s)" % (rir_s, tn - base, t, t - base, tc, lb, by / 1e9,
                                                                           by / tc / 1e6, fl / 1e9, fl / tc / 1e6))


if __name__ == "__main__":
    main()
