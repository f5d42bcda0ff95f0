#!/usr/bin/env python
"""pk_adam_clip and pk_bmuf_adam_update on the config-2 flat parameter buffer (91.4 M floats), timed with CUDA events after
warm-up, with the achieved bandwidth against the H100 SXM's 3.35 TB/s of HBM3.

Bytes per element, from what each kernel must read and write:
  * Adam step (clip on): read p, g, m, v; write p, m, v = 7 x 4 B (the absmax pass over g is timed separately);
  * Adam step with the second output (BlockAdamTrainer): + 1 write = 8 x 4 B;
  * BMUF-Adam sync update: read glob, dprev, m_g, v_g and the summed delta, m, v; write glob, local, dprev, m_g, v_g and the
    local m, v = 14 x 4 B.
Prints the card name and its power limit, which belong beside every number.

    python scripts/optim_bench.py [--n 91400000] [--iters 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pika_b200 import kernels as K  # noqa: E402

HBM_PEAK = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def timed(fn, iters, warmup):
    """median ms per call over ``iters`` individually event-timed calls"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in ev)
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=91_400_000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "optim_bench measures on the GPU"
    n = a.n
    gen = torch.Generator(device="cuda").manual_seed(0)
    p, g = torch.randn(n, device="cuda", generator=gen), 0.1 * torch.randn(n, device="cuda", generator=gen)
    m, v, out2 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.empty(n, device="cuda")
    am, flag = torch.zeros(1, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    K.absmax(g, am, flag)
    glob = p.clone()
    dprev, m_g, v_g = (torch.zeros(n, device="cuda") for _ in range(3))
    msg = 0.01 * torch.randn(3 * n, device="cuda", generator=gen).abs()

    def bmuf_adam():
        K.bmuf_adam_update(glob, p, dprev, m_g, v_g, msg, 8, 0.9, 1.0, 0.9 ** 8, 0.9 ** 7.2, 0.999 ** 8, 0.999 ** 7.2)

    rows = [("absmax (clip norm)", 1, lambda: K.absmax(g, am, flag)),
            ("adam_clip", 7, lambda: K.adam_clip(p, g, m, v, 1e-4, (0.9, 0.999), 1e-8, 10.0, 3.0, am, flag)),
            ("adam_clip + second output", 8, lambda: K.adam_clip(p, g, m, v, 1e-4, (0.9, 0.999), 1e-8, 10.0, -1.0, p_out2=out2)),
            ("bmuf_adam_update", 14, bmuf_adam)]
    name, pl = card()
    print("%s, power limit %s, n = %d floats (%.1f MB per buffer)" % (name, pl, n, 4 * n / 1e6))
    res = {}
    for label, words, fn in rows:
        ms = timed(fn, a.iters, a.warmup)
        gbs = words * 4 * n / (ms * 1e-3) / 1e9
        floor = words * 4 * n / HBM_PEAK * 1e3
        print("%-28s %8.3f ms  %6.2f GB moved  %7.1f GB/s  = %4.1f%% of 3.35 TB/s (floor %.3f ms)" %
              (label, ms, words * 4 * n / 1e9, gbs, 100 * gbs * 1e9 / HBM_PEAK, floor))
        res[label] = dict(ms=ms, gb_per_s=gbs, bytes=words * 4 * n)
    print(json.dumps(dict(device=name, power_limit=pl, n=n, results=res)))


if __name__ == "__main__":
    main()
