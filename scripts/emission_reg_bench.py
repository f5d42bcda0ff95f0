"""Train step with FastEmit and the delay penalty off and on, at the bench's config-2 shape.

    python scripts/emission_reg_bench.py [--steps 10] [--rounds 3] [--fastemit 0.01] [--delay 0.0015]

Runs bench.py's training step (B = 32, T = 1000 fbank frames -> T' = 240, U = 150, V = 6000, bf16, SpecAugment on) with the dense
joint and with --prune_range 5, each with the options off and on (--fastemit_lambda / --delay_penalty), alternating the four arms for
--rounds rounds in one process.  Prints one JSON line per arm: ms per step (CUDA events around --steps steps after warm-up) and the
in-step durations of the loss, the simple loss and the bounds (engine._Tap events).  Then the lattice kernel alone on the step's
tables (B = 32, T' = 240, U1 = 151), plain against regularised, 200 launches each, alternating; then the card's name and power limit.
Needs a GPU.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from pruned_bench import Arm, card  # noqa: E402  (the config-2 train step and the card query)
from pika_b200 import engine, kernels as K  # noqa: E402


def measure(args, dev, R, reg):
    torch.cuda.empty_cache()
    arm = Arm(args.batch, args.T, args.U, args.V, R, dev)
    arm.step.args.fastemit_lambda, arm.step.args.delay_penalty = reg
    ms, taps = arm.run(args.steps)
    del arm
    torch.cuda.empty_cache()
    return dict(prune_range=R, fastemit_lambda=reg[0], delay_penalty=reg[1], ms_per_step=round(ms, 3), taps_ms=taps)


def lattice_times(args, dev, reg, n=200):
    """the lattice kernel alone at the step's shape: mean ms per launch, plain (0, 0) and regularised, alternating in blocks of n"""
    B, T, U1 = args.batch, 240, args.U + 1
    g = torch.Generator(device=dev).manual_seed(0)
    lpb = -torch.rand(B, T + U1 - 1, U1, device=dev, generator=g) * 3
    lpl = -torch.rand(B, T + U1 - 1, U1, device=dev, generator=g) * 3
    fl = torch.full((B,), T, dtype=torch.int32, device=dev)
    ll = torch.full((B,), U1 - 1, dtype=torch.int32, device=dev)
    out = {"off": [], "on": []}
    for _ in range(3):
        for name, r in (("off", (0.0, 0.0)), ("on", reg)):
            for _ in range(5):
                K.rnnt_lattice(lpb, lpl, fl, ll, B, T, U1, fastemit_lambda=r[0], delay_penalty=r[1])
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(n):
                K.rnnt_lattice(lpb, lpl, fl, ll, B, T, U1, fastemit_lambda=r[0], delay_penalty=r[1])
            e.record()
            torch.cuda.synchronize()
            out[name].append(round(s.elapsed_time(e) / n, 4))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--T", type=int, default=1000)
    ap.add_argument("--U", type=int, default=150)
    ap.add_argument("--V", type=int, default=6000)
    ap.add_argument("--range", type=int, default=5, help="the pruned arms' --prune_range")
    ap.add_argument("--fastemit", type=float, default=0.01)
    ap.add_argument("--delay", type=float, default=0.0015)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("emission_reg_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    engine.set_precision("bf16")
    engine.set_seed(777)
    reg = (args.fastemit, args.delay)
    t0 = time.time()
    for rnd in range(args.rounds):
        for R in (0, args.range):
            for r in ((0.0, 0.0), reg):
                print(json.dumps(dict(round=rnd, **measure(args, dev, R, r))), flush=True)
    print(json.dumps(dict(lattice_ms=lattice_times(args, dev, reg))), flush=True)
    print(json.dumps(dict(card=card(), wall_s=round(time.time() - t0, 1))), flush=True)


if __name__ == "__main__":
    main()
