"""Forced alignment (engine.transducer_align) at the bench's config-2 shape, dense and pruned.

    python scripts/align_bench.py [--calls 10] [--rounds 2] [--ranges 5]

B = 32 utterances of T = 1000 spliced feature frames (T' = 240 after the TDNN-Transformer encoder), U = 150 labels, V = 6000, bf16,
the bench's model in eval mode.  The dense arm and every --ranges arm alternate for --rounds rounds in one process.  Prints one JSON
line per arm: utterances per second (CUDA events around --calls calls after two warm-up calls), the in-call durations of the Viterbi
kernel and of the costs-only lattice (engine._Tap events), and torch.cuda.max_memory_allocated; then the card's name and power limit.
Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (model_args, tprime: the bench's own workload)
from pika_b200 import engine  # noqa: E402
from pika_b200.model.transducer import Net  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:          # noqa: BLE001
        out = "nvidia-smi unavailable: %s" % e
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": out}


def measure(model, x, y, fl, ll, R, calls):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    run = lambda: engine.transducer_align(model, x, y, fl, ll, prune_range=R)      # noqa: E731
    for _ in range(2):
        run()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(calls):
        frames, vit, loglik = run()
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / calls
    engine.EVENT_TAPS = {}
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    taps = {k: round(sum(a.elapsed_time(b) for a, b in v) / len(v), 4) for k, v in engine.EVENT_TAPS.items() if v}
    engine.EVENT_TAPS = None
    B = x.shape[0]
    return dict(prune_range=R, ms_per_call=round(ms, 3), utt_per_s=round(B * 1000.0 / ms, 1), taps_ms=taps,
                max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2),
                mean_viterbi=round(float(vit.mean()), 3), mean_loglik=round(float(loglik.mean()), 3),
                finite=int(torch.isfinite(vit).sum()))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--ranges", default="5")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--T", type=int, default=1000)
    ap.add_argument("--U", type=int, default=150)
    ap.add_argument("--V", type=int, default=6000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("align_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    engine.set_precision("bf16")
    B, T, U, V = args.batch, args.T, args.U, args.V
    torch.manual_seed(777)
    margs = bench.model_args(V)
    margs.prune_range = max(int(r) for r in args.ranges.split(","))
    model = Net(margs, 240, V).to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(777)
    x = torch.randn(B, T, 240, device=dev, generator=g)
    y = torch.randint(1, V, (B, U), device=dev, generator=g)
    fl = torch.full((B,), bench.tprime(T), dtype=torch.int32, device=dev)
    ll = torch.full((B,), U, dtype=torch.int32, device=dev)
    arms = [0] + [int(r) for r in args.ranges.split(",")]
    t0 = time.time()
    for rnd in range(args.rounds):
        for R in arms:
            print(json.dumps(dict(round=rnd, batch=B, T_prime=int(fl[0]), U=U, V=V, **measure(model, x, y, fl, ll, R, args.calls))),
                  flush=True)
    print(json.dumps(dict(card=card(), wall_s=round(time.time() - t0, 1))), flush=True)


if __name__ == "__main__":
    main()
