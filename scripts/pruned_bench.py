"""Train step with the dense joint against the pruned RNN-T loss (--prune_range R), at the bench's config-2 shape.

    python scripts/pruned_bench.py [--steps 10] [--ranges 4,5,8] [--big-batch 96] [--smooth 0.25,0.0 [--smooth-range 5]]

Runs bench.py's training step (B = 32, T = 1000 fbank frames -> T' = 240, U = 150, V = 6000, bf16, SpecAugment on) with the dense
joint and with the pruned loss at every R, alternating the arms for --rounds rounds in one process.  Prints one JSON line per arm:
ms per step (CUDA events around --steps steps after warm-up), the in-step durations of the fc2 forward, the loss, the simple loss and
the bounds (engine._Tap events), and torch.cuda.max_memory_allocated; then the card's name and power limit.  --big-batch adds one
batch size (default 96) run pruned only, with the dense arm tried first to show whether it fits.  --smooth LM,AM adds one more arm
to every round: R = --smooth-range with the simple loss smoothed by --lm_only_scale LM and --am_only_scale AM.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (train_args, model_args, synth_pcm: the bench's own workload)
from pika_b200 import engine  # noqa: E402
from pika_b200.frontend import FbankOptions, Frontend  # noqa: E402
from pika_b200.model.transducer import Net  # noqa: E402
from pika_b200.trainer.bmuf import BmufTrainer  # noqa: E402
from pika_b200.trainer.flat import FlatParams, SgdNesterovClip  # noqa: E402
from pika_b200.trainer.step import TrainStep  # noqa: E402
from pika_b200.utils.spec_augment import SpecAugment  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:          # noqa: BLE001
        out = "nvidia-smi unavailable: %s" % e
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": out}


class Arm:
    def __init__(self, B, T, U, V, prune_range, dev, smooth=(0.0, 0.0)):
        ta = bench.train_args()
        ta.prune_range, ta.simple_loss_scale, ta.prune_warmup_batches = prune_range, 0.5, 0
        ta.lm_only_scale, ta.am_only_scale = smooth
        torch.manual_seed(777)
        margs = bench.model_args(V)
        margs.prune_range = prune_range
        self.model = Net(margs, 240, V).to(dev).train()
        flat = FlatParams(self.model)
        bmuf = BmufTrainer(0, 0, 1, self.model, ta.block_momentum, ta.block_lr, flat=flat)
        opt = SgdNesterovClip(flat, ta.initial_lr, ta.momentum, ta.grad_clip)
        fe = Frontend(FbankOptions(num_mel_bins=80, low_freq=40.0, high_freq=-200.0, dither=0.0, window_type="hamming"), 1, 1, dev)
        self.step = TrainStep(self.model, ta, fe, bmuf, opt, offset=torch.zeros(fe.D, device=dev), scale=torch.ones(fe.D, device=dev),
                              spec_augmentor=SpecAugment(ta.max_freq_span, ta.max_time_span))
        pcm = torch.from_numpy(bench.synth_pcm(B, T, 777)).to(dev)
        rng = np.random.default_rng(777)
        n = pcm.shape[1]
        new_len, frames = Frontend.lengths([n] * B, [1.0] * B)
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)          # noqa: E731
        self.batch = dict(pcm=pcm, target=torch.from_numpy(rng.integers(1, V, (B, U))).to(dev), n_samples=i32([n] * B),
                          new_len=i32(new_len), n_frames=i32(frames), ali_lens=i32([U] * B),
                          rate=torch.ones(B, device=dev), target_db=torch.full((B,), -25.0, device=dev), t_max=max(frames))

    def run(self, steps):
        for _ in range(2):
            self.step(self.batch)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(steps):
            self.step(self.batch)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e) / steps
        engine.EVENT_TAPS = {}
        for _ in range(3):
            self.step(self.batch)
        torch.cuda.synchronize()
        taps = {k: round(sum(a.elapsed_time(b) for a, b in v) / len(v), 3) for k, v in engine.EVENT_TAPS.items() if v}
        engine.EVENT_TAPS = None
        return ms, taps


def measure(B, R, steps, args, dev, smooth=(0.0, 0.0)):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    tag = dict(batch=B, prune_range=R, **(dict(lm_only_scale=smooth[0], am_only_scale=smooth[1]) if any(smooth) else {}))
    try:
        arm = Arm(B, args.T, args.U, args.V, R, dev, smooth)
        ms, taps = arm.run(steps)
        res = dict(tag, ms_per_step=round(ms, 3), taps_ms=taps, max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))
        del arm
    except torch.cuda.OutOfMemoryError as e:
        res = dict(tag, error="out of memory: %s" % str(e).split("\n")[0][:160])
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--ranges", default="4,5,8")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--big-batch", type=int, default=96)
    ap.add_argument("--T", type=int, default=1000)
    ap.add_argument("--U", type=int, default=150)
    ap.add_argument("--V", type=int, default=6000)
    ap.add_argument("--smooth", default="", help="LM,AM: add an arm with the simple loss smoothed by these scales")
    ap.add_argument("--smooth-range", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pruned_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    engine.set_precision("bf16")
    engine.set_seed(777)
    arms = [(0, (0.0, 0.0))] + [(int(r), (0.0, 0.0)) for r in args.ranges.split(",")]
    if args.smooth:
        arms.append((args.smooth_range, tuple(float(v) for v in args.smooth.split(","))))
    t0 = time.time()
    for rnd in range(args.rounds):
        for R, smooth in arms:
            print(json.dumps(dict(round=rnd, **measure(args.batch, R, args.steps, args, dev, smooth))), flush=True)
    if args.big_batch:
        for R in (0, 5):
            print(json.dumps(dict(round="big", **measure(args.big_batch, R, max(args.steps // 2, 3), args, dev))), flush=True)
    print(json.dumps(dict(card=card(), wall_s=round(time.time() - t0, 1))), flush=True)


if __name__ == "__main__":
    main()
