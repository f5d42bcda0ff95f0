"""Chunk-limited encoder attention (DESIGN.md "Chunked attention"): the fused attention and a whole train step, masked against full
context.

    python scripts/chunk_attn_bench.py [--iters 20] [--rounds 3] [--steps 10] [--step-chunk 16]

1. The fused attention forward + backward (engine.AttentionFn, allocations included as in the train step) at the encoder's shape
   (B = 32, T = 994, 16 heads, head dim 64, dropout 0.2 with keep bits) under layer 0's chunk mask (chunk_len 4C, offset 6) for
   C in {4, 16, 64} x left_chunks in {-1, 2}, each arm alternated with C = 0 (full context) for --rounds rounds in one process.  One
   JSON line per arm and round: ms per forward + backward from CUDA events over --iters calls, and the share of the 64 x 64 key tiles
   the masked kernels stream.
2. bench.py's config-2 train step (B = 32, T = 1000 fbank frames -> T' = 240, U = 150, V = 6000, bf16) with --chunk_size
   --step-chunk against full context, alternating; ms per step over --steps steps.
Then the card's name and power limit.  Needs a GPU.
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
from pika_b200 import engine  # noqa: E402


def tile_share(T, chunk):
    """share of the (128-row block, 64-key tile) pairs the forward streams: each block streams the tiles from its first row's lowest key
    to its last row's highest key"""
    if chunk is None:
        return 1.0
    L, off, left = chunk
    n_tiles, visited = (T + 63) // 64, 0
    for r0 in range(0, T, 128):
        r1 = min(r0 + 128, T) - 1
        lo = 0 if left < 0 else max(0, ((r0 + off) // L - left) * L - off)
        hi = min(T, ((r1 + off) // L + 1) * L - off)
        visited += (hi + 63) // 64 - lo // 64
    return visited / (n_tiles * ((T + 127) // 128))


def attention_ms(qkv, dy, heads, chunk, iters, p=0.2):
    def once():
        qkv.grad = None
        out = engine.AttentionFn.apply(qkv, heads, p, 1234, False, None, None, chunk)
        out.backward(dy)

    for _ in range(3):
        once()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        once()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--step-chunk", type=int, default=16)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("chunk_attn_bench.py needs a GPU")
    dev = torch.device("cuda", 0)
    engine.set_precision("bf16")
    engine.set_seed(777)
    t0 = time.time()
    B, T, heads = 32, 994, 16
    g = torch.Generator(device=dev).manual_seed(1)
    qkv = (torch.randn(B, T, 3 * heads * 64, generator=g, device=dev) * 0.5).bfloat16().requires_grad_()
    dy = torch.randn(B, T, heads * 64, generator=g, device=dev).bfloat16()
    for rnd in range(args.rounds):
        for C in (4, 16, 64):
            for left in (-1, 2):
                chunk = (4 * C, 6, left)
                full = attention_ms(qkv, dy, heads, None, args.iters)
                masked = attention_ms(qkv, dy, heads, chunk, args.iters)
                print(json.dumps(dict(round=rnd, C=C, left_chunks=left, chunk=chunk, ms_full=round(full, 3), ms_masked=round(masked, 3),
                                      tile_share=round(tile_share(T, chunk), 3))), flush=True)
    del qkv, dy
    torch.cuda.empty_cache()
    if not args.skip_step:
        for rnd in range(args.rounds):
            for C in (0, args.step_chunk):
                arm = Arm(32, 1000, 150, 6000, 0, dev)
                arm.model.encoder.chunk_size = C
                ms, _ = arm.run(args.steps)
                del arm
                torch.cuda.empty_cache()
                print(json.dumps(dict(round=rnd, step_chunk_size=C, ms_per_step=round(ms, 3))), flush=True)
    print(json.dumps(dict(card=card(), wall_s=round(time.time() - t0, 1))), flush=True)


if __name__ == "__main__":
    main()
