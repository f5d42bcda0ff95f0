"""Fused encoder self-attention at the bench shape (B=32, heads=16, head dim 64): forward, dQ and dK/dV timed separately.

    python scripts/attn_bench.py [--T 994] [--p 0,0.2] [--iters 20] [--dump DIR]

Each line is one JSON object: forward and backward milliseconds from CUDA events around engine.AttentionFn (allocations
included, as in the train step), then the per-kernel split of one more run of the same calls under torch.profiler.  The
achieved rate counts 9 T^2 * 64 multiply-adds per (batch, head) (2 forward, 3 dQ, 4 dK/dV).  --dump writes O, lse and
dQ|dK|dV of the seeded inputs to DIR (one .pt per p), so that two builds can be compared element by element."""
import argparse
import collections
import inspect
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from pika_b200 import engine as E  # noqa: E402
from pika_b200 import kernels as K  # noqa: E402


def inputs(B, T, heads):
    D = heads * 64
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = (torch.randn(B, T, 3 * D, generator=g, device="cuda") * 0.5).bfloat16()
    dy = torch.randn(B, T, D, generator=g, device="cuda").bfloat16()
    return qkv, dy


def outputs(qkv, dy, heads, p, seed):
    """O, lse and dQ|dK|dV through kernels.attention_fwd / _bwd (whichever keep-bits interface this build has)"""
    B, T, D3 = qkv.shape
    out = torch.empty(B, T, D3 // 3, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(B * heads * K.attention_lse_stride(T), device="cuda")
    alpha = 0.125
    dqkv = torch.empty_like(qkv)
    if "keep_bits" in inspect.signature(K.attention_bwd).parameters:
        bits = K.attention_keep_bits(B, T, heads, p, qkv.device)
        K.attention_fwd(qkv, out, lse, heads, alpha, p, seed, keep_bits=bits)
        K.attention_bwd(qkv, out, dy, lse, dqkv, heads, alpha, p, seed, keep_bits=bits)
    else:
        K.attention_fwd(qkv, out, lse, heads, alpha, p, seed)
        K.attention_bwd(qkv, out, dy, lse, dqkv, heads, alpha, p, seed)
    torch.cuda.synchronize()
    return dict(out=out, lse=lse, dqkv=dqkv)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--T", type=int, default=994)
    ap.add_argument("--heads", type=int, default=16)
    ap.add_argument("--p", default="0,0.2")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--tag", default="")
    ap.add_argument("--dump", default=None)
    a = ap.parse_args()
    E.set_precision("bf16")
    B, T, heads = a.B, a.T, a.heads
    qkv0, dy = inputs(B, T, heads)
    tflop = 9 * 2 * B * heads * T * T * 64 / 1e12
    seed = 99
    for p in (float(x) for x in a.p.split(",")):
        qkv = qkv0.clone().requires_grad_(True)

        def fwd():
            return E.AttentionFn.apply(qkv, heads, p, seed)

        for _ in range(3):
            fwd().backward(dy)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3 * a.iters)]
        for i in range(a.iters):
            ev[3 * i].record()
            out = fwd()
            ev[3 * i + 1].record()
            out.backward(dy)
            ev[3 * i + 2].record()
        torch.cuda.synchronize()
        f = sorted(ev[3 * i].elapsed_time(ev[3 * i + 1]) for i in range(a.iters))
        b = sorted(ev[3 * i + 1].elapsed_time(ev[3 * i + 2]) for i in range(a.iters))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fwd().backward(dy)
            torch.cuda.synchronize()
        kern = collections.defaultdict(float)
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "attention" in e.name:
                name = re.sub(r"\(.*", "", e.name).replace("void ", "").replace("pk::", "")
                kern[name] += e.device_time_total / 5 / 1000.0
        fm, bm = f[len(f) // 2], b[len(b) // 2]
        print(json.dumps(dict(tag=a.tag, B=B, T=T, heads=heads, p=p, fwd_ms=round(fm, 4), bwd_ms=round(bm, 4),
                              total_ms=round(fm + bm, 4), tflops=round(tflop / (fm + bm) * 1e3, 1),
                              kernels_ms={k: round(v, 4) for k, v in sorted(kern.items())})), flush=True)
        if a.dump:
            os.makedirs(a.dump, exist_ok=True)
            torch.save({k: v.cpu() for k, v in outputs(qkv0, dy, heads, p, seed).items()},
                       os.path.join(a.dump, "attn_T%d_p%g.pt" % (T, p)))


if __name__ == "__main__":
    main()
