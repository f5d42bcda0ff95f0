"""GEMM lab: the step's dominant shapes timed stand-alone with CUDA events (inputs >> L2, 3 warm-ups), one line per shape.
The first line names the build (pk_version), so that runs of two builds can be told apart:

    python scripts/gemm_lab.py fc2        # the three joint GEMMs
    python scripts/gemm_lab.py all

Each result is also spot-checked against torch on a few rows so that a fast-but-wrong variant cannot slip through.
Exploration tool, not a bench."""
import hashlib
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pika_b200 import kernels as K

torch.cuda.set_device(0)


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*s, generator=g, device="cuda") * scale).to(torch.bfloat16)


def timeit(fn, it=5):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(it):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / it


def check_rows(c, a, b, a_mn, b_mn, bias=None, rows=(0, 1, 77, -1)):
    af = (a.float().t() if a_mn else a.float())
    idx = torch.tensor([r % c.shape[0] for r in rows], device="cuda")
    ref = af[idx] @ (b.float() if b_mn else b.float().t())
    if bias is not None:
        ref = ref + bias
    got = c[idx].float()
    return ((got - ref).norm() / ref.norm().clamp_min(1e-20)).item()


def run(name, M, N, Kd, a_mn, b_mn, cdt, lse=False, bias=False, **kw):
    a = rnd(Kd, M, seed=1, scale=0.3) if a_mn else rnd(M, Kd, seed=1, scale=0.3)
    b = rnd(Kd, N, seed=2, scale=0.05) if b_mn else rnd(N, Kd, seed=2, scale=0.05)
    c = torch.empty(M, N, device="cuda", dtype=cdt)
    bs = torch.zeros(N, device="cuda") if bias else None
    parts = torch.empty(K.row_lse_parts(M, N, 256), M, 2, device="cuda") if lse else None
    extra = dict(block_n=256) if lse else {}
    fn = lambda: K.gemm(a, b, c, a_mn=a_mn, b_mn=b_mn, bias=bs, row_lse=parts, **extra, **kw)
    ms = timeit(fn)
    err = check_rows(c, a, b, a_mn, b_mn, bs)
    tf = 2.0 * M * N * Kd / ms / 1e9
    # fingerprint of every 97th output row: equal across two builds = bit-identical samples
    c_sha = hashlib.sha1(c[::97].contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()[:12]
    extra_out = {}
    if lse:   # natural-log LSE of sampled rows from the merged per-tile partials, against torch on the same rounded output
        idx = torch.arange(0, M, 9973, device="cuda")
        m, s = parts[:, idx, 0].double(), parts[:, idx, 1].double()
        got = torch.logsumexp((m + torch.log2(s)) * math.log(2.0), dim=0)
        extra_out["lse_abs_err"] = float("%.2e" % (got - torch.logsumexp(c[idx].double(), dim=1)).abs().max().item())
    del c
    torch.cuda.empty_cache()
    # yardstick only: torch.matmul (cuBLAS) on the same bf16 operands with a plain bf16 output (no bias, no LSE, no split-K)
    am, bm = (a.t() if a_mn else a), (b if b_mn else b.t())
    ms_ref = timeit(lambda: torch.matmul(am, bm))
    print(json.dumps(dict(shape=name, M=M, N=N, K=Kd, a_mn=int(a_mn), b_mn=int(b_mn), ms=round(ms, 4), tflops=round(tf, 1),
                          rel_err=float("%.2e" % err), lse=lse, c_sha=c_sha, **extra_out, cublas_ms=round(ms_ref, 4),
                          cublas_tflops=round(2.0 * M * N * Kd / ms_ref / 1e9, 1))), flush=True)
    del a, b
    torch.cuda.empty_cache()


R = 32 * 240 * 151
which = sys.argv[1] if len(sys.argv) > 1 else "all"
print(json.dumps(dict(config=dict(pk_version=int(K.lib.pk_version())))), flush=True)
bf, f32 = torch.bfloat16, torch.float32
if which in ("fc2", "all", "fwd"):
    run("fc2_fwd_plain", R, 6000, 1024, False, False, bf, bias=True)
    run("fc2_fwd_lse", R, 6000, 1024, False, False, bf, lse=True, bias=True)
if which == "lse":
    run("fc2_fwd_lse", R, 6000, 1024, False, False, bf, lse=True, bias=True)
if which in ("fc2", "all", "dgrad"):
    run("fc2_dgrad", R, 1024, 6000, False, True, bf)
if which in ("fc2", "all", "wgrad"):
    run("fc2_wgrad", 6000, 1024, R, True, True, f32)
if which in ("enc", "all"):
    run("ffn1_fwd", 31808, 4096, 1024, False, False, bf, bias=True)
    run("ffn2_fwd", 31808, 1024, 4096, False, False, bf, bias=True)
    run("ffn1_dgrad", 31808, 1024, 4096, False, True, bf)
    run("ffn2_dgrad", 31808, 4096, 1024, False, True, bf)
    run("qkv_fwd", 31808, 3072, 1024, False, False, bf, bias=True)
    run("enc_wgrad_1k_1k_31k", 1024, 1024, 31808, True, True, f32)
    run("enc_wgrad_4k_1k_31k", 4096, 1024, 31808, True, True, f32)
    run("enc_wgrad_1k_4k_31k", 1024, 4096, 31808, True, True, f32)
    run("enc_wgrad_1k_1k_7680", 1024, 1024, 7680, True, True, f32)
    run("enc_wgrad_4k_1k_7680", 4096, 1024, 7680, True, True, f32)
    run("joint_fc1_fwd", 7680, 2048, 1024, False, False, bf, bias=True)
if which in ("sq", "all"):
    run("sq8192", 8192, 8192, 8192, False, False, bf)
