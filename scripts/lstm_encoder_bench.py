"""LSTM encoder (--encoder_type rnn) timings on one GPU.

1. One bidirectional layer's recurrence at B=32, T=1000, H_dir=512 with ragged lengths spread over 800-1000, forward and backward
   timed separately: (a) both directions in one cooperative launch, (b) the same layer as two single-direction launches (run
   alternately with (a), several rounds), (c) cuDNN nn.LSTM in bf16 over the packed batch (the whole layer, including its input
   projection: a yardstick only).
2. A whole TrainStep (front end + encoder + prediction net + joint + loss + backward + clip/SGD) with --encoder_type rnn --brnn
   --rnn_size 1024 --enc_layers 2 at B=32, T=240 frames (T_out = 240), U=150, V=6000, bf16.

Prints the card and its power limit first.  Usage: python scripts/lstm_encoder_bench.py [--rounds 5]
"""
import argparse
import os
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return "%s | %s" % (torch.cuda.get_device_name(), q)


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def layer_bench(rounds, iters):
    from pika_b200 import kernels as K
    B, T, E, H = 32, 1000, 240, 512
    g = torch.Generator(device="cuda").manual_seed(1)
    lens = torch.linspace(1000, 800, B).round().int().cuda()
    gx = torch.randn(2, B, T, 4 * H, generator=g, device="cuda") * 0.5
    whh = (torch.randn(2 * 4 * H, H, generator=g, device="cuda") * 0.03).bfloat16()
    out = torch.empty(B, T, 2 * H, device="cuda", dtype=torch.bfloat16)
    gates = torch.empty(2, T, B, 4 * H, device="cuda")
    cs = torch.empty(2, T, B, H, device="cuda")
    dout = (torch.randn(B, T, 2 * H, generator=g, device="cuda") * 0.1).bfloat16()
    dG = torch.empty(2, T, B, 4 * H, device="cuda", dtype=torch.bfloat16)

    def one_fwd():
        K.lstm_seq_fwd_ex(gx, whh, out, gates, cs, lens)

    def one_bwd():
        K.lstm_seq_bwd_ex(dout, gates, cs, whh, dG, lens)

    def two_fwd():
        for d in range(2):
            K.lstm_seq_fwd_ex(gx[d:d + 1], whh[d * 4 * H:(d + 1) * 4 * H], out[:, :, d * H:(d + 1) * H], gates[d:d + 1], cs[d:d + 1], lens,
                              reverse=d == 1)

    def two_bwd():
        for d in range(2):
            K.lstm_seq_bwd_ex(dout[:, :, d * H:(d + 1) * H], gates[d:d + 1], cs[d:d + 1], whh[d * 4 * H:(d + 1) * 4 * H], dG[d:d + 1], lens,
                              reverse=d == 1)

    # both forms compute the same thing: check once (the backward's cross-warp partial sums are added in arrival order, so dG may
    # differ in the last bf16 bit from run to run, whichever form runs)
    one_fwd(); one_bwd()
    o1, g1 = out.clone(), dG.clone()
    two_fwd(); two_bwd()
    same = torch.equal(o1, out)
    dg_rel = ((g1.float() - dG.float()).norm() / dG.float().norm()).item()
    res = {"one_fwd": [], "one_bwd": [], "two_fwd": [], "two_bwd": []}
    for _ in range(rounds):
        res["one_fwd"].append(timed(one_fwd, iters))
        res["two_fwd"].append(timed(two_fwd, iters))
        res["one_bwd"].append(timed(one_bwd, iters))
        res["two_bwd"].append(timed(two_bwd, iters))
    # (c) cuDNN bf16 over the packed batch (whole layer: input projection included)
    lstm = torch.nn.LSTM(E, H, batch_first=True, bidirectional=True).cuda().bfloat16()
    x = torch.randn(B, T, E, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    lc = lens.cpu().long()

    def cudnn_fwd():
        o, _ = lstm(torch.nn.utils.rnn.pack_padded_sequence(x, lc, batch_first=True, enforce_sorted=False))
        return o

    cf = [timed(cudnn_fwd, iters) for _ in range(rounds)]
    o = cudnn_fwd()
    packed_dy = torch.randn_like(o.data)

    def cudnn_fwd_bwd():
        o = cudnn_fwd()
        torch.autograd.grad(o.data, [x] + list(lstm.parameters()), packed_dy)

    cfb = [timed(cudnn_fwd_bwd, iters) for _ in range(rounds)]
    steps = int(lens.max())
    print("1. one bidirectional layer's recurrence, B=%d T=%d H_dir=%d, lengths %d-%d (%d steps); ms per call, %d rounds x %d calls"
          % (B, T, H, int(lens.min()), int(lens.max()), steps, rounds, iters))
    print("   (a) and (b): forward outputs bit-identical: %s; dG relative difference %.2e" % (same, dg_rel))
    for k, label in (("one_fwd", "(a) one launch, forward "), ("two_fwd", "(b) two launches, forward"),
                     ("one_bwd", "(a) one launch, backward"), ("two_bwd", "(b) two launches, backward")):
        v = res[k]
        print("   %s  median %.3f ms (%.2f us/step)  runs %s" % (label, float(np.median(v)), float(np.median(v)) * 1e3 / steps,
                                                             " ".join("%.3f" % t for t in v)))
    for k in ("fwd", "bwd"):
        wins = sum(a < b for a, b in zip(res["one_" + k], res["two_" + k]))
        print("   %s: one launch faster in %d of %d rounds" % (k, wins, rounds))
    print("   (c) cuDNN bf16 packed, whole layer: forward median %.3f ms; forward+backward median %.3f ms (runs %s / %s)"
          % (float(np.median(cf)), float(np.median(cfb)), " ".join("%.3f" % t for t in cf), " ".join("%.3f" % t for t in cfb)))


def train_step_bench(steps, warmup):
    from pika_b200 import engine
    from pika_b200.frontend import FbankOptions, Frontend
    from pika_b200.model.transducer import Net
    from pika_b200.trainer.bmuf import BmufTrainer
    from pika_b200.trainer.flat import FlatParams, SgdNesterovClip
    from pika_b200.trainer.step import TrainStep
    dev = torch.device("cuda")
    B, T, U, V = 32, 240, 150, 6000
    engine.set_precision("bf16")
    engine.set_dropout_enabled(True)
    margs = types.SimpleNamespace(rnn_size=1024, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="rnn", embd_dim=100,
                                  padding_idx=V, dropout=0.3, dec_layers=2, enc_layers=2)
    ta = types.SimpleNamespace(cmn=True, model_lctx=0, model_rctx=0, model_stride=1, sync_period=5, initial_lr=4e-4, final_lr=4e-5,
                               momentum=0.9, grad_clip=3.0, num_epochs=15, num_batches_per_epoch=1000, epoch=0, block_momentum=0.9,
                               block_lr=1.0)
    torch.manual_seed(777)
    model = Net(margs, 240, V).to(dev).train()
    flat = FlatParams(model)
    bmuf = BmufTrainer(0, 0, 1, model, ta.block_momentum, ta.block_lr, flat=flat)
    opt = SgdNesterovClip(flat, ta.initial_lr, ta.momentum, ta.grad_clip)
    fe = Frontend(FbankOptions(num_mel_bins=80, low_freq=40.0, high_freq=-200.0, dither=0.0, window_type="hamming"), 1, 1, dev)
    step = TrainStep(model, ta, fe, bmuf, opt, offset=torch.zeros(fe.D, device=dev), scale=torch.ones(fe.D, device=dev))
    rng = np.random.default_rng(777)
    n = 400 + (T - 1) * 160
    pcm = torch.from_numpy(np.clip(np.round(rng.normal(0, 3000.0, (B, n))), -32768, 32767).astype(np.int16)).to(dev)
    new_len, frames = Frontend.lengths([n] * B, [1.0] * B)
    meta = torch.tensor([[n] * B, new_len, frames, [U] * B], dtype=torch.int32, device=dev)
    batch = dict(pcm=pcm, target=torch.from_numpy(rng.integers(1, V, (B, U))).to(dev), n_samples=meta[0], new_len=meta[1], n_frames=meta[2],
                 ali_lens=meta[3], rate=torch.ones(B, device=dev), target_db=torch.full((B,), -25.0, device=dev), t_max=max(frames))
    for _ in range(warmup):
        costs = step(batch)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        costs = step(batch)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    print("2. TrainStep, --encoder_type rnn --brnn --rnn_size 1024 --enc_layers 2, B=%d T=%d (T_out=%d) U=%d V=%d bf16: %.1f ms/step "
          "(%d steps after %d warm-up; mean cost %.3f)" % (B, T, max(frames), U, V, ms, steps, warmup, float(costs.detach().mean())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    print("card: %s" % card())
    layer_bench(a.rounds, a.iters)
    train_step_bench(a.steps, a.warmup)


if __name__ == "__main__":
    main()
