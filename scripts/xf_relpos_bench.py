"""Cost of relative-position self-attention in the transformer prediction net, m = 0 against m = 16 (H100, bf16):

1. the prediction net's attention alone (AttentionFn, causal + padding keys) at the config-2 label shape: B = 32, L = U + 1 = 151,
   8 heads, d_head = 64 -- forward and forward + backward, CUDA events over 50 calls after 10 warm-up calls;
2. a whole --decoder_type transformer train step (TDNN-Transformer encoder over T = 1000 frames -> T' = 240, the transformer
   prediction net, joint + fused RNN-T loss at V = 6000, backward, clip + SGD): 10 timed steps after 3 warm-up steps.
The two settings alternate within each measurement (A B A B ...) so that clock drift and neighbours hit both alike.  Prints one JSON
line per measurement with the card's name and power limit.  Writes nothing."""
import json
import os
import subprocess
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from pika_b200 import engine as E  # noqa: E402
from pika_b200.model.transducer import Net  # noqa: E402
from pika_b200.trainer.flat import FlatParams, SgdNesterovClip  # noqa: E402

M_REL = int(os.environ.get("M_REL", 16))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:                                  # the timing itself does not depend on it
        q = "unknown (%s)" % ex
    return q


def events(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def attention_only(gpu):
    B, L, heads, dh = 32, 151, 8, 64
    D = heads * dh
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv0 = (torch.randn(B, L, 3 * D, generator=g, device="cuda") * 0.5).bfloat16()
    dy = torch.randn(B, L, D, generator=g, device="cuda").bfloat16()
    lens = torch.randint(L // 2, L + 1, (B,), generator=g, device="cuda")
    key_pad = (torch.arange(L, device="cuda")[None, :] >= lens[:, None]).to(torch.uint8).contiguous()
    table = {0: None, M_REL: (torch.randn(2 * M_REL + 1, dh, generator=g, device="cuda") * 0.1).requires_grad_(True)}

    def fwd(m):
        return E.AttentionFn.apply(qkv0, heads, 0.0, 0, True, key_pad, table[m])

    def fwd_bwd(m):
        qkv = qkv0.clone().requires_grad_(True)
        E.AttentionFn.apply(qkv, heads, 0.0, 0, True, key_pad, table[m]).backward(dy)

    for name, fn in (("fwd", fwd), ("fwd+bwd", fwd_bwd)):
        res = {0: [], M_REL: []}
        for m in (0, M_REL):
            for _ in range(10):
                fn(m)
        torch.cuda.synchronize()
        for _ in range(5):
            for m in (0, M_REL):
                res[m].append(events(lambda: fn(m), 10))
        print(json.dumps({"what": "prednet attention " + name, "shape": "B=32 L=151 heads=8 d_head=64 causal+padding keys, bf16",
                          "gpu": gpu, "ms_m0": [round(v, 4) for v in sorted(res[0])],
                          "ms_m%d" % M_REL: [round(v, 4) for v in sorted(res[M_REL])]}), flush=True)


def train_step(gpu):
    B, T, U, V = 32, 1000, 150, 6000
    Tp = (T - 42 + 3) // 4
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(B, T, 240, generator=g, device="cuda")
    y = torch.randint(1, V, (B, U), generator=g, device="cuda")
    ulens = torch.randint(U // 2, U + 1, (B,), generator=g, device="cuda").int()
    ulens[0] = U
    for b in range(B):
        y[b, int(ulens[b]):] = V
    tlens = torch.full((B,), Tp, dtype=torch.int32, device="cuda")
    runs = {}
    for m in (0, M_REL):
        torch.manual_seed(777)
        a = types.SimpleNamespace(rnn_size=1024, local_rank=0, decoder_type="transformer", brnn=True, encoder_type="transformer",
                                  embd_dim=100, padding_idx=V, dropout=0.2, dec_layers=2, enc_layers=9, max_relative_positions=m)
        model = Net(a, 240, V).cuda().train()
        flat = FlatParams(model)
        runs[m] = (model, SgdNesterovClip(flat, 4e-4, 0.9, 3.0))
    E.assume_unit_loss_grad(True)

    def step(m):
        model, opt = runs[m]
        costs = E.transducer_loss(model, x, y, tlens, ulens)
        costs.sum().backward()
        opt.step()

    res = {0: [], M_REL: []}
    for m in (0, M_REL):
        for _ in range(3):
            step(m)
    torch.cuda.synchronize()
    for _ in range(5):
        for m in (0, M_REL):
            res[m].append(events(lambda: step(m), 2))
    print(json.dumps({"what": "transformer prediction-net train step", "shape": "B=32 T=1000 (T'=240) U=150 V=6000 bf16, dropout 0.2",
                      "gpu": gpu, "ms_m0": [round(v, 2) for v in sorted(res[0])], "ms_m%d" % M_REL: [round(v, 2) for v in sorted(res[M_REL])]}),
          flush=True)


if __name__ == "__main__":
    assert torch.cuda.is_available(), "xf_relpos_bench.py measures on the GPU"
    E.set_precision("bf16")
    gpu = card()
    attention_only(gpu)
    train_step(gpu)
