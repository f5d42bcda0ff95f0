"""Beam-search decoding with the transformer prediction net at the config-5 decode shape (H100, bf16): batch 64 x beam 16 = 1024 rows,
T' = 375 encoder frames, V = 6000, H = 1024, a 2-layer prediction net (d_model 512, 8 heads), max_len = T' + 100.  Seeded weights
(the default initialisation plus a wider embedding / output projection and a blank bias, so that hypotheses grow) and seeded
encoder outputs; nothing is read from disk and nothing is written.

1. whole decode_batch calls, without and with FST shallow fusion (a seeded back-off bigram over the 6000 labels): host clock around
   each call ending in a device synchronise, after one warm-up call (which captures the graph); ms per call and per beam step;
2. the prediction net's cost per beam step at history length L = 25 / 50 / 100 / 150: the incremental step (the KV-cached step the
   beam loop runs, on a pool filled as if every row had computed its L positions) against the full-history forward over
   [1024, L + 1] tokens that the earlier host-issued loop ran every step; CUDA events, the two alternating (A B A B ...).
Prints one JSON line per measurement with the card's name and power limit."""
import json
import os
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pika_b200 import engine  # noqa: E402
from pika_b200.decoder.beam_transducer import GlobalScorer  # noqa: E402
from pika_b200.decoder.sorted_matcher import SortedMatcher  # noqa: E402
from pika_b200.decoder.transducer_decoder import TransducerDecoder  # noqa: E402
from pika_b200.model.transducer import Net  # noqa: E402

B, BEAM, TP, V, H = 64, 16, 375, 6000, 1024
CALLS = int(os.environ.get("CALLS", 3))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:                                  # the timing itself does not depend on it
        q = "unknown (%s)" % ex
    return q


def model():
    torch.manual_seed(778)
    a = types.SimpleNamespace(rnn_size=H, local_rank=0, decoder_type="transformer", brnn=True, encoder_type="transformer", embd_dim=100,
                              padding_idx=V, dropout=0.0, dec_layers=2, enc_layers=9)
    m = Net(a, 240, V)
    g = torch.Generator().manual_seed(2025)
    with torch.no_grad():
        m.embed.weight.normal_(0, 1, generator=g)
        m.decoder.linear_out.weight *= 6.0
        for lin in (m.fc1, m.fc_gate):
            lin.weight.normal_(0, 0.05, generator=g)
        m.fc2.weight.normal_(0, 0.1, generator=g)
        m.fc2.bias[0] += 2.5
    return m.cuda().eval()


def backoff_lm(n_hist=64, seed=31):
    """seeded back-off bigram as a sorted arc table (ilabel = token + 1, label 1 = back-off): state 0 has an arc for every token"""
    rng = np.random.default_rng(seed)
    arcs = [sorted((y + 1, float(rng.uniform(0.1, 1.5)), int(rng.integers(0, n_hist + 1))) for y in range(1, V))]
    finals = [1.0]
    for s in range(1, n_hist + 1):
        toks = np.sort(rng.choice(np.arange(1, V), size=V // 20, replace=False))
        arcs.append([(1, float(rng.uniform(0.2, 1.5)), 0)] + [(int(y) + 1, float(rng.uniform(0.05, 1.0)), int(rng.integers(0, n_hist + 1)))
                                                              for y in toks])
        finals.append(float(rng.uniform(0.5, 2.0)) if s % 2 == 0 else float("inf"))
    return SortedMatcher((arcs, finals), max(len(a) for a in arcs), V + 2, 1, [])


def decode_calls(m, enc, tl, fst):
    kw = dict(lm_scorer=backoff_lm(), lm_scorer_scale=0.5) if fst else {}
    dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.45 if fst else 0.0)
    dec = TransducerDecoder(m, B, BEAM, n_best=BEAM, blk=0, global_scorer=GlobalScorer(), sm_scale=1.0, cuda=True, beam_prune=True,
                            args=dargs, **kw)
    ml = [int(t) + 100 for t in tl]
    ret, _ = dec.decode_batch(None, tl, max_len=ml, enc_out=enc)                 # warm-up: workspace, staging, graph capture
    times = []
    for _ in range(CALLS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ret, _ = dec.decode_batch(None, tl, max_len=ml, enc_out=enc)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    steps = int(dec._ws.step_ctx[0].item())
    labels = [sum(1 for t in ret["alignments"][b][0] if t != 0) for b in range(B)]
    return dec, dict(what="decode_batch", fst=fst, ms_per_call=float(np.median(times)), calls_ms=[round(t, 1) for t in times],
                     beam_steps=steps, ms_per_beam_step=float(np.median(times)) / steps, kernels_per_replay=dec.kernels_per_replay,
                     best_hyp_labels_mean=float(np.mean(labels)), best_hyp_labels_max=int(np.max(labels)))


def events(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def step_vs_recompute(dec, m, L, rounds=3, iters=10):
    """the incremental step on a workspace holding L cached positions per row vs the full-history forward over [rows, L + 1]"""
    ws = dec._ws
    rows, xf = ws.rows, ws.xf
    par = L & 1
    r = torch.arange(rows, dtype=torch.int32, device="cuda")
    j = torch.arange(L + 1, dtype=torch.int32, device="cuda")
    xf.slot.view(2, rows, -1)[par, :, :L + 1] = torch.where(j[None, :] == 0, 0, 1 + j[None, :] * rows + r[:, None])   # distinct entries
    g = torch.Generator(device="cuda").manual_seed(L)
    ws.hyp_tok.view(2, rows, -1)[par, :, :L] = torch.randint(1, V, (rows, L), generator=g, device="cuda", dtype=torch.int32)
    ws.hyp_len.view(2, rows)[par] = L
    ws.next_ys.view(-1, rows)[L] = ws.hyp_tok.view(2, rows, -1)[par, :, L - 1]
    ws.step_ctx.copy_(torch.tensor([L, 1], dtype=torch.int32))
    src = torch.cat((torch.zeros(rows, 1, dtype=torch.long, device="cuda"), ws.hyp_tok.view(2, rows, -1)[par, :, :L].long()), 1)
    new = lambda: xf.step(dec, ws.h[0])                                        # noqa: E731
    old = lambda: engine.conv_transformer_lm_forward_act(m.decoder, src)       # noqa: E731
    new(), old()
    a, b = [], []
    for _ in range(rounds):
        a.append(events(old, iters))
        b.append(events(new, iters))
    return dict(what="prednet_per_step", L=L, rows=rows, full_recompute_ms=float(np.median(a)), incremental_ms=float(np.median(b)),
                speedup=float(np.median(a) / np.median(b)))


@torch.no_grad()
def main():
    assert torch.cuda.is_available(), "xf_decode_bench.py measures on the GPU"
    engine.set_precision("bf16")
    gpu = card()
    m = model()
    g = torch.Generator(device="cuda").manual_seed(606)
    enc = torch.randn(B, TP, H, generator=g, device="cuda").bfloat16()
    tl = torch.from_numpy(np.random.default_rng(7).integers(TP * 3 // 4, TP + 1, B)).int()
    tl[0] = TP
    dec = None
    for fst in (False, True):
        d, res = decode_calls(m, enc, tl, fst)
        res["gpu"] = gpu
        print(json.dumps(res), flush=True)
        if not fst:
            dec = d
        else:
            del d
        torch.cuda.empty_cache()
    dec._ws.xf.pool.zero_()
    for L in (25, 50, 100, 150):
        res = step_vs_recompute(dec, m, L)
        res["gpu"] = gpu
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
