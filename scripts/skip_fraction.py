"""Fraction of the joint rows whose stored RNN-T gradient is all zeros, in the bench train step (B = 32, T = 1000, U = 150, V = 6000).

Such a row adds nothing to the fc2 dgrad, the fc2 wgrad or the fc2 bias gradient.  The script runs the dense joint backward and
counts, after each loss call, the rows of dlogits whose V entries are all +-0.  Env: B (batch), STEPS (counted steps).
"""
import os
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from pika_b200 import engine
from pika_b200 import kernels as K
from pika_b200.frontend import FbankOptions, Frontend
from pika_b200.model.transducer import Net
from pika_b200.trainer.bmuf import BmufTrainer
from pika_b200.trainer.flat import FlatParams, SgdNesterovClip
from pika_b200.trainer.step import TrainStep
from pika_b200.utils.spec_augment import SpecAugment

a = types.SimpleNamespace(batch=int(os.environ.get("B", 32)), T=1000, U=150, V=6000)
steps = int(os.environ.get("STEPS", 8))
dev = torch.device("cuda", 0)
engine.set_precision("bf16")
if hasattr(engine, "_COMPACT_GRAD"):
    engine._COMPACT_GRAD = False               # count on the dense gradient
ta = bench.train_args()
torch.manual_seed(777)
model = Net(bench.model_args(a.V), 240, a.V).to(dev)
model.train()
flat = FlatParams(model)
bmuf = BmufTrainer(0, 0, 1, model, ta.block_momentum, ta.block_lr, flat=flat)
opt = SgdNesterovClip(flat, ta.initial_lr, ta.momentum, ta.grad_clip)
fe = Frontend(FbankOptions(num_mel_bins=80, low_freq=40.0, high_freq=-200.0, dither=0.0, window_type="hamming"), 1, 1, dev)
step = TrainStep(model, ta, fe, bmuf, opt, spec_augmentor=SpecAugment(ta.max_freq_span, ta.max_time_span))
B = a.batch
torch.manual_seed(777)
np.random.seed(777)
pcm = torch.from_numpy(bench.synth_pcm(B, a.T, 777)).to(dev)
rng = np.random.default_rng(777)
n = pcm.shape[1]
new_len, frames = Frontend.lengths([n] * B, [1.0] * B)
i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)
batch = dict(pcm=pcm, target=torch.from_numpy(rng.integers(1, a.V, (B, a.U))).to(dev), n_samples=i32([n] * B), new_len=i32(new_len),
             n_frames=i32(frames), ali_lens=i32([a.U] * B), rate=torch.ones(B, device=dev), target_db=torch.full((B,), -25.0, device=dev),
             t_max=max(frames))

counts = []
_loss = K.rnnt_loss_fwd_bwd


def counting_loss(logits, *args, **kw):
    costs, dl = _loss(logits, *args, **kw)
    if dl is not None and kw.get("want_grad", True):
        V = kw.get("V") or dl.shape[-1]
        zero = 0
        for b in range(dl.shape[0]):            # one utterance at a time: a [T, U1] mask, not a 13.9 GB one
            zero += int((dl[b, ..., :V] == 0).all(dim=-1).sum())
        counts.append((zero, dl.shape[0] * dl.shape[1] * dl.shape[2]))
    return costs, dl


K.rnnt_loss_fwd_bwd = counting_loss
for _ in range(steps):
    step(batch)
torch.cuda.synchronize()
fr = [z / r for z, r in counts]
print("rows per step %d; all-zero gradient rows per step: %s" % (counts[0][1], " ".join("%.4f" % f for f in fr)))
print("skippable fraction: mean %.4f, min %.4f" % (sum(fr) / len(fr), min(fr)))
