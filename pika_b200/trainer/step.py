"""One RNN-T training batch on the GPU -- the body of run_one_epoch's hot loop
(trainer/train_transducer_bmuf_otfaug.py:71-130) with every numerically heavy stage replaced by the
sm_90a kernels: H2D of raw PCM -> on-GPU augmentation + fbank + splice + CMN/CMVN + SpecAugment ->
encoder / prediction net / fused joint+loss forward and backward -> inf-norm clip + Nesterov SGD ->
BMUF block sync every ``sync_period`` batches.
"""

import contextlib

import numpy as np

from .. import engine
from ..frontend import noise_rir_kwargs
from .flat import lr_at
from .bmuf import SUCCESS


def encoder_out_lens(lens, lctx, rctx, stride):
    """T' = ceil((T - lctx - rctx) / stride) (trainer/train_transducer_bmuf_otfaug.py:79-82)"""
    l = lens - lctx - rctx
    return l // stride + (l % stride != 0).to(l.dtype)


def encoder_out_max(t_max, lctx, rctx, stride):
    """max(encoder_out_lens) from the host-side longest input: the T_out of the packed LSTM encoder without a device read"""
    l = t_max - lctx - rctx
    return l // stride + (l % stride != 0)


def prune_loss_scales(args, i):
    """(simple_scale, pruned_scale) of the pruned RNN-T objective at global batch index i: (--simple_loss_scale, 1), or during the
    --prune_warmup_batches W warm-up 1 - (1 - simple_loss_scale) f and 0.1 + 0.9 f with f = min(i / W, 1)"""
    W = int(getattr(args, "prune_warmup_batches", 0))
    ss = float(getattr(args, "simple_loss_scale", 0.5))
    if W <= 0:
        return ss, 1.0
    f = min(i / W, 1.0)
    return 1.0 - (1.0 - ss) * f, 0.1 + 0.9 * f


def smoothing_scales(args):
    """the simple loss's smoothing keywords of engine.transducer_loss_pruned from --lm_only_scale / --am_only_scale (not ramped)"""
    return dict(lm_only_scale=float(getattr(args, "lm_only_scale", 0.0)), am_only_scale=float(getattr(args, "am_only_scale", 0.0)))


def emission_reg(args):
    """the FastEmit / delay-penalty keywords of engine.transducer_loss(_pruned) from --fastemit_lambda / --delay_penalty (not ramped)"""
    return dict(fastemit_lambda=float(getattr(args, "fastemit_lambda", 0.0)), delay_penalty=float(getattr(args, "delay_penalty", 0.0)))


def chunk_for_batch(args, index):
    """with --dynamic_chunk_max M, the encoder's chunk size for global batch ``index``: full context (0) with probability 1/2 and otherwise
    uniform in [1, M], from a generator of its own seeded by (--seed, rank, index), so the loader's, SpecAugment's and torch's random
    streams do not move.  None without the flag: the encoder keeps its own setting."""
    M = int(getattr(args, "dynamic_chunk_max", 0))
    if M <= 0:
        return None
    rng = np.random.default_rng([int(args.seed) & 0xFFFFFFFF, int(getattr(args, "local_rank", 0) or 0), int(index)])
    if rng.random() < 0.5:
        return 0
    return int(rng.integers(1, M + 1))


@contextlib.contextmanager
def encoder_chunk(model, chunk_size):
    """runs the block with the TDNN-Transformer encoder's chunk_size set to ``chunk_size`` (None: unchanged), and restores it after (so a
    checkpoint of a dynamically chunked model records its static setting)"""
    enc = model.encoder
    if chunk_size is None or not hasattr(enc, "chunk_masks"):
        yield
        return
    old = enc.chunk_size
    enc.chunk_size = chunk_size
    try:
        yield
    finally:
        enc.chunk_size = old


class TrainStep:
    def __init__(self, model, args, frontend, bmuf, optimizer, offset=None, scale=None, spec_augmentor=None):
        self.model, self.args, self.frontend, self.bmuf, self.opt = model, args, frontend, bmuf, optimizer
        self.offset, self.scale, self.spec = offset, scale, spec_augmentor
        self.num_done = 0

    def features(self, batch):
        """batch: dict of device tensors (pcm int16 [B,n], n_samples, rate, target_db, new_len, n_frames) + t_max (rows after the
        front end's stride), and the noise / reverberation draws when the loader made them (loader/otf_utt_loader.py: assemble)"""
        a = self.args
        sa = (0, 0, 0, 0)
        if self.spec is not None:
            sa = self.spec.draw(batch["t_max"], self.frontend.D)
        # the reference subtracts the utterance mean only inside ``if args.cmvn_stats:`` (:86-91), so --cmn without
        # --cmvn_stats is a no-op there; ``cmn_without_stats`` lets a caller that has no stats file (bench.py) keep CMN on
        cmn = bool(a.cmn) and (self.offset is not None or bool(getattr(a, "cmn_without_stats", False)))
        return self.frontend(batch["pcm"], batch["n_samples"], batch["rate"], batch["target_db"], batch["new_len"],
                             batch["n_frames"], batch["t_max"], out_dtype=engine.act_dtype(), cmn=cmn,
                             offset=self.offset, scale=self.scale, specaug=sa, **noise_rir_kwargs(batch))

    def __call__(self, batch):
        """-> per-utterance costs [B] (device).  Mirrors :71-123 of the reference trainer."""
        a = self.args
        self.opt.flat.zero_grad()                                         # optimizer.zero_grad()
        feats = self.features(batch)
        len_batch = encoder_out_lens(self.frontend.out_lens(batch["n_frames"]), a.model_lctx, a.model_rctx, a.model_stride)
        t_out = encoder_out_max(int(batch["t_max"]), a.model_lctx, a.model_rctx, a.model_stride)
        self.simple_costs = None
        with encoder_chunk(self.model, chunk_for_batch(a, a.epoch * a.num_batches_per_epoch + self.num_done)):
            costs, loss = self._loss(feats, batch, len_batch, t_out)
        engine.assume_unit_loss_grad(True)                                # loss = costs.sum() (:99): upstream gradient is exactly 1
        try:
            loss.backward()
        finally:
            engine.assume_unit_loss_grad(False)
        self.opt.step()                                                   # clip_grad_norm_(inf) + SGD(nesterov)
        self.end_of_item()
        return costs

    def _loss(self, feats, batch, len_batch, t_out):
        a = self.args
        if getattr(a, "prune_range", 0) > 0:
            ss, ps = prune_loss_scales(a, a.epoch * a.num_batches_per_epoch + self.num_done)
            simple, costs = engine.transducer_loss_pruned(self.model, feats, batch["target"], len_batch, batch["ali_lens"], a.prune_range,
                                                          ss, ps, x_len=len_batch, t_out=t_out, **smoothing_scales(a), **emission_reg(a))
            self.simple_costs = simple
            loss = (simple * ss + costs * ps).sum()                       # upstream gradients: exactly the scales passed above
        else:
            costs = engine.transducer_loss(self.model, feats, batch["target"], len_batch, batch["ali_lens"], x_len=len_batch, t_out=t_out,
                                           **emission_reg(a))
            loss = costs.sum()
        return costs, loss

    def skip(self):
        """An empty loader item (every utterance filtered, :100-101): no forward / backward / optimiser step, but the item
        still counts and still takes part in the periodic block sync (:112-123) -- a rank that skipped the collective
        while its peers entered it would pair their all-reduce with a later one."""
        self.end_of_item()

    def end_of_item(self):
        """``if num_done != 0 and num_done % sync_period == 0`` of the reference loop (:112-123): BMUF sync, new learning rate,
        fresh momentum buffer.  Runs for EVERY loader item, with or without data."""
        a = self.args
        if self.num_done != 0 and self.num_done % a.sync_period == 0:
            if self.bmuf.update_and_sync() != SUCCESS:
                raise FloatingPointError("BMUF: non-finite block delta")
            self.opt.reset(lr_at(a.initial_lr, a.final_lr, a.epoch * a.num_batches_per_epoch + self.num_done,
                                 a.num_epochs * a.num_batches_per_epoch))
        self.num_done += 1
