"""``warp_rnnt``-compatible loss entry point (the reference imports ``from warp_rnnt import RNNTLoss``,
trainer/train_transducer_bmuf_otfaug.py:25, and calls ``RNNTLoss(blank=0, reduction='sum').apply``, :58)."""
from .engine import RNNTLossFn, check_emission_reg


class RNNTLoss:
    """``RNNTLoss(blank=0, reduction='sum').apply(log_probs, labels, frame_lens, label_lens) -> costs [B]``.

    A plain callable object (not an instantiated autograd Function): ``apply`` forwards to ``RNNTLossFn.apply``.
    As at the reference call site the result is the per-utterance cost vector; the trainer sums it itself
    (:99), so ``reduction`` only validates ('sum' | 'none' give the same vector, 'mean' is not something the
    reference path ever asks for and is rejected rather than silently ignored).

    ``fastemit_lambda`` / ``delay_penalty`` (finite, >= 0; ValueError otherwise): FastEmit and the delay penalty (DESIGN.md "FastEmit
    and delay penalty").  Both 0 (the default) is the plain RNN-T loss."""

    def __init__(self, blank=0, reduction="sum", fastemit_lambda=0.0, delay_penalty=0.0):
        if blank != 0:
            raise ValueError("pika_b200 RNNTLoss: the reference path uses blank = 0 (got %r)" % (blank,))
        if reduction not in ("sum", "none"):
            raise ValueError("pika_b200 RNNTLoss: unsupported reduction %r" % (reduction,))
        self.blank, self.reduction = blank, reduction
        self.fastemit_lambda, self.delay_penalty = check_emission_reg(fastemit_lambda, delay_penalty)

    def apply(self, log_probs, labels, frame_lens, label_lens):
        return RNNTLossFn.apply(log_probs, labels, frame_lens, label_lens, self.fastemit_lambda, self.delay_penalty)

    __call__ = apply
