"""Flat fp32 parameter / gradient storage and the fused clip + Nesterov-SGD step.

All parameters of the model become views into ONE contiguous fp32 buffer (and their ``.grad`` views
into a second one), so that gradient clipping (inf-norm), the optimiser and the BMUF exchange are
single HBM streams over 91 M floats instead of ~200 small kernels plus
``parameters_to_vector`` / ``_copy_vec_to_param`` copies (trainer/bmuf.py:14-35,62-63,83-84,98).
"""
import math

import numpy as np
import torch

from .. import engine
from .. import kernels as K


class FlatParams:
    def __init__(self, model):
        params = [p for p in model.parameters()]
        assert all(p.dtype == torch.float32 for p in params), "model parameters must be fp32"
        # 16-byte aligned slots so that every parameter can be a TMA source / destination
        offs, n = [], 0
        for p in params:
            offs.append(n)
            n += (p.numel() + 3) // 4 * 4
        dev = params[0].device
        self.data = torch.zeros(n, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(n, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for p, o in zip(params, offs):
                self.data[o:o + p.numel()].copy_(p.detach().reshape(-1))
                p.data = self.data[o:o + p.numel()].view(p.shape)
                p.grad = self.grad[o:o + p.numel()].view(p.shape)
        self.params, self.offsets, self.numel = params, offs, n
        self.num_param = sum(p.numel() for p in params)
        engine.invalidate_weights()

    def zero_grad(self):
        self.grad.zero_()


def lr_at(initial_lr, final_lr, num_batches_processed, total_num_batches):
    """exponential decay (trainer/train_transducer_bmuf_otfaug.py:46-51,115-120)"""
    return initial_lr * math.exp(num_batches_processed * math.log(final_lr / initial_lr) / total_num_batches)


class SgdNesterovClip:
    """clip_grad_norm_(params, max_norm, norm_type=inf) + optim.SGD(lr, momentum, nesterov=True).step()
    (trainer/train_transducer_bmuf_otfaug.py:53-55,105-110) as two kernels over the flat buffers.
    ``reset()`` drops the momentum buffer, as re-creating the optimiser after every BMUF sync does in the
    reference (:121-123)."""

    def __init__(self, flat, lr, momentum=0.9, max_norm=-1.0):
        self.flat, self.lr, self.momentum, self.max_norm = flat, lr, momentum, max_norm
        self.buf = torch.zeros_like(flat.data)
        self.first = True
        self.absmax = torch.zeros(1, dtype=torch.float32, device=flat.data.device)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=flat.data.device)

    def reset(self, lr=None):
        self.first = True
        if lr is not None:
            self.lr = lr

    def step(self):
        f = self.flat
        if self.max_norm > 0:
            self.nan_flag.zero_()
            K.absmax(f.grad, self.absmax, self.nan_flag)
        K.sgd_nesterov_clip(f.data, f.grad, self.buf, self.lr, self.momentum, self.max_norm,
                            self.absmax if self.max_norm > 0 else None, self.first,
                            nan_flag=self.nan_flag if self.max_norm > 0 else None)
        self.first = False
        engine.invalidate_weights()


def f32(x):
    """round to float32: torch.optim.Adam keeps ``step`` in a float32 tensor, so its in-place updates round this way"""
    return float(np.float32(x))


class _AdamParamState(dict):
    """``state[p]`` of torch.optim.Adam for one parameter: ``exp_avg`` / ``exp_avg_sq`` are views into the flat moment buffers
    and ``step`` is the optimiser's single step count (one Adam step runs over the whole flat buffer, so every parameter
    shares it: assigning ``state[p]['step']`` sets it for all of them)."""

    def __init__(self, opt, exp_avg, exp_avg_sq):
        super().__init__(step=None, exp_avg=exp_avg, exp_avg_sq=exp_avg_sq)
        self._opt = opt

    def __getitem__(self, k):
        return self._opt.step_count if k == "step" else super().__getitem__(k)

    def __setitem__(self, k, value):
        if k == "step":
            self._opt.step_count = float(value)
        else:
            super().__setitem__(k, value)


class AdamClip:
    """clip_grad_norm_(params, max_norm, norm_type=inf) + optim.Adam(lr, betas, eps, weight_decay=0).step() as two kernels over the
    flat buffers (the optimiser BmufAdamTrainer drives, trainer/bmuf.py:191-215).  The moments live in two flat buffers with the
    parameters' slot layout.  ``reset(lr)`` only sets the learning rate: the moments and the step count persist.
    ``param_groups`` and ``state[p]`` look like torch.optim.Adam's, and ``state[p]['exp_avg']`` / ``['exp_avg_sq']`` are views
    of the flat moments, so code written against torch's Adam state reads and writes the same memory."""

    def __init__(self, flat, lr, betas=(0.9, 0.999), eps=1e-8, max_norm=-1.0, ops=None):
        # ``ops``: object with absmax / adam_clip; defaults to the CUDA kernels (the CPU-side gloo test injects numpy ones)
        self.ops = ops if ops is not None else K
        self.flat, self.max_norm = flat, max_norm
        self.param_groups = [dict(params=flat.params, lr=lr, betas=tuple(betas), eps=eps, weight_decay=0, amsgrad=False)]
        self.step_count = 0.0
        self.absmax = torch.zeros(1, dtype=torch.float32, device=flat.data.device)
        self.nan_flag = torch.zeros(1, dtype=torch.int32, device=flat.data.device)
        self.place_moments(torch.zeros_like(flat.data), torch.zeros_like(flat.data))

    lr = property(lambda self: self.param_groups[0]["lr"], lambda self, v: self.param_groups[0].__setitem__("lr", v))
    betas = property(lambda self: self.param_groups[0]["betas"])
    eps = property(lambda self: self.param_groups[0]["eps"])

    def place_moments(self, exp_avg, exp_avg_sq):
        """move the moments into caller-owned flat buffers (copying their values), e.g. slots of BMUF-Adam's exchange message"""
        if hasattr(self, "exp_avg"):
            exp_avg.copy_(self.exp_avg)
            exp_avg_sq.copy_(self.exp_avg_sq)
        self.exp_avg, self.exp_avg_sq = exp_avg, exp_avg_sq
        self.state = {}
        for p, o in zip(self.flat.params, self.flat.offsets):
            self.state[p] = _AdamParamState(self, exp_avg[o:o + p.numel()].view(p.shape), exp_avg_sq[o:o + p.numel()].view(p.shape))

    def reset(self, lr=None):
        if lr is not None:
            self.lr = lr

    def step(self):
        f = self.flat
        if self.max_norm > 0:
            self.nan_flag.zero_()
            self.ops.absmax(f.grad, self.absmax, self.nan_flag)
        self.step_count = f32(self.step_count + 1)
        self.ops.adam_clip(f.data, f.grad, self.exp_avg, self.exp_avg_sq, self.lr, self.betas, self.eps, self.step_count,
                           self.max_norm, self.absmax, self.nan_flag)
        engine.invalidate_weights()
