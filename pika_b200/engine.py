"""Execution engine: the transducer's forward/backward expressed as autograd Functions whose
bodies are calls into the hand-written sm_90a kernels (pika_b200/csrc) through the C ABI.

torch supplies device memory, streams and the autograd tape; no torch operator computes anything
on this path (boundary dtype casts and view/reshape bookkeeping aside).

Precision modes (``set_precision``):
  * "bf16" (production): activations and GEMM operands bf16, fp32 accumulation in registers, fp32
    statistics / master weights / gradients.
  * "fp32" (parity): activations fp32; every GEMM runs as three bf16 tensor-core products on hi/lo
    split operands (A_hi B_hi + A_hi B_lo + A_lo B_hi), i.e. fp32-class accuracy from the same kernel.

Reference semantics reproduced (paths relative to the reference root): trainer/model/transducer.py:74-112,
trainer/model/rnnt_tdnn_transformer.py:73-89, trainer/model/modules/{transformer.py:85-100,
multi_headed_attn.py:110-241, position_ffn.py:27-39}.
"""
import math
import weakref

import torch

from . import kernels as K

_PRECISION = "bf16"
_WEIGHT_EPOCH = 0           # bumped whenever parameters are modified through raw pointers
_SEED = [0x5EED]
_DROPOUT_ENABLED = True


def set_precision(p):
    global _PRECISION
    assert p in ("bf16", "fp32")
    _PRECISION = p


def get_precision():
    return _PRECISION


def act_dtype():
    return torch.bfloat16 if _PRECISION == "bf16" else torch.float32


def invalidate_weights():
    global _WEIGHT_EPOCH
    _WEIGHT_EPOCH += 1


def set_seed(seed):
    _SEED[0] = seed & 0x7FFFFFFF


def set_dropout_enabled(flag):
    """Parity runs disable dropout while BatchNorm stays in train mode (SURVEY.md section 7)."""
    global _DROPOUT_ENABLED
    _DROPOUT_ENABLED = bool(flag)


def _next_seed():
    _SEED[0] = (_SEED[0] * 1103515245 + 12345) & 0x7FFFFFFF
    return _SEED[0]


def _drop(p, training):
    return float(p) if (training and _DROPOUT_ENABLED and p > 0) else 0.0


# ------------------------------------------------------------------------------------------------
# operand staging
def stage_act(x):
    """Activation (act dtype, any shape, contiguous) -> GEMM operand parts [hi] or [hi, lo] (bf16)."""
    if x.dtype == torch.bfloat16:
        return [x]
    x2 = x.reshape(-1, x.shape[-1])
    hi = torch.empty(x2.shape, dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi)
    K.cast_split(x2, hi, lo)
    return [hi.view(x.shape), lo.view(x.shape)]


_wcache = {}


def _prune_wcache():
    if len(_wcache) > 512:
        for k in [k for k, v in _wcache.items() if any(r() is None for r in v[2])]:
            del _wcache[k]


def _same_objects(refs, params):
    """id() values are recycled: a cache entry only counts if its weak references still point at these very tensors
    (a freed parameter whose id, version and storage address all reappear would otherwise alias a stale staging)."""
    return len(refs) == len(params) and all(r() is p for r, p in zip(refs, params))


def stage_weight(params, cols_pad=None, scale=None):
    """Parameter(s) -> staged bf16 operand parts of the row-concatenated matrix [sum N_i, K(_pad)].
    Cached until the parameters change (torch version counter or ``invalidate_weights``)."""
    params = params if isinstance(params, (list, tuple)) else [params]
    key = (tuple(id(p) for p in params), _PRECISION, cols_pad)
    stamp = (tuple(p._version for p in params), _WEIGHT_EPOCH, tuple(p.data_ptr() for p in params))
    hit = _wcache.get(key)
    if hit is not None and hit[0] == stamp and _same_objects(hit[2], params):
        return hit[1]
    mats = [p.detach().reshape(p.shape[0], -1) for p in params]
    Kdim = mats[0].shape[1]
    kp = cols_pad or Kdim
    n = sum(m.shape[0] for m in mats)
    hi = torch.empty(n, kp, dtype=torch.bfloat16, device=mats[0].device)
    lo = torch.empty_like(hi) if _PRECISION == "fp32" else None
    r = 0
    for i, m in enumerate(mats):
        K.cast_split(m, hi[r:r + m.shape[0]], None if lo is None else lo[r:r + m.shape[0]], cols_pad=kp,
                     scale=1.0 if scale is None else scale[i])
        r += m.shape[0]
    parts = [hi] if lo is None else [hi, lo]
    _prune_wcache()
    _wcache[key] = (stamp, parts, tuple(weakref.ref(p) for p in params))
    return parts


def stage_conv1d_weight(weight, ld):
    """nn.Conv1d weight [N, C, Kw] -> staged bf16 parts of the tap-major matrix [N, Kw * ld] (tap k at columns [k*ld, k*ld + C),
    zero padding up to the activation pitch ``ld``): the B operand of the causal convolution written as one GEMM over
    overlapping (Toeplitz) activation rows.  Cached like ``stage_weight``."""
    key = (id(weight), _PRECISION, "conv1d", ld)
    stamp = (weight._version, _WEIGHT_EPOCH, weight.data_ptr())
    hit = _wcache.get(key)
    if hit is not None and hit[0] == stamp and _same_objects(hit[2], [weight]):
        return hit[1]
    N, C, Kw = weight.shape
    mat = torch.zeros(N, Kw, ld, dtype=torch.float32, device=weight.device)
    mat[:, :, :C] = weight.detach().permute(0, 2, 1)
    mat = mat.view(N, Kw * ld)
    hi = torch.empty(N, Kw * ld, dtype=torch.bfloat16, device=weight.device)
    lo = torch.empty_like(hi) if _PRECISION == "fp32" else None
    K.cast_split(mat, hi, lo)
    parts = [hi] if lo is None else [hi, lo]
    _prune_wcache()
    _wcache[key] = (stamp, parts, (weakref.ref(weight),))
    return parts


def _cat_bias(params):
    """Concatenated f32 bias for a row-concatenated weight (cached like the weights)."""
    if len(params) == 1:
        return params[0].detach()
    key = (tuple(id(p) for p in params), "bias")
    stamp = (tuple(p._version for p in params), _WEIGHT_EPOCH, tuple(p.data_ptr() for p in params))
    hit = _wcache.get(key)
    if hit is not None and hit[0] == stamp and _same_objects(hit[2], params):
        return hit[1]
    out = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=params[0].device)
    r = 0
    for p in params:
        out[r:r + p.numel()].copy_(p.detach())
        r += p.numel()
    _wcache[key] = (stamp, out, tuple(weakref.ref(p) for p in params))
    return out


def gemm_parts(a_taps, b_taps, c, **kw):
    """Accumulate sum over taps of A_tap @ B_tap^T where each tap is a parts list ([hi] | [hi, lo])."""
    A, Bm, aro, bro = [], [], [], []
    a_off = kw.pop("a_row_off", None)
    b_off = kw.pop("b_row_off", None)
    for t, (ap, bp) in enumerate(zip(a_taps, b_taps)):
        combos = [(0, 0)]
        if len(ap) > 1 and len(bp) > 1:
            combos += [(0, 1), (1, 0)]
        elif len(ap) > 1:
            combos += [(1, 0)]
        elif len(bp) > 1:
            combos += [(0, 1)]
        for (i, j) in combos:
            A.append(ap[i])
            Bm.append(bp[j])
            aro.append(a_off[t] if a_off else 0)
            bro.append(b_off[t] if b_off else 0)
    return K.gemm(A, Bm, c, a_row_off=aro, b_row_off=bro, **kw)


def grad_of(p):
    if p.grad is None:
        p.grad = torch.zeros_like(p, memory_format=torch.contiguous_format)
    return p.grad


def _new(shape, dtype=None, like=None, zero=False):
    dev = like.device if like is not None else "cuda"
    f = torch.zeros if zero else torch.empty
    return f(shape, dtype=dtype or act_dtype(), device=dev)


# ------------------------------------------------------------------------------------------------
class LinearFn(torch.autograd.Function):
    """y = dropout(act(x W^T + b)) + residual; W = row-concatenation of ``weights``."""

    @staticmethod
    def forward(ctx, x, residual, act, drop_p, seed, nw, premasked, mask_input_scale, *params):
        # premasked: the incoming gradient is already d(pre-activation) -- the consumer's backward applied this layer's
        #   ReLU(+dropout) mask (BatchNorm backward with relu_mask, or the next Linear's dgrad epilogue), so no mask pass runs here.
        # mask_input_scale (> 0): this layer's INPUT x is relu(+dropout) output of the previous Linear; its dgrad epilogue
        #   multiplies dx by (x != 0) * scale, i.e. hands the previous layer d(pre-activation) directly (AUX_MASK_NZ).
        weights = list(params[:nw])
        biases = list(params[nw:]) if len(params) > nw else None
        M, Kd = x.shape
        w_parts = stage_weight(weights, cols_pad=x.shape[1] if x.shape[1] != weights[0].shape[1] else None)
        N = w_parts[0].shape[0]
        y = _new((M, N), like=x)
        bias = _cat_bias(biases) if biases is not None else None
        a_parts = stage_act(x)
        gemm_parts([a_parts], [w_parts], y, bias=bias, act=K.ACT_RELU if act else K.ACT_NONE, drop_p=drop_p,
                   drop_seed=seed, aux=residual, aux_mode=K.AUX_ADD if residual is not None else K.AUX_NONE)
        ctx.weights, ctx.biases, ctx.act, ctx.drop_p, ctx.seed = weights, biases, act, drop_p, seed
        ctx.premasked, ctx.mask_input_scale = premasked, mask_input_scale
        ctx.has_res = residual is not None
        ctx.save_for_backward(x, y if act else None)
        ctx.a_parts, ctx.w_parts = a_parts, w_parts
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y = ctx.saved_tensors
        dy = dy.contiguous()
        M, N = dy.shape
        if ctx.premasked:
            dpre = dy
        elif ctx.act:
            dpre = torch.empty_like(dy)
            K.mask_nz(dy, y, dpre, 1.0 / (1.0 - ctx.drop_p) if ctx.drop_p > 0 else 1.0)
        elif ctx.drop_p > 0:
            dpre = torch.empty_like(dy)
            K.dropout(dy, dpre, ctx.drop_p, ctx.seed)
        else:
            dpre = dy
        d_parts = stage_act(dpre)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            # dx = dy @ W reads the staged W [N, K] as an MN-major B operand
            if ctx.mask_input_scale > 0:
                gemm_parts([d_parts], [ctx.w_parts], dx, b_mn=True, aux=x, aux_mode=K.AUX_MASK_NZ, aux_scale=ctx.mask_input_scale)
            else:
                gemm_parts([d_parts], [ctx.w_parts], dx, b_mn=True)
            if dx.shape[1] != x.shape[1]:
                dx = dx[:, :x.shape[1]]
        # dW_i = dpre[:, rows_i]^T x ; db_i = colsum(dpre)[rows_i]
        r = 0
        dbias = None
        if ctx.biases is not None:
            dbias = torch.empty(N, dtype=torch.float32, device=dy.device)
            K.colsum(dpre, dbias)
        for i, w in enumerate(ctx.weights):
            n_i = w.shape[0]
            g = grad_of(w).view(n_i, -1)
            gemm_parts([[p[:, r:r + n_i] for p in d_parts]], [[p[:, :g.shape[1]] for p in ctx.a_parts]], g, a_mn=True, b_mn=True)
            if ctx.biases is not None:
                grad_of(ctx.biases[i]).copy_(dbias[r:r + n_i])
            r += n_i
        n_par = len(ctx.weights) + (len(ctx.biases) if ctx.biases is not None else 0)
        return (dx, (dy if ctx.has_res else None), None, None, None, None, None, None) + (None,) * n_par


def linear(x, weights, biases=None, act=False, drop_p=0.0, residual=None, premasked=False, mask_input_scale=0.0):
    weights = list(weights) if isinstance(weights, (list, tuple)) else [weights]
    if biases is not None and not isinstance(biases, (list, tuple)):
        biases = [biases]
    params = weights + (list(biases) if biases is not None else [])
    if x.dtype != torch.bfloat16 or x.shape[1] % 8 != 0:
        mask_input_scale = 0.0                 # the epilogue mask reads x as a 16-byte-aligned aux operand of the activation dtype
    return LinearFn.apply(x, residual, act, drop_p, _next_seed() if drop_p > 0 else 0, len(weights), premasked, mask_input_scale, *params)


class TdnnFn(torch.autograd.Function):
    """relu(Conv2d(1, N, (3, C), dilation=(d,1), stride=(s,1))) on [B,T,C] as three accumulated GEMM
    taps over strided views (trainer/model/rnnt_tdnn_transformer.py:44-59, 81-82)."""

    @staticmethod
    def forward(ctx, x, weight, bias, dil, stride, premasked=False):
        B, T, C = x.shape
        ctx.premasked = premasked
        N = weight.shape[0]
        t_out = (T - 2 * dil - 1) // stride + 1
        w_parts = stage_weight(weight)                 # [N, 3*C] row-major == weight[:, 0, k, :] at cols k*C
        a_parts = stage_act(x)
        span = (t_out - 1) * stride + 1
        a_taps = [[p[:, k * dil: k * dil + span: stride, :] for p in a_parts] for k in range(3)]
        b_taps = [[p[:, k * C:(k + 1) * C] for p in w_parts] for k in range(3)]
        y = _new((B, t_out, N), like=x)
        gemm_parts(a_taps, b_taps, y, a_sel=(K.SEL_ZB0, K.SEL_ZERO), b_sel=(K.SEL_ZERO, K.SEL_ZERO), bias=bias.detach(),
                   act=K.ACT_RELU)
        ctx.save_for_backward(x, y)
        ctx.a_parts, ctx.w_parts, ctx.weight, ctx.bias = a_parts, w_parts, weight, bias
        ctx.dil, ctx.stride, ctx.t_out = dil, stride, t_out
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y = ctx.saved_tensors
        B, T, C = x.shape
        N = ctx.weight.shape[0]
        dil, stride, t_out = ctx.dil, ctx.stride, ctx.t_out
        if ctx.premasked:
            dpre = dy.contiguous()                  # BatchNormFn.backward already masked by (y > 0)
        else:
            dpre = torch.empty_like(y)
            K.mask_nz(dy.contiguous(), y, dpre, 1.0)
        d_parts = stage_act(dpre)
        b_taps = [[p[:, k * C:(k + 1) * C] for p in ctx.w_parts] for k in range(3)]
        dx = None
        if ctx.needs_input_grad[0]:
            if stride == 1:
                dx = torch.empty_like(x)
                gemm_parts([d_parts] * 3, b_taps, dx, b_mn=True, a_sel=(K.SEL_ZB0, K.SEL_ZERO),
                           b_sel=(K.SEL_ZERO, K.SEL_ZERO), a_row_off=[0, -dil, -2 * dil])
            else:
                # rows tau = k*dil + t*stride of the three taps are disjoint when the residues differ
                assert len({(k * dil) % stride for k in range(3)}) == 3, "overlapping strided taps not supported"
                dx = torch.zeros_like(x)
                span = (t_out - 1) * stride + 1
                for k in range(3):
                    gemm_parts([d_parts], [b_taps[k]], dx[:, k * dil: k * dil + span: stride, :], b_mn=True,
                               a_sel=(K.SEL_ZB0, K.SEL_ZERO), b_sel=(K.SEL_ZERO, K.SEL_ZERO))
        gw = grad_of(ctx.weight).view(N, 3 * C)
        span = (t_out - 1) * stride + 1
        for k in range(3):
            xt = [p[:, k * dil: k * dil + span: stride, :] for p in ctx.a_parts]
            gemm_parts([d_parts], [xt], gw[:, k * C:(k + 1) * C], a_mn=True, b_mn=True, a_sel=(K.SEL_KZ, K.SEL_ZERO),
                       b_sel=(K.SEL_KZ, K.SEL_ZERO), kz_count=B)
        K.colsum(dpre.view(B * t_out, N), grad_of(ctx.bias))
        return dx, None, None, None, None, None


class CausalConvFn(torch.autograd.Function):
    """relu(Conv1d(C, N, Kw, padding=Kw-1)(x)[..., :-(Kw-1)]) on [B,T,ld] (ld >= C, pad columns zero) -- the causal convolution of
    the transformer prediction net (trainer/model/rnnt_conv_transformer_lm.py:36-46, 74-75).
    Forward: ONE GEMM.  Row (b, t) of the im2col matrix is the window x[b, t-Kw+1 .. t, :], which is contiguous in a left-padded
    [B, T+Kw-1, ld] buffer, so the A operand is an overlapping strided view of that buffer (row pitch ld, K = Kw*ld) and the B
    operand the tap-major staged weight.  dgrad: Kw accumulated taps with row offsets (rows past T read as zero); wgrad: the same
    overlapping view read MN-major, one batched-reduction GEMM into the tap-major gradient, permuted into the [N, C, Kw] layout."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        B, T, ld = x.shape
        N, C, Kw = weight.shape
        assert ld >= C and ld % 8 == 0
        xp = _new((B, T + Kw - 1, ld), like=x, zero=True)
        xp[:, Kw - 1:, :] = x
        a_parts = [p.as_strided((B, T, Kw * ld), ((T + Kw - 1) * ld, ld, 1)) for p in stage_act(xp)]
        w_parts = stage_conv1d_weight(weight, ld)
        y = _new((B, T, N), like=x)
        gemm_parts([a_parts], [w_parts], y, a_sel=(K.SEL_ZB0, K.SEL_ZERO), b_sel=(K.SEL_ZERO, K.SEL_ZERO), bias=bias.detach(),
                   act=K.ACT_RELU)
        ctx.save_for_backward(y)
        ctx.a_parts, ctx.w_parts, ctx.weight, ctx.bias, ctx.shape = a_parts, w_parts, weight, bias, (B, T, ld, N, C, Kw)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        B, T, ld, N, C, Kw = ctx.shape
        dpre = torch.empty_like(y)
        K.mask_nz(dy.contiguous(), y, dpre, 1.0)
        d_parts = stage_act(dpre)
        dx = None
        if ctx.needs_input_grad[0]:
            # dx[t] = sum_k dpre[t + Kw-1-k] W_k; at most 9 (A,B) pairs per launch: 3 taps in the split-bf16 mode, all of them in bf16
            per = 3 if len(d_parts) > 1 else Kw
            dx = _new((B, T, ld), dtype=torch.float32 if len(d_parts) > 1 else None, like=y)
            for k0 in range(0, Kw, per):
                ks = list(range(k0, min(Kw, k0 + per)))
                b_taps = [[p[:, k * ld:(k + 1) * ld] for p in ctx.w_parts] for k in ks]
                gemm_parts([d_parts] * len(ks), b_taps, dx, b_mn=True, a_sel=(K.SEL_ZB0, K.SEL_ZERO), b_sel=(K.SEL_ZERO, K.SEL_ZERO),
                           a_row_off=[Kw - 1 - k for k in ks], accumulate=k0 > 0)
        gw = torch.empty(N, Kw * ld, dtype=torch.float32, device=y.device)
        gemm_parts([d_parts], [ctx.a_parts], gw, a_mn=True, b_mn=True, a_sel=(K.SEL_KZ, K.SEL_ZERO), b_sel=(K.SEL_KZ, K.SEL_ZERO),
                   kz_count=B)
        grad_of(ctx.weight).copy_(gw.view(N, Kw, ld)[:, :, :C].permute(0, 2, 1))
        K.colsum(dpre.view(B * T, N), grad_of(ctx.bias))
        return dx, None, None


class BatchNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bn, train, _w=None, _b=None, relu_input=False):
        # relu_input: x is a ReLU output whose producer was told ``premasked``; backward returns d(pre-ReLU) = dx * (x > 0)
        ctx.relu_input = relu_input
        rows, C = x.shape
        y = torch.empty_like(x)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        ws = torch.empty(2 * C, dtype=torch.float32, device=x.device)
        if train and bn.num_batches_tracked is not None:
            bn.num_batches_tracked += 1
        momentum = bn.momentum
        if momentum is None:            # nn.BatchNorm1d's cumulative average: 1 / num_batches_tracked after the increment (a host read)
            momentum = 1.0 / float(bn.num_batches_tracked) if train and bn.num_batches_tracked is not None else 0.0
        K.bn_fwd(x, y, bn.weight.detach(), bn.bias.detach(), bn.eps, train, momentum, bn.running_mean, bn.running_var, mean, rstd, ws)
        ctx.save_for_backward(x, mean, rstd)
        ctx.bn, ctx.train = bn, train
        return y

    @staticmethod
    def backward(ctx, dy):
        x, mean, rstd = ctx.saved_tensors
        dx = torch.empty_like(x)
        K.bn_bwd(dy.contiguous(), x, dx, ctx.bn.weight.detach(), mean, rstd, ctx.train, ctx.relu_input, grad_of(ctx.bn.weight),
                 grad_of(ctx.bn.bias))
        return dx, None, None, None, None, None


class LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ln, _w=None, _b=None):
        rows, C = x.shape
        y = torch.empty_like(x)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        K.layernorm_fwd(x, y, ln.weight.detach(), ln.bias.detach(), ln.eps, mean, rstd)
        ctx.save_for_backward(x, mean, rstd)
        ctx.ln = ln
        return y

    @staticmethod
    def backward(ctx, dy):
        x, mean, rstd = ctx.saved_tensors
        dx = torch.empty_like(x)
        K.layernorm_bwd(dy.contiguous(), x, dx, ctx.ln.weight.detach(), mean, rstd, grad_of(ctx.ln.weight), grad_of(ctx.ln.bias))
        return dx, None, None, None


_FUSED_ATTN = True          # tests/test_layers_gpu.py and scripts/attn_bench.py set False to run the materialised path on every shape


class AttentionFn(torch.autograd.Function):
    """Multi-head self-attention on a fused QKV tensor [B,T,3D] (q | k | v blocks):
    softmax((Q/sqrt(d)) K^T [masked]) -> dropout -> V   (trainer/model/modules/multi_headed_attn.py:199-223).
    Unmasked (the encoder): the fused wgmma kernels.  ``causal`` / ``key_pad`` (uint8 [B,T], 1 = padding key; the transformer
    prediction net, trainer/model/rnnt_conv_transformer_lm.py:66-70): batched GEMMs + the masked softmax kernel (short label
    sequences; the mask only enters the forward softmax -- a dropped key has probability 0, so its dS is 0 as well).
    ``rel``: the relative-position table R [2m+1, dh] (``self_attn.relative_positions_embeddings.weight``, multi_headed_attn.py:9-41,
    186-229), shared by the key and the value relations; it always takes the materialised path.  The band kernels
    (pk_softmax_masked_relpos_fwd / pk_softmax_relpos_bwd) add QR = (alpha Q) R^T to the scores and reduce Pd / dS onto the 2m+1
    buckets (Pb / dSb, token-major rows); the rest is GEMMs: out += Pb R, G = dO R^T, dQ += alpha dSb R, dR = dSb^T (alpha Q) + Pb^T dO.
    dR is written into ``grad_of(rel)`` (the engine's gradient contract), so no gradient is returned for it.
    ``chunk`` = (chunk_len, chunk_off, left_chunks): the streaming encoder's chunk mask (DESIGN.md "Chunked attention"), on the fused
    kernels' chunk instantiations (head dim 64, bf16) or the chunk-masked softmax; not combined with the other masks."""

    @staticmethod
    def forward(ctx, qkv, heads, drop_p, seed, causal=False, key_pad=None, rel=None, chunk=None):
        B, T, D3 = qkv.shape
        D = D3 // 3
        dh = D // heads
        masked = causal or key_pad is not None
        if chunk is not None and (masked or rel is not None):
            raise NotImplementedError("pika_b200: the chunk mask does not combine with causal / key_pad / relative positions")
        ctx.rel, ctx.chunk = rel, chunk
        ctx.fused = _FUSED_ATTN and qkv.dtype == torch.bfloat16 and dh == 64 and not masked and rel is None
        if ctx.fused:
            # scores / probabilities never leave the SM (pika_b200/csrc/attention_tc.cu)
            qkv = qkv.contiguous()
            out = _new((B, T, D), like=qkv)
            lse = torch.zeros(B * heads * K.attention_lse_stride(T), dtype=torch.float32, device=qkv.device)   # pad entries finite
            alpha = 1.0 / math.sqrt(dh)
            keep_bits = K.attention_keep_bits(B, T, heads, drop_p, qkv.device)   # dropout decisions, for the backward
            K.attention_fwd(qkv, out, lse, heads, alpha, drop_p, seed, keep_bits=keep_bits, chunk=chunk)
            ctx.save_for_backward(qkv, out, lse, keep_bits)
            ctx.meta = (B, T, D, heads, dh, 0, drop_p, seed, alpha)
            return out
        Tp = (T + 7) // 8 * 8
        parts = stage_act(qkv)

        def head_view(p, which):
            return p[:, :, which * D:(which + 1) * D].view(B, T, heads, dh).permute(0, 2, 1, 3)

        q, k, v = ([head_view(p, i) for p in parts] for i in range(3))
        S = torch.empty(B, heads, T, Tp, dtype=torch.float32, device=qkv.device)
        alpha = 1.0 / math.sqrt(dh)
        gemm_parts([q], [k], S[:, :, :, :T], alpha=alpha)
        P = _new((B, heads, T, Tp), like=qkv)
        Pd = _new((B, heads, T, Tp), like=qkv) if drop_p > 0 else P
        rel_out = {}
        if rel is not None:
            nb = rel.shape[0]                                   # 2m + 1 buckets
            r_parts = stage_weight(rel)
            # alpha Q, token-major [B*T*heads, dh]: the A operand of QR and the B operand of dR
            qc = [torch.empty(B * T, D, dtype=torch.bfloat16, device=qkv.device) for _ in parts]
            K.cast_split(qkv.view(B * T, D3)[:, :D], qc[0], qc[1] if len(qc) > 1 else None, scale=alpha)
            qc = [p.view(B * T * heads, dh) for p in qc]
            QR = torch.empty(B * T * heads, (nb + 7) // 8 * 8, dtype=torch.float32, device=qkv.device)
            gemm_parts([qc], [r_parts], QR[:, :nb])
            Pb = torch.empty_like(QR)
            K.softmax_masked_relpos_fwd(S, QR, P, Pd, Pb, T, heads, causal, key_pad, nb // 2, drop_p, seed)
            del QR
            pb_parts = [p[:, :nb] for p in stage_act(Pb)]
            Y = torch.empty(B * T * heads, dh, dtype=torch.float32, device=qkv.device)        # Pb R, added in the PV epilogue
            gemm_parts([pb_parts], [r_parts], Y, b_mn=True)
            rel_out = dict(aux=Y.view(B, T, heads, dh).permute(0, 2, 1, 3), aux_mode=K.AUX_ADD)
            ctx.r_parts, ctx.qc, ctx.pb_parts = r_parts, qc, pb_parts
        elif masked:
            K.softmax_masked_fwd(S, P, Pd, T, T, heads, causal, key_pad, drop_p, seed)
        elif chunk is not None:
            K.softmax_chunk_fwd(S, P, Pd, T, chunk, drop_p, seed)
        else:
            K.softmax_fwd(S, P, Pd, T, drop_p, seed)
        del S
        out = _new((B, T, D), like=qkv)
        pd_parts = stage_act(Pd)
        gemm_parts([[p[:, :, :, :T] for p in pd_parts]], [v], out.view(B, T, heads, dh).permute(0, 2, 1, 3), b_mn=True, **rel_out)
        ctx.save_for_backward(qkv, P)
        ctx.pd_parts, ctx.parts = pd_parts, parts
        ctx.meta = (B, T, D, heads, dh, Tp, drop_p, seed, alpha)
        return out

    @staticmethod
    def backward(ctx, dout):
        if ctx.fused:
            qkv, out, lse, keep_bits = ctx.saved_tensors
            B, T, D, heads, dh, _, drop_p, seed, alpha = ctx.meta
            dqkv = torch.empty_like(qkv)
            K.attention_bwd(qkv, out, dout.contiguous(), lse, dqkv, heads, alpha, drop_p, seed, keep_bits=keep_bits, chunk=ctx.chunk)
            return dqkv, None, None, None, None, None, None, None
        qkv, P = ctx.saved_tensors
        B, T, D, heads, dh, Tp, drop_p, seed, alpha = ctx.meta
        dout = dout.contiguous()

        def head_view(p, which, d=D):
            return p[:, :, which * d:(which + 1) * d].view(B, T, heads, dh).permute(0, 2, 1, 3)

        q, k, v = ([head_view(p, i) for p in ctx.parts] for i in range(3))
        do_parts = stage_act(dout)
        do = [p.view(B, T, heads, dh).permute(0, 2, 1, 3) for p in do_parts]
        dqkv = torch.empty_like(qkv)
        # dV = Pd^T dO
        gemm_parts([[p[:, :, :, :T] for p in ctx.pd_parts]], [do], head_view(dqkv, 2), a_mn=True, b_mn=True)
        # dPd = dO V^T
        dPd = torch.empty(B, heads, T, Tp, dtype=torch.float32, device=qkv.device)
        gemm_parts([do], [v], dPd[:, :, :, :T])
        dS = torch.empty_like(P)
        rel, rel_dq = ctx.rel, {}
        if rel is not None:
            nb = rel.shape[0]
            do2 = [p.view(B * T * heads, dh) for p in do_parts]
            G = torch.empty(B * T * heads, (nb + 7) // 8 * 8, dtype=torch.float32, device=qkv.device)
            gemm_parts([do2], [ctx.r_parts], G[:, :nb])
            dSb = torch.empty_like(G)
            K.softmax_relpos_bwd(dPd, G, P, dS, dSb, T, heads, nb // 2, drop_p, seed)
            del G
            dsb_parts = [p[:, :nb] for p in stage_act(dSb)]
            Z = torch.empty(B * T * heads, dh, dtype=torch.float32, device=qkv.device)        # alpha dSb R, added in the dQ epilogue
            gemm_parts([dsb_parts], [ctx.r_parts], Z, b_mn=True, alpha=alpha)
            rel_dq = dict(aux=Z.view(B, T, heads, dh).permute(0, 2, 1, 3), aux_mode=K.AUX_ADD)
            # dR = dSb^T (alpha Q) + Pb^T dO, reduced over every (sequence, query, head) row
            gemm_parts([dsb_parts, ctx.pb_parts], [ctx.qc, do2], grad_of(rel), a_mn=True, b_mn=True)
        else:
            K.softmax_bwd(dPd, P, dS, T, drop_p, seed)
        del dPd
        ds_parts = [p[:, :, :, :T] for p in stage_act(dS)]
        # dQ = alpha * dS K ; dK = alpha * dS^T Q
        gemm_parts([ds_parts], [k], head_view(dqkv, 0), b_mn=True, alpha=alpha, **rel_dq)
        gemm_parts([ds_parts], [q], head_view(dqkv, 1), a_mn=True, b_mn=True, alpha=alpha)
        return dqkv, None, None, None, None, None, None, None


class EmbeddingFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, idx, emb, ld, _w=None):
        n = idx.numel()
        out = _new((n, ld), like=emb.weight)
        K.embedding_fwd(idx.reshape(-1).contiguous(), emb.weight.detach(), out)
        ctx.idx, ctx.emb = idx.reshape(-1).contiguous(), emb
        return out

    @staticmethod
    def backward(ctx, dout):
        K.embedding_bwd(ctx.idx, dout.contiguous(), grad_of(ctx.emb.weight), ctx.emb.padding_idx)
        return None, None, None, None


def _lstm_step_maps(lens, B, U, rev):
    """Index maps of one direction's per-step path between time and processing step (step s of sequence b is time s, or
    L_b - 1 - s in reverse).  Returns (src, dsrc, to_time), all int32 [U, B] indexed [step or time, b]:
      src     -- row b*U + t of a [B*U, .] tensor that step s reads (clamped to t = 0 once the sequence has finished);
      dsrc    -- the same, but B*U (a zero row) once the sequence has finished;
      to_time -- row s*B + b of a step-major [U*B + 1, .] tensor that holds time t, or U*B (a zero row) for t >= L_b."""
    r = torch.arange(U, dtype=torch.int32, device=lens.device).view(U, 1)
    b = torch.arange(B, dtype=torch.int32, device=lens.device).view(1, B)
    L = lens.view(1, B).clamp(0, U)
    other = (L - 1 - r) if rev else r.expand(U, B)          # time of step r, or step of time r: the map is its own inverse
    live = r < L
    src = b * U + torch.where(live, other, torch.zeros_like(other))
    dsrc = torch.where(live, b * U + other, torch.full_like(other, B * U))
    to_time = torch.where(live, other * B + b, torch.full_like(other, U * B))
    return src, dsrc, to_time


class LstmLayerFn(torch.autograd.Function):
    """One nn.LSTM layer (batch_first, zero initial state) over x [B,U,E] -> [B,U,n_dir*H], for n_dir = 1 or 2 directions (params:
    w_ih, w_hh, b_ih, b_hh of each direction, direction 1 running backwards in time).  ``lens`` (int32 [B] on the device, or None):
    the pack_padded_sequence lengths -- sequence b runs over its first L_b steps, its reverse direction starts at L_b - 1, and
    outputs at t >= L_b are zero (pad_packed_sequence).  The input projection is one GEMM over all steps per direction; the
    recurrence is one cooperative launch for both directions (lstm_seq.cu), or per step a recurrent GEMM + a fused cell kernel
    (fp32-class mode, or shapes outside the persistent kernel's limits)."""

    @staticmethod
    def forward(ctx, x, lens, *params):
        B, U, E = x.shape
        n_dir = len(params) // 4
        dirs = [params[4 * d:4 * d + 4] for d in range(n_dir)]
        H = dirs[0][1].shape[1]
        G4 = 4 * H
        wih_parts = [stage_weight(p[0], cols_pad=E if E != p[0].shape[1] else None) for p in dirs]
        whh_parts = stage_weight([p[1] for p in dirs])                 # [n_dir*4H, H]
        x_parts = stage_act(x)
        gx = torch.empty(n_dir, B, U, G4, dtype=torch.float32, device=x.device)
        for d, (w_ih, w_hh, b_ih, b_hh) in enumerate(dirs):
            bsum = torch.empty(G4, dtype=torch.float32, device=x.device)
            K.add(b_ih.detach(), b_hh.detach(), bsum)
            gemm_parts([[p.view(B * U, E) for p in x_parts]], [wih_parts[d]], gx[d].view(B * U, G4), bias=bsum)
        out = _new((B, U, n_dir * H), like=x)
        gates = torch.empty(n_dir, U, B, G4, dtype=torch.float32, device=x.device)
        cs = torch.empty(n_dir, U, B, H, dtype=torch.float32, device=x.device)
        ctx.persistent = (x.dtype == torch.bfloat16 and H % 64 == 0 and
                          n_dir * H // 8 <= torch.cuda.get_device_properties(x.device).multi_processor_count)  # any batch: 32 sequences per cooperative launch
        if ctx.persistent:
            # whole recurrence of every direction in one cooperative launch (pika_b200/csrc/lstm_seq.cu)
            K.lstm_seq_fwd_ex(gx, whh_parts[0], out, gates, cs, lens)
        else:
            for d in range(n_dir):
                whh = [p[d * G4:(d + 1) * G4] for p in whh_parts]
                out_d = out[:, :, d * H:(d + 1) * H]
                if lens is None and d == 0:                           # step s is time s for every sequence
                    gx_s, h_s = (lambda t: gx[d][:, t, :]), (lambda t: out_d[:, t, :])
                else:
                    src, _, _ = _lstm_step_maps(lens if lens is not None else _full_lens(B, U, x.device), B, U, d == 1)
                    gxs = torch.empty(U * B, G4, dtype=torch.float32, device=x.device)
                    K.gather_rows(gx[d].view(B * U, G4), src.view(-1), gxs)
                    hs = _new((U * B + 1, H), like=x, zero=True)       # step-major; the last row stays zero
                    gx_s, h_s = (lambda t: gxs[t * B:(t + 1) * B]), (lambda t: hs[t * B:(t + 1) * B])
                gh = torch.empty(B, G4, dtype=torch.float32, device=x.device)
                for t in range(U):
                    if t > 0:
                        gemm_parts([stage_act_view(h_s(t - 1))], [whh], gh, block_n=64)
                    K.lstm_cell_fwd(gx_s(t), gh if t > 0 else None, cs[d][t - 1] if t > 0 else None, cs[d][t], h_s(t), gates[d][t], B, H)
                if not (lens is None and d == 0):
                    _, _, to_time = _lstm_step_maps(lens if lens is not None else _full_lens(B, U, x.device), B, U, d == 1)
                    ho = _new((B * U, H), like=x)
                    K.gather_rows(hs, to_time.t().contiguous().view(-1), ho)
                    out_d.copy_(ho.view(B, U, H))
        ctx.save_for_backward(x, out, gates, cs)
        ctx.x_parts, ctx.wih_parts, ctx.whh_parts = x_parts, wih_parts, whh_parts
        ctx.dirs, ctx.lens = dirs, lens
        return out

    @staticmethod
    def backward(ctx, dout):
        x, out, gates, cs = ctx.saved_tensors
        lens, dirs = ctx.lens, ctx.dirs
        n_dir = len(dirs)
        B, U, E = x.shape
        H = dirs[0][1].shape[1]
        G4 = 4 * H
        dout = dout.contiguous()
        dG = _new((n_dir, U, B, G4), like=out)             # time-major: dG[d][t] is a contiguous [B,4H] matrix; zero at t >= L_b
        if ctx.persistent:
            K.lstm_seq_bwd_ex(dout, gates, cs, ctx.whh_parts[0], dG, lens)
        else:
            dh_rec = torch.empty(B, H, dtype=torch.float32, device=x.device)
            dc = [torch.empty(B, H, dtype=torch.float32, device=x.device) for _ in range(2)]
            for d in range(n_dir):
                whh = [p[d * G4:(d + 1) * G4] for p in ctx.whh_parts]
                dout_d = dout[:, :, d * H:(d + 1) * H]
                if lens is None and d == 0:
                    do_s, dg_s = (lambda t: dout_d[:, t, :]), (lambda t: dG[d][t])
                else:
                    # step-major copies; a finished sequence reads a zero gradient, so its dG rows and dc stay exactly zero
                    _, dsrc, to_time = _lstm_step_maps(lens if lens is not None else _full_lens(B, U, x.device), B, U, d == 1)
                    dz = torch.zeros(B * U + 1, H, dtype=dout.dtype, device=x.device)
                    dz[:B * U].view(B, U, H).copy_(dout_d)
                    dos = torch.empty(U * B, H, dtype=dout.dtype, device=x.device)
                    K.gather_rows(dz, dsrc.view(-1), dos)
                    dgs = _new((U * B + 1, G4), like=out, zero=True)
                    do_s, dg_s = (lambda t: dos[t * B:(t + 1) * B]), (lambda t: dgs[t * B:(t + 1) * B])
                for t in range(U - 1, -1, -1):
                    last = (t == U - 1)
                    K.lstm_cell_bwd(do_s(t), None if last else dh_rec, None if last else dc[(t + 1) & 1], gates[d][t], cs[d][t],
                                    cs[d][t - 1] if t > 0 else None, dg_s(t), dc[t & 1], B, H)
                    if t > 0:
                        gemm_parts([stage_act_view(dg_s(t))], [whh], dh_rec, b_mn=True, block_n=64)
                if not (lens is None and d == 0):
                    K.gather_rows(dgs, to_time.view(-1), dG[d].view(U * B, G4))
        dg_all = stage_act(dG)                              # [n_dir,U,B,4H]
        out_parts = stage_act(out)                          # [B,U,n_dir*H]
        sel = dict(a_sel=(K.SEL_KZ, K.SEL_ZERO), b_sel=(K.SEL_KZ, K.SEL_ZERO))
        for d, (w_ih, w_hh, b_ih, b_hh) in enumerate(dirs):
            dg_parts = [p[d] for p in dg_all]
            h_parts = [p[:, :, d * H:(d + 1) * H].permute(1, 0, 2) for p in out_parts]       # [U,B,H]
            # dW_hh = sum_t dG[t]^T h[t-1] (forward) or dG[t]^T h[t+1] (reverse), reduced over batch rows, batched over t;
            # dG is zero past each length and h[L_b] is a zero output, so no masking
            if U > 1:
                a, b = ([p[1:] for p in dg_parts], [p[:-1] for p in h_parts]) if d == 0 else \
                       ([p[:-1] for p in dg_parts], [p[1:] for p in h_parts])
                gemm_parts([a], [b], grad_of(w_hh), a_mn=True, b_mn=True, kz_count=U - 1, **sel)
            else:
                grad_of(w_hh).zero_()
            gemm_parts([dg_parts], [[p.permute(1, 0, 2) for p in ctx.x_parts]], grad_of(w_ih), a_mn=True, b_mn=True, kz_count=U, **sel)
            K.colsum(dG[d].view(U * B, G4), grad_of(b_ih))
            grad_of(b_hh).copy_(b_ih.grad)
        dx = None
        if ctx.needs_input_grad[0]:
            # dx = sum_d dG_d W_ih_d: one GEMM over the directions' (A, B) pairs
            dx = torch.empty_like(x)
            taps = [[p[d] for p in dg_all] for d in range(n_dir)]
            gemm_parts(taps, ctx.wih_parts, dx.permute(1, 0, 2), b_mn=True, a_sel=(K.SEL_ZB0, K.SEL_ZERO), b_sel=(K.SEL_ZERO, K.SEL_ZERO))
        return (dx, None) + (None,) * (4 * n_dir)


def _full_lens(B, U, device):
    return torch.full((B,), U, dtype=torch.int32, device=device)


def stage_act_view(v):
    """stage a (possibly strided-row) 2-D activation view [B, H]."""
    if v.dtype == torch.bfloat16:
        return [v]
    hi = torch.empty(v.shape, dtype=torch.bfloat16, device=v.device)
    lo = torch.empty_like(hi)
    K.cast_split(v, hi, lo)
    return [hi, lo]


class DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p, seed):
        y = torch.empty_like(x)
        K.dropout(x.contiguous(), y, p, seed)
        ctx.p, ctx.seed = p, seed
        return y

    @staticmethod
    def backward(ctx, dy):
        dx = torch.empty_like(dy)
        K.dropout(dy.contiguous(), dx, ctx.p, ctx.seed)
        return dx, None, None


def _ldv(V):
    return (V + 7) // 8 * 8


# the fc2 GEMM epilogue does more work, and the 13.9 GB first pass of the loss goes away.  tests/test_layers_gpu.py sets False
# to compare against the stand-alone first pass
_FUSED_LSE = True


# bf16 training: store the joint gradient only for the rows where it is not all zeros and run the fc2 GEMMs and the gate backward
# on those rows alone (rnnt_loss_compact).  The dense path stays for the fp32-class mode; tests set False to compare the two
_COMPACT_GRAD = True


# measurement hook (bench.py): when set to a dict, single launches of the step are bracketed by CUDA events on the launching stream,
# e.g. EVENT_TAPS["fc2_fwd"] = [(start, end), ...] -- the duration of that kernel INSIDE a real step, not in a loop of its own
EVENT_TAPS = None


class _Tap:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if EVENT_TAPS is not None:
            self.s = torch.cuda.Event(enable_timing=True)
            self.s.record()

    def __exit__(self, *exc):
        if EVENT_TAPS is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            EVENT_TAPS.setdefault(self.name, []).append((self.s, e))


def joint_forward(enc, pred, model, want_lse=False, bounds=None, R=0, nodes=None):
    """The factored gated joint (trainer/model/transducer.py:96-108) over one of three row layouts -> (logits [rows, ldv] act dtype,
    saved state for ``joint_backward``):
      * the dense (b, t, u) grid (default): rows = B*T*U1 and the logits are shaped [B,T,U1,ldv];
      * ``bounds`` [B,T] int32 and ``R``: row (b, t, r) is the joint at (t, bounds[b,t] + r), rows = B*T*R (the pruned loss's windows);
      * ``nodes`` = (ex_idx, py_idx), int32 [rows]: row i joins row ex_idx[i] of enc [B,T,H] with row py_idx[i] of pred [B',U1,H] (the
        MBR alignment nodes); the logits are zero-filled.
    ``want_lse``: the fc2 GEMM also reduces every logits row to per-tile (max, sum-exp) pairs (state["row_lse"], else None) for the
    fused loss, in bf16 when V % 8 == 0."""
    H = enc.shape[-1]
    fc1, fcg, fc2 = model.fc1, model.fc_gate, model.fc2
    V = fc2.weight.shape[0]
    ldv = _ldv(V)
    wx = stage_weight([fc1.weight, fcg.weight])                       # [2H, 2H]; x half = cols [0,H), y half = [H,2H)
    enc_parts = stage_act(enc.reshape(-1, H))
    pred_parts = stage_act(pred.reshape(-1, H))
    ex = _new((enc_parts[0].shape[0], 2 * H), like=enc)
    py = _new((pred_parts[0].shape[0], 2 * H), like=enc)
    gemm_parts([enc_parts], [[p[:, :H] for p in wx]], ex, bias=_cat_bias([fc1.bias, fcg.bias]))
    gemm_parts([pred_parts], [[p[:, H:] for p in wx]], py)
    B, T, U1 = enc.shape[0], enc.shape[1], pred.shape[1]
    rows = nodes[0].shape[0] if nodes is not None else B * T * (R if bounds is not None else U1)
    h = _new((rows, H), like=enc)
    if nodes is not None:
        ex_g, py_g = _new((rows, 2 * H), like=enc), _new((rows, 2 * H), like=enc)
        K.gather_rows(ex, nodes[0], ex_g)
        K.gather_rows(py, nodes[1], py_g)
        ex, py = ex_g, py_g
        K.joint_gate_fwd(ex, py, h, rows, 1, 1, H)
    elif bounds is not None:
        K.joint_gate_pruned_fwd(ex, py, bounds, h, B, T, U1, R, H)
    else:
        K.joint_gate_fwd(ex, py, h, B, T, U1, H)
    w2 = stage_weight(fc2.weight)
    dense = nodes is None and bounds is None
    logits = _new((B, T, U1, ldv) if dense else (rows, ldv), like=enc, zero=(ldv != V or nodes is not None))
    h_parts = stage_act(h)
    del h
    row_lse = None
    if want_lse and _FUSED_LSE and logits.dtype == torch.bfloat16 and V % 8 == 0:
        row_lse = torch.empty(K.row_lse_parts(rows, V, 256), rows, 2, dtype=torch.float32, device=enc.device)
    with _Tap("fc2_fwd"):
        gemm_parts([h_parts], [w2], logits.view(rows, ldv)[:, :V], bias=fc2.bias.detach(), row_lse=row_lse,
                   **({"block_n": 256} if row_lse is not None else {}))
    state = dict(row_lse=row_lse, ex=ex, py=py, h_parts=h_parts, enc_parts=enc_parts, pred_parts=pred_parts, wx=wx,
                 enc_shape=enc.shape, pred_shape=pred.shape, bounds=bounds, R=R, nodes=nodes)
    return logits, state


def joint_backward(dlogits, st, model, need_enc=True, need_pred=True, db2=None, compact=None, accumulate=False):
    """dlogits (``joint_forward``'s logits shape, padding columns zero) -> (d_enc, d_pred) shaped like enc and pred; the joint's
    parameter gradients are written in place, or added to them with ``accumulate``.  db2: the column sums of dlogits when the loss
    kernel already formed them.  compact = (h_c, row_map, row_count) of rnnt_loss_compact (dense layout): dlogits and h_c hold only
    the kept rows, the fc2 GEMMs run over row_count of them and the gate backward reads dh through row_map.  The fc2 input is taken
    out of ``st`` and released before the gate backward."""
    h_parts, row_map, rows = st.pop("h_parts", None), None, None
    if compact is not None:
        h_c, row_map, rows = compact
        h_parts = [h_c]
    dh = _vocab_proj_backward(dlogits.view(-1, dlogits.shape[-1]), h_parts, model.fc2, db2, rows, accumulate)
    del h_parts
    dex, dpy = _gate_backward(st, dh, row_map)
    del dh
    return _gate_input_grads(dex, dpy, st, model, need_enc, need_pred, accumulate)


def _write_grad(p, g, accumulate):
    """p.grad = g, or p.grad += g with ``accumulate``"""
    if accumulate:
        K.add(p.grad, g, p.grad)
    else:
        grad_of(p).copy_(g)


def _vocab_proj_backward(d, x_parts, lin, db=None, a_rows_dev=None, accumulate=False):
    """d [rows, ldv] (act dtype, padding columns 0) = d(loss)/d(x W^T + b) of a projection ``lin`` to V, x staged as ``x_parts`` ->
    dx [rows, K]; dW and db written in place, or added to them with ``accumulate``.  db: the column sums of d if already formed;
    a_rows_dev: int32 device tensor [1], only that many leading rows of d and x take part."""
    V = lin.weight.shape[0]
    d_v = [p[:, :V] for p in stage_act(d)]
    dx = _new((d.shape[0], lin.weight.shape[1]), like=d)
    gemm_parts([d_v], [stage_weight(lin.weight)], dx, b_mn=True, a_rows_dev=a_rows_dev)
    gemm_parts([d_v], [x_parts], grad_of(lin.weight), a_mn=True, b_mn=True, a_rows_dev=a_rows_dev, accumulate=accumulate,
               k_splits=1 if accumulate else 0)
    if db is None:
        db = torch.empty(d.shape[1], dtype=torch.float32, device=d.device)
        K.colsum(d, db)
    _write_grad(lin.bias, db[:V], accumulate)
    return dx


def _gate_backward(st, dh, dh_map=None):
    """dh [rows, H] -> the gate-input gradients dex [B*T, 2H], dpy [B'*U1, 2H] through ``joint_forward``'s row layout (f32 for the
    node layout, whose rows are scatter-added; act dtype otherwise).  dh_map: the compacted rows' map (rnnt_loss_compact)."""
    ex, py, nodes = st["ex"], st["py"], st["nodes"]
    B, T, H = st["enc_shape"]
    U1 = st["pred_shape"][1]
    n_ex, n_py = st["enc_parts"][0].shape[0], st["pred_parts"][0].shape[0]
    if nodes is not None:
        rows = dh.shape[0]
        dex_g, dpy_g = _new((rows, 2 * H), like=dh), _new((rows, 2 * H), like=dh)
        K.joint_gate_bwd(ex, py, dh, dex_g, dpy_g, rows, 1, 1, H)
        dex = torch.zeros(n_ex, 2 * H, dtype=torch.float32, device=dh.device)
        dpy = torch.zeros(n_py, 2 * H, dtype=torch.float32, device=dh.device)
        K.scatter_add_rows(dex_g, nodes[0], dex)
        K.scatter_add_rows(dpy_g, nodes[1], dpy)
        return dex, dpy
    dex, dpy = _new((n_ex, 2 * H), like=dh), _new((n_py, 2 * H), like=dh)
    if st["bounds"] is not None:
        K.joint_gate_pruned_bwd(ex, py, st["bounds"], dh, dex, dpy, B, T, U1, st["R"], H)
    else:
        K.joint_gate_bwd(ex, py, dh, dex, dpy, B, T, U1, H, dh_map=dh_map)
    return dex, dpy


def _gate_input_grads(dex, dpy, st, model, need_enc, need_pred, accumulate):
    """gate-input gradients dex [B*T, 2H], dpy [B'*U1, 2H] -> (d_enc, d_pred); the fc1 / fc_gate gradients written in place, or
    added to them with ``accumulate``.  The GEMMs read dex / dpy in the activation dtype, the bias column sum as given."""
    H = st["enc_shape"][-1]
    fc1, fcg = model.fc1, model.fc_gate
    dex_parts, dpy_parts = stage_act(_to_act(dex)), stage_act(_to_act(dpy))
    g1, gg = grad_of(fc1.weight), grad_of(fcg.weight)
    acc = dict(accumulate=accumulate, k_splits=1 if accumulate else 0)
    for (dparts, xparts, lo) in ((dex_parts, st["enc_parts"], 0), (dpy_parts, st["pred_parts"], H)):
        gemm_parts([[p[:, :H] for p in dparts]], [xparts], g1[:, lo:lo + H], a_mn=True, b_mn=True, **acc)
        gemm_parts([[p[:, H:] for p in dparts]], [xparts], gg[:, lo:lo + H], a_mn=True, b_mn=True, **acc)
    dbx = torch.empty(2 * H, dtype=torch.float32, device=dex.device)
    K.colsum(dex, dbx)
    _write_grad(fc1.bias, dbx[:H], accumulate)
    _write_grad(fcg.bias, dbx[H:], accumulate)
    d_enc = d_pred = None
    if need_enc:
        d_enc = _new((dex.shape[0], H), like=dex)
        gemm_parts([dex_parts], [[p[:, :H] for p in st["wx"]]], d_enc, b_mn=True)
        d_enc = d_enc.view(st["enc_shape"])
    if need_pred:
        d_pred = _new((dpy.shape[0], H), like=dex)
        gemm_parts([dpy_parts], [[p[:, H:] for p in st["wx"]]], d_pred, b_mn=True)
        d_pred = d_pred.view(st["pred_shape"])
    return d_enc, d_pred


class JointFn(torch.autograd.Function):
    """enc [B,T,H], pred [B,U1,H] -> logits [B,T,U1,ldv] (trainer/model/transducer.py:96-108)."""

    @staticmethod
    def forward(ctx, enc, pred, model):
        logits, st = joint_forward(enc, pred, model)
        ctx.st, ctx.model = st, model
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        # a copy: joint_backward takes the fc2 input out of the state it is given, and a retained graph may run this again
        d_enc, d_pred = joint_backward(dlogits.contiguous(), dict(ctx.st), ctx.model, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return d_enc, d_pred, None


_UNIT_LOSS_GRAD = False


def assume_unit_loss_grad(flag):
    """The training step calls ``costs.sum().backward()`` (trainer/train_transducer_bmuf_otfaug.py:97-103), i.e. the upstream
    gradient of every cost is exactly 1.  TrainStep declares that here so JointLossFn.backward does no re-scaling work;
    any other caller gets the general (scaled) backward.  For the pruned loss (transducer_loss_pruned) the declaration is that the
    upstream gradients are exactly the simple / pruned scales it was called with."""
    global _UNIT_LOSS_GRAD
    _UNIT_LOSS_GRAD = bool(flag)


class JointLossFn(torch.autograd.Function):
    """Fused joint + log-softmax + RNN-T loss: the logits tensor is produced, consumed by the loss
    kernels and overwritten IN PLACE by d(loss)/d(logits); the joint backward then runs immediately, so
    only one [B,T,U1,V] tensor ever exists.  Returns costs [B].

    Gradient contract (one place): every Function of this engine OVERWRITES the ``.grad`` of the parameters it owns
    (EmbeddingFn zero-fills, then scatters), so one forward + one backward per ``zero_grad`` is the supported pattern, as in
    the reference loop (:74, :103).  The joint's parameter gradients are produced here in forward for an upstream gradient
    of 1 per utterance; ``backward`` re-scales them (and d_enc / d_pred) when the upstream gradient is a different UNIFORM
    scalar, and scales d_enc / d_pred per utterance otherwise -- per-utterance weights on the joint's OWN parameters are not
    representable after the fact and raise.  With grad mode off (``need_grad`` False: the eval branch of run_one_epoch) only the
    costs are computed and no gradient buffer is touched."""

    @staticmethod
    def forward(ctx, enc, pred, model, labels, frame_lens, label_lens, need_grad=True, fastemit_lambda=0.0, delay_penalty=0.0):
        logits, st = joint_forward(enc, pred, model, want_lse=True)
        V = model.fc2.weight.shape[0]
        ctx.need_grad = need_grad
        reg = dict(fastemit_lambda=fastemit_lambda, delay_penalty=delay_penalty)
        if not need_grad:
            costs, _ = K.rnnt_loss_fwd_bwd(logits, labels, frame_lens, label_lens, V=V, want_grad=False, row_lse=st.pop("row_lse"), **reg)
            return costs
        db2 = torch.empty(logits.shape[-1], dtype=torch.float32, device=logits.device)
        compact = None
        if _COMPACT_GRAD and logits.dtype == torch.bfloat16:
            with _Tap("rnnt_loss"):
                costs, dz_c, h_c, row_map, rows = K.rnnt_loss_compact(logits, labels, frame_lens, label_lens, st["h_parts"][0], V=V,
                                                                      colsum=db2, row_lse=st.pop("row_lse"), **reg)
            logits, compact = dz_c, (h_c, row_map, rows)          # the logits and h are released here: dz_c and h_c replace them
            del dz_c, h_c
            st.pop("h_parts")
        else:
            with _Tap("rnnt_loss"):
                costs, _ = K.rnnt_loss_fwd_bwd(logits, labels, frame_lens, label_lens, V=V, dlogits=logits, colsum=db2,
                                               row_lse=st.pop("row_lse"), **reg)
        d_enc, d_pred = joint_backward(logits, st, model, db2=db2, compact=compact)
        del compact
        del logits, st
        ctx.save_for_backward(d_enc, d_pred)
        ctx.model = model
        return costs

    @staticmethod
    def backward(ctx, dcosts):
        if not ctx.need_grad:
            raise RuntimeError("JointLossFn: forward ran with grad mode off; there is nothing to back-propagate")
        d_enc, d_pred = ctx.saved_tensors
        if not _UNIT_LOSS_GRAD:
            w = dcosts.detach().float()
            if not bool((w == w[0]).all()):
                raise RuntimeError("JointLossFn: per-utterance loss weights are not supported by the fused joint backward "
                                   "(its parameter gradients were formed for a uniform upstream gradient)")
            if float(w[0]) != 1.0:
                m = ctx.model
                for p in (m.fc1.weight, m.fc1.bias, m.fc_gate.weight, m.fc_gate.bias, m.fc2.weight, m.fc2.bias):
                    p.grad.mul_(w[0])
                d_enc = d_enc * w[0].to(d_enc.dtype)
                d_pred = d_pred * w[0].to(d_pred.dtype)
        return d_enc, d_pred, None, None, None, None, None, None, None


class RNNTLossFn(torch.autograd.Function):
    """warp_rnnt.RNNTLoss.apply-compatible: log_probs [B,T,U1,V] -> costs [B] (reference call site
    trainer/train_transducer_bmuf_otfaug.py:58,97-98).  ``fastemit_lambda`` / ``delay_penalty``: check_emission_reg."""

    @staticmethod
    def forward(ctx, log_probs, labels, frame_lens, label_lens, fastemit_lambda=0.0, delay_penalty=0.0):
        fastemit_lambda, delay_penalty = check_emission_reg(fastemit_lambda, delay_penalty)
        lp = log_probs.contiguous()
        B, T, U1, V = lp.shape
        ldv = V if (V % (8 if lp.dtype == torch.bfloat16 else 4) == 0) else None
        if ldv is None:
            ldv = _ldv(V)
            buf = torch.zeros(B, T, U1, ldv, dtype=lp.dtype, device=lp.device)
            buf[..., :V].copy_(lp)
            lp = buf
        costs, grads = K.rnnt_loss_fwd_bwd(lp, labels.int().contiguous(), frame_lens.int().contiguous(),
                                           label_lens.int().contiguous(), V=V, fastemit_lambda=fastemit_lambda, delay_penalty=delay_penalty)
        ctx.save_for_backward(grads[..., :V])
        return costs

    @staticmethod
    def backward(ctx, dcosts):
        (g,) = ctx.saved_tensors
        return g * dcosts.view(-1, 1, 1, 1).to(g.dtype), None, None, None, None, None


# ------------------------------------------------------------------------------------------------
# model assembly
def _to_act(x):
    x = x.contiguous()
    if x.dtype == act_dtype():
        return x
    if act_dtype() == torch.bfloat16:
        x2 = x.reshape(-1, x.shape[-1]).float()
        out = torch.empty(x2.shape, dtype=torch.bfloat16, device=x.device)
        K.cast_split(x2, out)
        return out.view(x.shape)
    return x.float()


def transformer_layer(layer, x2, B, T, training, causal=False, key_pad=None, chunk=None):
    """x2 [B*T, D] -> [B*T, D]   (pre-LN attention block + position-wise FFN); ``causal`` / ``key_pad``, ``chunk`` and the layer's
    relative-position table (when it has one): see AttentionFn.  A chunk mask that admits every key runs the unmasked path."""
    if chunk is not None and K.attention_chunk_admits_all(T, chunk):
        chunk = None
    att, ff = layer.self_attn, layer.feed_forward
    p = _drop(layer.dropout_p, training)
    ln = LayerNormFn.apply(x2, layer.layer_norm, layer.layer_norm.weight, layer.layer_norm.bias)
    qkv = linear(ln, [att.linear_query.weight, att.linear_keys.weight, att.linear_values.weight],
                 [att.linear_query.bias, att.linear_keys.bias, att.linear_values.bias])
    rel = att.relative_positions_embeddings.weight if getattr(att, "max_relative_positions", 0) > 0 else None
    ctxv = AttentionFn.apply(qkv.view(B, T, -1), att.head_count, p, _next_seed() if p > 0 else 0, causal, key_pad, rel, chunk)
    h1 = linear(ctxv.view(B * T, -1), att.final_linear.weight, att.final_linear.bias, drop_p=p, residual=x2)
    ln2 = LayerNormFn.apply(h1, ff.layer_norm, ff.layer_norm.weight, ff.layer_norm.bias)
    fold = ln2.dtype == torch.bfloat16
    inter = linear(ln2, ff.w_1.weight, ff.w_1.bias, act=True, drop_p=p, premasked=fold)
    # w_2's dgrad epilogue applies w_1's ReLU(+dropout) mask: inter != 0 <=> active and kept
    return linear(inter, ff.w_2.weight, ff.w_2.bias, drop_p=p, residual=h1,
                  mask_input_scale=(1.0 / (1.0 - p) if p > 0 else 1.0) if fold else 0.0)


def encoder_forward_act(enc, x, x_len=None, t_out=None):
    """x [B,T,D] -> [B,T',H] in the activation dtype.  An nn.LSTM encoder runs over the packed lengths ``x_len`` (see
    lstm_encoder_forward_act); the TDNN-Transformer encoder ignores them, as the reference does (pack_seq is False).  Its attention
    layers run under the chunk masks of ``enc.chunk_size`` / ``enc.left_chunks`` (Net.chunk_masks; full context at chunk_size 0)."""
    if isinstance(enc, torch.nn.LSTM):
        return lstm_encoder_forward_act(enc, x, x_len, t_out)
    training = enc.training
    B, T, D = x.shape
    C = enc.tdnn_nhid
    if T < 43:
        raise ValueError("encoder input has %d frames; the TDNN stack needs at least 43 (receptive field 21+1+21)" % T)
    chunks = enc.chunk_masks()
    # ReLU masks ride in the BatchNorm backward (pk_bn_bwd relu_mask) instead of separate passes
    h = linear(_to_act(x).view(B * T, D), enc.fc_in.weight, enc.fc_in.bias, act=True, premasked=True)
    h = BatchNormFn.apply(h, enc.bn_in, training, enc.bn_in.weight, enc.bn_in.bias, True)
    for l, (conv, bn) in enumerate(zip(enc.hidden_conv, enc.hidden_bn)):
        dil, stride = enc.TDNN_DIL_STRIDE[l]
        h3 = TdnnFn.apply(h.view(B, T, C), conv.weight, conv.bias, dil, stride, True)
        T = h3.shape[1]
        h = BatchNormFn.apply(h3.view(B * T, C), bn, training, bn.weight, bn.bias, True)
        if (l + 1) % 3 == 0:
            h = transformer_layer(enc.transformer[l // 3], h, B, T, training, chunk=chunks[l // 3])
    h = BatchNormFn.apply(h, enc.bn_final, training, enc.bn_final.weight, enc.bn_final.bias)
    h = linear(h, enc.fc_out.weight, enc.fc_out.bias)
    return h.view(B, T, -1)


def encoder_forward(enc, x):
    return encoder_forward_act(enc, x).float()


def _lstm_layer_params(lstm, l):
    names = ["weight_ih_l%d", "weight_hh_l%d", "bias_ih_l%d", "bias_hh_l%d"]
    sfx = ["", "_reverse"] if lstm.bidirectional else [""]
    return [getattr(lstm, n % l + x) for x in sfx for n in names]


def lstm_encoder_forward_act(lstm, x, x_len=None, t_out=None):
    """The LSTM encoder (trainer/model/transducer.py:38-44,82-86): nn.LSTM (batch_first, optionally bidirectional) over
    pack_padded_sequence(x, x_len, enforce_sorted=False), unpacked again: x [B,T,D] -> [B,T_out,n_dir*H] in the activation dtype,
    zero at t >= x_len[b].  T_out = max(x_len), as pad_packed_sequence returns; a caller that knows it on the host passes ``t_out``
    (the lengths are then not read back), otherwise it is read once.  ``x_len = None``: every sequence runs all T frames (the
    reference's unpacked forward).  Lengths may come in any order.  nn.LSTM's inter-layer dropout runs in training mode only,
    never after the last layer."""
    if lstm.batch_first is not True or not lstm.bias or lstm.proj_size:
        raise NotImplementedError("pika_b200: the LSTM encoder expects nn.LSTM(batch_first=True, bias=True, proj_size=0)")
    B, T, D = x.shape
    lens = None
    if x_len is None:
        t_out = T
    else:
        x_len = torch.as_tensor(x_len)
        if x_len.shape != (B,):
            raise ValueError("x_len must hold one length per sequence (%d), got shape %s" % (B, tuple(x_len.shape)))
        if t_out is None or not x_len.is_cuda:
            lo, hi = (int(v) for v in torch.stack((x_len.min(), x_len.max())).tolist())
            if lo < 1 or hi > T:
                raise ValueError("x_len must lie in [1, %d] (the frames of x); got [%d, %d]" % (T, lo, hi))
            t_out = hi if t_out is None else t_out
        if not 1 <= t_out <= T:
            raise ValueError("t_out = %d must lie in [1, %d]" % (t_out, T))
        lens = x_len.to(device=x.device, dtype=torch.int32).contiguous()
    ld = (D + 7) // 8 * 8
    h = _to_act(x[:, :t_out])
    if ld != D:
        hp = _new((B, t_out, ld), like=h, zero=True)
        hp[:, :, :D] = h
        h = hp
    p = _drop(lstm.dropout, lstm.training)
    for l in range(lstm.num_layers):
        h = LstmLayerFn.apply(h, lens, *_lstm_layer_params(lstm, l))
        if p > 0 and l < lstm.num_layers - 1:
            h = DropoutFn.apply(h, p, _next_seed())
    return h


def prednet_forward_act(model, y):
    """y [B,U] int64 -> [B,U+1,H]: SOS(blank=0) prepend, embedding, LSTM stack with inter-layer dropout
    (trainer/model/transducer.py:90-95)."""
    B, U = y.shape
    sos = torch.zeros(B, 1, dtype=torch.long, device=y.device)
    yy = torch.cat((sos, y.long()), dim=1).contiguous()
    if getattr(model, "decoder_type", "rnn") != "rnn":
        return conv_transformer_lm_forward_act(model.decoder, yy)                  # trainer/model/transducer.py:96-97
    E = model.embed.weight.shape[1]
    ld = (E + 7) // 8 * 8
    h = EmbeddingFn.apply(yy, model.embed, ld, model.embed.weight).view(B, U + 1, ld)
    lstm = model.decoder
    p = _drop(lstm.dropout, lstm.training)
    for l in range(lstm.num_layers):
        h = LstmLayerFn.apply(h, None, *_lstm_layer_params(lstm, l))
        if p > 0 and l < lstm.num_layers - 1:
            h = DropoutFn.apply(h, p, _next_seed())
    return h


def conv_transformer_lm_forward_act(dec, src):
    """Transformer prediction net (trainer/model/rnnt_conv_transformer_lm.py:59-80): src [B,L] int64 (SOS already prepended) ->
    [B,L,output_dim].  Embedding -> num_layers x (causal Conv1d(k=5) + ReLU -> pre-LN transformer layer under the causal +
    padding-key mask, with relative-position attention when ``max_relative_positions`` > 0) -> LayerNorm -> linear_out."""
    B, L = src.shape
    emb = dec.embeddings
    ld = (emb.weight.shape[1] + 7) // 8 * 8
    src = src.contiguous()
    h = EmbeddingFn.apply(src, emb, ld, emb.weight).view(B, L, ld)
    key_pad = src.eq(emb.padding_idx).to(torch.uint8).contiguous() if emb.padding_idx is not None else None     # :66-68
    training = dec.training
    for conv, layer in zip(dec.conv, dec.transformer):
        assert conv.kernel_size[0] - 1 == conv.padding[0] and conv.dilation[0] == 1 and conv.stride[0] == 1
        h = CausalConvFn.apply(h, conv.weight, conv.bias)                          # :74-75
        h = transformer_layer(layer, h.view(B * L, -1), B, L, training, causal=True, key_pad=key_pad).view(B, L, -1)
    hn = LayerNormFn.apply(h.reshape(B * L, -1), dec.layer_norm, dec.layer_norm.weight, dec.layer_norm.bias)
    return linear(hn, dec.linear_out.weight, dec.linear_out.bias).view(B, L, -1)


def model_encoder_forward_act(model, x, x_len=None, t_out=None):
    """The transducer's encoder as Net.forward runs it: over the packed lengths ``x_len`` when ``model.pack_seq`` (the LSTM
    encoder; ``t_out`` = max(x_len) if the caller knows it on the host), over all frames otherwise."""
    if getattr(model, "pack_seq", False):
        return encoder_forward_act(model.encoder, x, x_len, t_out)
    return encoder_forward_act(model.encoder, x)


def transducer_forward(model, x, y, softmax=True, x_len=None, t_out=None):
    """Net.forward drop-in: -> [B,T',U+1,V] fp32 log-probs (softmax=True) or logits.  ``x_len`` / ``t_out``: the packed lengths of
    an LSTM encoder (lstm_encoder_forward_act); ignored by the TDNN-Transformer encoder."""
    enc = model_encoder_forward_act(model, x, x_len, t_out)
    pred = prednet_forward_act(model, y)
    logits = JointFn.apply(enc, pred, model)
    V = model.fc2.weight.shape[0]
    if not softmax:
        return logits[..., :V].float()
    return LogSoftmaxFn.apply(logits, V)


class LogSoftmaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, V):
        out = torch.empty(logits.shape[:-1] + (V,), dtype=torch.float32, device=logits.device)
        K.log_softmax(logits, out, V)
        ctx.save_for_backward(out)
        ctx.ldv, ctx.dt = logits.shape[-1], logits.dtype
        return out

    @staticmethod
    def backward(ctx, dlp):
        # d logits = dlp - softmax * sum(dlp); boundary op of the compatibility API only (the training
        # path uses JointLossFn, which never materialises log-probs)
        (lp,) = ctx.saved_tensors
        g = dlp - lp.exp() * dlp.sum(-1, keepdim=True)
        out = torch.zeros(lp.shape[:-1] + (ctx.ldv,), dtype=ctx.dt, device=lp.device)
        out[..., :lp.shape[-1]] = g.to(ctx.dt)
        return out, None


def check_emission_reg(fastemit_lambda, delay_penalty):
    """-> (fastemit_lambda, delay_penalty) as floats; ValueError unless both are finite and >= 0 (DESIGN.md "FastEmit and delay
    penalty")"""
    lam_f, lam_d = float(fastemit_lambda), float(delay_penalty)
    if not (math.isfinite(lam_f) and math.isfinite(lam_d) and lam_f >= 0.0 and lam_d >= 0.0):
        raise ValueError("emission regularisation needs finite fastemit_lambda >= 0 and delay_penalty >= 0 (got %r, %r)"
                         % (fastemit_lambda, delay_penalty))
    return lam_f, lam_d


def transducer_loss(model, x, y, frame_lens, label_lens, x_len=None, t_out=None, fastemit_lambda=0.0, delay_penalty=0.0):
    """Fused training path: costs [B] with gradients wired to every parameter.  ``x_len`` / ``t_out`` as in transducer_forward
    (the trainer passes the encoder output lengths, which are also ``frame_lens``).  ``fastemit_lambda`` / ``delay_penalty``: FastEmit
    and the delay penalty (DESIGN.md "FastEmit and delay penalty"); the costs are then the delay-penalised ones, and with FastEmit the
    gradients are not those of the costs.  Out-of-range values raise ValueError before any work."""
    lam_f, lam_d = check_emission_reg(fastemit_lambda, delay_penalty)
    enc = model_encoder_forward_act(model, x, x_len, t_out)
    pred = prednet_forward_act(model, y)
    return JointLossFn.apply(enc, pred, model, y.int().contiguous(), frame_lens.int().contiguous(), label_lens.int().contiguous(),
                             torch.is_grad_enabled(), lam_f, lam_d)


# ------------------------------------------------------------------------------------------------
# pruned RNN-T loss (DESIGN.md "Pruned RNN-T"): a simple joiner am[t] + lm[u] gives a full lattice cheaply, its occupancies choose a
# window of R label positions per frame, and the gated joint + fc2 run on those B*T*R rows only.
def _scaled_grads_backward(ctx, dcosts, params, who):
    """Shared backward of the two pruned-loss Functions: their gradients were formed in forward for an upstream gradient equal to
    ``ctx.scale`` per utterance.  TrainStep declares exactly that (assume_unit_loss_grad); any other caller's uniform upstream
    gradient is re-scaled here, and per-utterance weights raise, as in JointLossFn."""
    if not ctx.need_grad:
        raise RuntimeError("%s: forward ran with grad mode off; there is nothing to back-propagate" % who)
    d_enc, d_pred = ctx.saved_tensors
    if not _UNIT_LOSS_GRAD:
        w = dcosts.detach().float()
        if not bool((w == w[0]).all()):
            raise RuntimeError("%s: per-utterance loss weights are not supported (its parameter gradients were formed for a uniform "
                               "upstream gradient)" % who)
        f = float(w[0])
        if f != ctx.scale:
            if ctx.scale == 0.0:
                raise RuntimeError("%s: forward ran with scale 0, so no gradient was formed; pass the scale the loss is weighted by" % who)
            r = f / ctx.scale
            for p in params:
                p.grad.mul_(r)
            d_enc = d_enc * r
            d_pred = d_pred * r
    return d_enc, d_pred


def check_smoothing_scales(lm_only_scale, am_only_scale):
    """-> (lm_only_scale, am_only_scale) as floats; ValueError unless both are >= 0 and their sum is < 1"""
    lam_l, lam_a = float(lm_only_scale), float(am_only_scale)
    if not (lam_l >= 0.0 and lam_a >= 0.0 and lam_l + lam_a < 1.0):
        raise ValueError("simple-loss smoothing needs lm_only_scale >= 0, am_only_scale >= 0 and lm_only_scale + am_only_scale < 1 "
                         "(got %r, %r)" % (lm_only_scale, am_only_scale))
    return lam_l, lam_a


def simple_loss(am, lm, V, B, T, U1, labels, frame_lens, label_lens, R, scale=1.0, need_grad=True, lm_only_scale=0.0, am_only_scale=0.0,
                delay_penalty=0.0):
    """The simple joiner's RNN-T loss from its two projections am [B*T, ldv], lm [B*U1, ldv] (f32, V valid columns) -> (costs [B],
    bounds [B,T] int32 for windows of R, dam, dlm) with dam [B*T, ldv], dlm [B*U1, ldv] (activation dtype, padding columns 0) the
    gradients of sum_b scale * cost_b, or None when ``need_grad`` is False.  R = 0: no bounds (None).
    ``lm_only_scale`` / ``am_only_scale`` (lam_l, lam_a): the lattice's log-probs become mu * full + lam_l * LM-only + lam_a * AM-only,
    mu = 1 - lam_l - lam_a (DESIGN.md "Pruned RNN-T"); costs and bounds are then the smoothed ones.  Both 0: the unsmoothed kernels.
    ``delay_penalty``: the lattice's label arcs carry the delay penalty (DESIGN.md "FastEmit and delay penalty"), so the costs, the bounds
    and the gradients are the penalised ones."""
    lam_l, lam_a = check_smoothing_scales(lm_only_scale, am_only_scale)
    _, lam_d = check_emission_reg(0.0, delay_penalty)
    smooth = lam_l > 0.0 or lam_a > 0.0
    ldv = am.shape[1]
    U1p = (U1 + 7) // 8 * 8
    dev = am.device
    split = _PRECISION == "fp32"

    def parts(rows, cols):
        return [torch.empty(rows, cols, dtype=torch.bfloat16, device=dev) for _ in range(2 if split else 1)]
    E, P = parts(B * T, ldv), parts(B * U1p, ldv)
    am_max = K.rnnt_simple_prep(am, V, B, T, T, E[0], E[1] if split else None)
    lm_max = K.rnnt_simple_prep(lm, V, B, U1, U1p, P[0], P[1] if split else None)
    E3 = [e.view(B, T, ldv) for e in E]
    P3 = [p.view(B, U1p, ldv) for p in P]
    S = torch.empty(B, T, U1p, dtype=torch.float32, device=dev)
    with _Tap("simple_loss"):
        gemm_parts([E3], [P3], S)                                   # S[t,u] = E[t] . P[u]
        if smooth:
            Nl, logq, Na = K.rnnt_simple_smooth_stats(am, lm, V, am_max, lm_max, frame_lens, label_lens, B, T, U1)
            lpb, lpl = K.rnnt_simple_tables_smooth(am, lm, am_max, lm_max, S.view(B * T, U1p), labels, frame_lens, label_lens, B, T, U1,
                                                   Nl, logq, Na, lam_l, lam_a)
        else:
            lpb, lpl = K.rnnt_simple_tables(am, lm, am_max, lm_max, S.view(B * T, U1p), labels, frame_lens, label_lens, B, T, U1)
        costs, gb, gl = K.rnnt_lattice(lpb, lpl, frame_lens, label_lens, B, T, U1, delay_penalty=lam_d)
    del lpb, lpl
    bounds = None
    if R:
        with _Tap("prune_bounds"):
            bounds = K.rnnt_prune_bounds(gb, gl, frame_lens, label_lens, R)
    if not need_grad:
        return costs, bounds, None, None
    scale_t = torch.full((B,), float(scale), dtype=torch.float32, device=dev)
    scale_w = scale_t
    if smooth:                  # the full term's share of the gradient: W = mu * scale * gamma / S, mu in f32 as the kernels form it
        f32 = lambda v: torch.tensor(v, dtype=torch.float32)                 # noqa: E731
        mu = f32(1.0) - f32(lam_l) - f32(lam_a)
        scale_w = torch.full((B,), float(f32(float(scale)) * mu), dtype=torch.float32, device=dev)
    W = parts(B * T, U1p)
    K.rnnt_simple_w(gb, gl, S.view(B * T, U1p), frame_lens, label_lens, scale_w, W[0], W[1] if split else None)
    W3 = [w.view(B, T, U1p) for w in W]
    WP = torch.empty(B, T, ldv, dtype=torch.float32, device=dev)
    WtE = torch.empty(B, U1p, ldv, dtype=torch.float32, device=dev)
    gemm_parts([W3], [P3], WP, b_mn=True)                           # (W P)[t]   = sum_u W[t,u] P[u]
    gemm_parts([W3], [E3], WtE, a_mn=True, b_mn=True)               # (W^T E)[u] = sum_t W[t,u] E[t]
    del W, W3, E, E3, P, P3, S
    dam = _new((B * T, ldv), like=am)
    dlm = _new((B * U1, ldv), like=am)
    if smooth:
        K.rnnt_simple_grad_smooth(am, V, am_max, WP.view(B * T, ldv), T, 0, gb, gl, labels, frame_lens, label_lens, scale_t, logq, Na,
                                  lam_l, lam_a, dam)
        K.rnnt_simple_grad_smooth(lm, V, lm_max, WtE.view(B * U1p, ldv), U1p, 1, gb, gl, labels, frame_lens, label_lens, scale_t, logq, Nl,
                                  lam_l, lam_a, dlm)
    else:
        K.rnnt_simple_grad(am, V, am_max, WP.view(B * T, ldv), T, 0, gb, gl, labels, frame_lens, label_lens, scale_t, dam)
        K.rnnt_simple_grad(lm, V, lm_max, WtE.view(B * U1p, ldv), U1p, 1, gb, gl, labels, frame_lens, label_lens, scale_t, dlm)
    return costs, bounds, dam, dlm


class SimpleLossFn(torch.autograd.Function):
    """Simple-joiner RNN-T loss and the pruning bounds: enc [B,T,H], pred [B,U1,H] -> (costs [B], bounds [B,T] int32).
    am = simple_am_proj(enc), lm = simple_lm_proj(pred) in f32; z[t,u] = am[t] + lm[u] is never formed: the normaliser is
    log(E.P^T) + the row maxes (pk_rnnt_simple_*), the lattice runs on the resulting tables (pk_rnnt_lattice) and its occupancies give the
    bounds (pk_rnnt_prune_bounds).  The gradients (for an upstream gradient of ``scale`` per utterance) are formed here in forward:
    dam = E (.) (W P) and dlm = P (.) (W^T E) plus the blank / label terms, W = scale * occupancy / (E.P^T).  ``lm_only_scale`` /
    ``am_only_scale`` smooth the lattice and ``delay_penalty`` penalises its label arcs, as in simple_loss."""

    @staticmethod
    def forward(ctx, enc, pred, model, labels, frame_lens, label_lens, R, scale, need_grad, lm_only_scale=0.0, am_only_scale=0.0,
                delay_penalty=0.0):
        B, T, H = enc.shape
        U1 = pred.shape[1]
        am_p, lm_p = model.simple_am_proj, model.simple_lm_proj
        V = am_p.weight.shape[0]
        ldv = _ldv(V)
        enc_parts = stage_act(enc.reshape(B * T, H))
        pred_parts = stage_act(pred.reshape(B * U1, H))
        am = torch.zeros(B * T, ldv, dtype=torch.float32, device=enc.device)
        lm = torch.zeros(B * U1, ldv, dtype=torch.float32, device=enc.device)
        gemm_parts([enc_parts], [stage_weight(am_p.weight)], am[:, :V], bias=am_p.bias.detach())
        gemm_parts([pred_parts], [stage_weight(lm_p.weight)], lm[:, :V], bias=lm_p.bias.detach())
        costs, bounds, dam, dlm = simple_loss(am, lm, V, B, T, U1, labels, frame_lens, label_lens, R, scale, need_grad, lm_only_scale,
                                              am_only_scale, delay_penalty)
        del am, lm
        ctx.mark_non_differentiable(bounds)
        ctx.need_grad, ctx.scale, ctx.model = need_grad, float(scale), model
        if need_grad:
            d_enc = _vocab_proj_backward(dam, enc_parts, am_p).view(B, T, H)
            d_pred = _vocab_proj_backward(dlm, pred_parts, lm_p).view(B, U1, H)
            ctx.save_for_backward(d_enc, d_pred)
        return costs, bounds

    @staticmethod
    def backward(ctx, dcosts, _dbounds):
        m = ctx.model
        d_enc, d_pred = _scaled_grads_backward(ctx, dcosts, (m.simple_am_proj.weight, m.simple_am_proj.bias, m.simple_lm_proj.weight,
                                                             m.simple_lm_proj.bias), "SimpleLossFn")
        return d_enc, d_pred, None, None, None, None, None, None, None, None, None, None


class PrunedJointLossFn(torch.autograd.Function):
    """Pruned joint + RNN-T loss: row (b, t, r) of the joint is the gated joint at (t, bounds[b,t] + r) (pk_joint_gate_pruned_fwd),
    fc2 runs on the B*T*R rows (with the row log-sum-exp epilogue in bf16), the loss and its gradient come from pk_rnnt_pruned_loss
    (in place over the logits), and the joint backward runs at once, as in JointLossFn.  Gradients are formed for an upstream
    gradient of ``scale`` per utterance.  ``fastemit_lambda`` / ``delay_penalty`` as in transducer_loss."""

    @staticmethod
    def forward(ctx, enc, pred, model, labels, frame_lens, label_lens, bounds, R, scale, need_grad, fastemit_lambda=0.0, delay_penalty=0.0):
        U1 = pred.shape[1]
        V = model.fc2.weight.shape[0]
        logits, st = joint_forward(enc, pred, model, want_lse=True, bounds=bounds, R=R)
        row_lse = st.pop("row_lse")
        ctx.need_grad, ctx.scale, ctx.model = need_grad, float(scale), model
        reg = dict(fastemit_lambda=fastemit_lambda, delay_penalty=delay_penalty)
        if not need_grad:
            return K.rnnt_pruned_loss(logits, labels, frame_lens, label_lens, bounds, U1, R, V, row_lse=row_lse, **reg)
        scale_t = torch.full((enc.shape[0],), float(scale), dtype=torch.float32, device=enc.device)
        db2 = torch.empty(logits.shape[-1], dtype=torch.float32, device=enc.device)
        with _Tap("rnnt_loss"):
            costs = K.rnnt_pruned_loss(logits, labels, frame_lens, label_lens, bounds, U1, R, V, grad_scale=scale_t, dlogits=logits,
                                       colsum=db2, row_lse=row_lse, **reg)
        del row_lse
        d_enc, d_pred = joint_backward(logits, st, model, db2=db2)
        ctx.save_for_backward(d_enc, d_pred)
        return costs

    @staticmethod
    def backward(ctx, dcosts):
        m = ctx.model
        d_enc, d_pred = _scaled_grads_backward(ctx, dcosts, (m.fc1.weight, m.fc1.bias, m.fc_gate.weight, m.fc_gate.bias, m.fc2.weight,
                                                             m.fc2.bias), "PrunedJointLossFn")
        return d_enc, d_pred, None, None, None, None, None, None, None, None, None, None


def check_prune_feasible(frame_lens, label_lens, prune_range):
    """Raise ValueError naming every utterance with U > T (R - 1): no path through the lattice fits in windows of R label positions
    (each frame advances a window by at most R - 1).  Reads the lengths on the host."""
    R = int(prune_range)
    if R < 2:
        raise ValueError("prune_range must be >= 2 (got %d)" % R)
    fl = torch.as_tensor(frame_lens).long().cpu()
    ll = torch.as_tensor(label_lens).long().cpu()
    bad = torch.nonzero(ll > fl * (R - 1)).flatten().tolist()
    if bad:
        raise ValueError("pruned RNN-T loss: utterance(s) %s have more labels than frames x (prune_range - 1) = %s; no alignment fits "
                         "in windows of %d label positions (raise --prune_range or drop them)"
                         % (bad, ["U=%d > T=%d x %d" % (int(ll[i]), int(fl[i]), R - 1) for i in bad], R))


def transducer_loss_pruned(model, x, y, frame_lens, label_lens, prune_range, simple_scale, pruned_scale, x_len=None, t_out=None,
                           lm_only_scale=0.0, am_only_scale=0.0, fastemit_lambda=0.0, delay_penalty=0.0):
    """Pruned RNN-T training path -> (simple_costs [B], pruned_costs [B]).  The gradients wired to every parameter are those of
    sum_b (simple_scale * simple_b + pruned_scale * pruned_b); back-propagate exactly that sum (TrainStep does).  Refuses, before any
    work, an utterance that has no path inside the windows.  With grad mode off only the costs are computed.  ``model`` needs the
    simple projections (Net with prune_range > 0).  ``lm_only_scale`` / ``am_only_scale`` smooth the simple loss (simple_loss); its
    costs and the bounds are then the smoothed ones.  ``delay_penalty`` applies to both losses (so the bounds come from the penalised
    simple lattice) and ``fastemit_lambda`` to the pruned loss only (DESIGN.md "FastEmit and delay penalty").  Out-of-range scales raise
    ValueError before any work."""
    lam_l, lam_a = check_smoothing_scales(lm_only_scale, am_only_scale)
    lam_f, lam_d = check_emission_reg(fastemit_lambda, delay_penalty)
    check_prune_feasible(frame_lens, label_lens, prune_range)
    if not hasattr(model, "simple_am_proj"):
        raise ValueError("the pruned RNN-T loss needs the simple joiner: build Net with prune_range > 0")
    R = int(prune_range)
    fl, ll = frame_lens.int().contiguous(), label_lens.int().contiguous()
    labels = y.int().contiguous()
    need = torch.is_grad_enabled()
    enc = model_encoder_forward_act(model, x, x_len, t_out)
    pred = prednet_forward_act(model, y)
    simple_costs, bounds = SimpleLossFn.apply(enc, pred, model, labels, fl, ll, R, float(simple_scale), need, lam_l, lam_a, lam_d)
    pruned_costs = PrunedJointLossFn.apply(enc, pred, model, labels, fl, ll, bounds, R, float(pruned_scale), need, lam_f, lam_d)
    return simple_costs, pruned_costs


# ------------------------------------------------------------------------------------------------
# forced alignment (DESIGN.md "Forced alignment")
def transducer_align(model, x, y, frame_lens, label_lens, x_len=None, t_out=None, prune_range=0):
    """Viterbi alignment of known transcripts -> (emit_frames [B, Umax] int32, viterbi [B] f32, loglik [B] f32), Umax = y.shape[1].
    emit_frames[b, u] is the encoder frame on which the best path through the RNN-T lattice emits label u (-1 from label_lens[b] on, and
    everywhere when no path has a finite score), viterbi[b] that path's log-probability (-inf when there is none) and loglik[b] =
    log P(y | x) summed over every path.  Runs without gradients; ``x_len`` / ``t_out`` as in transducer_forward.
    ``prune_range`` R >= 2: the lattice is the pruned loss's, with the simple joiner's windows of R label positions per frame (the model
    needs simple_am_proj; an utterance with no path inside the windows raises ValueError before any work) and loglik the
    log-likelihood over the windows.  0: the dense joint."""
    R = int(prune_range)
    if R != 0:
        check_prune_feasible(frame_lens, label_lens, R)
        if not hasattr(model, "simple_am_proj"):
            raise ValueError("alignment with prune_range needs the simple joiner: build Net with prune_range > 0")
    fl, ll = frame_lens.int().contiguous(), label_lens.int().contiguous()
    labels = y.int().contiguous()
    with torch.no_grad():
        enc = model_encoder_forward_act(model, x, x_len, t_out)
        pred = prednet_forward_act(model, y)
        B, T, _ = enc.shape
        U1 = pred.shape[1]
        V = model.fc2.weight.shape[0]
        if R:
            _, bounds = SimpleLossFn.apply(enc, pred, model, labels, fl, ll, R, 1.0, False)
            logits, st = joint_forward(enc, pred, model, want_lse=True, bounds=bounds, R=R)
            lpb, lpl = K.rnnt_pruned_tables(logits, labels, fl, ll, bounds, U1, R, V, row_lse=st["row_lse"])
        else:
            logits, st = joint_forward(enc, pred, model, want_lse=True)
            lpb, lpl = K.rnnt_tables(logits, labels, fl, ll, V=V, row_lse=st["row_lse"])
        del logits, st
        with _Tap("lattice"):
            loglik = -K.rnnt_lattice_costs(lpb, lpl, fl, ll, B, T, U1)
        with _Tap("viterbi"):
            viterbi, frames = K.rnnt_viterbi(lpb, lpl, fl, ll, B, T, U1, ld_emit=y.shape[1])
    return frames, viterbi, loglik
