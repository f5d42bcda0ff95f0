"""Every engine layer in the bf16 training precision, with dropout on, against float64 at the shapes bench.py trains (B = 32, T = 1000
input frames, d_model 1024, d_ff 4096, heads 16 / 16 / 8, H = 1024, U1 = 151, V = 6000).

tests/test_layers_gpu.py checks the same Functions in the fp32-class mode at small shapes; the bf16 mode takes other code: bf16 operands
with no lo part, bf16 GEMM epilogues (bias, ReLU, dropout, residual, the AUX_MASK_NZ dgrad mask), the FFN fold (w_1 premasked, its
ReLU + dropout mask applied in w_2's dgrad epilogue), the one-launch causal-convolution dgrad, the fused attention with keep bits, and
the joint loss's fused row log-sum-exp and compacted gradient.

Each Function is checked in isolation against tests/layers_bf16_oracle.py: the reference takes the engine's own bf16 inputs and
incoming gradients, the weights rounded to bf16 as stage_weight rounds them, and the masks the engine drew (ReLU: y != 0; GEMM-epilogue
and stand-alone dropout: pk_dropout on ones with the seed the layer drew; attention: the keep bits).  The bounds are element-wise
(see the oracle's docstring) and every case states the largest |got - ref| / bound measured on an H100.  The composed cases (the
transformer block, and fc_in -> BatchNorm(relu_input)) run the engine's whole graph and check each Function's forward and backward from
the tensors it saw, so a mask moved from one Function into another is checked where it lands.

Every case also asserts, through a recording proxy for pika_b200.kernels.lib, that the path it claims ran, before any numeric check.
Where a case claims split-K in a weight gradient, it also observes it: the same GEMM launched without split-K gives other bits.
f32 gradients whose reference reads the engine's exact operands are also held to a norm-relative bound (NREL_F32), which the
element-wise gamma_K bound at K = 32 000 is too loose to replace; every output's norm-relative error is printed with -s.

Measured on an H100 80GB HBM3 (700 W), largest |got - ref| / bound per test (the module prints them all with -s; 42 tests, 33 s):
  bf16 outputs reach up to 1.0 where the accumulation error is far below half an ulp, because the final rounding's half ulp is
  attained (and autograd's bf16 sum of two bf16 gradients lands on rounding ties); the f32 weight and bias gradients, whose bound is
  the gamma_K accumulation term, stay below 3e-3 (the joint's fc2 gradients, which carry the loss gradient's bound, 0.064):
    test_linear             y 0.994, dx 0.882, dW 7.8e-4, db 1.7e-5
    test_tdnn               y 0.498, dx 0.756, dW 2.7e-4, db 7.1e-6
    test_fc_in_batchnorm    BN y 1.0, dx 1.0, dw 3.3e-6, db 7.4e-7; fc_in y 0.978, dx 0.892, dW 2.6e-5
    test_layernorm          y 0.973, dx 0.955, dw 2.5e-5, db 5.3e-6
    test_attention          out 0.84, dqkv 0.753 (causal + key_pad); fused 0.31 / 0.50; chunk 0.54 / 0.73
    test_transformer_layer  block input gradient 1.0 (a bf16 sum), stage outputs <= 0.99, d(pre) of w_1 through the fold 0.53,
                            weight gradients <= 2.5e-3
    test_embedding_dropout  0 (bit-exact)
    test_causal_conv        y 0.938, dx 0.759, dW 4.0e-4, db 7.9e-6
    test_joint_loss         ex / py / h / logits <= 0.889, cost 6.2e-4, fc2 dW 0.063, fc2 db 0.036, fc1 / fc_gate <= 2.8e-3,
                            d_enc / d_pred 2.2e-3
    test_log_softmax        log-probabilities 0.105, dz 1.0 (the bf16 cast of an f32 value)
    test_joint_fn           ex / py / h / logits <= 0.889, fc2 dW 1.2e-4, db 4.0e-7, fc1 / fc_gate <= 4.1e-4, d_enc / d_pred 2.8e-4
    test_simple_and_pruned_loss  simple am / lm 2.7e-3, simple cost 5.3e-3, simple projections' dW 0.032; pruned ex / py / h /
                            logits <= 0.888, cost 5.0e-4, fc2 dW 0.118, fc2 db 0.071, fc1 / fc_gate <= 0.011, d_enc 0.014, d_pred 0.087
    test_attention_relpos   out 0.283, dq 0.066, dk 0.029, dv 0.227, dR 3.1e-4
    test_lstm_prednet       recurrence: gates <= 0.52, c 0.64, h 1.0 (half ulp attained), dG 0.992; gx 0.014, dx 0.517,
                            dW_ih / dW_hh <= 2.3e-3, biases 2.4e-5
"""
import math

import pytest
import torch
import torch.nn as nn

import layers_bf16_oracle as O

pytestmark = pytest.mark.gpu

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False

B, T_IN, D, DFF, H, U1, V = 32, 1000, 1024, 4096, 1024, 151, 6000
XF_T = {0: 994, 1: 976, 2: 240}          # frames seen by the three encoder attention layers (after TDNN 3, 6 and 9)
_WORST = {}
_NREL = {}
# norm-relative bound for f32 gradients whose reference reads exactly the operands the engine's GEMM or reduction read: fp32
# accumulation over K <= 32 000 rows of random-signed terms moves them by a few sqrt(K) u32 (measured on an H100: at most 3.7e-5),
# while one lost or doubled row of 32 000 random rows moves them by about 1 / sqrt(32 000) ~ 6e-3
NREL_F32 = 2e-4


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _WORST:
        print("\nlargest err / bound: " + ", ".join("%s %.3g" % kv for kv in sorted(_WORST.items())))
        print("\nnorm-relative error: " + ", ".join("%s %.3g" % kv for kv in sorted(_NREL.items())))


@pytest.fixture(autouse=True)
def bf16_mode():
    from pika_b200 import engine as E
    prev, drop = E.get_precision(), E._DROPOUT_ENABLED
    E.set_precision("bf16")
    E.set_dropout_enabled(True)
    try:
        yield E
    finally:
        E.set_precision(prev)
        E.set_dropout_enabled(drop)
        torch.cuda.empty_cache()


def check(name, got, ref, bound, nrel=None):
    """|got - ref| <= bound element by element, and ||got - ref|| <= nrel ||ref|| when given; records the worst ratio and the
    norm-relative error under ``name``"""
    assert got.shape == ref.shape, (name, tuple(got.shape), tuple(ref.shape))
    r = O.worst(got, ref, bound)
    n = O.norm_rel(got, ref)
    _WORST[name] = max(_WORST.get(name, 0.0), r)
    _NREL[name] = max(_NREL.get(name, 0.0), n)
    assert r <= 1.0, "%s: |got - ref| reaches %.3g of the bound (norm-relative error %.3g)" % (name, r, n)
    assert nrel is None or n <= nrel, "%s: norm-relative error %.3g above %.3g" % (name, n, nrel)
    return r


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def randn(*shape, seed, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device="cuda", generator=gen(seed)) * scale).to(dtype)


def w16(p):
    """a parameter as stage_weight stages it"""
    return p.detach().bfloat16().double()


def f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------ path recording
class Recorder:
    """stands in for pika_b200.kernels.lib: every C ABI call goes through, and is recorded as its name and, for pk_gemm_bf16, the
    descriptor fields that select a path"""

    def __init__(self, lib):
        self._lib, self.calls, self.on = lib, [], True

    def stop(self):
        """stop recording: the reference computations that follow call kernels of their own (pk_dropout for the masks)"""
        self.on = False

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*args):
            if not self.on:
                return fn(*args)
            rec = {"name": name}
            if name == "pk_gemm_bf16":
                d = args[0]
                K = d.a[0].dim[1] if d.a_mn_major else d.a[0].dim[0]
                rec.update(n_pairs=d.n_pairs, M=d.c.dim[1], N=d.c.dim[0], zb=d.c.dim[2] * d.c.dim[3], K=K, kz=d.kz_count,
                           a_mn=d.a_mn_major, b_mn=d.b_mn_major, c_f32=d.c_dtype == 0, acc=d.c_accumulate, bias=bool(d.bias),
                           act=d.act, drop_p=d.drop_p, aux_mode=d.aux_mode if d.aux else 0, aux_scale=d.aux_scale,
                           block_n=d.block_n, k_splits=d.k_splits, row_lse=bool(d.row_lse), a_rows=bool(d.a_rows_dev))
            self.calls.append(rec)
            return fn(*args)
        return call

    def names(self):
        return [c["name"] for c in self.calls]

    def gemms(self, **match):
        return [c for c in self.calls if c["name"] == "pk_gemm_bf16" and all(c[k] == v for k, v in match.items())]


def auto_splits(g):
    """the split-K count pk_gemm_bf16 chooses for a recorded call (gemm.cu: a plain f32 2-D C whose grid is short of 6 waves and
    whose reduction has >= 16 k-blocks is split in the count that wastes the least of the last wave)"""
    if g["k_splits"] > 0:
        return g["k_splits"]
    bn = g["block_n"] or (64 if g["N"] <= 64 else 128 if g["N"] <= 128 else 256)
    tiles = -(-g["M"] // 128) * -(-g["N"] // bn) * g["zb"]
    iters = g["n_pairs"] * g["kz"] * -(-g["K"] // 64)
    w = torch.cuda.get_device_properties(0).multi_processor_count
    plain = not g["bias"] and g["act"] == 0 and g["drop_p"] == 0 and g["aux_mode"] == 0
    if not (g["c_f32"] and plain and g["zb"] == 1 and iters >= 16 and tiles < 6 * w and (not g["a_rows"] or g["a_mn"])):
        return 1
    best, sp_best = 0.0, 1
    for sp in range(1, min(16, iters // 8) + 1):
        units = tiles * sp
        eff = units / (-(-units // w) * w)
        if eff > best + 0.02:
            best, sp_best = eff, sp
    return sp_best


@pytest.fixture
def rec(monkeypatch):
    from pika_b200 import kernels as K
    r = Recorder(K.lib)
    monkeypatch.setattr(K, "lib", r)
    return r


class Spy:
    """stands in for an engine autograd Function: records (args, output) of every apply and retains the output's gradient"""

    def __init__(self, fn, log):
        self.fn, self.log = fn, log

    def apply(self, *args):
        for a in args:
            if isinstance(a, torch.Tensor) and a.requires_grad and not a.is_leaf:
                a.retain_grad()
        out = self.fn.apply(*args)
        if out.requires_grad:
            out.retain_grad()
        self.log.append((self.fn.__name__, args, out))
        return out


@pytest.fixture
def spy(monkeypatch):
    from pika_b200 import engine as E
    from pika_b200 import kernels as K
    log, bits = [], []
    for name in ("LinearFn", "LayerNormFn", "AttentionFn", "BatchNormFn", "TdnnFn", "CausalConvFn", "DropoutFn", "EmbeddingFn",
                 "LstmLayerFn"):
        monkeypatch.setattr(E, name, Spy(getattr(E, name), log))
    real_bits = K.attention_keep_bits

    def keep_bits(*a):
        t = real_bits(*a)
        bits.append(t)
        return t
    monkeypatch.setattr(K, "attention_keep_bits", keep_bits)
    return log, bits


def keep_scaled(M, N, p, seed):
    """the dropout keep mask times its scale that the GEMM epilogue and pk_dropout draw for an [M, N] tensor with ``seed``"""
    from pika_b200 import kernels as K
    ones = torch.ones(M, N, device="cuda")
    out = torch.empty_like(ones)
    K.dropout(ones, out, p, seed)
    return out.double()


class Grads:
    """float64 gradient contributions per input tensor, summed as autograd sums them (bf16 adds: one more rounding per add)"""

    def __init__(self):
        self.ref, self.bound, self.n = {}, {}, {}

    def add(self, t, ref, bound):
        k = id(t)
        if k in self.ref:
            self.ref[k] = self.ref[k] + ref
            self.bound[k] = self.bound[k] + bound
        else:
            self.ref[k], self.bound[k] = ref, bound
        self.n[k] = self.n.get(k, 0) + 1

    def check(self, name, t):
        k = id(t)
        ref, bound = self.ref[k], self.bound[k]
        if self.n[k] > 1 and t.grad.dtype == torch.bfloat16:
            bound = bound + O.half_ulp(ref.abs() + bound, torch.bfloat16) * (self.n[k] - 1)
        return check(name, t.grad.view(ref.shape), ref, bound)


# ------------------------------------------------------------------------------------------------ per-Function checks
def check_linear(tag, args, out, grads, mask_input_scale=None):
    """forward of one LinearFn call, its parameter gradients, and its input / residual gradient contributions.  mask_input_scale: the
    scale the reference applies with the (x != 0) dgrad mask, when the caller derives it (default: the one the call was given)"""
    x, residual, act, drop_p, seed, nw, premasked, mis = args[:8]
    params = args[8:]
    weights, biases = params[:nw], params[nw:]
    x64 = x.detach().double()
    M, Kx = x64.shape
    W = torch.cat([w16(w).reshape(w.shape[0], -1) for w in weights])
    Kw = W.shape[1]
    if Kx != Kw:
        W = torch.cat([W, W.new_zeros(W.shape[0], Kx - Kw)], 1)
    N = W.shape[0]
    b = torch.cat([p.detach().double() for p in biases]) if biases else None
    keep = keep_scaled(M, N, drop_p, seed) if drop_p > 0 else None
    res = residual.detach().double() if residual is not None else None
    y, inner = O.linear_fwd(x64, W, b, act, keep, res)
    check(tag + " y", out, y, O.stored(y, inner, torch.bfloat16))
    del y, inner
    dy = out.grad.double()
    if premasked:
        dpre = dy
    elif act:
        dpre = O.bf16r(dy * (out != 0) * (f32(1.0 / (1.0 - drop_p)) if drop_p > 0 else 1.0))
    elif drop_p > 0:
        dpre = O.bf16r(dy * keep)
    else:
        dpre = dy
    del keep
    if mask_input_scale is not None:
        mis = mask_input_scale
    xm = (x64 != 0) * f32(mis) if mis > 0 else None
    (dx, dxi), (dw, dwi), (db, dbi) = O.linear_bwd(dpre, x64, W, xm)
    if x.requires_grad:
        grads.add(x, dx, O.stored(dx, dxi, torch.bfloat16))
    if residual is not None and residual.requires_grad:
        grads.add(residual, dy, torch.full_like(dy, O.TINY))
    r = 0
    for i, w in enumerate(weights):
        n = w.shape[0]
        g, gi = dw[r:r + n, :Kw], dwi[r:r + n, :Kw]
        check(tag + " dW", w.grad.view(n, -1), g, O.stored(g, gi, torch.float32), NREL_F32)
        if biases:
            check(tag + " db", biases[i].grad, db[r:r + n], O.stored(db[r:r + n], dbi[r:r + n], torch.float32), NREL_F32)
        r += n


def check_layernorm(tag, args, out, grads):
    x, ln = args[0], args[1]
    x64 = x.detach().double()
    y, inner, st = O.norm_fwd(x64, ln.weight.detach().double(), ln.bias.detach().double(), ln.eps, 1)
    check(tag + " y", out, y, O.stored(y, inner, torch.bfloat16))
    (dx, dxi), (dw, dwi), (db, dbi) = O.norm_bwd(out.grad.double(), st, ln.weight.detach().double(), 1, True)
    grads.add(x, dx, O.stored(dx, dxi, torch.bfloat16))
    check(tag + " dw", ln.weight.grad, dw, O.stored(dw, dwi, torch.float32), NREL_F32)
    check(tag + " db", ln.bias.grad, db, O.stored(db, dbi, torch.float32), NREL_F32)


def check_batchnorm(tag, args, out, grads, stats):
    """stats: (running_mean, running_var) as they were before the forward, for eval mode"""
    x, bn, train = args[0], args[1], args[2]
    relu_input = args[5] if len(args) > 5 else False
    x64 = x.detach().double()
    w, b = bn.weight.detach().double(), bn.bias.detach().double()
    if train:
        y, inner, st = O.norm_fwd(x64, w, b, bn.eps, 0)
    else:
        y, inner, st = O.norm_fwd(x64, w, b, bn.eps, 0, stats[0].double()[None], stats[1].double()[None])
    check(tag + " y", out, y, O.stored(y, inner, torch.bfloat16))
    del y, inner
    (dx, dxi), (dw, dwi), (db, dbi) = O.norm_bwd(out.grad.double(), st, w, 0, train)
    if relu_input:
        dx, dxi = dx * (x64 > 0), dxi * (x64 > 0)
    grads.add(x, dx, O.stored(dx, dxi, torch.bfloat16))
    check(tag + " dw", bn.weight.grad, dw, O.stored(dw, dwi, torch.float32), NREL_F32)
    check(tag + " db", bn.bias.grad, db, O.stored(db, dbi, torch.float32), NREL_F32)


def check_attention(tag, args, out, grads, bits):
    """one AttentionFn call: per group of (sequence, head) pairs, the float64 forward and backward of test_attention_kernels_gpu with
    the engine's dropout mask -- decoded from the keep bits on the fused path, drawn from the shared generator on the materialised one"""
    from test_attention_kernels_gpu import attention_tols, drop_mask, drop_params, ref_attention_bwd
    from test_attention_keep_bits_gpu import decode_keep_bits
    qkv, heads, p, seed, causal, key_pad, rel, chunk = args
    assert rel is None
    Bq, T, D3 = qkv.shape
    Dm = D3 // 3
    dh = Dm // heads
    alpha = 1.0 / math.sqrt(dh)
    scale = drop_params(p)[1]
    fused = dh == 64 and not causal and key_pad is None
    if p > 0:
        M = decode_keep_bits(bits, Bq * heads, T) if fused else drop_mask(Bq * heads * T, T, p, seed).view(Bq * heads, T, T)
    allowed = None
    if chunk is not None:
        from chunk_oracle import allowed as chunk_allowed
        allowed = chunk_allowed(T, *chunk).cuda()[None]

    def heads_of(t, i):
        return t[:, :, i * Dm:(i + 1) * Dm].reshape(Bq, T, heads, dh).permute(0, 2, 1, 3).reshape(Bq * heads, T, dh)
    q, k, v = (heads_of(qkv.detach(), i).double() for i in range(3))
    o = out.detach().view(Bq, T, heads, dh).permute(0, 2, 1, 3).reshape(Bq * heads, T, dh)
    do = out.grad.view(Bq, T, heads, dh).permute(0, 2, 1, 3).reshape(Bq * heads, T, dh)
    dq_ref = torch.empty(3, Bq * heads, T, dh, dtype=torch.float64, device="cuda")
    dq_bnd = torch.empty_like(dq_ref)
    step = max(1, (1 << 25) // (T * T))
    r_o = 0.0
    for s in range(0, Bq * heads, step):
        e = min(Bq * heads, s + step)
        sc = alpha * q[s:e] @ k[s:e].transpose(1, 2)
        if causal or key_pad is not None or allowed is not None:
            ok = torch.ones(e - s, T, T, dtype=torch.bool, device="cuda")
            if causal:
                ok &= torch.ones(T, T, dtype=torch.bool, device="cuda").tril()[None]
            if key_pad is not None:
                ok &= (key_pad.repeat_interleave(heads, 0)[s:e] == 0)[:, None, :]
            if allowed is not None:
                ok &= allowed
            sc = sc.masked_fill(~ok, -math.inf)
        lse = torch.logsumexp(sc, -1)
        P = torch.exp(sc - lse[..., None])
        del sc
        Mk = M[s:e] if p > 0 else None
        Pd = P if Mk is None else P * Mk * scale
        O_ref = Pd @ v[s:e]
        tol, _ = attention_tols(P, Pd, v[s:e], O_ref, lse)
        if not fused and p > 0:
            # the softmax kernels round P to bf16 and drop from the rounded value, so Pd is rounded twice (one more 2^-8 relative)
            tol = tol + 2.0 ** -8 * (Pd @ v[s:e].abs())
        r_o = max(r_o, O.worst(o[s:e], O_ref, tol))
        res = ref_attention_bwd(q[s:e], k[s:e], v[s:e], P, Pd, do[s:e].double(), o[s:e].double(), alpha, Mk, scale)
        for j, (ref, bnd) in enumerate(res):
            dq_ref[j, s:e], dq_bnd[j, s:e] = ref, bnd
        if not fused and p > 0:
            dq_bnd[2, s:e] += 2.0 ** -8 * (Pd.transpose(1, 2) @ do[s:e].double().abs())
        if not fused:
            # the materialised backward forms D = sum_j Pd dPd from the stored bf16 Pd (2^-8 relative per term) rather than from dO and
            # O, so dS = P (dPd - D) carries up to 2^-8 P sum_j |Pd dPd| more
            dPabs = do[s:e].double().abs() @ v[s:e].abs().transpose(1, 2)
            if Mk is not None:
                dPabs = dPabs * Mk * scale
            eD = 2.0 ** -8 * P * (Pd * dPabs).sum(-1, keepdim=True)
            dq_bnd[0, s:e] += alpha * eD @ k[s:e].abs()
            dq_bnd[1, s:e] += alpha * eD.transpose(1, 2) @ q[s:e].abs()
            del dPabs, eD
        del P, Pd, res
    _WORST[tag + " out"] = max(_WORST.get(tag + " out", 0.0), r_o)
    assert r_o <= 1.0, "%s out: %.3g of the bound" % (tag, r_o)

    def back(t):
        return t.view(Bq, heads, T, dh).permute(0, 2, 1, 3).reshape(Bq, T, Dm)
    grads.add(qkv, torch.cat([back(dq_ref[j]) for j in range(3)], -1), torch.cat([back(dq_bnd[j]) for j in range(3)], -1))


def check_tdnn(tag, args, out, grads):
    x, weight, bias, dil, stride = args[:5]
    premasked = args[5] if len(args) > 5 else False
    N = weight.shape[0]
    C = x.shape[-1]
    W = w16(weight).view(N, 3, C)
    x64 = x.detach().double()
    pre, inner = O.tdnn_fwd(x64, W, bias.detach().double(), dil, stride)
    y = pre.clamp_min(0)
    check(tag + " y", out, y, O.stored(y, inner, torch.bfloat16))
    del pre, y, inner
    dy = out.grad.double()
    dpre = dy if premasked else dy * (out != 0)
    (dx, dxi), (dw, dwi), (db, dbi) = O.tdnn_bwd(dpre, x64, W, dil, stride)
    if x.requires_grad:
        grads.add(x, dx, O.stored(dx, dxi, torch.bfloat16))
    check(tag + " dW", weight.grad.view(N, 3, C), dw, O.stored(dw, dwi, torch.float32), NREL_F32)
    check(tag + " db", bias.grad, db, O.stored(db, dbi, torch.float32), NREL_F32)


def check_grads(tag, grads, *tensors):
    for i, t in enumerate(tensors):
        grads.check("%s dx%d" % (tag, i), t)


# ------------------------------------------------------------------------------------------------ LinearFn
def _lin(K_in, N, seed):
    lin = nn.Linear(K_in, N).cuda()
    with torch.no_grad():
        lin.bias.copy_(torch.randn(N, device="cuda", generator=gen(seed)) * 0.1)
    return lin


def _relu_drop_input(M, K_in, p, seed):
    """a bf16 ReLU(+dropout) output, as the previous layer hands it to a layer with mask_input_scale"""
    x = randn(M, K_in, seed=seed).float().clamp_min(0)
    if p > 0:
        x = x * (torch.rand(M, K_in, device="cuda", generator=gen(seed + 1)) >= p) / (1 - p)
    return x.bfloat16()


# name: (M, K, N, n weights, bias, act, drop_p, residual, premasked, mask_input_scale p (None: off), x columns)
LINEAR_CASES = {
    "plain": (32000, 1024, 1024, 1, True, False, 0.0, False, False, None, None),
    "relu": (32000, 1024, 4096, 1, True, True, 0.0, False, False, None, None),
    "relu_dropout": (32000, 1024, 4096, 1, True, True, 0.2, False, False, None, None),
    "dropout_residual": (32000, 4096, 1024, 1, True, False, 0.2, True, False, None, None),
    "qkv": (32000, 1024, 1024, 3, True, False, 0.0, False, False, None, None),
    "premasked": (32000, 1024, 4096, 1, True, True, 0.2, False, True, None, None),
    "mask_input_p02": (32000, 4096, 1024, 1, True, False, 0.2, True, False, 0.2, None),
    "mask_input_p0": (32000, 4096, 1024, 1, True, False, 0.0, True, False, 0.0, None),
    "cols_pad": (32 * U1, 100, 4096, 1, True, False, 0.0, False, False, None, 104),
    "fc_in": (32000, 240, 1024, 1, True, True, 0.0, False, False, None, None),
    "ragged_m_n_tail": (4001, 1024, 6000, 1, True, False, 0.0, False, False, None, None),
}


# weight gradients of 1024 x 1024 and 1024 x 240 over K = 32 000 rows fill under a wave of output tiles: split-K is chosen
SPLIT_K_CASES = ("plain", "qkv", "fc_in")


@pytest.mark.parametrize("case", sorted(LINEAR_CASES))
def test_linear(case, bf16_mode, rec, spy):
    """LinearFn alone, forward and backward.  Measured on an H100: see the module's report (largest err / bound per output)."""
    E = bf16_mode
    M, Kin, N, nw, has_b, act, p, has_res, premasked, mis_p, xcols = LINEAR_CASES[case]
    log, _ = spy
    lins = [_lin(Kin, N, 10 + i) for i in range(nw)]
    if mis_p is not None:
        x = _relu_drop_input(M, Kin, mis_p, 3)
    else:
        x = randn(M, xcols or Kin, seed=3)
        if xcols:
            x[:, Kin:] = 0                               # the pad columns of an ld-padded activation
    x.requires_grad_(True)
    res = randn(M, nw * N, seed=4).requires_grad_(True) if has_res else None
    mis = (1.0 / (1.0 - mis_p) if mis_p > 0 else 1.0) if mis_p is not None else 0.0
    y = E.linear(x, [l.weight for l in lins], [l.bias for l in lins] if has_b else None, act=act, drop_p=p, residual=res,
                 premasked=premasked, mask_input_scale=mis)
    y.backward(randn(M, nw * N, seed=5))
    rec.stop()
    # the path: one forward GEMM with the claimed epilogue, one dgrad, and a wgrad per weight with split-K chosen
    fwd, dgrad = rec.gemms(b_mn=0)[0], rec.gemms(a_mn=0, b_mn=1)[0]
    assert fwd["act"] == int(act) and abs(fwd["drop_p"] - p) < 1e-7 and fwd["aux_mode"] == (1 if has_res else 0) and not fwd["c_f32"]
    assert dgrad["aux_mode"] == (2 if mis > 0 else 0) and (mis == 0 or abs(dgrad["aux_scale"] - mis) < 1e-6)
    assert ("pk_mask_nz" in rec.names()) == (act and not premasked)
    wg = rec.gemms(a_mn=1, b_mn=1)
    assert len(wg) == nw
    if case in SPLIT_K_CASES:
        assert all(auto_splits(g) > 1 for g in wg), [auto_splits(g) for g in wg]
    (name, args, out), = log
    grads = Grads()
    check_linear("linear " + case, args, out, grads)
    check_grads("linear " + case, grads, x, *([res] if has_res else []))
    if p == 0 and mis_p is None:
        # observe the split-K choice: the same weight gradient launched with k_splits = 1 has the engine's bits exactly when the
        # engine's launch did not split (one summation order), and other bits when it did
        from pika_b200 import kernels as K
        dpre = (out.grad * (out != 0)).bfloat16() if act and not premasked else out.grad
        for i, (l, g) in enumerate(zip(lins, wg)):
            g1 = torch.empty_like(l.weight.grad)
            K.gemm(dpre[:, i * N:(i + 1) * N], x.detach()[:, :Kin], g1, a_mn=True, b_mn=True, k_splits=1)
            assert torch.equal(g1, l.weight.grad) == (auto_splits(g) == 1), (case, auto_splits(g))


# ------------------------------------------------------------------------------------------------ TdnnFn / BatchNormFn
@pytest.mark.parametrize("dil,stride", [(1, 1), (3, 1), (3, 4)])
@pytest.mark.parametrize("premasked", [False, True])
def test_tdnn(dil, stride, premasked, bf16_mode, rec, spy):
    """TdnnFn at B = 32, T = 1000, C = 1024: the three-tap forward, the kz_count = B batched wgrad, the row-offset dgrad (stride 1)
    and the three disjoint strided dgrads (stride 4)."""
    E = bf16_mode
    log, _ = spy
    conv = nn.Conv2d(1, D, (3, D), dilation=(dil, 1), stride=(stride, 1)).cuda()
    x = randn(B, T_IN, D, seed=7).requires_grad_(True)
    y = E.TdnnFn.apply(x, conv.weight, conv.bias, dil, stride, premasked)
    y.backward(randn(*y.shape, seed=8))
    rec.stop()
    wg = rec.gemms(a_mn=1, b_mn=1)
    assert len(wg) == 3 and all(g["kz"] == B for g in wg)
    assert len(rec.gemms(a_mn=0, b_mn=1)) == (1 if stride == 1 else 3)
    assert ("pk_mask_nz" in rec.names()) != premasked
    grads = Grads()
    check_tdnn("tdnn", log[0][1], log[0][2], grads)
    check_grads("tdnn", grads, x)


@pytest.mark.parametrize("train", [True, False])
def test_fc_in_batchnorm_relu_input(train, bf16_mode, rec, spy):
    """fc_in (240 -> 1024, ReLU, premasked) -> BatchNormFn(relu_input=True) over 32 000 rows, as the encoder composes them: the ReLU
    mask of the linear rides in the BatchNorm backward.  Train and eval statistics."""
    E = bf16_mode
    log, _ = spy
    lin = _lin(240, D, 20)
    bn = nn.BatchNorm1d(D).cuda()
    with torch.no_grad():
        bn.weight.copy_(1 + 0.2 * torch.randn(D, device="cuda", generator=gen(21)))
        bn.bias.copy_(0.2 * torch.randn(D, device="cuda", generator=gen(22)))
        bn.running_mean.copy_(0.3 + 0.1 * torch.randn(D, device="cuda", generator=gen(23)))
        bn.running_var.copy_(0.3 + torch.rand(D, device="cuda", generator=gen(24)))
    stats = (bn.running_mean.clone(), bn.running_var.clone())
    x = randn(B * T_IN, 240, seed=25).requires_grad_(True)
    h = E.linear(x, lin.weight, lin.bias, act=True, premasked=True)
    y = E.BatchNormFn.apply(h, bn, train, bn.weight, bn.bias, True)
    y.backward(randn(*y.shape, seed=26))
    rec.stop()
    assert "pk_mask_nz" not in rec.names() and "pk_bn_bwd" in rec.names()
    grads = Grads()
    (_, la, lo), (_, ba, bo) = log
    check_batchnorm("bn relu_input", ba, bo, grads, stats)
    check_grads("bn relu_input", grads, lo)
    check_linear("fc_in premasked", la, lo, grads)
    check_grads("fc_in premasked", grads, x)


# ------------------------------------------------------------------------------------------------ LayerNormFn
@pytest.mark.parametrize("rows", [32000, 7777])
def test_layernorm(rows, bf16_mode, rec, spy):
    E = bf16_mode
    log, _ = spy
    ln = nn.LayerNorm(D, eps=1e-6).cuda()
    with torch.no_grad():
        ln.weight.copy_(1 + 0.2 * torch.randn(D, device="cuda", generator=gen(30)))
        ln.bias.copy_(0.2 * torch.randn(D, device="cuda", generator=gen(31)))
    x = (randn(rows, D, seed=32).float() * 2 + 0.5).bfloat16().requires_grad_(True)
    y = E.LayerNormFn.apply(x, ln, ln.weight, ln.bias)
    y.backward(randn(rows, D, seed=33))
    rec.stop()
    grads = Grads()
    check_layernorm("layernorm", log[0][1], log[0][2], grads)
    check_grads("layernorm", grads, x)


# ------------------------------------------------------------------------------------------------ AttentionFn
ATTN_CASES = {
    "fused_h16_T994": (32, 994, 16, 0.2, dict()),
    "fused_h16_T976_p0": (32, 976, 16, 0.0, dict()),
    "materialised_h8_T240": (32, 240, 8, 0.2, dict()),
    "causal_keypad_h8": (32, 152, 8, 0.2, dict(causal=True, key_pad=True)),
    "chunk_h16": (8, 994, 16, 0.2, dict(chunk=(64, 10, 2))),
}


@pytest.mark.parametrize("case", sorted(ATTN_CASES))
def test_attention(case, bf16_mode, rec, spy):
    """AttentionFn: the fused kernels at head dim 64 (T = 994, 976; keep bits with dropout), the materialised path at head dim 128
    (T' = 240), the causal + padding-key softmax of the transformer prediction net, and the fused chunk-mask kernels."""
    E = bf16_mode
    log, bits = spy
    Bq, T, heads, p, kw = ATTN_CASES[case]
    qkv = randn(Bq, T, 3 * D, seed=40).requires_grad_(True)
    key_pad = None
    if kw.get("key_pad"):
        lens = torch.randint(T // 2, T + 1, (Bq,), generator=torch.Generator().manual_seed(41)).cuda()
        key_pad = (torch.arange(T, device="cuda")[None] >= lens[:, None]).to(torch.uint8).contiguous()
    out = E.AttentionFn.apply(qkv, heads, p, 4242, kw.get("causal", False), key_pad, None, kw.get("chunk"))
    out.backward(randn(Bq, T, D, seed=42))
    rec.stop()
    names = rec.names()
    if "chunk" in kw:
        assert "pk_attention_fwd_chunk" in names and "pk_attention_bwd_chunk" in names
    elif D // heads == 64 and not kw:
        assert ("pk_attention_fwd_bits" if p > 0 else "pk_attention_fwd") in names
        assert ("pk_attention_bwd_bits" if p > 0 else "pk_attention_bwd") in names
        assert not any(n.startswith("pk_softmax") for n in names)
    else:
        assert ("pk_softmax_masked_fwd" if kw else "pk_softmax_fwd") in names and "pk_softmax_bwd" in names
        assert not any(n.startswith("pk_attention_fwd") for n in names)
    grads = Grads()
    check_attention("attention " + case, log[0][1], log[0][2], grads, bits[0] if bits else None)
    check_grads("attention " + case, grads, qkv)


def test_attention_relpos(bf16_mode, rec):
    """AttentionFn with a relative-position table (the transformer prediction net with max_relative_positions m = 16: B = 32,
    L = 151, d_model 512, 8 heads, causal + padding keys, dropout 0.2) on the band kernels, against float64 autograd of
    softmax(alpha (q k^T + q R_b(i,j)^T)) with out = Pd v + sum_j Pd R_b(i,j), b(i, j) = clamp(j - i, -m, m) + m.
    Bounds, from the engine's operand roundings: the scores carry the bf16 rounding of alpha q in QR (2^-8 alpha |q||R_b|) and the f32
    products; P is rounded to bf16 and dropout scales the rounded value (two roundings of Pd); the bucket sums Pb and dSb are f32 sums
    rounded to bf16 for their GEMMs; dS is rounded to bf16 and its row term D reads the stored probabilities."""
    from test_attention_kernels_gpu import drop_mask, drop_params, ref_bucket
    E = bf16_mode
    Bq, T, Dm, heads, mr, p = 32, U1, 512, 8, 16, 0.2
    dh = Dm // heads
    nb = 2 * mr + 1
    alpha = 1.0 / math.sqrt(dh)
    qkv = randn(Bq, T, 3 * Dm, seed=110).requires_grad_(True)
    rel = nn.Parameter((torch.randn(nb, dh, device="cuda", generator=gen(111)) * 0.5))
    lens = torch.randint(T // 2, T + 1, (Bq,), generator=torch.Generator().manual_seed(112)).cuda()
    key_pad = (torch.arange(T, device="cuda")[None] >= lens[:, None]).to(torch.uint8).contiguous()
    out = E.AttentionFn.apply(qkv, heads, p, 5151, True, key_pad, rel, None)
    dout = randn(Bq, T, Dm, seed=113)
    out.backward(dout)
    rec.stop()
    names = rec.names()
    assert "pk_softmax_masked_relpos_fwd" in names and "pk_softmax_relpos_bwd" in names
    assert not any(n.startswith("pk_attention") for n in names)
    scale = drop_params(p)[1]
    M = drop_mask(Bq * heads * T, T, p, 5151).view(Bq * heads, T, T).double()
    bk = ref_bucket(T, mr)
    Rw = w16(rel)
    ok = torch.ones(T, T, dtype=torch.bool, device="cuda").tril()[None] & (key_pad.repeat_interleave(heads, 0) == 0)[:, None, :]

    def heads_of(t, i):
        return t[:, :, i * Dm:(i + 1) * Dm].reshape(Bq, T, heads, dh).permute(0, 2, 1, 3).reshape(Bq * heads, T, dh)
    q, k, v = (heads_of(qkv.detach(), i).double() for i in range(3))
    do = dout.view(Bq, T, heads, dh).permute(0, 2, 1, 3).reshape(Bq * heads, T, dh).double()
    o_got = out.detach().view(Bq, T, heads, dh).permute(0, 2, 1, 3).reshape(Bq * heads, T, dh)
    g_got = [heads_of(qkv.grad, i) for i in range(3)]
    U8 = 2.0 ** -8
    dR, dR_b = torch.zeros_like(Rw), torch.zeros_like(Rw)
    Rg, Rga = Rw[bk], Rw.abs()[bk]                                               # [T, T, dh]

    def bucket_sums(X):
        return torch.zeros(X.shape[0], T, nb, dtype=X.dtype, device="cuda").scatter_add_(-1, bk.expand_as(X), X)
    step = 32
    for s0 in range(0, Bq * heads, step):
        sl = slice(s0, min(Bq * heads, s0 + step))
        qs, ks, vs = (t[sl].clone().requires_grad_(True) for t in (q, k, v))
        Rs = Rw.clone().requires_grad_(True)
        Rgs = Rs[bk]
        sc = alpha * (qs @ ks.transpose(1, 2) + torch.einsum("hid,ijd->hij", qs, Rgs))
        P = torch.softmax(sc.masked_fill(~ok[sl], -math.inf), -1)
        Pd = P * M[sl] * scale
        o = Pd @ vs + torch.einsum("hij,ijd->hid", Pd, Rgs)
        gq, gk, gv, gR = torch.autograd.grad(o, [qs, ks, vs, Rs], do[sl])
        P, Pd, o = P.detach(), Pd.detach(), o.detach()
        qa, ka, va, doa = q[sl].abs(), k[sl].abs(), v[sl].abs(), do[sl].abs()
        # scores: f32 products over dh and the bf16 alpha q of QR; P's relative error is twice the row's largest score error
        eS = alpha * (O.acc(2 * dh, qa @ ka.transpose(1, 2) + torch.einsum("hid,ijd->hij", qa, Rga)) + U8 * torch.einsum("hid,ijd->hij", qa, Rga))
        eP = 2 * eS.masked_fill(~ok[sl], 0).amax(-1, keepdim=True) + 1e-5
        Pb_abs = bucket_sums(Pd)
        mag_o = Pd @ va + Pb_abs @ Rw.abs()
        inner = (2 * U8 + eP) * mag_o + U8 * (Pb_abs @ Rw.abs()) + O.acc(T + nb, mag_o)
        check("attention relpos out", o_got[sl], o, O.stored(o, inner, torch.bfloat16))
        mag_dP = doa @ va.transpose(1, 2) + torch.einsum("hid,ijd->hij", doa, Rga)
        dP = do[sl] @ v[sl].transpose(1, 2) + torch.einsum("hid,ijd->hij", do[sl], Rg)
        dS = P * (M[sl] * scale * dP - (Pd * dP).sum(-1, keepdim=True))
        EdS = (U8 * dS.abs() + (2 * U8 + eP) * P * (M[sl] * scale * mag_dP + (Pd * mag_dP).sum(-1, keepdim=True))
               + P * O.acc(2 * dh, M[sl] * scale * mag_dP))
        dSb_abs, EdSb = bucket_sums(dS.abs()), bucket_sums(EdS)
        bq = alpha * (EdS @ ka + (EdSb + U8 * dSb_abs) @ Rw.abs()) + O.acc(T + nb, alpha * (dS.abs() @ ka + dSb_abs @ Rw.abs()))
        bk_ = alpha * EdS.transpose(1, 2) @ qa + O.acc(T, alpha * dS.abs().transpose(1, 2) @ qa)
        bv = (Pd * (2 * U8 + eP)).transpose(1, 2) @ doa + O.acc(T, Pd.transpose(1, 2) @ doa)
        for j, (ref, bnd) in enumerate(((gq, bq), (gk, bk_), (gv, bv))):
            check("attention relpos d" + "qkv"[j], g_got[j][sl], ref, O.stored(ref, bnd, torch.bfloat16))
        dR += gR
        # dR = dSb^T (alpha q) + Pb^T dO over every (sequence, head, query) row, f32
        dR_b += ((EdSb + 2 * U8 * dSb_abs).transpose(1, 2) @ (alpha * qa)).sum(0) \
            + (((2 * U8 + eP) * Pb_abs + U8 * Pb_abs).transpose(1, 2) @ doa).sum(0) \
            + O.acc(Bq * heads * T, (dSb_abs.transpose(1, 2) @ (alpha * qa) + Pb_abs.transpose(1, 2) @ doa).sum(0))
    check("attention relpos dR", rel.grad, dR, O.stored(dR, dR_b, torch.float32))


# ------------------------------------------------------------------------------------------------ transformer_layer
@pytest.mark.parametrize("layer", [0, 1, 2])
@pytest.mark.parametrize("p", [0.2, 0.0])
def test_transformer_layer(layer, p, bf16_mode, rec, spy):
    """The whole encoder block of attention layer ``layer`` (16 / 16 / 8 heads at T = 994 / 976 / 240, B = 32) in training mode: every
    Function checked from the tensors it saw, so with p = 0.2 the fold -- w_1 premasked, its ReLU and dropout mask applied with scale
    1 / (1 - p) by w_2's AUX_MASK_NZ dgrad epilogue -- is checked against w_1's float64 d(pre-activation)."""
    from pika_b200.model.rnnt_tdnn_transformer import Net, _TransformerLayerParams
    E = bf16_mode
    log, bits = spy
    heads, T = Net.HEADS[layer], XF_T[layer]
    torch.manual_seed(50 + layer)
    blk = _TransformerLayerParams(D, heads, DFF, 0.2).cuda()
    blk.dropout_p = p
    with torch.no_grad():
        for ln in (blk.layer_norm, blk.feed_forward.layer_norm):
            ln.weight.copy_(1 + 0.2 * torch.randn(D, device="cuda"))
            ln.bias.copy_(0.2 * torch.randn(D, device="cuda"))
    x = randn(B * T, D, seed=51).requires_grad_(True)
    y = E.transformer_layer(blk, x, B, T, True)
    y.backward(randn(B * T, D, seed=52))
    rec.stop()
    # the fold: w_1 premasked, no mask pass, w_2's dgrad applies (inter != 0) * 1/(1-p)
    assert log[5][1][6] is True and "pk_mask_nz" not in rec.names()
    masked = rec.gemms(aux_mode=2)
    assert len(masked) == 1 and abs(masked[0]["aux_scale"] - f32(1.0 / (1.0 - p))) < 1e-7
    assert ("pk_attention_fwd_bits" in rec.names()) == (heads == 16 and p > 0)
    assert any(auto_splits(g) > 1 for g in rec.gemms(a_mn=1, b_mn=1))
    grads = Grads()
    tag = "block%d p%g " % (layer, p)
    kinds = [n for n, _, _ in log]
    assert kinds == ["LayerNormFn", "LinearFn", "AttentionFn", "LinearFn", "LayerNormFn", "LinearFn", "LinearFn"], kinds
    names = ["ln", "qkv", "attn", "final", "ln2", "w_1", "w_2"]
    for (kind, args, out), nm in zip(log, names):
        if kind == "LinearFn":
            # w_2's dgrad mask is w_1's ReLU and dropout: scale 1 / (1 - p) from w_1's own drop probability, not w_2's arguments
            check_linear(tag + nm, args, out, grads,
                         (1.0 / (1.0 - log[5][1][3]) if log[5][1][3] > 0 else 1.0) if nm == "w_2" else None)
        elif kind == "LayerNormFn":
            check_layernorm(tag + nm, args, out, grads)
        else:
            check_attention(tag + nm, args, out, grads, bits[0] if bits else None)
    for (kind, args, out), nm in zip(log, names):
        if args[0] is not x:
            grads.check(tag + "d_in " + nm, args[0])
    grads.check(tag + "dx", x)


# ------------------------------------------------------------------------------------------------ EmbeddingFn / DropoutFn
def test_embedding_dropout(bf16_mode, rec, spy):
    """EmbeddingFn at the prediction net's shape (B = 32, U1 = 151, 100-wide embedding at ld 104, padding index V) and DropoutFn with
    p = 0.2 on its output"""
    E = bf16_mode
    log, _ = spy
    emb = nn.Embedding(V + 1, 100, padding_idx=V).cuda()
    idx = torch.randint(0, V + 1, (B, U1), generator=torch.Generator().manual_seed(60)).cuda()
    idx[:, -20:] = V
    idx[0, :5] = 7                                               # one row gathered several times
    seed = 1234
    h = E.EmbeddingFn.apply(idx, emb, 104, emb.weight)
    y = E.DropoutFn.apply(h, 0.2, seed)
    dy = randn(*y.shape, seed=61)
    y.backward(dy)
    rec.stop()
    assert rec.names().count("pk_dropout") == 2 and "pk_embedding_bwd" in rec.names()
    table = emb.weight.detach().double()
    ref_h = torch.zeros(B * U1, 104, dtype=torch.float64, device="cuda")
    ref_h[:, :100] = O.bf16r(table[idx.view(-1)])
    check("embedding y", h, ref_h, torch.full_like(ref_h, O.TINY))
    keep = keep_scaled(B * U1, 104, 0.2, seed)
    ref_y = O.bf16r(ref_h * keep)
    check("dropout y", y, ref_y, torch.full_like(ref_y, O.TINY))
    dh = O.bf16r(dy.double() * keep)
    check("dropout dx", h.grad, dh, torch.full_like(dh, O.TINY))
    g = torch.zeros_like(table)
    g.index_add_(0, idx.view(-1), dh[:, :100])
    g[V] = 0
    cnt = torch.zeros(V + 1, dtype=torch.float64, device="cuda").index_add_(0, idx.view(-1), torch.ones(B * U1, dtype=torch.float64,
                                                                                                        device="cuda"))
    mag = torch.zeros_like(table).index_add_(0, idx.view(-1), dh[:, :100].abs())
    check("embedding dW", emb.weight.grad, g, O.stored(g, O.acc(1, mag) * cnt[:, None], torch.float32))


# ------------------------------------------------------------------------------------------------ CausalConvFn
def test_causal_conv(bf16_mode, rec, spy):
    """CausalConvFn (Kw = 5, d_model 512, B = 32, L = 152, input at ld 104 from the 100-wide embedding, and 512 -> 512): the
    overlapping-window forward, the tap-major wgrad and the bf16 dgrad with all five taps in one launch"""
    E = bf16_mode
    log, _ = spy
    L = U1 + 1
    for C, ld, seed in ((100, 104, 70), (512, 512, 72)):
        log.clear()
        rec.calls.clear()
        rec.on = True
        conv = nn.Conv1d(C, 512, 5, padding=4).cuda()
        x = randn(B, L, ld, seed=seed)
        x[:, :, C:] = 0
        x.requires_grad_(True)
        y = E.CausalConvFn.apply(x, conv.weight, conv.bias)
        y.backward(randn(*y.shape, seed=seed + 1))
        rec.stop()
        dg = rec.gemms(a_mn=0, b_mn=1)
        assert len(dg) == 1 and dg[0]["n_pairs"] == 5 and not dg[0]["c_f32"]
        Wk = w16(conv.weight)
        x64 = x.detach().double()[:, :, :C]
        pre, inner = O.causal_conv_fwd(x64, Wk, conv.bias.detach().double())
        yr = pre.clamp_min(0)
        check("causal conv y", y, yr, O.stored(yr, inner, torch.bfloat16))
        dpre = y.grad.double() * (y != 0)
        (dx, dxi), (dw, dwi), (db, dbi) = O.causal_conv_bwd(dpre, x64, Wk)
        dxf = torch.zeros_like(x.detach(), dtype=torch.float64)
        dxb = torch.full_like(dxf, O.TINY)
        dxf[:, :, :C], dxb[:, :, :C] = dx, O.stored(dx, dxi, torch.bfloat16)
        check("causal conv dx", x.grad, dxf, dxb)
        check("causal conv dW", conv.weight.grad, dw, O.stored(dw, dwi, torch.float32), NREL_F32)
        check("causal conv db", conv.bias.grad, db, O.stored(db, dbi, torch.float32), NREL_F32)


# ------------------------------------------------------------------------------------------------ JointLossFn
class _Joint(nn.Module):
    def __init__(self, V_):
        super().__init__()
        self.fc1, self.fc_gate, self.fc2 = nn.Linear(2 * H, H), nn.Linear(2 * H, H), nn.Linear(H, V_)


@pytest.mark.parametrize("V_", [V, 5997])
def test_joint_loss(V_, bf16_mode, rec, monkeypatch):
    """JointLossFn at B = 4, T' = 240, U1 = 151, H = 1024: the fc1 / fc_gate forward, the gate, fc2 (with the row log-sum-exp epilogue
    when V % 8 == 0), the loss against oracle/rnnt.py's lattice on the engine's logits, and the compacted gradient's fc2 bias (its column
    sums), fc2, fc1 and fc_gate gradients and d_enc / d_pred against float64 from the engine's logits.

    The loss gradient's bound: each log-probability carries the fp32 log-sum-exp error e_lse (a sum of <= 320 exponentials per partial,
    ex2.approx), so a node occupancy exp(alpha + beta + lp - ll) is within e_path = 2 (T + U + 1) e_lse relatively; dz = g - p G then
    has |d dz| <= e_path |g| + (e_path + 2 e_lse) p G, and is stored in bf16."""
    from pika_b200 import engine as E
    torch.manual_seed(80)
    m = _Joint(V_).cuda()
    Bj, T = 4, 240
    enc = randn(Bj, T, H, seed=81).requires_grad_(True)
    pred = randn(Bj, U1, H, seed=82).requires_grad_(True)
    labels = torch.randint(1, V_, (Bj, U1 - 1), generator=torch.Generator().manual_seed(83)).int().cuda()
    fl = torch.tensor([T, T - 17, T - 60, 190], dtype=torch.int32, device="cuda")
    ll = torch.tensor([U1 - 1, U1 - 9, 80, 131], dtype=torch.int32, device="cuda")
    cap = {}
    real = E.joint_forward

    def joint_forward(*a, **k):
        logits, st = real(*a, **k)
        cap.update(logits=logits.clone(), h=st["h_parts"][0].clone(), ex=st["ex"].clone(), py=st["py"].clone(),
                   row_lse=st["row_lse"] is not None)
        return logits, st
    monkeypatch.setattr(E, "joint_forward", joint_forward)
    costs = E.JointLossFn.apply(enc, pred, m, labels, fl, ll)
    costs.sum().backward()
    rec.stop()
    # the path: fc2 with the row-LSE epilogue exactly when V % 8 == 0, the compacted gradient either way
    names = rec.names()
    assert cap["row_lse"] == (V_ % 8 == 0)
    assert len(rec.gemms(row_lse=True)) == (1 if V_ % 8 == 0 else 0)
    assert "pk_rnnt_loss_fwd_bwd_compact" in names and not any(n.startswith("pk_rnnt_loss_fwd_bwd_lse") for n in names)
    assert len(rec.gemms(a_rows=True)) == 2
    tag = "joint V%d " % V_
    e_lse = 2 * 320 * O.U24 + 2.0 ** -21

    def dz_of(b, z):
        zb = z.double()
        Tb, Ub = int(fl[b]), int(ll[b])
        cost, dz, occ = O.rnnt_from_logits(zb, labels[b], Tb, Ub)
        lse = torch.logsumexp(zb, -1)
        e_lp = e_lse + 2 * O.U24 * (zb.abs().amax(-1) + lse.abs())
        n_arcs = Tb + Ub + 1
        bound = n_arcs * float(e_lp[:Tb, :Ub + 1].max()) + 4 * n_arcs * O.U24 * abs(cost)
        r = abs(float(costs[b]) - cost) / bound
        _WORST[tag + "cost"] = max(_WORST.get(tag + "cost", 0.0), r)
        assert r <= 1.0, (b, float(costs[b]), cost, bound)
        e_path = 2 * n_arcs * float(e_lp[:Tb, :Ub + 1].max())
        g_abs = (dz + torch.softmax(zb, -1) * (-occ)[..., None]).abs()           # |g| (g = dz + p G with G = sum g = -occ)
        dz_err = e_path * g_abs + (e_path + 2 * e_lse) * torch.softmax(zb, -1) * occ[..., None]
        dz_err = dz_err + O.half_ulp(dz.abs() + dz_err, torch.bfloat16)
        del g_abs, zb
        return dz, dz_err

    check_joint(tag, m, enc, pred, cap, dz_of)


def check_joint(tag, m, enc, pred, cap, dz_of, py_idx=None, extra=None):
    """the gated joint from the tensors joint_forward left in ``cap``: ex / py, h and the logits forward, then its backward from
    dz_of(b, logits of utterance b) -> (d logits [T', U1, V] float64, element-wise bound on the engine's stored d logits): the fc2
    bias (column sums) and weight gradients, the gate backward, the fc1 / fc_gate gradients and d_enc / d_pred.
    py_idx [B, T', Rn] int64: the pred row each logits row (b, t, r) joins (the pruned windows); None: the dense grid (Rn = U1).
    extra: {"d_enc" | "d_pred": (reference, bound)} of another Function's gradient that autograd adds (in bf16) to the input's"""
    Bj, T = enc.shape[0], enc.shape[1]
    if py_idx is None:
        py_idx = torch.arange(U1, device="cuda").view(1, 1, U1).expand(Bj, T, U1)
    Rn = py_idx.shape[2]
    V_ = m.fc2.weight.shape[0]
    # forward stages
    Wx = torch.cat([w16(m.fc1.weight), w16(m.fc_gate.weight)])               # [2H, 2H]
    bx = torch.cat([m.fc1.bias, m.fc_gate.bias]).detach().double()
    e64, p64 = enc.detach().double().view(-1, H), pred.detach().double().view(-1, H)
    ex, exi = O.linear_fwd(e64, Wx[:, :H], bx)
    check(tag + "ex", cap["ex"], ex, O.stored(ex, exi, torch.bfloat16))
    py, pyi = O.linear_fwd(p64, Wx[:, H:])
    check(tag + "py", cap["py"], py, O.stored(py, pyi, torch.bfloat16))
    del ex, exi, py, pyi
    W2, b2 = w16(m.fc2.weight), m.fc2.bias.detach().double()
    exg, pyg = cap["ex"].double().view(Bj, T, 2 * H), cap["py"].double().view(Bj, U1, 2 * H)
    hg = cap["h"].view(Bj, T, Rn, H)
    lg = cap["logits"].view(Bj, T, Rn, -1)
    assert bool((lg[..., V_:] == 0).all())
    db2 = torch.zeros(V_, dtype=torch.float64, device="cuda")
    db2_b = torch.zeros_like(db2)
    dW2 = torch.zeros(V_, H, dtype=torch.float64, device="cuda")
    dW2_b = torch.zeros_like(dW2)
    dex = torch.zeros(Bj, T, 2 * H, dtype=torch.float64, device="cuda")
    dex_b, dpy, dpy_b = torch.zeros_like(dex), torch.zeros_like(pyg), torch.zeros_like(pyg)
    for b in range(Bj):
        pyb = pyg[b][py_idx[b]]                                                  # [T', Rn, 2H]
        h_ref, h_in = O.joint_gate(exg[b][:, None], pyb)
        check(tag + "h", hg[b], h_ref, O.stored(h_ref, h_in, torch.bfloat16))
        del h_ref, h_in
        h = hg[b].double().view(-1, H)
        z, zi = O.linear_fwd(h, W2, b2)
        check(tag + "logits", lg[b, ..., :V_].reshape(-1, V_), z, O.stored(z, zi, torch.bfloat16))
        del z, zi
        dz, dz_err = dz_of(b, lg[b, ..., :V_])
        dz2, dze2 = dz.view(-1, V_), dz_err.view(-1, V_)
        rows = dz2.shape[0]
        db2 += dz2.sum(0)
        db2_b += dze2.sum(0) + O.acc(rows, dz2.abs().sum(0))
        dW2 += dz2.t() @ h
        dW2_b += dze2.t() @ h.abs() + O.acc(rows, dz2.abs().t() @ h.abs())
        dh = dz2 @ W2
        dh_b = dze2 @ W2.abs() + O.acc(V_, dz2.abs() @ W2.abs())
        dh_b = dh_b + O.half_ulp(dh.abs() + dh_b, torch.bfloat16)
        del dz, dz_err, dz2, dze2, h
        dag, dag_b = O.joint_gate_bwd(exg[b][:, None], pyb, dh.view(T, Rn, H))
        # |s (1 - t^2)| <= 1 and |t s (1 - s)| <= 1/4: the error dh carries passes to each half at most once
        dag_b = dag_b + torch.cat([dh_b, dh_b], -1).view(T, Rn, 2 * H)
        dex[b], dex_b[b] = dag.sum(1), dag_b.sum(1) + O.acc(Rn, dag.abs().sum(1))
        ix = py_idx[b].reshape(-1)
        dpy[b].index_add_(0, ix, dag.view(-1, 2 * H))
        dpy_b[b].index_add_(0, ix, dag_b.view(-1, 2 * H) + O.acc(T, dag.abs().view(-1, 2 * H)))
        del dag, dag_b, dh, dh_b
    check(tag + "fc2 db", m.fc2.bias.grad, db2, O.stored(db2, db2_b, torch.float32))
    check(tag + "fc2 dW", m.fc2.weight.grad, dW2, O.stored(dW2, dW2_b, torch.float32))
    # dex / dpy are stored in bf16 before the fc1 / fc_gate GEMMs read them
    dex, dpy = dex.view(-1, 2 * H), dpy.view(-1, 2 * H)
    dex_b = O.stored(dex, dex_b.view(-1, 2 * H), torch.bfloat16)
    dpy_b = O.stored(dpy, dpy_b.view(-1, 2 * H), torch.bfloat16)
    gw = torch.cat([dex.t() @ e64, dpy.t() @ p64], 1)
    gw_b = torch.cat([dex_b.t() @ e64.abs() + O.acc(dex.shape[0], dex.abs().t() @ e64.abs()),
                      dpy_b.t() @ p64.abs() + O.acc(dpy.shape[0], dpy.abs().t() @ p64.abs())], 1)
    check(tag + "fc1 dW", m.fc1.weight.grad, gw[:H], O.stored(gw[:H], gw_b[:H], torch.float32))
    check(tag + "fc_gate dW", m.fc_gate.weight.grad, gw[H:], O.stored(gw[H:], gw_b[H:], torch.float32))
    gb = dex.sum(0)
    gb_b = dex_b.sum(0) + O.acc(dex.shape[0], dex.abs().sum(0))
    check(tag + "fc1 db", m.fc1.bias.grad, gb[:H], O.stored(gb[:H], gb_b[:H], torch.float32))
    check(tag + "fc_gate db", m.fc_gate.bias.grad, gb[H:], O.stored(gb[H:], gb_b[H:], torch.float32))
    for nm, d, db_, t, wx in (("d_enc", dex, dex_b, enc, Wx[:, :H]), ("d_pred", dpy, dpy_b, pred, Wx[:, H:])):
        r = d @ wx
        rb = O.stored(r, db_ @ wx.abs() + O.acc(2 * H, d.abs() @ wx.abs()), torch.bfloat16)
        if extra and nm in extra:
            r, rb = r + extra[nm][0], rb + extra[nm][1]
            rb = rb + O.half_ulp(r.abs() + rb, torch.bfloat16)
        check(tag + nm, t.grad.view(-1, H), r, rb)




def test_joint_fn(bf16_mode, rec, monkeypatch):
    """JointFn on its own at B = 4, T' = 240, U1 = 151, H = 1024, V = 6000: the forward, and joint_backward from a bf16 d logits with
    no loss in between -- the dense (not compacted) fc2 dgrad / wgrad over every row, the fc2 bias column sums and the dense gate
    backward"""
    from pika_b200 import engine as E
    torch.manual_seed(84)
    m = _Joint(V).cuda()
    Bj, T = 4, 240
    enc = randn(Bj, T, H, seed=85).requires_grad_(True)
    pred = randn(Bj, U1, H, seed=86).requires_grad_(True)
    cap = {}
    real = E.joint_forward

    def joint_forward(*a, **k):
        logits, st = real(*a, **k)
        cap.update(logits=logits.clone(), h=st["h_parts"][0].clone(), ex=st["ex"].clone(), py=st["py"].clone())
        return logits, st
    monkeypatch.setattr(E, "joint_forward", joint_forward)
    logits = E.JointFn.apply(enc, pred, m)
    dy = randn(*logits.shape, seed=87, scale=1e-3)
    logits.backward(dy)
    rec.stop()
    names = rec.names()
    assert not any(n.startswith("pk_rnnt") for n in names) and "pk_joint_gate_bwd" in names and "pk_colsum" in names
    assert not rec.gemms(row_lse=True) and not rec.gemms(a_rows=True)
    check_joint("joint_fn ", m, enc, pred, cap, lambda b, z: (dy[b].double(), torch.zeros_like(z, dtype=torch.float64)))


def test_simple_and_pruned_loss(bf16_mode, rec, monkeypatch):
    """SimpleLossFn + PrunedJointLossFn at B = 4, T' = 240, U1 = 151, H = 1024, V = 6000, R = 5 (the pruned training path):
      * the simple joiner's projections am / lm (f32) against float64, its costs against tests/pruned_rnnt_oracle.py on the engine's
        am / lm, its window starts against the windows' guarantees, and the projections' weight and bias gradients and input
        gradients from the engine's dam / dlm;
      * the pruned joint at the engine's windows: ex / py, h at (t, s_t + r), the logits, the pruned costs against the oracle's lattice
        on the engine's logits, and the whole joint backward (check_joint) from the float64 pruned d logits; enc and pred receive the
        sum of both Functions' gradients.
    The simple loss's E and P operands are bf16 (S = E P^T), so each of its log-probabilities is within 2 2^-8 + 2e-4 of float64."""
    import numpy as np

    import pruned_rnnt_oracle as PO
    from pika_b200 import engine as E
    torch.manual_seed(100)
    m = _Joint(V).cuda()
    m.simple_am_proj, m.simple_lm_proj = nn.Linear(H, V).cuda(), nn.Linear(H, V).cuda()
    Bj, T, R_ = 4, 240, 5
    enc = randn(Bj, T, H, seed=101).requires_grad_(True)
    pred = randn(Bj, U1, H, seed=102).requires_grad_(True)
    labels = torch.randint(1, V, (Bj, U1 - 1), generator=torch.Generator().manual_seed(103)).int().cuda()
    fl = torch.tensor([T, T - 17, T - 60, 190], dtype=torch.int32, device="cuda")
    ll = torch.tensor([U1 - 1, U1 - 9, 80, 131], dtype=torch.int32, device="cuda")
    cap, scap = {}, {}
    real_jf, real_sl = E.joint_forward, E.simple_loss

    def joint_forward(*a, **k):
        logits, st = real_jf(*a, **k)
        cap.update(logits=logits.clone(), h=st["h_parts"][0].clone(), ex=st["ex"].clone(), py=st["py"].clone(),
                   row_lse=st["row_lse"] is not None)
        return logits, st

    def simple_loss(am, lm, *a, **k):
        out = real_sl(am, lm, *a, **k)
        scap.update(am=am.clone(), lm=lm.clone(), dam=out[2], dlm=out[3])
        return out
    monkeypatch.setattr(E, "joint_forward", joint_forward)
    monkeypatch.setattr(E, "simple_loss", simple_loss)
    sc, bounds = E.SimpleLossFn.apply(enc, pred, m, labels, fl, ll, R_, 1.0, True)
    pc = E.PrunedJointLossFn.apply(enc, pred, m, labels, fl, ll, bounds, R_, 1.0, True)
    (sc.sum() + pc.sum()).backward()
    rec.stop()
    names = rec.names()
    for n in ("pk_rnnt_simple_tables", "pk_rnnt_lattice", "pk_rnnt_prune_bounds", "pk_joint_gate_pruned_fwd", "pk_joint_gate_pruned_bwd",
              "pk_rnnt_pruned_loss"):
        assert n in names, n
    assert cap["row_lse"] and len(rec.gemms(row_lse=True)) == 1 and "pk_joint_gate_fwd" not in names
    tag = "pruned "
    e64, p64 = enc.detach().double().view(-1, H), pred.detach().double().view(-1, H)
    # the simple joiner
    extra = {}
    for nm, x64, proj, a_, d_, rows in (("am", e64, m.simple_am_proj, scap["am"], scap["dam"], "d_enc"),
                                          ("lm", p64, m.simple_lm_proj, scap["lm"], scap["dlm"], "d_pred")):
        W = w16(proj.weight)
        ref, inner = O.linear_fwd(x64, W, proj.bias.detach().double())
        check(tag + "simple " + nm, a_[:, :V], ref, O.stored(ref, inner, torch.float32))
        d = d_[:, :V].double()
        (dx, dxi), (dw, dwi), (db, dbi) = O.linear_bwd(d, x64, W)
        check(tag + "simple " + nm + " dW", proj.weight.grad, dw, O.stored(dw, dwi, torch.float32), NREL_F32)
        check(tag + "simple " + nm + " db", proj.bias.grad, db, O.stored(db, dbi, torch.float32), NREL_F32)
        extra[rows] = (dx, O.stored(dx, dxi, torch.bfloat16))
    am, lm = scap["am"].view(Bj, T, -1), scap["lm"].view(Bj, U1, -1)
    s_all = bounds.cpu().numpy()
    for b in range(Bj):
        Tb, Ub = int(fl[b]), int(ll[b])
        y = labels[b, :Ub].cpu().numpy()
        cost = PO.simple_loss(am[b, :Tb, :V].double().cpu().numpy(), lm[b, :Ub + 1, :V].double().cpu().numpy(), y, fast=True)[0]
        n_arcs = Tb + Ub + 1
        bound = n_arcs * (2 * 2.0 ** -8 + 2e-4) + 4 * n_arcs * O.U24 * abs(cost)
        r = abs(float(sc[b]) - cost) / bound
        _WORST[tag + "simple cost"] = max(_WORST.get(tag + "simple cost", 0.0), r)
        assert r <= 1.0, (b, float(sc[b]), cost, bound)
        PO.check_bounds_properties(s_all[b], Tb, Ub, R_)
    # the pruned joint and its loss
    py_idx = (bounds.long()[..., None] + torch.arange(R_, device="cuda")).clamp(max=U1 - 1)
    e_lse = 2 * 320 * O.U24 + 2.0 ** -21

    def dz_of(b, z):
        zb = z.double()                                                          # [T', R, V]
        Tb, Ub = int(fl[b]), int(ll[b])
        s = s_all[b]
        y = labels[b, :Ub].long()
        lp = torch.log_softmax(zb, -1)
        lpb = np.full((Tb, Ub + 1), -np.inf)
        lpl = np.full((Tb, max(Ub, 1)), -np.inf)
        lpc = lp[:Tb].cpu().numpy()
        yc = y.cpu().numpy()
        for t in range(Tb):
            for r in range(R_):
                u = s[t] + r
                if u <= Ub:
                    lpb[t, u] = lpc[t, r, 0]
                if u < Ub:
                    lpl[t, u] = lpc[t, r, yc[u]]
        cost, gb, gl = PO.pruned_cost(lpb, lpl[:, :Ub], s[:Tb], R_, fast=True)
        lse = torch.logsumexp(zb, -1)
        e_lp = e_lse + 2 * O.U24 * (zb.abs().amax(-1) + lse.abs())
        n_arcs = Tb + Ub + 1
        bound = n_arcs * float(e_lp[:Tb].max()) + 4 * n_arcs * O.U24 * abs(cost)
        rr = abs(float(pc[b]) - cost) / bound
        _WORST[tag + "cost"] = max(_WORST.get(tag + "cost", 0.0), rr)
        assert rr <= 1.0, (b, float(pc[b]), cost, bound)
        g = torch.zeros_like(zb)
        tt = torch.arange(Tb, device="cuda")
        st = torch.from_numpy(s[:Tb]).cuda().long()
        gbt, glt = torch.from_numpy(gb).cuda(), torch.from_numpy(gl).cuda()
        for r in range(R_):
            u = st + r
            ok = u <= Ub
            g[tt[ok], r, 0] = gbt[tt[ok], u[ok]]
            ok2 = u < Ub
            if Ub > 0:
                g[tt[ok2], r, y[u[ok2]]] += glt[tt[ok2], u[ok2]]
        occ = g.abs().sum(-1)
        p_ = torch.softmax(zb, -1)
        dz = g - p_ * g.sum(-1, keepdim=True)
        e_path = 2 * n_arcs * float(e_lp[:Tb].max())
        dz_err = e_path * g.abs() + (e_path + 2 * e_lse) * p_ * occ[..., None]
        return dz, dz_err + O.half_ulp(dz.abs() + dz_err, torch.bfloat16)

    check_joint(tag, m, enc, pred, cap, dz_of, py_idx, extra)


# ------------------------------------------------------------------------------------------------ LstmLayerFn
def test_lstm_prednet(bf16_mode, rec, spy, monkeypatch):
    """The benchmark's prediction net: embedding (100 wide at ld 104) -> two LstmLayerFn layers at B = 32, U1 = 151, H = 1024 with
    DropoutFn (p = 0.2) between them, on the persistent recurrence kernels.  The recurrence of each layer (gates, c, h and the
    backward's dG) is checked step by step against test_lstm_seq_gpu's float64 restatement on the tensors the engine handed the
    kernels; the layer's own GEMMs -- the input projection with the summed biases, dx, dW_ih, dW_hh (h of the previous step) and the
    bias gradients -- against the float64 references from the engine's dG."""
    import types

    import test_lstm_seq_gpu as LS
    from pika_b200 import engine as E
    from pika_b200 import kernels as K
    log, _ = spy
    ls_worst = {}
    monkeypatch.setattr(LS, "_WORST", ls_worst)                  # the restatement's ratios, reported here
    calls = {"fwd": [], "bwd": []}
    for kind, name in (("fwd", "lstm_seq_fwd_ex"), ("bwd", "lstm_seq_bwd_ex")):
        def wrap(*a, _real=getattr(K, name), _kind=kind):
            calls[_kind].append(a)
            return _real(*a)
        monkeypatch.setattr(K, name, wrap)
    torch.manual_seed(95)
    emb = nn.Embedding(V + 1, 100, padding_idx=V).cuda()
    lstm = nn.LSTM(100, H, num_layers=2, batch_first=True, dropout=0.2).cuda().train()
    y = torch.randint(1, V, (B, U1 - 1), generator=torch.Generator().manual_seed(96)).cuda()
    out = E.prednet_forward_act(types.SimpleNamespace(embed=emb, decoder=lstm), y)
    out.backward(randn(B, U1, H, seed=97))
    rec.stop()
    names = rec.names()
    assert names.count("pk_lstm_seq_fwd_ex") == 2 and names.count("pk_lstm_seq_bwd_ex") == 2
    assert not any(n.startswith("pk_lstm_cell") for n in names)
    layers = [(args, o) for n, args, o in log if n == "LstmLayerFn"]
    drops = [(args, o) for n, args, o in log if n == "DropoutFn"]
    assert len(layers) == 2 and len(drops) == 1
    (dx_in, dp, dseed), d_out = drops[0]
    keep = keep_scaled(B * U1, H, dp, dseed).view(B, U1, H)
    check("lstm dropout y", d_out, O.bf16r(dx_in.detach().double() * keep), torch.full(d_out.shape, O.TINY, device="cuda"))
    check("lstm dropout dx", dx_in.grad, O.bf16r(d_out.grad.double() * keep), torch.full(d_out.shape, O.TINY, device="cuda"))
    G4 = 4 * H
    for l, ((args, o), fa, ba) in enumerate(zip(layers, calls["fwd"], calls["bwd"][::-1])):
        tag = "lstm layer%d " % l
        x, _, w_ih, w_hh, b_ih, b_hh = args
        gx, whh, _, gates, cs, _ = fa
        dout, _, _, _, dG, _ = ba
        assert fa[2] is o and whh.dtype == torch.bfloat16
        # the recurrence, step by step on the engine's own h, c and dG
        p = types.SimpleNamespace(B=B, U=U1, H=H, G4=G4, nd=1, L=[U1] * B, gx=gx, w=whh, dt=torch.bfloat16, dout=dout)
        LS.check_forward(p, o, gates.view(-1), cs.view(-1), 0, False)
        LS.check_backward(p, gates.view(-1), cs.view(-1), dG.view(-1), 0, False)
        # the layer's GEMMs
        Bx, U, Ex = x.shape
        E_ = w_ih.shape[1]
        x2 = x.detach().double().reshape(B * U, Ex)
        Wih = w16(w_ih)
        if Ex != E_:
            Wih = torch.cat([Wih, Wih.new_zeros(G4, Ex - E_)], 1)
        bsum = b_ih.detach().double() + b_hh.detach().double()
        g_ref, g_in = O.linear_fwd(x2, Wih, bsum)
        g_in = g_in + O.U24 * bsum.abs()                                        # the f32 add of b_ih + b_hh
        check(tag + "gx", gx[0].reshape(B * U, G4), g_ref, O.stored(g_ref, g_in, torch.float32))
        dG2 = dG[0].permute(1, 0, 2).reshape(B * U, G4).double()
        (dx, dxi), (dwi, dwii), (db, dbi) = O.linear_bwd(dG2, x2, Wih)
        check(tag + "dx", x.grad.reshape(B * U, Ex), dx, O.stored(dx, dxi, torch.bfloat16))
        check(tag + "dW_ih", w_ih.grad, dwi[:, :E_], O.stored(dwi[:, :E_], dwii[:, :E_], torch.float32), NREL_F32)
        check(tag + "db_ih", b_ih.grad, db, O.stored(db, dbi, torch.float32), NREL_F32)
        check(tag + "db_hh", b_hh.grad, db, O.stored(db, dbi, torch.float32), NREL_F32)
        hp = torch.zeros(B, U, H, dtype=torch.float64, device="cuda")
        hp[:, 1:] = o.detach()[:, :-1].double()
        _, (dwh, dwhi), _ = O.linear_bwd(dG2, hp.reshape(B * U, H), w16(w_hh))
        check(tag + "dW_hh", w_hh.grad, dwh, O.stored(dwh, dwhi, torch.float32), NREL_F32)
    for k, v in ls_worst.items():
        _WORST["lstm recurrence " + k] = max(_WORST.get("lstm recurrence " + k, 0.0), v)


# ------------------------------------------------------------------------------------------------ LogSoftmaxFn
@pytest.mark.parametrize("V_", [V, 5997])
def test_log_softmax(V_, bf16_mode, rec):
    """LogSoftmaxFn (the compatibility path's log-probabilities) on bf16 logits [1, 240, 151, 6000] with V = 6000 and with V = 5997
    inside the 6000-column pitch.  The kernel sums exp over a row lane-strided (V / 32 terms per lane and a 5-level tree) with expf, so
    the row's log-sum-exp is within gamma_(V/32 + 8) plus a few ulp of log; the backward is torch f32 arithmetic stored in bf16."""
    E = bf16_mode
    z = randn(1, 240, U1, 6000, seed=90, scale=3.0)
    z[..., V_:] = 0
    z.requires_grad_(True)
    lp = E.LogSoftmaxFn.apply(z, V_)
    dlp = torch.randn(lp.shape, device="cuda", generator=gen(91))
    lp.backward(dlp)
    rec.stop()
    assert "pk_log_softmax" in rec.names()
    tag = "log_softmax V%d " % V_
    z64 = z.detach()[..., :V_].double()
    lse = torch.logsumexp(z64, -1, keepdim=True)
    ref = z64 - lse
    e_l = O.acc(V_ // 32 + 8, 1.0) + 4 * O.U24 * (lse.abs() + 1)
    check(tag + "y", lp, ref, O.stored(ref, e_l.expand_as(ref), torch.float32))
    del z64
    p = ref.exp()
    d64 = dlp.double()
    S = d64.sum(-1, keepdim=True)
    g = d64 - p * S
    inner = p * S.abs() * (e_l + 4 * O.U24) + p * O.acc(V_, d64.abs().sum(-1, keepdim=True)) + 2 * O.U24 * (d64.abs() + p * S.abs())
    check(tag + "dz", z.grad[..., :V_], g, O.stored(g, inner, torch.bfloat16))
    assert bool((z.grad[..., V_:] == 0).all())
