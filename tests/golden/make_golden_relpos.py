#!/usr/bin/env python
"""Generate tests/golden/model_xf_relpos.npz and decode_xf_relpos.npz by EXECUTING THE REFERENCE's own transducer Net with the
convolutional-transformer prediction net and relative-position self-attention (``max_relative_positions`` m > 0,
trainer/model/modules/multi_headed_attn.py:9-41,105-108,186-229), imported from /root/reference through tests/golden/ref_shim.py,
with torchaudio's RNN-T loss standing in for warp_rnnt (as in make_golden.py).

The reference Net never passes ``max_relative_positions`` to its prediction net (trainer/model/transducer.py:62-68), so the
generator swaps in ``decoder_transformer(..., max_relative_positions=m)`` at the constructor call: the module is created at the
same point of the seeded construction as the drop-in's, so both draw the same initial weights.

Run in the build container only:   python tests/golden/make_golden_relpos.py
The GPU box never runs this script.
"""
import functools
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from fixture_utils import decode_fixture_reinit_xf, grad_fingerprint  # noqa: E402

ref_shim.install()
torch.set_num_threads(8)

# m = 3: every label sequence (L = U + 1 = 10 with SOS) is longer than m, so both end buckets collect several keys;
# m = 16: no distance reaches m, every key has a bucket of its own
MODEL_M = (3, 16)
DECODE_M = 4


def build_ref_model_xf_relpos(V, m, seed=778, embd=100, dec_layers=2):
    """reference transducer with the transformer prediction net (trainer/model/transducer.py:62-68), its decoder built with
    max_relative_positions = m"""
    import trainer.model.transducer as rt
    a = ref_shim.model_args(V, embd_dim=embd, dec_layers=dec_layers)
    a.decoder_type = "transformer"
    orig = rt.decoder_transformer
    rt.decoder_transformer = functools.partial(orig, max_relative_positions=m)
    try:
        torch.manual_seed(seed)
        return rt.Net(a, 240, V)
    finally:
        rt.decoder_transformer = orig


def xf_inputs(seed, B, Tp, H=1024):
    return np.random.default_rng(seed).standard_normal((B, Tp, H)).astype(np.float32)


def weight_fingerprint(model):
    out = {}
    for k, v in model.state_dict().items():
        if v.dtype.is_floating_point:
            out[k] = np.array([v.double().sum().item(), v.double().abs().sum().item(), float(v.flatten()[0]), float(v.flatten()[-1])])
    return out


def golden_model_xf_relpos():
    """Per m: seeded initial weights and state_dict keys, then prediction net + joint forward and (torchaudio-loss) backward with
    dropout off.  The encoder is replaced by seeded outputs; everything from the embedding to the loss is the reference's own code.
    Label rows of unequal length, padded with the padding id (= V, embed.padding_idx)."""
    import torchaudio
    V, B, Tp, U = 40, 3, 20, 9
    res = dict(dims=np.array([V, B, Tp, U]), seed=np.array(707), ms=np.array(MODEL_M))
    g = torch.Generator().manual_seed(99)
    y = torch.randint(1, V, (B, U), generator=g)
    ulens = torch.tensor([U, U - 3, U - 5], dtype=torch.int32)
    for b in range(B):
        y[b, int(ulens[b]):] = V
    tl = torch.tensor([Tp, Tp - 4, Tp - 7], dtype=torch.int32)
    res.update(y=y.numpy().astype(np.int64), ulens=ulens.numpy(), tlens=tl.numpy())
    for m_rel in MODEL_M:
        pre = "m%d_" % m_rel
        m = build_ref_model_xf_relpos(V, m_rel)
        m.train()
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
        res[pre + "keys"] = np.array([k for k in m.state_dict() if not k.startswith("encoder.")])
        for k, v in weight_fingerprint(m).items():
            if not k.startswith("encoder."):
                res[pre + "w_" + k] = v
        enc = torch.from_numpy(xf_inputs(707, B, Tp)).requires_grad_(True)
        sos = torch.zeros(B, 1).long()
        pred = m.decoder(torch.cat((sos, y), dim=1))                       # trainer/model/transducer.py:96-97
        T_, U1 = enc.size(1), pred.size(1)
        out = torch.cat((enc.unsqueeze(2).expand(-1, -1, U1, -1), pred.unsqueeze(1).expand(-1, T_, -1, -1)), dim=-1)
        logits = m.fc2(torch.tanh(m.fc1(out)) * torch.sigmoid(m.fc_gate(out)))
        yl = y.clone()
        yl[yl == V] = 0                                                     # label values past label_lens are never read by the loss
        costs = torchaudio.functional.rnnt_loss(F.log_softmax(logits, -1), yl.int(), tl, ulens, blank=0, reduction="none",
                                                fused_log_softmax=False)
        costs.sum().backward()
        res.update({pre + "pred": pred.detach().numpy(), pre + "costs": costs.detach().numpy(),
                    pre + "denc": grad_fingerprint(enc.grad, 512)})
        for k, p in m.named_parameters():
            if not k.startswith("encoder."):
                res[pre + "gs_" + k] = grad_fingerprint(p.grad if p.grad is not None else torch.zeros_like(p), 512)
        print("model_xf_relpos m=%d: costs %s, pred %s, |dR0| %.4g" % (m_rel, costs.tolist(), tuple(pred.shape),
              m.decoder.transformer[0].self_attn.relative_positions_embeddings.weight.grad.norm().item()))
    np.savez_compressed(os.path.join(HERE, "model_xf_relpos.npz"), **res)


def golden_decode_xf_relpos():
    """Reference decode_batch with the relative-position transformer prediction net (decoder/transducer_decoder.py:117-120,151-171),
    beam 4 and 8, on seeded encoder outputs; torch.cuda.LongTensor pointed at torch.LongTensor for the CPU run, as in
    make_golden.py:golden_decode_xf."""
    ref_shim.load_beam_module()
    from decoder.transducer_decoder import TransducerDecoder
    import decoder.beam_transducer as bt
    V, B, Tp = 40, 4, 24
    m = build_ref_model_xf_relpos(V, DECODE_M)
    m.eval()
    decode_fixture_reinit_xf(m)
    enc_t = torch.from_numpy(xf_inputs(809, B, Tp))

    class FixedEncoder(torch.nn.Module):
        def forward(self, x):
            return enc_t

    m.encoder = FixedEncoder()
    tl = torch.tensor([24, 21, 17, 9])
    cases = {}
    saved = torch.cuda.LongTensor
    torch.cuda.LongTensor = torch.LongTensor
    try:
        for name, beam, nbest in [("b4n2", 4, 2), ("b8n4", 8, 4)]:
            dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.0)
            dec = TransducerDecoder(m, B, beam, n_best=nbest, blk=0, global_scorer=bt.GlobalScorer(), sm_scale=1.0, cuda=False,
                                    beam_prune=True, args=dargs)
            with torch.no_grad():
                ret, _ = dec.decode_batch(torch.zeros(B, 1, 240), tl, max_len=[int(t) + 30 for t in tl])
            for b in range(B):
                for n in range(nbest):
                    cases["%s_pred_%d_%d" % (name, b, n)] = np.array([int(t) for t in ret["predictions"][b][n]], np.int64)
                    cases["%s_score_%d_%d" % (name, b, n)] = np.array(float(ret["scores"][b][n]))
            print("decode_xf_relpos", name, [len(cases["%s_pred_%d_0" % (name, b)]) for b in range(B)],
                  [float(ret["scores"][b][0]) for b in range(B)])
    finally:
        torch.cuda.LongTensor = saved
    np.savez_compressed(os.path.join(HERE, "decode_xf_relpos.npz"), seed=np.array(809), tlens=tl.numpy(), dims=np.array([V, B, Tp]),
                        m=np.array(DECODE_M), **cases)


if __name__ == "__main__":
    golden_model_xf_relpos()
    golden_decode_xf_relpos()
