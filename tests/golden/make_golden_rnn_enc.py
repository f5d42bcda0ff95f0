#!/usr/bin/env python
"""Generate tests/golden/model_rnn_enc.npz by EXECUTING THE REFERENCE's own transducer Net with its default LSTM encoder
(``encoder_type='rnn'``), imported from /root/reference through tests/golden/ref_shim.py, with torchaudio's RNN-T loss standing in
for warp_rnnt (as in make_golden.py).

Run in the build container only:   python tests/golden/make_golden_rnn_enc.py
The GPU box never runs this script.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from fixture_utils import grad_fingerprint  # noqa: E402

ref_shim.install()
torch.set_num_threads(8)

CONFIGS = {"bi": dict(brnn=True, rnn_size=256, enc_layers=2), "uni": dict(brnn=False, rnn_size=256, enc_layers=2)}


def weight_fingerprint(model):
    """[sum, abs-sum, first, last] of every floating-point state_dict entry"""
    out = {}
    for k, v in model.state_dict().items():
        if v.dtype.is_floating_point:
            out[k] = np.array([v.double().sum().item(), v.double().abs().sum().item(),
                               float(v.flatten()[0]), float(v.flatten()[-1])])
    return out


def golden_model_rnn_enc():
    """Forward through pack / unpack exactly as trainer/model/transducer.py:82-86 (enforce_sorted=True, so the lengths are sorted
    descending, and max(len) < T), then the prediction net and joint of :89-108 with the hard-coded SOS.cuda() (:91) left out,
    torchaudio RNN-T loss, backward.  Dropout off.  Two encoders: bidirectional and unidirectional."""
    import torchaudio
    from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence
    from trainer.model.transducer import Net
    V, B, T, U = 40, 3, 40, 6
    g = torch.Generator().manual_seed(4321)
    x = torch.randn(B, T, 240, generator=g)
    y = torch.randint(1, V, (B, U), generator=g)
    lens = torch.tensor([36, 29, 17], dtype=torch.int32)
    ulens = torch.tensor([U, U - 2, U - 1], dtype=torch.int32)
    out = dict(x=x.numpy(), y=y.numpy().astype(np.int32), lens=lens.numpy(), ulens=ulens.numpy(), V=np.array(V))
    for c, kw in CONFIGS.items():
        a = ref_shim.model_args(V, rnn_size=kw["rnn_size"], dropout=0.3)
        a.encoder_type, a.brnn, a.enc_layers = "rnn", kw["brnn"], kw["enc_layers"]
        torch.manual_seed(779)
        m = Net(a, 240, V)
        for k, v in weight_fingerprint(m).items():
            out["w_%s_%s" % (c, k)] = v
        for k, v in m.state_dict().items():
            out["shape_%s_%s" % (c, k)] = np.array(v.shape, np.int64)
        m.train()
        m.encoder.dropout = 0.0
        m.decoder.dropout = 0.0
        packed, _ = m.encoder(pack_padded_sequence(x, lens, batch_first=True, enforce_sorted=True))
        enc = pad_packed_sequence(packed, batch_first=True)[0]
        yy = torch.cat((torch.zeros(B, 1).long(), y), dim=1)
        pred, _ = m.decoder(m.embed(yy))
        Te, U1 = enc.size(1), pred.size(1)
        j = torch.cat((enc.unsqueeze(2).expand(-1, -1, U1, -1), pred.unsqueeze(1).expand(-1, Te, -1, -1)), dim=-1)
        logits = m.fc2(torch.tanh(m.fc1(j)) * torch.sigmoid(m.fc_gate(j)))
        costs = torchaudio.functional.rnnt_loss(F.log_softmax(logits, -1), y.int(), lens, ulens, blank=0, reduction="none",
                                                fused_log_softmax=False)
        costs.sum().backward()
        out["enc_" + c] = enc.detach().numpy()
        out["logits_" + c] = logits.detach().numpy()
        out["costs_" + c] = costs.detach().numpy()
        for k, p in m.named_parameters():
            out["g_%s_%s" % (c, k)] = np.array([p.grad.double().norm().item(), p.grad.double().abs().max().item()])
            out["gs_%s_%s" % (c, k)] = grad_fingerprint(p.grad, 512)
        print("model_rnn_enc[%s]: costs %s, enc %s, logits %s" % (c, costs.tolist(), tuple(enc.shape), tuple(logits.shape)))
    np.savez_compressed(os.path.join(HERE, "model_rnn_enc.npz"), **out)


if __name__ == "__main__":
    golden_model_rnn_enc()
