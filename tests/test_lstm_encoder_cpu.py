"""The reference's default encoder (``--encoder_type rnn``) builds on the CPU: nn.LSTM of rnn_size // (2 if brnn) units per
direction, the reference's construction order (so seeded initial weights and state_dict keys match its own Net, run by
tests/golden/make_golden_rnn_enc.py), and ``pack_seq`` set."""
import os
import types

import numpy as np
import pytest
import torch

CONFIGS = {"bi": dict(brnn=True, rnn_size=256, enc_layers=2), "uni": dict(brnn=False, rnn_size=256, enc_layers=2)}


def build(cfg, V=40):
    from pika_b200.model.transducer import Net
    torch.manual_seed(779)
    args = types.SimpleNamespace(rnn_size=cfg["rnn_size"], local_rank=0, decoder_type="rnn", brnn=cfg["brnn"], encoder_type="rnn",
                                 embd_dim=100, padding_idx=V, dropout=0.3, dec_layers=2, enc_layers=cfg["enc_layers"])
    return Net(args, 240, V)


@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_rnn_encoder_net_matches_reference_construction(golden_dir, cfg):
    d = np.load(os.path.join(golden_dir, "model_rnn_enc.npz"))
    m = build(CONFIGS[cfg])
    assert m.pack_seq is True
    assert isinstance(m.encoder, torch.nn.LSTM)
    assert m.encoder.bidirectional == CONFIGS[cfg]["brnn"] and m.encoder.num_layers == 2 and m.encoder.batch_first
    assert m.encoder.dropout == 0.3
    sd = m.state_dict()
    ref_keys = sorted(k[len("shape_%s_" % cfg):] for k in d.files if k.startswith("shape_%s_" % cfg))
    assert sorted(sd) == ref_keys
    for k, v in sd.items():
        assert tuple(v.shape) == tuple(d["shape_%s_%s" % (cfg, k)]), k
        if v.dtype.is_floating_point:
            ref = d["w_%s_%s" % (cfg, k)]
            got = np.array([v.double().sum().item(), v.double().abs().sum().item(), float(v.flatten()[0]), float(v.flatten()[-1])])
            np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-6, err_msg=k)


def test_rnn_encoder_output_width():
    for cfg, per_dir in (("bi", 128), ("uni", 256)):
        m = build(CONFIGS[cfg])
        assert m.encoder.hidden_size == per_dir
        assert m.fc1.weight.shape == (256, 512)


def test_trainer_parser_defaults_build_an_rnn_encoder_model():
    """the trainer's own defaults (``--encoder_type rnn``, ``--enc_layers 2``, ``--rnn_size 512``, no ``--brnn``) give a model"""
    from pika_b200.model.transducer import Net
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    args = T.build_parser().parse_args(["transducer", "data.lst", "log", "out"])
    assert args.encoder_type == "rnn"
    m = Net(args, 240, 60)
    assert m.pack_seq and isinstance(m.encoder, torch.nn.LSTM)
    assert m.encoder.hidden_size == args.rnn_size and m.encoder.num_layers == args.enc_layers
    assert m.encoder.bidirectional == bool(args.brnn)
