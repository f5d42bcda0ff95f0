"""Chunk-limited attention of the TDNN-Transformer encoder on the CPU: the per-layer geometry against the receptive field measured by
perturbation on the oracle encoder, the dependency bound in float64, the trainers' and the decoder's flag checks, and the dynamic
chunk draws (their own generator: no other random stream moves)."""
import random
import types

import numpy as np
import pytest
import torch
from chunk_oracle import allowed, dependency_end, encoder_forward


def _small_encoder(nhid=32, input_dim=8, output_dim=16, seed=3):
    from pika_b200.model.rnnt_tdnn_transformer import Net
    torch.manual_seed(seed)
    enc = Net(input_dim, 0, output_dim, nhid, 9)
    sd = {"encoder." + k: v.double() for k, v in enc.state_dict().items()}
    g = torch.Generator().manual_seed(seed)
    for k in sd:                                   # running statistics away from (0, 1), so eval mode is not the identity
        if k.endswith("running_mean"):
            sd[k] = torch.randn(sd[k].shape, generator=g, dtype=torch.float64) * 0.1
        elif k.endswith("running_var"):
            sd[k] = torch.rand(sd[k].shape, generator=g, dtype=torch.float64) + 0.5
    return enc, sd


def test_geometry_of_the_shipped_table():
    enc, _ = _small_encoder()
    assert enc.attention_geometry() == [(1, 6), (1, 24), (4, 42)]
    for C in (1, 4, 16):
        assert enc.chunk_masks(C, 2) == [(4 * C, 6, 2), (4 * C, 24, 2), (C, 10, 2)]
    assert enc.chunk_masks(0, -1) == [None, None, None]
    enc.chunk_size, enc.left_chunks = 8, -1
    assert enc.chunk_masks() == [(32, 6, -1), (32, 24, -1), (8, 10, -1)]
    with pytest.raises(ValueError):
        enc.chunk_masks(-1, -1)
    with pytest.raises(ValueError):
        enc.chunk_masks(4, -2)


def _attention_inputs(sd, x):
    """the inputs of the three attention layers of the oracle encoder in eval mode, with every attention reduced to the frame itself
    (a chunk of one frame and no earlier chunk): their dependence on x is then the TDNN stack's alone"""
    taps = []
    import chunk_oracle

    orig = chunk_oracle.transformer_layer

    def tap(h, *a, **kw):
        taps.append(h)
        return orig(h, *a, **kw)

    chunk_oracle.transformer_layer = tap
    try:
        encoder_forward(sd, x, train=False, chunks=[(1, 0, 0)] * 3)
    finally:
        chunk_oracle.transformer_layer = orig
    return taps


def test_geometry_matches_the_measured_receptive_field():
    """r_l(i), the rightmost input frame that moves frame i of attention layer l's input, is s_l * i + o_l"""
    enc, sd = _small_encoder()
    T = 90
    x = torch.randn(1, T, 8, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    base = _attention_inputs(sd, x)
    r = [torch.full((h.shape[1],), -1, dtype=torch.long) for h in base]
    for p in range(T):
        xp = x.clone()
        xp[:, p] += 1.0
        for l, h in enumerate(_attention_inputs(sd, xp)):
            moved = (h - base[l]).abs().amax(-1)[0] > 0
            r[l][moved] = p
    for (s, o), rl in zip(enc.attention_geometry(), r):
        i = torch.arange(rl.numel())
        assert torch.equal(rl, s * i + o)


@pytest.mark.parametrize("C,left", [(1, -1), (2, 1), (3, 0), (5, 2)])
def test_dependency_bound_float64(C, left):
    """output frame t' depends on input frames [0, W (floor((4 t' + 42) / W) + 1)) only, W = 4C: perturbing every input frame from p
    on leaves each output frame whose bound ends at or before p exactly unchanged, and moves at least one later frame"""
    enc, sd = _small_encoder()
    chunks = enc.chunk_masks(C, left)
    T = 120
    g = torch.Generator().manual_seed(C * 10 + left)
    x = torch.randn(2, T, 8, dtype=torch.float64, generator=g)
    y = encoder_forward(sd, x, train=False, chunks=chunks)
    W = 4 * C
    ends = torch.tensor([dependency_end(t, W) for t in range(y.shape[1])])
    for p in (43, 50, 61, 77, 100):
        xp = x.clone()
        xp[:, p:] = torch.randn(2, T - p, 8, dtype=torch.float64, generator=g)
        yp = encoder_forward(sd, xp, train=False, chunks=chunks)
        keep = ends <= p
        assert torch.equal(y[:, keep], yp[:, keep]), p
        assert bool((y[:, ~keep] != yp[:, ~keep]).any()), p
    # full context for comparison: the first output frame already sees the last input frame
    xp = x.clone()
    xp[:, -1] += 1.0
    assert bool((encoder_forward(sd, xp, train=False)[:, 0] != encoder_forward(sd, x, train=False)[:, 0]).any())


def test_allowed_mask_rule():
    A = allowed(10, 3, 1, 1)
    c = [(i + 1) // 3 for i in range(10)]
    for i in range(10):
        for j in range(10):
            assert bool(A[i, j]) == (c[i] - 1 <= c[j] <= c[i])


def test_chunk_attributes_are_not_state():
    from pika_b200.model.transducer import Net
    torch.manual_seed(0)
    opt = types.SimpleNamespace(rnn_size=64, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="transformer", embd_dim=8,
                                padding_idx=10, dropout=0.0, dec_layers=1, enc_layers=9, chunk_size=4, left_chunks=2)
    m = Net(opt, 8, 10)
    assert (m.encoder.chunk_size, m.encoder.left_chunks) == (4, 2)
    opt0 = types.SimpleNamespace(**{**vars(opt), "chunk_size": 0, "left_chunks": -1})
    torch.manual_seed(0)
    m0 = Net(opt0, 8, 10)
    assert list(m.state_dict()) == list(m0.state_dict())
    del m.encoder.chunk_size, m.encoder.left_chunks              # an encoder pickled before the attributes existed
    assert (m.encoder.chunk_size, m.encoder.left_chunks) == (0, -1) and m.encoder.chunk_masks() == [None] * 3


def _train_parser(mbr=False):
    if mbr:
        from pika_b200.trainer.train_transducer_mbr_bmuf_otfaug import build_parser
    else:
        from pika_b200.trainer.train_transducer_bmuf_otfaug import build_parser
    return build_parser()


@pytest.mark.parametrize("mbr", [False, True])
def test_trainer_flag_checks(mbr):
    from pika_b200.trainer.train_transducer_bmuf_otfaug import check_chunk_args
    pos = ["transducer", "data.lst", "log", "out"]
    bad = [["--encoder_type", "rnn", "--chunk_size", "4"], ["--encoder_type", "rnn", "--dynamic_chunk_max", "4"],
           ["--encoder_type", "rnn", "--chunk_size", "4", "--left_chunks", "2"], ["--encoder_type", "transformer", "--chunk_size", "-1"],
           ["--encoder_type", "transformer", "--dynamic_chunk_max", "-2"],
           ["--encoder_type", "transformer", "--chunk_size", "4", "--left_chunks", "-2"],
           ["--encoder_type", "transformer", "--chunk_size", "4", "--dynamic_chunk_max", "8"],
           ["--encoder_type", "transformer", "--left_chunks", "2"]]
    for flags in bad:
        p = _train_parser(mbr)
        args = p.parse_args(pos + flags)
        with pytest.raises(SystemExit):
            check_chunk_args(p, args)
    good = [[], ["--encoder_type", "transformer", "--chunk_size", "4", "--left_chunks", "2"],
            ["--encoder_type", "transformer", "--dynamic_chunk_max", "8"],
            ["--encoder_type", "transformer", "--dynamic_chunk_max", "8", "--left_chunks", "0"], ["--encoder_type", "rnn"]]
    for flags in good:
        p = _train_parser(mbr)
        args = p.parse_args(pos + flags)
        check_chunk_args(p, args)
    args = _train_parser(mbr).parse_args(pos)
    assert (args.chunk_size, args.left_chunks, args.dynamic_chunk_max) == (0, -1, 0)


def test_decoder_and_aligner_overrides():
    from pika_b200.decoder import align_transducer, decode_transducer
    from pika_b200.model.rnnt_tdnn_transformer import Net as Enc
    pos = ["model", "feats", "labels", "out"]
    for build in (decode_transducer.build_parser, align_transducer.build_parser):
        p = build()
        args = p.parse_args(pos)
        assert args.chunk_size is None and args.left_chunks is None
        model = types.SimpleNamespace(encoder=Enc(8, 0, 16, 32, 9))
        model.encoder.chunk_size, model.encoder.left_chunks = 6, 1
        decode_transducer.apply_chunk_args(p, args, model)                     # as trained
        assert (model.encoder.chunk_size, model.encoder.left_chunks) == (6, 1)
        decode_transducer.apply_chunk_args(p, p.parse_args(pos + ["--chunk_size", "0"]), model)
        assert (model.encoder.chunk_size, model.encoder.left_chunks) == (0, 1)
        decode_transducer.apply_chunk_args(p, p.parse_args(pos + ["--chunk_size", "3", "--left_chunks", "-1"]), model)
        assert (model.encoder.chunk_size, model.encoder.left_chunks) == (3, -1)
        for flags in (["--chunk_size", "-1"], ["--left_chunks", "-2"]):
            with pytest.raises(SystemExit):
                decode_transducer.apply_chunk_args(p, p.parse_args(pos + flags), model)
        lstm = types.SimpleNamespace(encoder=torch.nn.LSTM(8, 8))
        with pytest.raises(SystemExit):
            decode_transducer.apply_chunk_args(p, p.parse_args(pos + ["--chunk_size", "4"]), lstm)


def test_dynamic_chunk_draws_leave_other_streams_alone():
    from pika_b200.trainer.step import chunk_for_batch, encoder_chunk
    torch.manual_seed(5)
    np.random.seed(5)
    random.seed(5)
    states = (torch.get_rng_state(), np.random.get_state()[1].copy(), random.getstate())
    args = types.SimpleNamespace(seed=777, local_rank=0, chunk_size=0, dynamic_chunk_max=8)
    draws = [chunk_for_batch(args, i) for i in range(4000)]
    assert torch.equal(torch.get_rng_state(), states[0])
    assert np.array_equal(np.random.get_state()[1], states[1]) and random.getstate() == states[2]
    assert all(0 <= c <= 8 for c in draws)
    full = sum(c == 0 for c in draws) / len(draws)
    assert 0.45 < full < 0.55
    counts = np.bincount([c for c in draws if c], minlength=9)[1:]
    assert counts.min() > 0.7 * counts.mean()
    assert draws == [chunk_for_batch(args, i) for i in range(4000)]              # reproducible per (seed, rank, index)
    other = types.SimpleNamespace(**{**vars(args), "local_rank": 1})
    assert draws[:200] != [chunk_for_batch(other, i) for i in range(200)]
    static = types.SimpleNamespace(seed=777, local_rank=0, chunk_size=6, dynamic_chunk_max=0)
    assert chunk_for_batch(static, 3) is None                                     # the encoder keeps its own setting
    # the setting holds inside the block only, so a checkpoint records the static chunk size
    from pika_b200.model.rnnt_tdnn_transformer import Net as Enc
    model = types.SimpleNamespace(encoder=Enc(8, 0, 16, 32, 9))
    with encoder_chunk(model, 5):
        assert model.encoder.chunk_size == 5
    assert model.encoder.chunk_size == 0
    with encoder_chunk(model, None):
        assert model.encoder.chunk_size == 0
