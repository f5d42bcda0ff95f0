"""The chunked TDNN-Transformer encoder on the GPU: forward and every parameter gradient against the float64 restatement with the same
per-layer masks (tests/chunk_oracle.py), the dependency bound bit for bit, the admit-all mask bit-identical to full context, decoding
and alignment equal to running them on the masked encoder output, and the trainers, the decoder and one MBR step from the command
line."""
import os
import types

import numpy as np
import pytest
import torch
from chunk_oracle import dependency_end, encoder_forward as ref_encoder_forward

pytestmark = pytest.mark.gpu


def rel(a, b):
    a = torch.as_tensor(a).double().cpu(); b = torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _encoder(seed=777):
    from pika_b200.model.rnnt_tdnn_transformer import Net
    torch.manual_seed(seed)
    return Net(240, 0, 1024, 1024, 9).cuda()


@pytest.mark.parametrize("precision,tol_act", [("fp32", 1e-3), ("bf16", 6e-2)])
def test_chunked_encoder_forward_and_gradients(precision, tol_act):
    """train mode (batch statistics), dropout off: C = 4 with two left chunks, so every layer's mask is partial"""
    from pika_b200 import engine
    engine.set_precision(precision)
    engine.set_dropout_enabled(False)
    try:
        enc = _encoder()
        enc.train()
        enc.chunk_size, enc.left_chunks = 4, 2
        g = torch.Generator().manual_seed(3)
        x = torch.randn(2, 200, 240, generator=g)
        y = engine.encoder_forward(enc, x.cuda())
        R = torch.randn(y.shape, generator=g)
        (y * R.cuda()).sum().backward()
        sd = {"encoder." + k: v.detach().cpu().double().requires_grad_(v.dtype.is_floating_point) for k, v in enc.state_dict().items()}
        y_ref = ref_encoder_forward(sd, x.double(), train=True, chunks=enc.chunk_masks())
        (y_ref * R.double()).sum().backward()
        assert rel(y, y_ref) < tol_act
        # the mask matters: full context is far from the chunked output
        y_full = ref_encoder_forward(sd, x.double(), train=True)
        assert rel(y_full, y_ref) > 3 * rel(y, y_ref)
        errs = {}
        for k, p in enc.named_parameters():
            ref = sd["encoder." + k].grad
            # analytically zero: a bias in front of a BatchNorm, and the key bias (softmax is invariant to a shift of a query's scores);
            # in bf16 these hold the rounding noise of the batch statistics, so they are bounded in the fp32-class mode only
            if ref.norm() < 1e-6 * max(1.0, float(sd["encoder." + k].detach().norm())):
                if precision == "fp32":
                    assert float(p.grad.abs().max()) < 1e-5, k
                continue
            errs[k] = rel(p.grad, ref)
        e = sorted(errs.values())
        worst = max(errs.items(), key=lambda kv: kv[1])
        # the bounds of tests/test_model_gpu.py's gradient samples (DESIGN.md section 4)
        assert worst[1] < (3e-2 if precision == "fp32" else 0.5), worst
        assert e[len(e) // 2] < (1.5e-2 if precision == "fp32" else 0.35), e[len(e) // 2]
    finally:
        engine.set_precision("bf16")
        engine.set_dropout_enabled(True)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("C,left", [(1, -1), (4, 2), (16, 0)])
def test_dependency_bound_bit_for_bit(precision, C, left):
    """eval mode: perturbing every input frame from p on leaves output frame t' bit-identical whenever W (floor((4 t' + 42) / W) + 1)
    <= p, W = 4C"""
    from pika_b200 import engine
    engine.set_precision(precision)
    try:
        enc = _encoder()
        enc.eval()
        enc.chunk_size, enc.left_chunks = C, left
        g = torch.Generator().manual_seed(C)
        T = 400
        x = torch.randn(3, T, 240, generator=g).cuda()
        with torch.no_grad():
            y = engine.encoder_forward(enc, x)
            W = 4 * C
            ends = torch.tensor([dependency_end(t, W) for t in range(y.shape[1])])
            for p in (64, 150, 257, 333):
                xp = x.clone()
                xp[:, p:] = torch.randn(3, T - p, 240, generator=g).cuda()
                yp = engine.encoder_forward(enc, xp)
                keep = (ends <= p).cuda()
                assert int(keep.sum()) > 0
                assert torch.equal(y[:, keep], yp[:, keep]), (p, int(keep.sum()))
                assert not torch.equal(y[:, ~keep], yp[:, ~keep])
    finally:
        engine.set_precision("bf16")


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_admit_all_chunk_is_full_context(precision):
    """a chunk wider than the utterance runs the unmasked path: same launches, bit-identical outputs, and gradients bit-identical
    wherever two full-context runs are (the LayerNorm weight gradients are summed with atomics, so their order may vary; elsewhere the
    difference stays within a few times that of the two full-context runs)"""
    from pika_b200 import _lib, engine
    engine.set_precision(precision)
    engine.set_dropout_enabled(False)
    try:
        g = torch.Generator().manual_seed(9)
        x = torch.randn(2, 300, 240, generator=g).cuda()
        R = torch.randn(2, 65, 1024, generator=g).cuda()           # sum(y) would have a zero gradient behind the final BatchNorm
        runs = []
        for C in (0, 0, 1000):
            enc = _encoder()
            enc.train()
            enc.chunk_size = C
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            y = engine.encoder_forward(enc, x)
            (y * R).sum().backward()
            torch.cuda.synchronize()
            runs.append((y, {k: p.grad.clone() for k, p in enc.named_parameters()}, _lib.launch_count() - n0))
        (y0, g0, n0), (_, g0b, _), (y1, g1, n1) = runs
        assert torch.equal(y0, y1) and n0 == n1
        for k in g0:
            if torch.equal(g0[k], g0b[k]):
                assert torch.equal(g0[k], g1[k]), k
            else:
                assert rel(g1[k], g0[k]) <= 4 * rel(g0b[k], g0[k]) + 1e-7, k
    finally:
        engine.set_precision("bf16")
        engine.set_dropout_enabled(True)


def _net(V=40, chunk_size=0, left_chunks=-1, prune_range=0):
    from pika_b200.model.transducer import Net
    torch.manual_seed(777)
    o = types.SimpleNamespace(rnn_size=1024, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="transformer", embd_dim=64,
                              padding_idx=V, dropout=0.0, dec_layers=2, enc_layers=9, prune_range=prune_range, chunk_size=chunk_size,
                              left_chunks=left_chunks)
    m = Net(o, 240, V).cuda().eval()
    with torch.no_grad():
        m.fc2.bias[0] += 2.0                  # blank-heavy, so decodes emit a few labels per utterance
    return m


def test_decode_and_align_use_the_masked_encoder():
    from pika_b200 import engine
    from pika_b200.decoder.beam_transducer import GlobalScorer
    from pika_b200.decoder.transducer_decoder import TransducerDecoder
    V = 40
    m = _net(V, chunk_size=4, left_chunks=1, prune_range=2)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(3, 240, 240, generator=g).cuda()
    tl = torch.tensor([50, 44, 38])
    with torch.no_grad():
        enc = engine.model_encoder_forward_act(m, x)
    m_full = _net(V, prune_range=2)
    with torch.no_grad():
        assert not torch.equal(enc, engine.model_encoder_forward_act(m_full, x))
    dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.0)
    dec = TransducerDecoder(m, 3, 4, n_best=2, blk=0, global_scorer=GlobalScorer(), sm_scale=1.0, cuda=True, beam_prune=True, args=dargs)
    ret, enc_d = dec.decode_batch(x, tl, max_len=[int(t) + 40 for t in tl])
    ret2, _ = dec.decode_batch(None, tl, max_len=[int(t) + 40 for t in tl], enc_out=enc)
    assert torch.equal(enc_d.to(enc.dtype), enc[:, :enc_d.shape[1]])
    for b in range(3):
        for h1, h2 in zip(ret["predictions"][b], ret2["predictions"][b]):
            assert [int(t) for t in h1] == [int(t) for t in h2]
        assert [float(s) for s in ret["scores"][b]] == [float(s) for s in ret2["scores"][b]]
    y = torch.randint(1, V, (3, 6), generator=g).cuda()
    ll = torch.tensor([6, 4, 5]).cuda()
    for R in (0, 2):
        got = engine.transducer_align(m, x, y, tl.cuda(), ll, prune_range=R)
        orig = engine.model_encoder_forward_act
        engine.model_encoder_forward_act = lambda *a, **kw: enc
        try:
            want = engine.transducer_align(m_full, x, y, tl.cuda(), ll, prune_range=R)
        finally:
            engine.model_encoder_forward_act = orig
        assert all(torch.equal(a, b) for a, b in zip(got, want)), R


def _cli_args(tmp_path, lst, cfg, extra):
    return ["transducer", lst, str(tmp_path / "log.WORKER-ID"), str(tmp_path / "out"), "--cuda", "--local_rank", "0", "--encoder_type",
            "transformer", "--decoder_type", "rnn", "--rnn_size", "1024", "--embd_dim", "100", "--output_dim", "60", "--padding_idx", "60",
            "--padding_tgt", "60", "--dec_layers", "2", "--dropout", "0.0", "--brnn", "--model_lctx", "21", "--model_rctx", "21",
            "--model_stride", "4", "--lctx", "1", "--rctx", "1", "--feats_dim", "80", "--feat_config", str(cfg), "--batch_size", "2",
            "--num_workers", "1", "--batch_first", "--max_len", "1600", "--TU_limit", "50000", "--gain_range", "25,25", "--speed_rate", "1.0",
            "--grad_clip", "3.0", "--initial_lr", "1e-3", "--final_lr", "1e-3", "--momentum", "0.9", "--num_epochs", "1",
            "--num_batches_per_epoch", "2", "--sync_period", "1", "--seed", "777"] + extra


def test_training_decoding_and_mbr_from_the_command_line(tmp_path):
    from test_loader_cpu import make_dataset
    from pika_b200.decoder import decode_transducer as D
    from pika_b200.loader.kaldi_io import write_float_matrix_ark
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T, train_transducer_mbr_bmuf_otfaug as M
    lst, _ = make_dataset(tmp_path, n_utts=4, shards=1, n_lo=14000, n_hi=18000)
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--window-type=hamming\n--sample-frequency=16000\n--dither=0\n--low-freq=40\n--high-freq=-200\n--num-mel-bins=80\n")
    os.environ.setdefault("WORLD_SIZE", "1")
    models = {}
    for name, extra in (("static", ["--chunk_size", "4", "--left_chunks", "2"]), ("dynamic", ["--dynamic_chunk_max", "8"])):
        (tmp_path / "out").mkdir(exist_ok=True)
        T.main(_cli_args(tmp_path, lst, cfg, extra))
        text = open(str(tmp_path / "log.0")).read()
        losses = [float(l.split("Loss:")[1].split()[0]) for l in text.splitlines() if "Overall Avg Loss" in l]
        assert "Training Finished" in text and len(losses) == 1 and np.isfinite(losses).all()
        models[name] = torch.load(str(tmp_path / "out" / "model.epoch.0.0"), weights_only=False)
        os.rename(str(tmp_path / "out" / "model.epoch.0.0"), str(tmp_path / ("%s.model" % name)))
    assert (models["static"].encoder.chunk_size, models["static"].encoder.left_chunks) == (4, 2)
    assert (models["dynamic"].encoder.chunk_size, models["dynamic"].encoder.left_chunks) == (0, -1)   # checkpoints record chunk size 0

    # decoding: an override on the dynamically trained model equals a model pickled with that setting
    rng = np.random.default_rng(2)
    feats = [("u%d" % i, rng.standard_normal((n, 80)).astype(np.float32)) for i, n in enumerate((180, 150, 120, 200))]
    write_float_matrix_ark(str(tmp_path / "feats.ark"), feats)
    (tmp_path / "labels.ark").write_text("".join("%s 1 2 3\n" % k for k, _ in feats))
    (tmp_path / "symbols.txt").write_text("".join("<%d> %d\n" % (i, i) for i in range(61)))
    m = models["dynamic"]
    m.encoder.chunk_size, m.encoder.left_chunks = 2, 1
    torch.save(m, str(tmp_path / "pickled_2_1.model"))

    def decode(model, out, extra=()):
        D.main([str(tmp_path / model), "ark:%s" % (tmp_path / "feats.ark"), "ark,t:%s" % (tmp_path / "labels.ark"), str(tmp_path / out),
                "--loader", "utt", "--cuda", "--batch_first", "--batch_size", "2", "--lctx", "1", "--rctx", "1", "--feats_dim", "80",
                "--max_len", "1000", "--padding_tgt", "60", "--symbols_map", str(tmp_path / "symbols.txt"), "--beam_size", "4",
                "--model_lctx", "21", "--model_rctx", "21", "--model_stride", "4", "--output_scores"] + list(extra))
        return (tmp_path / out).read_text()

    a = decode("dynamic.model", "a.txt", ["--chunk_size", "2", "--left_chunks", "1"])
    b = decode("pickled_2_1.model", "b.txt")
    c = decode("pickled_2_1.model", "c.txt", ["--chunk_size", "0"])
    d = decode("dynamic.model", "d.txt")
    assert a == b and c == d and len(a.splitlines()) == 4

    # one MBR step from the chunked model, with the flags inherited from the RNN-T trainer
    (tmp_path / "out").mkdir(exist_ok=True)
    M.main(_cli_args(tmp_path, lst, cfg, ["--init_model", str(tmp_path / "static.model"), "--chunk_size", "4", "--left_chunks", "2",
                                          "--num_batches_per_epoch", "1", "--beam_size", "4", "--rnnt_scale", "0.5"]))
    text = open(str(tmp_path / "log.0")).read()
    assert "Overall Avg MBR Loss" in text and "Training Finished" in text
    m = torch.load(str(tmp_path / "out" / "model.epoch.0.0"), weights_only=False)
    assert bool(torch.isfinite(m.fc2.weight).all()) and (m.encoder.chunk_size, m.encoder.left_chunks) == (4, 2)
