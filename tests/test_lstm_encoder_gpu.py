"""The LSTM encoder (``--encoder_type rnn``) on the GPU: the ragged, (bi)directional persistent LSTM kernels and the layer around
them against torch's nn.LSTM over pack_padded_sequence, the whole model against the reference's own Net
(tests/golden/model_rnn_enc.npz), and the decoder, MBR and trainer entry points with that encoder."""
import copy
import os
import types

import numpy as np
import pytest
import torch
import torch.nn as nn
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_tf32():
    """the torch references run in true fp32 (cuDNN's RNN would otherwise use TF32 tensor cores)"""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def rel(a, b):
    a = torch.as_tensor(a).float().cpu(); b = torch.as_tensor(b).float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def ragged_lens(B, T, seed):
    """unsorted lengths with ties, one length-1 sequence and max(len) < T"""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(2, T - 2, (B,), generator=g)
    lens[0] = T - 3
    lens[B // 2] = 1
    lens[-1] = lens[1]
    return lens.int()


def torch_packed(lstm, x, lens):
    out, _ = lstm(pack_padded_sequence(x, lens.cpu().long(), batch_first=True, enforce_sorted=False))
    return pad_packed_sequence(out, batch_first=True)[0]


def layer_case(precision, H, bi, B, T=40, E=240, seed=0):
    from pika_b200 import engine as E_
    E_.set_precision(precision)
    try:
        torch.manual_seed(seed)
        lstm = nn.LSTM(E, H, num_layers=1, batch_first=True, bidirectional=bi).cuda()
        with torch.no_grad():
            for p in lstm.parameters():
                p.copy_(p.to(torch.bfloat16).float())
        lens = ragged_lens(B, T, seed)
        Tout = int(lens.max())
        x = torch.randn(B, T, E, device="cuda").to(torch.bfloat16).float()
        ref_lstm = copy.deepcopy(lstm)
        xr = x.clone().requires_grad_(True)
        ref = torch_packed(ref_lstm, xr, lens)
        assert ref.shape[1] == Tout
        dy = torch.randn(ref.shape, device="cuda") * 0.1
        grads = torch.autograd.grad(ref, [xr] + list(ref_lstm.parameters()), dy)
        # the encoder entry: T_out = max(len) < T, exact zeros past every length
        enc = E_.lstm_encoder_forward_act(lstm, x, lens.cuda())
        assert enc.shape == (B, Tout, (2 if bi else 1) * H) and enc.dtype == E_.act_dtype()
        # the layer itself, with a gradient for its input
        xa = x[:, :Tout].to(E_.act_dtype()).contiguous().requires_grad_(True)
        out = E_.LstmLayerFn.apply(xa, lens.cuda(), *E_._lstm_layer_params(lstm, 0))
        assert rel(out, enc) < 1e-5
        for p in lstm.parameters():
            p.grad = None
        out.backward(dy.to(out.dtype))
        return lens, out, ref, xa.grad, grads, lstm
    finally:
        E_.set_precision("bf16")


def check_case(lens, out, ref, dx, grads, lstm, tol_out, tol_grad):
    B = out.shape[0]
    for b in range(B):
        assert bool((out[b, int(lens[b]):] == 0).all()), "padded outputs must be exactly zero"
    assert rel(out, ref) < tol_out, rel(out, ref)
    Tout = out.shape[1]
    assert rel(dx, grads[0][:, :Tout]) < tol_grad, rel(dx, grads[0][:, :Tout])
    for (name, p), gr in zip(lstm.named_parameters(), grads[1:]):
        assert rel(p.grad, gr) < tol_grad, (name, rel(p.grad, gr))


@pytest.mark.parametrize("B", [5, 32, 45])
@pytest.mark.parametrize("bi", [False, True])
@pytest.mark.parametrize("H", [128, 256, 512, 200])
def test_ragged_lstm_layer_bf16_matches_packed_torch(H, bi, B):
    """bf16 production path: one cooperative launch for both directions (B > 32: several launches); H = 200 (not a multiple of
    64) takes the bf16 per-step path instead, a recurrent GEMM and a fused cell kernel per step.  Same bounds as
    test_lstm_persistent_kernel_bf16"""
    check_case(*layer_case("bf16", H, bi, B, seed=H + B + int(bi)), tol_out=2e-2, tol_grad=6e-2)


@pytest.mark.parametrize("B", [5, 45])
@pytest.mark.parametrize("bi", [False, True])
def test_ragged_lstm_layer_fp32_matches_packed_torch(bi, B):
    """fp32-class mode: the length-aware per-step path (gathered step-major rows, split-bf16 GEMMs)"""
    check_case(*layer_case("fp32", 128, bi, B, seed=7 + B), tol_out=1e-3, tol_grad=1e-3)


def test_lstm_encoder_rejects_bad_lengths():
    from pika_b200 import engine as E_
    lstm = nn.LSTM(16, 64, batch_first=True).cuda()
    x = torch.randn(2, 10, 16, device="cuda")
    for bad in ([0, 5], [11, 3]):
        with pytest.raises(ValueError):
            E_.lstm_encoder_forward_act(lstm, x, torch.tensor(bad))
    assert E_.lstm_encoder_forward_act(lstm, x, None).shape == (2, 10, 64)


def build_rnn(cfg, V=40):
    from test_lstm_encoder_cpu import CONFIGS, build
    return build(CONFIGS[cfg], V).cuda()


@pytest.mark.parametrize("cfg", ["bi", "uni"])
@pytest.mark.parametrize("precision,tol_act,tol_loss", [("fp32", 1e-3, 1e-3), ("bf16", 6e-2, 1e-3)])
def test_rnn_encoder_model_matches_reference(golden_dir, cfg, precision, tol_act, tol_loss):
    from fixture_utils import grad_fingerprint
    from pika_b200 import engine
    d = np.load(os.path.join(golden_dir, "model_rnn_enc.npz"))
    engine.set_precision(precision)
    engine.set_dropout_enabled(False)
    try:
        x = torch.from_numpy(d["x"]).cuda()
        y = torch.from_numpy(d["y"]).long().cuda()
        lens, ulens = torch.from_numpy(d["lens"]).cuda(), torch.from_numpy(d["ulens"]).cuda()
        m = build_rnn(cfg); m.train()
        enc = engine.model_encoder_forward_act(m, x, lens)
        assert rel(enc, d["enc_" + cfg]) < tol_act, rel(enc, d["enc_" + cfg])
        logits = m.forward(x, y, lens, softmax=False)
        assert tuple(logits.shape) == d["logits_" + cfg].shape
        assert rel(logits, d["logits_" + cfg]) < tol_act, rel(logits, d["logits_" + cfg])
        m3 = build_rnn(cfg); m3.train()
        costs = engine.transducer_loss(m3, x, y, lens, ulens, x_len=lens, t_out=int(d["lens"].max()))
        np.testing.assert_allclose(costs.detach().cpu().numpy(), d["costs_" + cfg], rtol=tol_loss)
        costs.sum().backward()
        worst = {}
        for k, p in m3.named_parameters():
            ref = d["gs_%s_%s" % (cfg, k)]
            assert p.grad is not None, k
            got = grad_fingerprint(p.grad.cpu(), 512)
            rn = np.linalg.norm(ref[3:])
            if rn < 1e-3 * ref[2]:
                continue
            err = np.linalg.norm(got[3:] - ref[3:]) / rn
            cos = float(np.dot(got[3:], ref[3:]) / (np.linalg.norm(got[3:]) * rn + 1e-30))
            worst[k] = (err, cos)
        errs = sorted(v[0] for v in worst.values())
        top = sorted(worst.items(), key=lambda kv: -kv[1][0])[:6]
        assert max(errs) < (3e-2 if precision == "fp32" else 0.5), top
        assert min(v[1] for v in worst.values()) > (0.9995 if precision == "fp32" else 0.9), top
        assert errs[len(errs) // 2] < (1.5e-2 if precision == "fp32" else 0.35), top
    finally:
        engine.set_precision("bf16")
        engine.set_dropout_enabled(True)


def _decoder(m, B, beam):
    from pika_b200.decoder.beam_transducer import GlobalScorer
    from pika_b200.decoder.transducer_decoder import TransducerDecoder
    dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.0)
    return TransducerDecoder(m, B, beam, n_best=beam, blk=0, global_scorer=GlobalScorer(), sm_scale=1.0, cuda=True, beam_prune=False,
                             args=dargs)


def _blank_friendly(m):
    with torch.no_grad():
        m.fc2.bias[0] += 3.0
    return m


def test_decode_batch_packs_the_rnn_encoder(golden_dir):
    from pika_b200 import engine
    d = np.load(os.path.join(golden_dir, "model_rnn_enc.npz"))
    engine.set_precision("fp32")
    try:
        m = _blank_friendly(build_rnn("bi")); m.eval()
        x = torch.from_numpy(d["x"]).cuda()
        lens = torch.from_numpy(d["lens"])
        ml = [int(t) + 10 for t in lens]
        ret, _ = _decoder(m, 3, 4).decode_batch(x, lens, max_len=ml)
        with torch.no_grad():
            enc_ref = torch_packed(m.encoder, x, lens)
        ret_ref, _ = _decoder(m, 3, 4).decode_batch(None, lens, max_len=ml, enc_out=enc_ref)
        toks = [[[int(t) for t in h] for h in row] for row in ret["predictions"]]
        toks_ref = [[[int(t) for t in h] for h in row] for row in ret_ref["predictions"]]
        assert toks == toks_ref
        sc = np.array([[float(v) for v in row] for row in ret["scores"]])
        sc_ref = np.array([[float(v) for v in row] for row in ret_ref["scores"]])
        np.testing.assert_allclose(sc, sc_ref, atol=1e-3, rtol=1e-3)
    finally:
        engine.set_precision("bf16")


def test_mbr_with_rnn_encoder(golden_dir):
    from pika_b200 import engine
    from pika_b200.trainer.mbr import mbr_forward_backward
    d = np.load(os.path.join(golden_dir, "model_rnn_enc.npz"))
    engine.set_precision("fp32")
    engine.set_dropout_enabled(False)
    try:
        V, beam = 40, 4
        m = _blank_friendly(build_rnn("bi"))
        x = torch.from_numpy(d["x"]).cuda()
        tl = torch.from_numpy(d["lens"]).int()
        ul = torch.from_numpy(d["ulens"]).int()
        target = torch.full((3, int(ul.max())), V, dtype=torch.long)
        y = torch.from_numpy(d["y"]).long()
        for i in range(3):
            target[i, :ul[i]] = y[i, :ul[i]]
        m.eval()
        ret, _ = _decoder(m, 3, beam).decode_batch(x, tl, max_len=[int(t) + int(u) + 3 for t, u in zip(tl, ul)])
        m.train()
        for p in m.parameters():
            p.grad = None
        mbr_loss, rnnt_costs = mbr_forward_backward(m, x, target.cuda(), tl.cuda(), ul.cuda(), ret, blk=0, rnnt_scale=0.5, sm_scale=1.0)
        assert np.isfinite(mbr_loss)
        for k, p in m.encoder.named_parameters():
            assert p.grad is not None and bool(torch.isfinite(p.grad).all()) and float(p.grad.abs().max()) > 0, k
        with torch.no_grad():
            costs = engine.transducer_loss(m, x, target.cuda(), tl.cuda(), ul.cuda(), x_len=tl.cuda())
        np.testing.assert_allclose(rnnt_costs.detach().cpu().numpy(), 0.5 * costs.cpu().numpy(), rtol=1e-4)
    finally:
        engine.set_precision("bf16")
        engine.set_dropout_enabled(True)


def test_train_cli_rnn_encoder_one_epoch(tmp_path):
    from test_loader_cpu import make_dataset
    from pika_b200.model.transducer import Net
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    lst, utts = make_dataset(tmp_path, n_utts=6, shards=1, n_lo=8000, n_hi=16000)
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--window-type=hamming\n--sample-frequency=16000\n--dither=1\n--low-freq=40\n--high-freq=-200\n--num-mel-bins=80\n")
    out = tmp_path / "out"
    out.mkdir()
    log = tmp_path / "log.WORKER-ID"
    argv = ["transducer", lst, str(log), str(out), "--cuda", "--local_rank", "0", "--encoder_type", "rnn", "--brnn", "--enc_layers", "2",
            "--decoder_type", "rnn", "--rnn_size", "512", "--embd_dim", "100", "--output_dim", "60", "--padding_idx", "60", "--padding_tgt", "60",
            "--dec_layers", "1", "--dropout", "0.3", "--model_lctx", "0", "--model_rctx", "0", "--model_stride", "1",
            "--lctx", "1", "--rctx", "1", "--feats_dim", "80", "--feat_config", str(cfg), "--batch_size", "3", "--num_workers", "1", "--batch_first", "--max_len", "1600",
            "--TU_limit", "50000", "--gain_range", "25,25", "--speed_rate", "1.0", "--grad_clip", "3.0", "--initial_lr", "0.002",
            "--final_lr", "0.001", "--momentum", "0.9", "--num_epochs", "1", "--num_batches_per_epoch", "2", "--sync_period", "1",
            "--block_momentum", "0.9", "--block_lr", "1.0", "--seed", "777"]
    os.environ.setdefault("WORLD_SIZE", "1")
    T.main(argv)
    text = open(str(log).replace("WORKER-ID", "0")).read()
    losses = [float(l.split("Loss:")[1].split()[0]) for l in text.splitlines() if "Overall Avg Loss" in l]
    assert "Training Finished" in text and losses and np.isfinite(losses).all()
    saved = torch.load(str(out / "model.epoch.0.0"), weights_only=False)
    args = types.SimpleNamespace(rnn_size=512, local_rank=0, decoder_type="rnn", brnn=True, encoder_type="rnn", embd_dim=100,
                                 padding_idx=60, dropout=0.3, dec_layers=1, enc_layers=2)
    fresh = Net(args, saved.input_dim, 60)
    fresh.load_state_dict({k: v.cpu() for k, v in saved.state_dict().items()})
    assert saved.pack_seq and isinstance(saved.encoder, nn.LSTM)
