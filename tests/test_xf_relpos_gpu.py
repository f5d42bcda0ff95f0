"""Relative-position self-attention in the transformer prediction net (``max_relative_positions`` m > 0) on the GPU, against
fixtures produced by executing the reference's own modules (tests/golden/model_xf_relpos.npz, decode_xf_relpos.npz;
make_golden_relpos.py): training forward / backward through the joint and the loss in both precision modes, beam search, the
dropout path, one MBR step, and m = 0 left exactly as it was.

Tolerances are test_xf_prednet_gpu.py's: fp32-class 1e-3 norm-relative on the prediction-net output, loss and every gradient;
bf16 3e-2 on activations and 0.12 on gradients."""
import os
import types

import numpy as np
import pytest
import torch

from test_oracle_xf_prednet import xf_inputs
from test_oracle_xf_relpos import build_xf_relpos

pytestmark = pytest.mark.gpu

REL_KEYS = ["decoder.transformer.%d.self_attn.relative_positions_embeddings.weight" % l for l in range(2)]


def rel(a, b):
    a = torch.as_tensor(a).float().cpu(); b = torch.as_tensor(b).float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _loss(m, y, enc, tl, ul):
    from pika_b200 import engine
    pred = engine.prednet_forward_act(m, y)
    costs = engine.JointLossFn.apply(engine._to_act(enc), pred, m, y.int().contiguous(), tl, ul, True)
    return pred, costs


@pytest.mark.parametrize("m_rel", [3, 16])
@pytest.mark.parametrize("precision,tol_act,tol_grad", [("fp32", 1e-3, 1e-3), ("bf16", 3e-2, 0.12)])
def test_relpos_train_matches_reference(golden_dir, precision, tol_act, tol_grad, m_rel):
    from fixture_utils import grad_fingerprint
    from pika_b200 import engine
    d = np.load(os.path.join(golden_dir, "model_xf_relpos.npz"))
    V, B, Tp, U = [int(v) for v in d["dims"]]
    pre = "m%d_" % m_rel
    engine.set_precision(precision)
    engine.set_dropout_enabled(False)
    try:
        m = build_xf_relpos(V, m_rel).cuda().train()
        y = torch.from_numpy(d["y"]).cuda()
        enc = torch.from_numpy(xf_inputs(int(d["seed"]), B, Tp)).cuda().requires_grad_(precision == "fp32")
        pred, costs = _loss(m, y, enc, torch.from_numpy(d["tlens"]).cuda(), torch.from_numpy(d["ulens"]).cuda())
        assert rel(pred, d[pre + "pred"]) < tol_act
        np.testing.assert_allclose(costs.detach().cpu().numpy(), d[pre + "costs"], rtol=1e-3)
        costs.sum().backward()
        worst = {}
        for k, p in m.named_parameters():
            if k.startswith("encoder."):
                continue
            ref = d[pre + "gs_" + k]
            assert p.grad is not None, k
            got = grad_fingerprint(p.grad.cpu(), 512)
            rn = np.linalg.norm(ref[3:])
            if ref[2] < 1e-7 or rn < 1e-3 * ref[2]:
                continue
            worst[k] = float(np.linalg.norm(got[3:] - ref[3:]) / rn)
            assert abs(got[2] - ref[2]) < tol_grad * ref[2], (k, got[2], ref[2])
        top = sorted(worst.items(), key=lambda kv: -kv[1])[:5]
        assert len(worst) > 40 and top[0][1] < tol_grad, top
        assert all(k in worst for k in REL_KEYS + ["embed.weight"]), sorted(worst)
        if precision == "fp32":
            ref = d[pre + "denc"]
            got = grad_fingerprint(enc.grad.cpu(), 512)
            assert np.linalg.norm(got[3:] - ref[3:]) / np.linalg.norm(ref[3:]) < tol_grad
    finally:
        engine.set_precision("bf16")
        engine.set_dropout_enabled(True)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_relpos_zero_table_equals_m0_and_m0_is_unchanged(precision):
    """With a zero table the band kernels add exact zeros (QR = 0, Pb R = 0, G = 0, dSb R = 0), so the prediction-net output and the
    costs must be bit-identical to the m = 0 model, which runs the unchanged masked-softmax path.  m = 0 modules carry no table, and
    the engine gives them the same output as modules built without the attribute at all.  Gradients agree to summation order: the
    embedding and LayerNorm parameter gradients are reduced with atomics, so they differ in the last bits between any two runs."""
    from pika_b200 import engine
    V, B, Tp, U = 40, 3, 14, 11
    g = torch.Generator().manual_seed(5)
    y = torch.randint(1, V, (B, U), generator=g)
    y[1, 7:] = V
    y[2, 4:] = V
    y = y.cuda()
    enc = torch.from_numpy(xf_inputs(21, B, Tp)).cuda()
    tl = torch.tensor([Tp, Tp - 2, Tp - 5], dtype=torch.int32, device="cuda")
    ul = torch.tensor([U, 7, 4], dtype=torch.int32, device="cuda")
    engine.set_precision(precision)
    engine.set_dropout_enabled(False)
    try:
        runs = []
        sd0 = build_xf_relpos(V, 0).state_dict()
        for m_rel in (0, 0, 5):
            m = build_xf_relpos(V, m_rel)
            if m_rel > 0:                                # the table shifts the seeded draws: take the m = 0 weights, a zero table
                assert sorted(m.load_state_dict(sd0, strict=False).missing_keys) == REL_KEYS
                with torch.no_grad():
                    for k in REL_KEYS:
                        m.get_parameter(k).zero_()
            m = m.cuda().train()
            if m_rel == 0 and runs:                                   # second m = 0 model: strip the attribute, as modules built before it existed
                for layer in m.decoder.transformer:
                    del layer.self_attn.max_relative_positions
                del m.decoder.max_relative_positions
            pred, costs = _loss(m, y, enc, tl, ul)
            costs.sum().backward()
            grads = {k: p.grad.clone() for k, p in m.named_parameters() if not k.startswith("encoder.") and k not in REL_KEYS}
            runs.append((pred.detach().clone(), costs.detach().clone(), grads))
            if m_rel > 0:
                assert all(float(m.get_parameter(k).grad.norm()) > 0 for k in REL_KEYS)
        for other in runs[1:]:
            assert torch.equal(runs[0][0], other[0]) and torch.equal(runs[0][1], other[1])
            assert runs[0][2].keys() == other[2].keys()
            for k in runs[0][2]:
                if k.endswith("linear_keys.bias"):       # analytically zero (the softmax's shift invariance): rounding noise only
                    continue
                assert rel(other[2][k], runs[0][2][k]) < 1e-5, (k, rel(other[2][k], runs[0][2][k]))
    finally:
        engine.set_precision("bf16")
        engine.set_dropout_enabled(True)


def test_relpos_dropout_path_runs():
    """training mode with dropout on (attention probabilities, residual, FFN): finite loss and gradients, the tables included"""
    from pika_b200 import engine
    V, B, Tp, U = 40, 2, 12, 7
    m = build_xf_relpos(V, 4).cuda().train()
    g = torch.Generator().manual_seed(3)
    y = torch.randint(1, V, (B, U), generator=g).cuda()
    enc = torch.from_numpy(xf_inputs(11, B, Tp)).cuda()
    _, costs = _loss(m, y, enc, torch.full((B,), Tp, dtype=torch.int32, device="cuda"), torch.full((B,), U, dtype=torch.int32, device="cuda"))
    costs.sum().backward()
    assert bool(torch.isfinite(costs).all())
    for k, p in m.named_parameters():
        if k.startswith("decoder."):
            assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k
    assert all(float(m.get_parameter(k).grad.norm()) > 0 for k in REL_KEYS)


@pytest.mark.parametrize("name,beam,nbest", [("b4n2", 4, 2), ("b8n4", 8, 4)])
def test_relpos_decode_matches_reference(golden_dir, name, beam, nbest):
    """fp32-class mode: every hypothesis bit-exact against the reference's decode_batch (the fixture's closest n-best neighbours are
    2e-2 apart), every score within 1e-3 relative"""
    from fixture_utils import decode_fixture_reinit_xf
    from pika_b200 import engine
    from pika_b200.decoder.beam_transducer import GlobalScorer
    from pika_b200.decoder.transducer_decoder import TransducerDecoder
    d = np.load(os.path.join(golden_dir, "decode_xf_relpos.npz"))
    V, B, Tp = [int(v) for v in d["dims"]]
    engine.set_precision("fp32")
    try:
        m = build_xf_relpos(V, int(d["m"]))
        decode_fixture_reinit_xf(m)
        m = m.cuda().eval()
        dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.0)
        dec = TransducerDecoder(m, B, beam, n_best=nbest, blk=0, global_scorer=GlobalScorer(), sm_scale=1.0, cuda=True, beam_prune=True,
                                args=dargs)
        enc = torch.from_numpy(xf_inputs(int(d["seed"]), B, Tp)).cuda()
        tl = torch.from_numpy(d["tlens"])
        ret, _ = dec.decode_batch(None, tl, max_len=[int(t) + 30 for t in tl], enc_out=enc)
    finally:
        engine.set_precision("bf16")
    for b in range(B):
        for n in range(nbest):
            sc, ref_sc = float(ret["scores"][b][n]), float(d["%s_score_%d_%d" % (name, b, n)])
            assert abs(sc - ref_sc) <= 1e-3 * abs(ref_sc), (b, n, sc, ref_sc)
            hyp = [int(t.item()) for t in ret["predictions"][b][n]]
            assert hyp == d["%s_pred_%d_%d" % (name, b, n)].tolist(), (b, n)


def test_relpos_mbr_step_runs():
    """one MBR step (N-best generation with the relative-position prediction net, RNN-T and MBR branches): finite loss and
    gradients, the tables receive a gradient"""
    from fixture_utils import decode_fixture_reinit_xf
    from pika_b200 import engine
    from pika_b200.decoder.beam_transducer import GlobalScorer
    from pika_b200.decoder.transducer_decoder import TransducerDecoder
    from pika_b200.trainer.mbr import mbr_forward_backward
    V, beam = 40, 4
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decode_small.npz"))
    x = torch.from_numpy(d["x"]).cuda()
    tl = torch.from_numpy(d["tlens"]).int()
    ul = torch.tensor([5, 3, 4], dtype=torch.int32)
    g = torch.Generator().manual_seed(11)
    target = torch.full((3, 5), V, dtype=torch.long)
    for i in range(3):
        target[i, :ul[i]] = torch.randint(1, V, (int(ul[i]),), generator=g)
    m = build_xf_relpos(V, 4)
    decode_fixture_reinit_xf(m)
    m = m.cuda().eval()
    engine.set_dropout_enabled(False)
    try:
        dargs = types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=0.0)
        dec = TransducerDecoder(m, 3, beam, n_best=beam, blk=0, global_scorer=GlobalScorer(), sm_scale=0.8, cuda=True, beam_prune=False,
                                args=dargs)
        ret, _ = dec.decode_batch(x, tl, max_len=[int(t) + int(u) + 3 for t, u in zip(tl, ul)])
        m.train()
        mbr_loss, rnnt_costs = mbr_forward_backward(m, x, target.cuda(), tl.cuda(), ul.cuda(), ret, blk=0, rnnt_scale=0.5, sm_scale=0.8)
    finally:
        engine.set_dropout_enabled(True)
    assert np.isfinite(mbr_loss) and bool(torch.isfinite(rnnt_costs).all())
    for k, p in m.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k
    assert all(float(m.get_parameter(k).grad.norm()) > 0 for k in REL_KEYS)


def test_train_cli_relpos_loss_decreases(tmp_path):
    """``--decoder_type transformer --max_relative_positions 16`` through the training entry point on a tiny synthetic corpus:
    finite losses that go down, and a pickled model that carries the tables"""
    from test_loader_cpu import make_dataset
    from pika_b200.trainer import train_transducer_bmuf_otfaug as T
    lst, _ = make_dataset(tmp_path, n_utts=8, shards=1, n_lo=14000, n_hi=22000)
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--window-type=hamming\n--sample-frequency=16000\n--dither=0\n--low-freq=40\n--high-freq=-200\n--num-mel-bins=80\n")
    out = tmp_path / "out"
    out.mkdir()
    log = tmp_path / "log.WORKER-ID"
    argv = ["transducer", lst, str(log), str(out), "--cuda", "--local_rank", "0", "--encoder_type", "transformer",
            "--decoder_type", "transformer", "--max_relative_positions", "16", "--rnn_size", "1024", "--embd_dim", "100",
            "--output_dim", "60", "--padding_idx", "60", "--padding_tgt", "60", "--dec_layers", "2", "--dropout", "0.0", "--brnn",
            "--model_lctx", "21", "--model_rctx", "21", "--model_stride", "4", "--lctx", "1", "--rctx", "1", "--feats_dim", "80",
            "--feat_config", str(cfg), "--batch_size", "4", "--num_workers", "1", "--batch_first", "--max_len", "1600", "--TU_limit", "50000",
            "--gain_range", "25,25", "--speed_rate", "1.0", "--grad_clip", "3.0", "--initial_lr", "0.002", "--final_lr", "0.001",
            "--momentum", "0.9", "--num_epochs", "5", "--num_batches_per_epoch", "2", "--sync_period", "1", "--block_momentum", "0.9",
            "--block_lr", "1.0", "--seed", "777"]
    os.environ.setdefault("WORLD_SIZE", "1")
    T.main(argv)
    text = open(str(log).replace("WORKER-ID", "0")).read()
    assert "Training Finished" in text
    losses = [float(l.split("Loss:")[1].split()[0]) for l in text.splitlines() if "Overall Avg Loss" in l]
    assert len(losses) == 5 and np.isfinite(losses).all() and min(losses[-2:]) < losses[0], losses
    m = torch.load(str(out / "model.epoch.4.0"), weights_only=False)
    tab = m.decoder.transformer[0].self_attn.relative_positions_embeddings.weight
    assert tuple(tab.shape) == (33, 64) and bool(torch.isfinite(tab).all())
