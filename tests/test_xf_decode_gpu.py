"""Beam search with the transformer prediction net on its incremental KV-cached step (pika_b200/csrc/beam_xf.cu,
decoder/transducer_decoder.py:_XfBuffers), replayed from a CUDA graph, with and without FST shallow fusion.

* FST fusion against tests/golden/decode_xf_fst.npz (make_golden_xf_fst.py: the reference's own TransducerDecoder + SortedMatcher).
* The incremental step against the full-history forward (engine.conv_transformer_lm_forward_act) on seeded histories, m = 0 / 3,
  both precisions, including rows that share prefixes through a permuted slot table.
* Graph vs eager issue, workspace reuse, the documented limits and the command-line entry point with ``--fst_lm``."""
import os
import types

import numpy as np
import pytest
import torch

from test_oracle_xf_prednet import build_xf, xf_inputs
from test_oracle_xf_relpos import build_xf_relpos

pytestmark = pytest.mark.gpu
V = 40


def _dargs(reward):
    return types.SimpleNamespace(las_rescorer=None, las_rescorer_bw=None, bilas_rescorer=None, nonblk_reward=reward)


def _model(m_rel, reinit=True):
    from fixture_utils import decode_fixture_reinit_xf
    m = build_xf(V) if m_rel == 0 else build_xf_relpos(V, m_rel)
    if reinit:
        decode_fixture_reinit_xf(m)
    return m.cuda().eval()


def _matcher():
    from make_inputs import toy_backoff_lm
    from pika_b200.decoder.sorted_matcher import SortedMatcher
    arcs, finals = toy_backoff_lm(V)
    return SortedMatcher((arcs, finals), max(len(a) for a in arcs), V + 2, 1, [])


def _decoder(m, B, beam, nbest, fst=True):
    from pika_b200.decoder.beam_transducer import GlobalScorer
    from pika_b200.decoder.transducer_decoder import TransducerDecoder
    kw = dict(lm_scorer=_matcher(), lm_scorer_scale=0.5) if fst else {}
    return TransducerDecoder(m, B, beam, n_best=nbest, blk=0, global_scorer=GlobalScorer(), sm_scale=1.0, cuda=True, beam_prune=True,
                             args=_dargs(0.45 if fst else 0.0), **kw)


def _hyps(ret):
    return [[[int(t) for t in h] for h in row] for row in ret["predictions"]], [[float(s) for s in row] for row in ret["scores"]]


@pytest.mark.parametrize("case", range(3))
def test_xf_fst_decode_matches_reference(golden_dir, case):
    """tokens bit-exact for n = 0 and wherever the reference's n-best neighbours are more than 5e-3 apart, every score within 1e-3
    (the criterion of the existing decode tests); fp32-class mode"""
    from pika_b200 import engine
    f = np.load(os.path.join(golden_dir, "decode_xf_fst.npz"))
    name, beam, nbest, m_rel = str(f["cases"][case]), int(f["beams"][case]), int(f["nbests"][case]), int(f["rel_m"][case])
    _, B, Tp = [int(v) for v in f["dims"]]
    engine.set_precision("fp32")
    try:
        dec = _decoder(_model(m_rel), B, beam, nbest)
        enc = torch.from_numpy(xf_inputs(int(f["seed"]), B, Tp)).cuda()
        tl = torch.from_numpy(f["tlens"])
        ret, _ = dec.decode_batch(None, tl, max_len=[int(t) + 30 for t in tl], enc_out=enc)
    finally:
        engine.set_precision("bf16")
    assert dec.last_replays > 0
    exact = 0
    for b in range(B):
        ref_scores = [float(f["%s_score_%d_%d" % (name, b, n)]) for n in range(nbest)]
        for n in range(nbest):
            sc = float(ret["scores"][b][n])
            assert abs(sc - ref_scores[n]) < 1e-3 * abs(sc) + 1e-3, (name, b, n, sc, ref_scores[n])
            gap = min([abs(ref_scores[n] - ref_scores[j]) for j in (n - 1, n + 1) if 0 <= j < nbest])
            hyp = [int(t.item()) for t in ret["predictions"][b][n]]
            ref = f["%s_pred_%d_%d" % (name, b, n)].tolist()
            if gap > 5e-3 or n == 0:
                assert hyp == ref, (name, b, n, gap, hyp[:30], ref[:30])
                exact += 1
    assert exact >= B * nbest - 3


# history lengths: empty, the conv taps' edge (4, 5), past m, around the attention kernel's 32-key rounds, long
_LENS = [0, 1, 4, 5, 2, 31, 32, 33, 63, 64, 65, 300]


def _full_last(m, hists):
    """the full-history forward's output at every history's last position"""
    from pika_b200 import engine
    L = max(len(h) for h in hists) + 1
    src = torch.full((len(hists), L), V, dtype=torch.long)                  # padding id = V
    src[:, 0] = 0
    for r, h in enumerate(hists):
        src[r, 1:len(h) + 1] = torch.tensor(h, dtype=torch.long)
    out = engine.conv_transformer_lm_forward_act(m.decoder, src.cuda())
    return torch.stack([out[r, len(h)] for r, h in enumerate(hists)]).float()


def _row_err(got, ref):
    return ((got.float() - ref).norm(dim=1) / ref.norm(dim=1)).max().item()


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-4), ("bf16", 3e-2)])   # measured on an H100: fp32 9.5e-6, bf16 7.9e-3 (worst row)
@pytest.mark.parametrize("m_rel", [0, 3])
def test_xf_incremental_step_matches_full_recompute(m_rel, precision, tol):
    """dec_hid of the incremental step == the full-history forward at the last position, per row (norm-relative): the histories are built
    one step at a time (rows of unequal length, so other rows are masked meanwhile), then rows continue other rows' prefixes of
    several lengths through a permuted slot table"""
    from pika_b200 import engine
    B, beam, S = 3, 4, 320
    rows = B * beam
    rng = np.random.default_rng(41 + m_rel)
    engine.set_precision(precision)
    try:
        m = _model(m_rel, reinit=False)
        dec = _decoder(m, B, beam, 1, fst=False)
        ws = dec._workspace(B, 4, S, engine.act_dtype(), torch.device("cuda", torch.cuda.current_device()))
        ws.stage(dec)
        ws.reset(dec, torch.zeros(B, 4, ws.H, device="cuda"), [4] * B, [S - 2] * B)
        xf = ws.xf
        ws.xf.step(dec, ws.h[0], init=True)
        next_ys, hyp_tok, hyp_len = ws.next_ys.view(-1, rows), ws.hyp_tok.view(2, rows, -1), ws.hyp_len.view(2, rows)
        slot = xf.slot.view(2, rows, -1)
        hists = [rng.integers(1, V, n).tolist() for n in _LENS]

        def run_step(t, toks, lens):
            par = t & 1
            if t > 0:
                slot[par].copy_(slot[par ^ 1])
            ws.step_ctx.copy_(torch.tensor([t, 1], dtype=torch.int32))
            next_ys[t].copy_(torch.tensor(toks, dtype=torch.int32))
            hyp_len[par].copy_(torch.tensor(lens, dtype=torch.int32))
            for r, n in enumerate(lens):
                if n > 0:
                    hyp_tok[par, r, :n] = torch.tensor(cur[r][:n], dtype=torch.int32)
            xf.step(dec, ws.h[0])

        cur = hists
        T1 = max(_LENS)
        for t in range(T1):
            run_step(t, [h[t] if t < len(h) else 0 for h in hists], [min(t + 1, len(h)) for h in hists])
        err1 = _row_err(ws.h[0], _full_last(m, hists))
        # continue other rows' prefixes: row r takes src[r]'s first k positions (SOS + k - 1 labels) and appends a new label
        src = rng.integers(0, rows, rows)
        src[:4] = _LENS.index(300)                                            # four rows share one long history
        keep = [int(rng.integers(0, len(hists[s]) + 1)) if r % 3 else len(hists[s]) for r, s in enumerate(src)]
        keep[:4] = [300, 64, 63, 0]
        old = slot[(T1 - 1) & 1].clone()
        new = [hists[s][:k] + [int(rng.integers(1, V))] for s, k in zip(src, keep)]
        par = T1 & 1
        for r, (s, k) in enumerate(zip(src, keep)):
            slot[par ^ 1, r, :k + 1] = old[s, :k + 1]                          # run_step copies parity par ^ 1 into par
        cur = new
        run_step(T1, [h[-1] for h in new], [len(h) for h in new])
        err2 = _row_err(ws.h[0], _full_last(m, new))
    finally:
        engine.set_precision("bf16")
    assert err1 < tol and err2 < tol, (err1, err2)


@pytest.mark.parametrize("fst", [False, True])
def test_xf_graph_replay_matches_eager(fst):
    """the same batch decoded with every launch issued from the host and from the captured graph: identical tokens and scores"""
    from pika_b200.decoder import transducer_decoder as td
    d_B, Tp, beam = 4, 24, 8
    m = _model(4)
    enc = torch.from_numpy(xf_inputs(808, d_B, Tp)).cuda()
    tl = torch.tensor([24, 21, 17, 9])
    ml = [int(t) + 30 for t in tl]
    saved = td._USE_GRAPH
    try:
        td._USE_GRAPH = False
        eager = _decoder(m, d_B, beam, 4, fst)
        r0, _ = eager.decode_batch(None, tl, max_len=ml, enc_out=enc)
        td._USE_GRAPH = True
        graph = _decoder(m, d_B, beam, 4, fst)
        r1, _ = graph.decode_batch(None, tl, max_len=ml, enc_out=enc)
        r2, _ = graph.decode_batch(None, tl, max_len=ml, enc_out=enc)                  # replay of the stored graph
    finally:
        td._USE_GRAPH = saved
    assert eager._ws.graph is None and graph._ws.graph is not None
    assert graph.last_replays > 0 and graph.kernels_per_replay > 0
    assert _hyps(r0) == _hyps(r1) == _hyps(r2)
    assert any(len(h) > 20 for row in _hyps(r0)[0] for h in row)


def test_xf_workspace_reuse_equals_fresh_decoders():
    """two different batches (the second with more frames, so the workspace grows) through one decoder == each through a fresh one"""
    m = _model(0)
    B, beam = 4, 4
    batches = [(torch.from_numpy(xf_inputs(808, B, 24)).cuda(), torch.tensor([24, 21, 17, 9]), 30),
               (torch.from_numpy(xf_inputs(909, B, 31)).cuda(), torch.tensor([12, 31, 25, 7]), 10),
               (torch.from_numpy(xf_inputs(808, B, 24)).cuda(), torch.tensor([24, 21, 17, 9]), 30)]
    one = _decoder(m, B, beam, 2)
    for enc, tl, extra in batches:
        ml = [int(t) + extra for t in tl]
        got, _ = one.decode_batch(None, tl, max_len=ml, enc_out=enc)
        want, _ = _decoder(m, B, beam, 2).decode_batch(None, tl, max_len=ml, enc_out=enc)
        assert _hyps(got) == _hyps(want)


def test_xf_limits_raise_before_any_launch():
    from pika_b200 import _lib
    from pika_b200._lib import PikaError
    m = _model(0)
    n0 = _lib.launch_count()
    dec = _decoder(m, 2, 4, 1)
    with pytest.raises(PikaError, match="max_size"):
        dec.decode_batch(None, torch.tensor([10, 8]), max_len=[100, 4999], enc_out=torch.zeros(2, 10, 1024, device="cuda"))
    for layer in m.decoder.transformer:
        layer.self_attn.head_count = 4                                      # d_model 512 / 4 heads: head size 128
    with pytest.raises(PikaError, match="head size of 64"):
        _decoder(m, 2, 4, 1)
    assert _lib.launch_count() == n0


def _write_fst_text(path):
    from make_inputs import toy_backoff_lm
    arcs, finals = toy_backoff_lm(V)
    with open(path, "w") as f:
        for s, a in enumerate(arcs):
            for il, w, ns in a:
                f.write("%d\t%d\t%d\t%d\t%r\n" % (s, ns, il, il, w))
        for s, w in enumerate(finals):
            if np.isfinite(w):
                f.write("%d\t%r\n" % (s, w))
    return max(len(a) for a in arcs)


def test_xf_decode_cli_with_fst_end_to_end(tmp_path):
    """decoder/decode_transducer.py with a transformer-prediction-net model and ``--fst_lm`` (OpenFst text form): the N-best lines must be
    what a direct TransducerDecoder call with the same SortedMatcher gives on the same processed features"""
    from fixture_utils import decode_fixture_reinit_xf
    from pika_b200 import engine
    from pika_b200.decoder import decode_transducer as D
    from pika_b200.decoder.beam_transducer import GlobalScorer
    from pika_b200.decoder.sorted_matcher import SortedMatcher, read_fst_text
    from pika_b200.decoder.transducer_decoder import TransducerDecoder
    from pika_b200.loader import utt_loader as UL
    from pika_b200.loader.kaldi_io import write_float_matrix_ark
    from pika_b200.model.transducer import Net
    nutt, bs, beam, nbest = 4, 2, 4, 2
    torch.manual_seed(777)
    margs = types.SimpleNamespace(rnn_size=1024, local_rank=0, decoder_type="transformer", brnn=True, encoder_type="transformer",
                                  embd_dim=100, padding_idx=V, dropout=0.2, dec_layers=2, enc_layers=9)
    m = Net(margs, 240, V)
    decode_fixture_reinit_xf(m)
    torch.save(m, str(tmp_path / "model.pt"))
    rng = np.random.default_rng(6)
    feats = [("u%d" % i, rng.standard_normal((int(rng.integers(90, 131)), 80)).astype(np.float32)) for i in range(nutt)]
    write_float_matrix_ark(str(tmp_path / "feats.ark"), feats)
    (tmp_path / "labels.ark").write_text("".join("%s 1 2\n" % k for k, _ in feats))
    (tmp_path / "symbols.txt").write_text("".join("<%d> %d\n" % (i, i) for i in range(V + 1)))
    max_arcs = _write_fst_text(str(tmp_path / "G.txt"))
    out = tmp_path / "hyp.txt"
    argv = [str(tmp_path / "model.pt"), "ark:%s" % (tmp_path / "feats.ark"), "ark,t:%s" % (tmp_path / "labels.ark"), str(out), "--loader", "utt",
            "--cuda", "--batch_first", "--batch_size", str(bs), "--beam_size", str(beam), "--n_best", str(nbest), "--lctx", "1", "--rctx", "1",
            "--feats_dim", "80", "--max_len", "400", "--padding_tgt", str(V), "--symbols_map", str(tmp_path / "symbols.txt"),
            "--model_lctx", "21", "--model_rctx", "21", "--model_stride", "4", "--min_len", "60", "--output_scores",
            "--fst_lm", str(tmp_path / "G.txt"), "--fst_lm_scale", "0.5", "--nonblk_reward", "0.45", "--max_num_arcs", str(max_arcs),
            "--max_id", str(V + 2), "--backoff_id", "1"]
    prec = engine.get_precision()
    engine.set_precision("fp32")
    try:
        D.main(argv)
        lines = out.read_text().splitlines()
        assert len(lines) == nutt * nbest
        la = types.SimpleNamespace(lctx=1, rctx=1, max_len=400, batch_size=bs, padding_tgt=V, feats_dim=80, batch_first=True, stride=1,
                                   queue_size=8, cuda=True, local_rank=0, ctc_target=False)
        mg = m.cuda().eval()
        matcher = SortedMatcher(read_fst_text(str(tmp_path / "G.txt")), max_arcs, V + 2, 1, [])
        dec = TransducerDecoder(mg, bs, beam, n_best=nbest, blk=0, global_scorer=GlobalScorer(), sm_scale=1.0, cuda=True, beam_prune=True,
                                lm_scorer=matcher, lm_scorer_scale=0.5, args=_dargs(0.45))
        want = []
        for data, _, lens, _ in UL.dataloader("ark,t:%s" % (tmp_path / "labels.ark"), "ark:%s" % (tmp_path / "feats.ark"), False, la):
            tl = torch.from_numpy(lens).cuda() - 42
            tl = tl // 4 + torch.ne(tl % 4, 0).int()
            ret, _ = dec.decode_batch(data, tl, (tl + 100).tolist())
            for i in range(bs):
                for j in range(nbest):
                    want.append("".join("<%d>" % int(e.item()) for e in ret["predictions"][i][j] if e != 0))
        got = [l.split(" ")[0] for l in lines]
        assert got == want and any(len(g) > 0 for g in got)
        assert all(np.isfinite(float(l.split(" ")[1])) for l in lines)
    finally:
        engine.set_precision(prec)
