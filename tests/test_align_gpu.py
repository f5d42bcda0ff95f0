"""Forced alignment on the GPU (pk_rnnt_tables, pk_rnnt_pruned_tables, pk_rnnt_lattice_costs, pk_rnnt_viterbi, engine.transducer_align
and the align_transducer CLI) against the float64 oracle (tests/viterbi_oracle.py) and float64 restatements of the model."""
import copy
import math
import types

import numpy as np
import pytest
import torch

import viterbi_oracle as VO

pytestmark = pytest.mark.gpu

PRECS = ["bf16", "fp32"]


@pytest.fixture
def prec(request):
    from pika_b200 import engine
    old = engine.get_precision()
    engine.set_precision(request.param)
    yield request.param
    engine.set_precision(old)


def _lens(*v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def _random_tables(rng, Ts, Us, grid=None, p_inf=0.0):
    """natural [B, T, U1] f32 tables; ``grid``: dyadic values (exact sums, built ties); ``p_inf``: share of -inf nodes"""
    B, T, U1 = len(Ts), max(Ts), max(Us) + 1
    lpb = rng.uniform(-4.0, 0.0, (B, T, U1))
    lpl = rng.uniform(-4.0, 0.0, (B, T, U1))
    if grid is not None:
        lpb, lpl = np.round(lpb / grid) * grid, np.round(lpl / grid) * grid
    if p_inf:
        lpb[rng.random(lpb.shape) < p_inf] = -np.inf
        lpl[rng.random(lpl.shape) < p_inf] = -np.inf
    return lpb.astype(np.float32), lpl.astype(np.float32)


def _run_kernel(lpb, lpl, Ts, Us, ld=None):
    from pika_b200 import kernels as K
    B, T, U1 = lpb.shape
    sb = torch.from_numpy(VO.to_skew(lpb, T, U1)).cuda()
    sl = torch.from_numpy(VO.to_skew(lpl, T, U1)).cuda()
    fl, ll = _lens(*Ts), _lens(*Us)
    score, emit, dec = K.rnnt_viterbi(sb, sl, fl, ll, B, T, U1, ld_emit=ld, want_decisions=True)
    costs = K.rnnt_lattice_costs(sb, sl, fl, ll, B, T, U1)
    return score.cpu().numpy(), emit.cpu().numpy(), dec.cpu().numpy(), -costs.cpu().numpy()


# (Ts, Us): every cells-per-thread path (U1 <= 512: 1, <= 1024: 2, <= 1536: 3, <= 2048: 4), T = 1, U = 0, ragged batches
KERNEL_CASES = [
    ((1,), (0,)),
    ((1, 3, 2), (0, 2, 4)),
    ((7, 40, 23), (31, 32, 5)),
    ((50, 37), (63, 64)),
    ((6, 9), (511, 300)),
    ((5, 4), (700, 1023)),
    ((4, 3), (1100, 1535)),
    ((3, 4), (2047, 1600)),
]


@pytest.mark.parametrize("Ts,Us", KERNEL_CASES)
@pytest.mark.parametrize("kind", ["random", "ties", "inf"])
def test_viterbi_kernel_against_oracle(Ts, Us, kind):
    """decisions and emit_frames bit-equal to the oracle, the score its f64 value rounded to f32; consistency with the tables and the
    total log-likelihood; two runs bit-identical"""
    rng = np.random.default_rng(sum(Us) * 7 + len(kind))
    grid, p_inf = {"random": (None, 0.0), "ties": (0.5, 0.0), "inf": (0.25, 0.15)}[kind]
    lpb, lpl = _random_tables(rng, Ts, Us, grid, p_inf)
    ld = max(Us) + 3                                          # padding past U1 - 1 is written -1 too
    score, emit, dec, loglik = _run_kernel(lpb, lpl, Ts, Us, ld)
    again = _run_kernel(lpb, lpl, Ts, Us, ld)
    for a, b in zip((score, emit, dec, loglik), again):
        np.testing.assert_array_equal(a, b)
    n_found = 0
    for b, (T, U) in enumerate(zip(Ts, Us)):
        s, d, frames = VO.viterbi(lpb[b], lpl[b], T, U)
        np.testing.assert_array_equal(VO.decision_bits(dec[b], T, U), d, err_msg="decisions of utterance %d" % b)
        np.testing.assert_array_equal(emit[b, :U], frames)
        assert (emit[b, U:] == -1).all()
        assert score[b] == np.float32(s), (b, score[b], s)
        if s == -np.inf:
            assert (emit[b] == -1).all() and loglik[b] == -np.inf
            continue
        n_found += 1
        # the tables summed along the returned path (f64, path order) are the score; the best path is at most the total
        arcs, t = [], 0
        for f in emit[b, :U]:
            arcs += [0] * (int(f) - t) + [1]
            t = int(f)
        arcs += [0] * (T - 1 - t)
        assert np.float32(VO.path_score(lpb[b], lpl[b], arcs)) == score[b]
        assert score[b] <= loglik[b] + 1e-5 * abs(loglik[b])
    if kind != "inf":
        assert n_found == len(Ts)


def test_viterbi_kernel_no_path_and_padding():
    """an utterance whose lattice has no finite path (a -inf blank on the last frame) scores -inf and gets -1 frames; T = 0 too"""
    rng = np.random.default_rng(3)
    Ts, Us = (5, 5, 4), (3, 2, 1)
    lpb, lpl = _random_tables(rng, Ts, Us)
    lpb[0, 4, 3] = -np.inf                                      # the final blank of utterance 0
    score, emit, dec, loglik = _run_kernel(lpb, lpl, Ts, Us)
    assert score[0] == -np.inf and loglik[0] == -np.inf and (emit[0] == -1).all()
    assert np.isfinite(score[1:]).all()
    score, emit, _, _ = _run_kernel(lpb, lpl, (0, 5, 4), Us)
    assert score[0] == -np.inf and (emit[0] == -1).all() and np.isfinite(score[1:]).all()


# ------------------------------------------------------------------------------------------------ the engine against float64
def _net(encoder_type, decoder_type, V, prune_range=0, m_rel=0):
    from pika_b200.model.transducer import Net
    torch.manual_seed(777)
    o = types.SimpleNamespace(rnn_size=256, local_rank=0, decoder_type=decoder_type, brnn=True, encoder_type=encoder_type, embd_dim=64,
                              padding_idx=V, dropout=0.0, dec_layers=2, enc_layers=2, prune_range=prune_range,
                              max_relative_positions=m_rel)
    return Net(o, 40, V).cuda().eval()


def _batch(V, Tin, Us, D=40, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(len(Tin), max(Tin), D, generator=g)
    y = torch.randint(1, V, (len(Us), max(max(Us), 1)), generator=g)
    for b, U in enumerate(Us):
        y[b, U:] = V                                            # padding id
    return x, y


def _f64_log_probs(m, x, y, x_len, m_rel):
    """log-probs [B, T', U1, V] of the restatement: oracle/model.py, whose attention (the TDNN-Transformer encoder, the transformer
    prediction net; relative positions as in tests/test_oracle_xf_relpos.py) keeps the reference's f32 scores, so those two run on f32
    weights; the LSTM encoder is a float64 nn.LSTM over the packed lengths, the LSTM prediction net, the joint and the log-softmax are
    float64"""
    from oracle import model as om
    sd = {k: v.detach().double().cpu() for k, v in m.state_dict().items()}
    sd32 = {k: v.float() for k, v in sd.items()}
    dt = torch.get_default_dtype()
    try:
        with torch.no_grad():
            if m.pack_seq:
                lstm = copy.deepcopy(m.encoder).double().cpu()
                pk = torch.nn.utils.rnn.pack_padded_sequence(x.double(), torch.as_tensor(x_len).cpu(), batch_first=True, enforce_sorted=False)
                enc = torch.nn.utils.rnn.pad_packed_sequence(lstm(pk)[0], batch_first=True)[0]
            else:
                enc = om.encoder_forward(sd32, x.float(), train=False).double()
            if m.decoder_type == "rnn":
                torch.set_default_dtype(torch.float64)          # the oracle LSTM's zero state
                pred = om.prednet_forward(sd, y)
            elif m_rel:
                from test_oracle_xf_relpos import relpos_prednet_forward
                pred = relpos_prednet_forward(sd32, y, m_rel).double()
            else:
                pred = om.prednet_forward(sd32, y).double()
            return om.joint_forward(sd, enc, pred).numpy()
    finally:
        torch.set_default_dtype(dt)


def _oracle_tables(lp, y, T, U):
    lpb = lp[:T, :U + 1, 0]
    lpl = np.stack([lp[:T, u, int(y[u])] for u in range(U)], 1) if U else np.zeros((T, 1))
    return lpb, lpl


def _two_best(lpb, lpl, T, U):
    """scores of the best and the second-best path (float64 2-best Viterbi)"""
    top = [[None] * (U + 1) for _ in range(T)]
    for t in range(T):
        for u in range(U + 1):
            if t == 0 and u == 0:
                top[t][u] = [0.0, -np.inf]
                continue
            c = []
            if t > 0:
                c += [v + lpb[t - 1, u] for v in top[t - 1][u]]
            if u > 0:
                c += [v + lpl[t, u - 1] for v in top[t][u - 1]]
            top[t][u] = sorted(c, reverse=True)[:2] + [-np.inf] * max(0, 2 - len(c))
    return [v + lpb[T - 1, U] for v in top[T - 1][U]]


def _loglik(lpb, lpl, T, U):
    from oracle import rnnt as orc
    alpha, _ = orc.rnnt_alpha_beta(lpb, lpl, T, U)
    return alpha[T - 1, U] + lpb[T - 1, U]


NETS = [("transformer", "rnn", 0), ("transformer", "transformer", 0), ("rnn", "rnn", 0), ("rnn", "transformer", 4)]


@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("enc_type,dec_type,m_rel", NETS)
def test_engine_align_against_float64_model(prec, enc_type, dec_type, m_rel):
    from pika_b200 import engine
    from oracle.model import frame_lens_after_encoder
    V = 48
    if enc_type == "transformer":                              # the TDNN encoder: 21 + 21 context frames, stride 4
        Tin = (90, 75, 62)
        Ts = frame_lens_after_encoder(torch.tensor(Tin)).tolist()
    else:
        Tin = Ts = (17, 12, 6)
    Us = (7, 4, 0)
    x, y = _batch(V, Tin, Us)
    m = _net(enc_type, dec_type, V, m_rel=m_rel)
    with torch.no_grad():
        m.fc2.weight.mul_(20.0)                                 # a peakier joint: wider margins between the best path and the rest
    fl, ll = _lens(*Ts), _lens(*Us)
    frames, vit, loglik = engine.transducer_align(m, x.cuda(), y.cuda(), fl, ll, x_len=fl, t_out=max(Ts))
    assert frames.shape == (3, y.shape[1]) and frames.dtype == torch.int32
    frames, vit, loglik = frames.cpu().numpy(), vit.cpu().numpy(), loglik.cpu().numpy()
    lp = _f64_log_probs(m, x, y, Ts, m_rel)
    rtol, atol = (3e-2, 0.5) if prec == "bf16" else (1e-4, 2e-3)
    n_cmp = 0
    for b, (T, U) in enumerate(zip(Ts, Us)):
        lpb, lpl = _oracle_tables(lp[b], y[b].numpy(), T, U)
        s, _, want = VO.viterbi(lpb, lpl, T, U)
        best, second = _two_best(lpb, lpl, T, U)
        assert best == s
        np.testing.assert_allclose(vit[b], s, rtol=rtol, atol=atol)
        np.testing.assert_allclose(loglik[b], _loglik(lpb, lpl, T, U), rtol=rtol, atol=atol)
        assert vit[b] <= loglik[b] + 1e-5 * abs(loglik[b])
        assert (frames[b, U:] == -1).all() and (np.diff(frames[b, :U]) >= 0).all() and (frames[b, :U] < T).all()
        # the returned path is (near-)optimal in the float64 model; it is the oracle's wherever that one wins by more than the tolerance
        arcs, t = [], 0
        for f in frames[b, :U]:
            arcs += [0] * (int(f) - t) + [1]
            t = int(f)
        arcs += [0] * (T - 1 - t)
        assert VO.path_score(lpb, lpl, arcs) >= s - 2 * (atol + rtol * abs(s))
        if s - second > atol + rtol * abs(s):
            np.testing.assert_array_equal(frames[b, :U], want)
            n_cmp += 1
    assert n_cmp >= 1                                          # U = 0 always has a single path


# ------------------------------------------------------------------------------------------------ pruned
@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("dec_type", ["rnn", "transformer"])
def test_pruned_align_full_windows_equal_dense(prec, dec_type):
    """R = U_max + 1 keeps every node: the same frames and (to rounding) the same scores as the dense alignment"""
    from pika_b200 import engine
    V, Ts, Us = 60, (17, 12, 9), (6, 3, 0)
    x, y = _batch(V, Ts, Us, seed=2)
    m = _net("rnn", dec_type, V, prune_range=max(Us) + 1)
    fl, ll = _lens(*Ts), _lens(*Us)
    fd, vd, ld = engine.transducer_align(m, x.cuda(), y.cuda(), fl, ll, x_len=fl)
    fp, vp, lpr = engine.transducer_align(m, x.cuda(), y.cuda(), fl, ll, x_len=fl, prune_range=max(Us) + 1)
    rtol = 2e-2 if prec == "bf16" else 1e-4
    torch.testing.assert_close(vp, vd, rtol=rtol, atol=rtol)
    torch.testing.assert_close(lpr, ld, rtol=rtol, atol=rtol)
    for b in range(len(Ts)):
        if float(vp[b]) == float(vd[b]):                        # the same tables (the bf16 row log-sum-exp merge): the same path
            assert torch.equal(fp[b], fd[b])


@pytest.mark.parametrize("prec", PRECS, indirect=True)
@pytest.mark.parametrize("R", [2, 3])
def test_pruned_align_stays_in_windows_and_matches_pruned_loss(prec, R):
    from pika_b200 import engine
    V, Ts, Us = 61, (19, 14, 8), (9, 6, 3)
    x, y = _batch(V, Ts, Us, seed=3)
    m = _net("rnn", "rnn", V, prune_range=R)
    fl, ll = _lens(*Ts), _lens(*Us)
    xc, yc = x.cuda(), y.cuda()
    frames, vit, loglik = engine.transducer_align(m, xc, yc, fl, ll, x_len=fl, prune_range=R)
    again = engine.transducer_align(m, xc, yc, fl, ll, x_len=fl, prune_range=R)
    for a, b in zip((frames, vit, loglik), again):
        assert torch.equal(a, b)
    with torch.no_grad():
        _, pruned = engine.transducer_loss_pruned(m, xc, yc, fl, ll, R, 0.5, 1.0, x_len=fl)
        enc = engine.model_encoder_forward_act(m, xc, fl)
        pred = engine.prednet_forward_act(m, yc)
        _, bounds = engine.SimpleLossFn.apply(enc, pred, m, yc.int(), fl, ll, R, 1.0, False)
    torch.testing.assert_close(loglik, -pruned, rtol=1e-6, atol=1e-5)
    assert bool((vit <= loglik + 1e-5 * loglik.abs()).all()) and bool(torch.isfinite(vit).all())
    s = bounds.cpu().numpy()
    for b, (T, U) in enumerate(zip(Ts, Us)):
        t = u = 0
        nodes = [(0, 0)]
        for f in frames[b, :U].tolist():
            while t < f:
                t += 1
                nodes.append((t, u))
            u += 1
            nodes.append((t, u))
        while t < T - 1:
            t += 1
            nodes.append((t, u))
        assert nodes[-1] == (T - 1, U)
        for (t, u) in nodes:
            assert s[b, t] <= u < s[b, t] + R, (b, t, u, s[b, t])
    with pytest.raises(ValueError, match=r"\[0\]"):
        engine.transducer_align(m, xc, yc, _lens(4, 14, 8), ll, x_len=_lens(4, 14, 8), prune_range=2)   # U = 9 > 4 x 1
    m_dense = _net("rnn", "rnn", V)
    with pytest.raises(ValueError, match="simple joiner"):
        engine.transducer_align(m_dense, xc, yc, fl, ll, x_len=fl, prune_range=R)


# ------------------------------------------------------------------------------------------------ the CLI
def test_align_cli_end_to_end(tmp_path):
    """5 utterances in batches of 2 (a tail of 1): every utterance gets its CTM lines and a score line, times are non-decreasing, and
    under --prune_range 2 the utterance with more labels than frames is reported with -inf, not dropped"""
    from pika_b200 import engine
    from pika_b200.decoder import align_transducer as A
    from pika_b200.loader.kaldi_io import write_float_matrix_ark
    V = 40
    m = _net("rnn", "rnn", V, prune_range=2).cpu()
    torch.save(m, str(tmp_path / "model.pt"))
    rng = np.random.default_rng(11)
    n_frames = [30, 22, 3, 26, 18]
    n_labels = [6, 4, 5, 3, 7]                                  # utterance u2: 5 labels on 3 frames
    feats = [("u%d" % i, rng.standard_normal((n, 40)).astype(np.float32)) for i, n in enumerate(n_frames)]
    write_float_matrix_ark(str(tmp_path / "feats.ark"), feats)
    labels = {k: rng.integers(1, V, n).tolist() for (k, _), n in zip(feats, n_labels)}
    (tmp_path / "labels.ark").write_text("".join("%s %s\n" % (k, " ".join(map(str, labels[k]))) for k, _ in feats))
    (tmp_path / "symbols.txt").write_text("".join("<%d> %d\n" % (i, i) for i in range(V + 1)))
    prec = engine.get_precision()
    try:
        for R, precision in ((0, "fp32"), (2, "bf16")):
            ctm, sc = tmp_path / ("out%d.ctm" % R), tmp_path / ("scores%d.txt" % R)
            A.main([str(tmp_path / "model.pt"), "ark:%s" % (tmp_path / "feats.ark"), "ark,t:%s" % (tmp_path / "labels.ark"), str(ctm),
                    "--loader", "utt", "--cuda", "--batch_first", "--batch_size", "2", "--lctx", "0", "--rctx", "0", "--feats_dim", "40",
                    "--max_len", "100", "--padding_tgt", str(V), "--symbols_map", str(tmp_path / "symbols.txt"), "--precision", precision,
                    "--prune_range", str(R), "--scores", str(sc), "--frame_shift_ms", "10"])
            rows = [l.split() for l in sc.read_text().splitlines()]
            assert [r[0] for r in rows] == [k for k, _ in feats]
            ctm_rows = [l.split() for l in ctm.read_text().splitlines()]
            for (k, _), n, U, r in zip(feats, n_frames, n_labels, rows):
                assert (int(r[1]), int(r[2])) == (n, U)
                mine = [c for c in ctm_rows if c[0] == k]
                if R and U > n * (R - 1):
                    assert r[3:] == ["-inf", "-inf", "-inf"] and not mine
                    continue
                vit, ll, per = float(r[3]), float(r[4]), float(r[5])
                assert math.isfinite(vit) and vit <= ll + 1e-3 and abs(per - vit / n) < 1e-5
                assert [c[4] for c in mine] == ["<%d>" % t for t in labels[k]]
                starts = [float(c[2]) for c in mine]
                assert all(c[1] == "1" and c[3] == "0.010" for c in mine)
                assert starts == sorted(starts) and 0.0 <= starts[0] and starts[-1] <= (n - 1) * 0.01 + 1e-9
            if R == 0:
                assert len(ctm_rows) == sum(n_labels)
    finally:
        engine.set_precision(prec)
