"""Forced alignment on the CPU: the float64 Viterbi oracle (tests/viterbi_oracle.py) against brute force over every monotone path, the
CTM / score line formats of the alignment CLI, its argument checks, and the utt loader's opt-in tail batch."""
import types

import numpy as np
import pytest

import viterbi_oracle as VO


def _tables(rng, T, U, grid, lo=-3.0, p_inf=0.0):
    """dyadic log-probs (multiples of ``grid``): every sum is exact in f64, so ties are exact ties"""
    lpb = np.round(rng.uniform(lo, 0.0, (T, U + 1)) / grid) * grid
    lpl = np.round(rng.uniform(lo, 0.0, (T, max(U, 1))) / grid) * grid
    if p_inf:
        lpb[rng.random(lpb.shape) < p_inf] = -np.inf
        lpl[rng.random(lpl.shape) < p_inf] = -np.inf
    return lpb.astype(np.float32), lpl.astype(np.float32)


@pytest.mark.parametrize("grid,p_inf", [(2.0 ** -20, 0.0), (0.5, 0.0), (1.0, 0.0), (0.25, 0.2), (1.0, 0.35)])
def test_oracle_equals_brute_force(grid, p_inf):
    """same best score and the same path under the tie rule, on every T <= 6, U <= 4 (coarse grids make ties; -inf nodes too)"""
    rng = np.random.default_rng(int(grid * 1000) + int(p_inf * 100))
    n_ties = n_inf = 0
    for T in range(1, 7):
        for U in range(0, 5):
            for _ in range(6):
                lpb, lpl = _tables(rng, T, U, grid, p_inf=p_inf)
                s, dec, frames = VO.viterbi(lpb, lpl, T, U)
                bs, bframes = VO.brute_force(lpb, lpl, T, U)
                assert s == bs, (T, U, s, bs)
                np.testing.assert_array_equal(frames, bframes)
                if s == -np.inf:
                    n_inf += 1
                    assert (frames == -1).all()
                else:
                    assert (np.diff(frames) >= 0).all() and (frames >= 0).all() and (frames < T).all()
                    assert VO.path_score(lpb, lpl, _arcs(frames, T, U)) == s
                n_ties += int(_n_best(lpb, lpl, T, U) > 1)
    if grid >= 0.5:
        assert n_ties > (20 if p_inf == 0 else 5)        # the coarse grids do exercise the tie rule
    if p_inf >= 0.35:
        assert n_inf > 5


def _arcs(frames, T, U):
    """frames of the label arcs -> the arc sequence (0 blank, 1 label) from (0, 0) to (T-1, U)"""
    arcs, t = [], 0
    for f in frames:
        arcs += [0] * (int(f) - t) + [1]
        t = int(f)
    return arcs + [0] * (T - 1 - t)


def _n_best(lpb, lpl, T, U):
    import itertools
    n = T - 1 + U
    scores = []
    for pos in itertools.combinations(range(n), U):
        arcs = [0] * n
        for p in pos:
            arcs[p] = 1
        scores.append(VO.path_score(lpb, lpl, arcs))
    best = max(scores)
    return sum(1 for s in scores if s == best and best > -np.inf)


def test_tie_rule_on_a_built_tie():
    """all-zero tables: every path scores 0; the label arc is taken only when strictly better, so every node past frame 0 comes in by
    blank, the back-trace walks back through the blanks first and every label is emitted on frame 0"""
    T, U = 4, 3
    s, dec, frames = VO.viterbi(np.zeros((T, U + 1), np.float32), np.zeros((T, U), np.float32), T, U)
    assert s == 0.0 and not dec[1:, :].any() and dec[0, 1:].all()
    np.testing.assert_array_equal(frames, [0] * U)


def test_skew_round_trip():
    rng = np.random.default_rng(0)
    nat = rng.standard_normal((2, 5, 4)).astype(np.float32)
    np.testing.assert_array_equal(VO.from_skew(VO.to_skew(nat, 5, 4), 5, 4), nat)


def test_ctm_times_and_format():
    from pika_b200.decoder import align_transducer as A
    lines = A.ctm_lines("utt1", [0, 3, 3, 10], ["a", "b", "c", "d"], model_lctx=21, model_stride=4, stride=1, frame_shift_ms=10.0)
    assert lines == ["utt1 1 0.210 0.040 a", "utt1 1 0.330 0.040 b", "utt1 1 0.330 0.040 c", "utt1 1 0.610 0.040 d"]
    # the loader's stride and the frame shift scale both start and duration: (2 + 5 * 3) * 2 * 0.008 = 0.272, 3 * 2 * 0.008 = 0.048
    assert A.ctm_lines("u", [5], ["x"], model_lctx=2, model_stride=3, stride=2, frame_shift_ms=8.0) == ["u 1 0.272 0.048 x"]
    assert A.ctm_lines("u", [], [], 0, 1, 1, 10.0) == []
    assert A.score_line("u", 50, 3, -12.5, -11.25) == "u 50 3 -12.5000 -11.2500 -0.250000"
    assert A.score_line("u", 50, 3, -np.inf, -np.inf) == "u 50 3 -inf -inf -inf"


@pytest.mark.parametrize("bad", [["--prune_range", "1"], ["--prune_range", "-1"], ["--prune_range", "-4"], ["--model_stride", "0"],
                                 ["--frame_shift_ms", "0"], ["--precision", "fp16"]])
def test_cli_refuses_bad_arguments(bad, tmp_path):
    from pika_b200.decoder import align_transducer as A
    argv = ["m.pt", "ark:f.ark", "ark,t:l.ark", str(tmp_path / "out.ctm")] + bad
    with pytest.raises(SystemExit) as e:
        A.main(argv)
    assert e.value.code == 2                       # argparse's usage error, before any file is read


def test_cli_accepts_dense_and_pruned_ranges():
    from pika_b200.decoder import align_transducer as A
    p = A.build_parser()
    for r in ("0", "2", "5"):
        a = p.parse_args(["m", "f", "l", "o", "--prune_range", r])
        A.check_args(p, a)
    a = p.parse_args(["m", "f", "l", "o"])
    assert (a.prune_range, a.frame_shift_ms, a.precision, a.scores) == (0, 10.0, "bf16", None)


def _write_archive(tmp_path, n_utt, D=8, seed=0):
    from pika_b200.loader.kaldi_io import write_float_matrix_ark
    rng = np.random.default_rng(seed)
    feats = [("utt%02d" % i, rng.standard_normal((int(rng.integers(5, 12)), D)).astype(np.float32)) for i in range(n_utt)]
    labels = [(k, list(rng.integers(1, 9, int(rng.integers(1, 5))))) for k, _ in feats]
    write_float_matrix_ark(str(tmp_path / "feats.ark"), feats)
    (tmp_path / "labels.ark").write_text("".join("%s %s\n" % (k, " ".join(str(v) for v in y)) for k, y in labels))
    return feats, labels


def _loader_args(bs, D=8):
    return types.SimpleNamespace(lctx=0, rctx=0, max_len=100, batch_size=bs, padding_tgt=9, feats_dim=D, batch_first=True, stride=1,
                                 queue_size=4, cuda=False, local_rank=0, ctc_target=False)


@pytest.mark.parametrize("n_utt,bs", [(7, 3), (6, 3), (2, 4)])
def test_utt_loader_keep_tail(tmp_path, n_utt, bs):
    """keep_tail yields every utterance (the last batch holds what is left), with_ids names them; the default still drops the tail"""
    from pika_b200.loader import utt_loader as UL
    feats, labels = _write_archive(tmp_path, n_utt)
    fr, lr = "ark:%s" % (tmp_path / "feats.ark"), "ark,t:%s" % (tmp_path / "labels.ark")
    a = _loader_args(bs)
    full = list(UL.dataloader(lr, fr, False, a))
    assert len(full) == n_utt // bs and all(len(item) == 4 and item[0].shape[0] == bs for item in full)
    kept = list(UL.dataloader(lr, fr, False, a, keep_tail=True, with_ids=True))
    assert len(kept) == -(-n_utt // bs)
    ids = [i for item in kept for i in item[4]]
    assert ids == [k for k, _ in feats]
    feat_of, lab_of = dict(feats), dict(labels)
    for (data, target, lens, ali_lens, names), dense in zip(kept, full + [None]):
        assert data.shape[0] == target.shape[0] == len(lens) == len(ali_lens) == len(names)
        for b, k in enumerate(names):
            n, u = int(lens[b]), int(ali_lens[b])
            np.testing.assert_array_equal(data[b, :n].numpy(), feat_of[k])
            assert target[b, :u].tolist() == list(lab_of[k]) and (target[b, u:] == 9).all()
            assert n == feat_of[k].shape[0] and (data[b, n:] == data[b, n - 1]).all()
        if dense is not None:                      # the full batches are what the default mode yields
            for x, y in zip(dense, (data, target, lens, ali_lens)):
                np.testing.assert_array_equal(np.asarray(x), np.asarray(y))
