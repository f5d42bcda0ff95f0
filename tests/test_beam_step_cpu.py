"""Pins tests/beam_step_oracle.py, the one-step restatement of pk_beam_advance[_lm] in the kernel's data layout, to
oracle.decode.Beam.advance (itself pinned to the reference by test_oracle_decode.py): multi-step runs at every beam width the
kernel has, with and without duplicate pruning and with and without an FST that has disambiguation arcs, a depth-3 back-off chain,
repeated input labels, a label with no arc and a state with no reachable final state.  The tie rule and the device-only limits
(cap, L, max_states) are checked against hand-built values."""
import math

import numpy as np
import pytest
import torch

import beam_step_oracle as bso
from oracle.decode import Beam, SortedMatcher

BLK = 0


def _log_softmax(x):
    x = x.astype(np.float64)
    return (x - x.max(1, keepdims=True) - np.log(np.exp(x - x.max(1, keepdims=True)).sum(1, keepdims=True))).astype(np.float32)


def _matcher(V):
    arcs, finals, bo, dis = bso.fusion_lm(V)
    return SortedMatcher(arcs, finals, bo, dis)


def _compare(beam, st, b, step, lm):
    K = beam.size
    pn = (step & 1) ^ 1
    assert st["next_ys"][step + 1, b].tolist() == beam.next_ys[-1].tolist()
    assert st["prev_ks"][step, b].tolist() == beam.prev_ks[-1].tolist()
    assert st["scores"][b].tobytes() == beam.scores.numpy().astype(np.float32).tobytes(), (st["scores"][b], beam.scores)
    for i in range(K):
        n = int(st["hyp_len"][pn, b, i])
        assert st["hyp_tok"][pn, b, i, :n].tolist() == beam.cur_hyp[i], (i, n)
    n = int(st["fin_count"][b])
    got = [(float(st["fin_score"][b, j]), int(st["fin_step"][b, j]), int(st["fin_k"][b, j])) for j in range(n)]
    assert got == beam.finished
    assert bool(st["eos_top"][b]) == beam.eos_top and bool(st["done"][b]) == beam.done()
    if lm:
        assert st["lm_scores"][b].tobytes() == beam.lm_scores.numpy().tobytes()
        for i in range(K):
            n = int(st["set_n"][pn, b, i])
            got = list(zip(st["set_state"][pn, b, i, :n].tolist(), st["set_cost"][pn, b, i, :n].tolist()))
            assert got == list(beam.state_sets[i].items()), (i, got, list(beam.state_sets[i].items()))


def _run(K, prune, use_lm, seed, steps=36, V=20, n_best=2):
    rng = np.random.default_rng(seed)
    nf, ml = [5, 12, 24], [10000, 22, 10000]
    B = len(nf)
    L, cap, MS = steps + 1, steps * K, 8
    m = _matcher(V) if use_lm else None
    lm = bso.Lm(m, 0.6, 0.25) if use_lm else None
    st = bso.init_state(B, K, steps, L, cap, BLK, MS if use_lm else None)
    beams = [Beam(K, BLK, n_best, ml[b], prune, m, 0.6 if use_lm else 1.0, 0.25 if use_lm else 0.0) for b in range(B)]
    t_idx = np.full(B * K, -1, np.int64)
    live, compared = set(range(B)), np.zeros(B, int)
    for step in range(steps):
        t_idx = t_idx + (st["next_ys"][step].reshape(-1) == BLK)
        logits = 2.0 * rng.standard_normal((B * K, V))
        logits[:, 0] += 1.0
        wp = _log_softmax(logits)
        new, ties = bso.advance(st, wp, t_idx, nf, ml, step, BLK, n_best, prune, lm)
        for b in sorted(live):
            if ties[b]:                           # torch.topk leaves the order of ties unspecified
                live.discard(b)
                continue
            try:
                beams[b].advance(torch.from_numpy(wp[b * K:(b + 1) * K]), torch.from_numpy(t_idx[b * K:(b + 1) * K]), nf[b])
            except ValueError:                    # min() over the final costs of an empty state set (see beam_step_oracle)
                live.discard(b)
                continue
            _compare(beams[b], new, b, step, use_lm)
            compared[b] += 1
            if (new["next_ys"][step + 1, b] == bso.EOS).all():
                live.discard(b)
        t_idx = t_idx.reshape(B, K)[np.arange(B)[:, None], new["prev_ks"][step]].reshape(-1)
        st = new
    assert st["not_done_total"][0] == B - int(st["done"].sum())
    return compared, st


@pytest.mark.parametrize("use_lm", [False, True], ids=["nolm", "lm"])
@pytest.mark.parametrize("prune", [1, 0])
@pytest.mark.parametrize("K", [1, 2, 4, 8, 16])
def test_layout_oracle_equals_beam_advance(K, prune, use_lm):
    compared, st = _run(K, prune, use_lm, seed=100 * K + 10 * prune + use_lm)
    assert compared.max() >= 30, compared                 # one utterance runs the whole way
    assert st["fin_count"].sum() > 0                      # and some finish (on the last frame or on max_len)


def test_fusion_lm_reaches_every_branch():
    """the FST of the fusion tests has what the kernel's search must handle"""
    V = 20
    m = _matcher(V)
    arcs, finals, bo, dis = bso.fusion_lm(V)
    assert len(dis) == 2
    assert any(a[i][0] == a[i + 1][0] for a in arcs for i in range(len(a) - 1))                  # repeated input label
    depth, s = 0, 3
    while m.search(s, bo) is not None:
        s, depth = m.search(s, bo)[2], depth + 1
    assert depth == 3
    assert m.get_scores(0, V) == ([], [])                                                        # token V-1 has no arc
    assert math.isinf(m.final_score(5)[0][0])                                                    # no final state reachable
    no_dis = SortedMatcher(arcs, finals, bo, [])
    assert len(m.get_scores(4, 3)[1]) > len(no_dis.get_scores(4, 3)[1])                         # the disambig arcs add paths


def test_tie_rule_is_value_desc_index_asc():
    v = np.array([1, 3, 3, -1e20, 3, 2, -1e20], np.float32)
    vals, ids = bso.stable_topk(v, np.arange(7), 7)
    assert ids.tolist() == [1, 2, 4, 5, 0, 3, 6]
    # every row of the utterance finished: K*V candidates at -1e20, the first K flat indices win (row 0, tokens 0..K-1)
    K, V = 4, 5
    st = bso.init_state(1, K, 4, 6, 8, BLK)
    st["next_ys"][2, 0] = bso.EOS
    st["scores"][0] = [-3, -4, -5, -6]
    new, ties = bso.advance(st, np.zeros((K, V), np.float32), np.zeros(K, np.int64), [50], [100], 2, BLK, 1, 1)
    assert ties[0]
    assert new["prev_ks"][2, 0].tolist() == [0, 0, 0, 0]
    assert new["next_ys"][3, 0].tolist() == [0, 1, 2, 3]
    assert new["scores"][0].tolist() == [np.float32(-1e20)] * K


def test_saturation_of_cap_L_and_max_states():
    K, V, L, cap = 4, 6, 2, 2
    st = bso.init_state(1, K, 4, L, cap, BLK, max_states=1)
    st["next_ys"][1, 0] = [3, 4, 5, 2]
    st["hyp_len"][1, 0] = [2, 2, 1, 0]
    st["hyp_tok"][1, 0] = [[3, 3], [4, 4], [5, 0], [0, 0]]
    st["set_n"][1, 0] = 1
    st["scores"][0] = [-1, -2, -3, -4]
    wp = np.full((K, V), -30, np.float32)
    wp[0, 0], wp[1, 0], wp[2, 0], wp[0, 2] = -0.5, -0.25, -0.125, -1.0          # three blanks on the last frame, one label
    m = _matcher(V)
    new, _ = bso.advance(st, wp, np.array([9, 9, 9, 0]), [10], [100], 1, BLK, 1, 1, bso.Lm(m, 1.0, 0.0))
    assert new["prev_ks"][1, 0].tolist() == [0, 0, 1, 2]
    assert new["next_ys"][2, 0].tolist() == [-1, 2, -1, -1]
    assert new["fin_count"][0] == cap and new["fin_k"][0].tolist() == [0, 2] and new["fin_step"][0].tolist() == [2, 2]
    assert new["eos_top"][0] == 1 and new["done"][0] == 1 and new["not_done_total"][0] == 0
    assert new["hyp_len"][0, 0].tolist() == [2, 2, 1, 0]          # row 1 = row 0 (already L tokens) + label 2: stays at L
    assert new["hyp_tok"][0, 0, 1].tolist() == [3, 3]
    # label 2 from state 0 (set of row 0: {0}) reaches one state; max_states 1 holds it, the blank rows copy theirs
    assert new["set_n"][0, 0].tolist() == [1, 1, 1, 1] and new["err"][0] == 0
    # two states reached from one: the second overflows max_states = 1
    st2 = bso.init_state(1, K, 4, L, cap, BLK, max_states=1)
    st2["next_ys"][1, 0] = [3, 3, 3, 3]
    st2["set_n"][1, 0] = 1
    st2["set_state"][1, 0, :, 0] = 4
    wp2 = np.full((K, V), -30, np.float32)
    wp2[0, 2] = -0.1
    new2, _ = bso.advance(st2, wp2, np.zeros(K, np.int64), [10], [100], 1, BLK, 1, 0, bso.Lm(m, 1.0, 0.0))
    assert len(m.get_scores(4, 3)[1]) > 1
    assert new2["set_n"][0, 0, 0] == 1 and new2["err"][0] == 1
