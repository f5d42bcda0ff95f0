"""LM FST scorer for on-the-fly shallow fusion -- drop-in for decoder/sorted_matcher.py (reference).

Same constructor (``SortedMatcher(vector_fst, max_num_arcs, max_id, backoff_id, disambig_ids)``) and the same ``get_scores`` /
``final_score`` results.  The reference walks a PyKaldi ``VectorFst`` arc iterator from Python once per (beam, active state,
back-off level) and step; here the FST is flattened ONCE into a CSR arc table (arcs of a state sorted by input label) that
lives in HBM, and the whole per-beam search (binary search for the label, back-off chain, disambiguation arcs, state-set
update, final costs) runs inside ``pk_beam_advance_lm`` (pika_b200/csrc/beam.cu) for all utterances of the batch.

``vector_fst`` may be anything exposing the slice of the OpenFst interface the reference uses -- ``num_states()``,
``arcs(state)`` (iterable of arcs with ``ilabel``, ``weight.value``, ``nextstate``) and ``final(state).value`` -- or a ready
``(arcs, finals)`` pair: ``arcs[state]`` = list of ``(ilabel, weight, nextstate)``, ``finals[state]`` = cost (inf = not final).
"""
import math

import numpy as np
import torch

from .._lib import LmFst


class SortedMatcher(object):
    def __init__(self, vector_fst, max_num_arcs=None, max_id=None, backoff_id=0, disambig_ids=()):
        self.fst, self.max_num_arcs, self.max_id = vector_fst, max_num_arcs, max_id
        self.backoff_id, self.disambig_ids = int(backoff_id), [int(d) for d in disambig_ids]
        if len(self.disambig_ids) > 4:
            raise ValueError("pika_b200 SortedMatcher: at most 4 disambiguation labels")
        if isinstance(vector_fst, (tuple, list)) and len(vector_fst) == 2:
            arcs, finals = vector_fst
        else:
            n = vector_fst.num_states()
            arcs = [[(a.ilabel, a.weight.value, a.nextstate) for a in vector_fst.arcs(s)] for s in range(n)]
            finals = [vector_fst.final(s).value for s in range(n)]
        off = np.zeros(len(arcs) + 1, np.int32)
        for s, a in enumerate(arcs):
            if any(a[i][0] > a[i + 1][0] for i in range(len(a) - 1)):
                raise ValueError("pika_b200 SortedMatcher: the arcs of state %d are not sorted by input label" % s)
            off[s + 1] = off[s] + len(a)
        flat = [t for a in arcs for t in a]
        self._off = off
        self._il = np.array([t[0] for t in flat], np.int32)
        self._w = np.array([float(t[1]) for t in flat], np.float64)
        self._ns = np.array([t[2] for t in flat], np.int32)
        self._fin = np.array([float(f) for f in finals], np.float64)
        self._dev = {}

    # ------------------------------------------------------------------ device tables
    def device_tables(self, device):
        """-> (LmFst struct for the C ABI, tensors that keep the arrays alive)"""
        key = str(device)
        if key not in self._dev:
            t = [torch.from_numpy(a).to(device) for a in (self._off, self._il, self._w, self._ns, self._fin)]
            st = LmFst()
            st.arc_off, st.arc_ilabel, st.arc_weight, st.arc_next, st.finals = (x.data_ptr() for x in t)
            st.backoff_id, st.n_disambig = self.backoff_id, len(self.disambig_ids)
            for i, d in enumerate(self.disambig_ids):
                st.disambig_ids[i] = d
            self._dev[key] = (st, t)
        return self._dev[key]

    # ------------------------------------------------------------------ host-side API of the reference class (small tables only)
    def search(self, state_id, ilabel):
        lo, hi = int(self._off[state_id]), int(self._off[state_id + 1])
        end = hi
        while lo < hi:
            mid = (lo + hi) // 2
            if self._il[mid] >= ilabel:
                hi = mid
            else:
                lo = mid + 1
        return lo if (lo < end and self._il[lo] == ilabel) else None

    def get_scores_wodisambig(self, state_id, ilabel, init_score=0.0):
        scores, states, bf, cur = [], [], init_score, state_id
        while True:
            a = self.search(cur, ilabel)
            if a is not None:
                scores.append(bf + float(self._w[a])); states.append(int(self._ns[a]))
            b = self.search(cur, self.backoff_id)
            if b is None:
                return scores, states
            bf += float(self._w[b]); cur = int(self._ns[b])

    def get_scores(self, state_id, ilabel):
        init = [(0.0, state_id)]
        for lab in self.disambig_ids:
            a = self.search(state_id, lab)
            if a is not None:
                init.append((float(self._w[a]), int(self._ns[a])))
        scores, states = [], []
        for s0, st0 in init:
            sc, st = self.get_scores_wodisambig(st0, ilabel, s0)
            scores.extend(sc); states.extend(st)
        return scores, states

    def final_score(self, state_id):
        init = [(0.0, state_id)]
        for lab in self.disambig_ids:
            a = self.search(state_id, lab)
            if a is not None:
                init.append((float(self._w[a]), int(self._ns[a])))
        fs, fst = [], []
        for score, cur in init:
            while True:
                f = float(self._fin[cur])
                if math.isinf(f):
                    b = self.search(cur, self.backoff_id)
                    if b is None:
                        score, cur = float("inf"), None
                        break
                    score += float(self._w[b]); cur = int(self._ns[b])
                else:
                    score += f
                    break
            fs.append(score); fst.append(cur)
        return fs, fst


def read_fst_text(path):
    """An acceptor / transducer in OpenFst TEXT form (``fstprint`` output: ``src dst ilabel [olabel] [weight]`` arc lines, ``state
    [weight]`` final lines) -> the ``(arcs, finals)`` pair ``SortedMatcher`` takes, arcs of a state sorted by input label (``fstarcsort``
    order).  Stands in for ``kaldi.fstext.StdVectorFst.read`` (decoder/decode_transducer.py:85), which needs PyKaldi: print the binary
    LM once with ``fstprint`` and point ``--fst_lm`` at the text file."""
    arcs, finals = {}, {}
    n_states = 0
    for line in open(path):
        f = line.split()
        if not f:
            continue
        if len(f) >= 3:
            src, dst, il = int(f[0]), int(f[1]), int(f[2])
            w = float(f[4]) if len(f) >= 5 else (float(f[3]) if len(f) == 4 and not f[3].lstrip("-").isdigit() else 0.0)
            arcs.setdefault(src, []).append((il, w, dst))
            n_states = max(n_states, src + 1, dst + 1)
        else:
            st = int(f[0])
            finals[st] = float(f[1]) if len(f) == 2 else 0.0
            n_states = max(n_states, st + 1)
    return ([sorted(arcs.get(s, []), key=lambda a: a[0]) for s in range(n_states)], [finals.get(s, math.inf) for s in range(n_states)])
