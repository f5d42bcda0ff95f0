"""Oracle: batched transducer beam search on the CPU -- a restatement of
decoder/transducer_decoder.py:66-217 (TransducerDecoder.decode_batch / _beam_update / _from_beam) and
decoder/beam_transducer.py:82-243 (BeamMergeTransducer.advance / sort_finished / get_hyp), with the optional on-the-fly FST
scorer of decoder/beam_transducer.py:135-159,167-176 and decoder/sorted_matcher.py:24-111.

TEST INFRASTRUCTURE / REPORTED BASELINE ONLY (see oracle/__init__.py): the checker of the device beam search at shapes the
committed fixtures do not cover, and the ``cpu_baseline`` of ``bench.py --workload decode``.  Pinned (tests/test_oracle_decode.py)
against the reference's own decode_batch outputs in tests/golden/decode_small.npz and decode_big.npz: bit-exact tokens.

All paths relative to /root/reference.  torch-CPU fp32 for the dense layers (prediction net, joint), Python for the
per-utterance beam bookkeeping, exactly as the reference does it.
"""
import math
from collections import defaultdict

import torch
import torch.nn.functional as F

from . import model as om

EOS = -1


class Beam:
    """BeamMergeTransducer (decoder/beam_transducer.py:10-243) for one utterance."""

    def __init__(self, size, blk, n_best, max_len, beam_prune, lm_scorer=None, lm_scorer_scale=1.0, nonblk_reward=0.0):
        self.size, self.blk, self.n_best, self.max_len, self.beam_prune = size, blk, n_best, max_len, beam_prune
        self.scores = torch.zeros(size)
        self.prev_ks, self.next_ys = [], [torch.full((size,), blk, dtype=torch.long)]
        self.eos_top, self.finished = False, []
        self.prev_hyp = [[] for _ in range(size)]
        self.cur_hyp = [[] for _ in range(size)]
        self.lm, self.lm_scale, self.nonblk_reward = lm_scorer, lm_scorer_scale, nonblk_reward
        self.state_sets = [defaultdict(lambda: float("inf")) for _ in range(size)]      # :62-66
        for sm in self.state_sets:
            sm[0] = 0.0
        self.lm_scores = torch.zeros(size)

    def advance(self, word_probs, t_idx, num_frames):
        """:82-187"""
        V = word_probs.size(1)
        if self.prev_ks:
            beam_scores = word_probs + self.scores.unsqueeze(1) + self.lm_scale * self.lm_scores.unsqueeze(1)     # :94-97
            seen = {}
            for i in range(self.size):
                if self.next_ys[-1][i] == EOS:
                    beam_scores[i] = -1e20                                            # :103-104
                elif self.beam_prune:
                    key = str(self.cur_hyp[i])
                    if len(key) > 2:                                                   # non-empty partial hypothesis
                        if key in seen:
                            beam_scores[i] = -1e20                                     # :110-112
                        else:
                            seen[key] = i
            self.prev_hyp = [list(h) for h in self.cur_hyp]                            # :116
        else:
            beam_scores = word_probs[0]                                                # :118
        best, ids = beam_scores.reshape(-1).topk(self.size, 0, True, True)            # :120-121
        prev_k = ids // V                                                              # :125 (floor division, pre-1.5 torch semantics)
        self.prev_ks.append(prev_k)
        self.next_ys.append(ids - prev_k * V)
        self.scores = best - self.lm_scale * self.lm_scores[prev_k]                    # :131-132
        if self.lm is not None:                                                        # :135-159
            nxt = [defaultdict(lambda: float("inf")) for _ in range(self.size)]
            for i in range(self.size):
                y = int(self.next_ys[-1][i])
                src = self.state_sets[int(prev_k[i])]
                if y != self.blk:
                    for state in list(src.keys()):
                        sc, st = self.lm.get_scores(state, y + 1)
                        for ns, cost in zip(st, sc):
                            c = src[state] + cost
                            if c < nxt[i][ns]:
                                nxt[i][ns] = c - self.nonblk_reward
                else:
                    for k, v in src.items():
                        nxt[i][k] = v
                self.lm_scores[i] = -min(nxt[i].values()) if nxt[i] else -1e20
            self.state_sets = nxt
        for i in range(self.size):                                                     # :161-183
            y = int(self.next_ys[-1][i])
            if (y == self.blk and int(t_idx[int(prev_k[i])]) == num_frames - 1) or len(self.next_ys) > self.max_len:
                s = self.scores[i]                                                     # a view: the final LM term lands in self.scores
                self.next_ys[-1][i] = EOS
                if self.lm is not None:                                                # :167-176
                    fin = defaultdict(lambda: float("inf"))
                    for state in list(self.state_sets[i].keys()):
                        fs, fst = self.lm.final_score(state)
                        for f_s, cost in zip(fst, fs):
                            c = self.state_sets[i][state] + cost
                            if c < fin[f_s]:
                                fin[f_s] = c
                    s += self.lm_scale * (-min(fin.values()))
                self.finished.append((float(s), len(self.next_ys) - 1, i))             # GlobalScorer.score is the identity (:246-258)
            else:                                                                      # update_partial_hyp :224-232
                k0 = int(self.prev_ks[-1][i])
                if i != k0:
                    self.cur_hyp[i] = list(self.prev_hyp[k0])
                if y != self.blk:
                    self.cur_hyp[i].append(y)
        if self.next_ys[-1][0] == EOS:
            self.eos_top = True                                                        # :185-187

    def done(self):
        return self.eos_top and len(self.finished) >= self.n_best                     # :190-194

    def sort_finished(self, minimum):
        """:196-217"""
        i = 0
        while len(self.finished) < minimum:
            self.finished.append((float(self.scores[i]), len(self.next_ys) - 1, i))
        self.finished.sort(key=lambda a: -a[0])
        return [s for s, _, _ in self.finished], [(t, k) for _, t, k in self.finished]

    def get_hyp(self, timestep, k):
        """:236-243"""
        hyp = []
        for j in range(len(self.prev_ks[:timestep]) - 1, -1, -1):
            hyp.append(int(self.next_ys[j + 1][k]))
            k = int(self.prev_ks[j][k])
        return hyp[::-1]


class SortedMatcher:
    """decoder/sorted_matcher.py:3-111 over a plain arc table instead of a PyKaldi VectorFst:
    ``arcs[state]`` = list of (ilabel, weight, nextstate) sorted by ilabel, ``finals[state]`` = final cost (inf = none)."""

    def __init__(self, arcs, finals, backoff_id, disambig_ids=()):
        self.arcs, self.finals, self.backoff_id, self.disambig_ids = arcs, finals, backoff_id, list(disambig_ids)

    def search(self, state, ilabel):
        """:24-50 (binary search for the FIRST arc with this ilabel)"""
        a = self.arcs[state]
        lo, hi = 0, len(a)
        while lo < hi:
            mid = (lo + hi) // 2
            if a[mid][0] >= ilabel:
                hi = mid
            else:
                lo = mid + 1
        if lo < len(a) and a[lo][0] == ilabel:
            return a[lo]
        return None

    def _wo_disambig(self, state, ilabel, init):
        """:52-68"""
        scores, states, bf, cur = [], [], init, state
        while True:
            arc = self.search(cur, ilabel)
            if arc is not None:
                scores.append(bf + arc[1]); states.append(arc[2])
            b = self.search(cur, self.backoff_id)
            if b is None:
                return scores, states
            bf += b[1]; cur = b[2]

    def get_scores(self, state, ilabel):
        """:70-85"""
        init_s, init_st = [0.0], [state]
        for lab in self.disambig_ids:
            arc = self.search(state, lab)
            if arc is not None:
                init_s.append(arc[1]); init_st.append(arc[2])
        scores, states = [], []
        for s0, st0 in zip(init_s, init_st):
            sc, st = self._wo_disambig(st0, ilabel, s0)
            scores.extend(sc); states.extend(st)
        return scores, states

    def final_score(self, state):
        """:87-111"""
        fs, fst = [0.0], [state]
        for lab in self.disambig_ids:
            arc = self.search(state, lab)
            if arc is not None:
                fs.append(arc[1]); fst.append(arc[2])
        for i in range(len(fs)):
            score, cur = fs[i], fst[i]
            while True:
                f = self.finals[cur]
                if math.isinf(f):
                    b = self.search(cur, self.backoff_id)
                    if b is None:
                        score, cur = float("inf"), None
                        break
                    score += b[1]; cur = b[2]
                else:
                    score += f
                    break
            fs[i], fst[i] = score, cur
        return fs, fst


@torch.no_grad()
def decode_batch(sd, enc_out, x_len, beam_size, n_best=1, blk=0, max_len=None, sm_scale=1.0, beam_prune=True,
                 lm_scorer=None, lm_scorer_scale=1.0, nonblk_reward=0.0):
    """decoder/transducer_decoder.py:66-217 from the encoder outputs on (``enc_out`` [B,T',H] fp32 = ``self.model.encoder(x)``,
    :102).  ``sd``: state_dict with the reference's key names.  Returns {"predictions": B x n_best token lists (EOS stripped),
    "scores": B x n_best floats}."""
    B, Tenc, H = enc_out.shape
    K = beam_size
    beams = [Beam(K, blk, n_best, max_len[i] if max_len and max_len[i] else 10000, beam_prune, lm_scorer, lm_scorer_scale, nonblk_reward)
             for i in range(B)]
    x = enc_out.repeat(K, 1, 1)                                                        # :106 rows = k * B + b
    t_idx = torch.zeros(K, B, dtype=torch.long) - 1                                    # :109
    emb_w = sd["embed.weight"]
    blk_sos = torch.full((B * K, 1), blk, dtype=torch.long)
    xf = "decoder.conv.0.weight" in sd                 # transformer prediction net: the state is its last output row (:117-120)
    if xf:
        pad = emb_w.shape[0] - 1                       # embed.padding_idx (-1 -> last row)
        dec = om.conv_transformer_lm_forward(sd, blk_sos)[:, -1, :].clone()
    else:
        _, (h, c) = om.lstm_forward(sd, F.embedding(blk_sos, emb_w))                   # :116
        h, c = h.clone(), c.clone()
    rows = torch.arange(B * K)
    while not all(b.done() for b in beams):                                            # :123
        inp = torch.stack([b.next_ys[-1] for b in beams]).t()                          # [K, B]
        t_idx = t_idx + inp.eq(blk).long()                                             # :129
        flat = inp.contiguous().view(-1)
        enc_hid = x[rows, t_idx.contiguous().view(-1).clamp(max=Tenc - 1), :]          # :133-134
        nonblk = flat.gt(blk)                                                          # :139
        if int(nonblk.sum()) > 0 and xf:                                               # :151-171: the whole partial hypothesis again
            idx = rows[nonblk].tolist()
            hyps = [[blk] + beams[k % B].cur_hyp[k // B] for k in idx]
            lens = [len(hp) for hp in hyps]
            src = torch.tensor([hp + [pad] * (max(lens) - len(hp)) for hp in hyps], dtype=torch.long)
            dec[nonblk] = om.conv_transformer_lm_forward(sd, src)[torch.arange(len(idx)), torch.tensor(lens) - 1, :]
        elif int(nonblk.sum()) > 0:                                                    # :140-150
            _, (hn, cn) = om.lstm_forward(sd, F.embedding(flat[nonblk].view(-1, 1), emb_w), state=(h[:, nonblk], c[:, nonblk]))
            h[:, nonblk], c[:, nonblk] = hn, cn
        z = torch.cat((enc_hid, dec if xf else h[-1]), -1)                             # :173
        out = om.linear(torch.tanh(om.linear(z, sd, "fc1")) * torch.sigmoid(om.linear(z, sd, "fc_gate")), sd, "fc2")
        out = F.log_softmax(sm_scale * out, -1).view(K, B, -1)                         # :177-178
        for j, b in enumerate(beams):                                                  # :181-183
            b.advance(out[:, j], t_idx[:, j], int(x_len[j]))
            pos = b.prev_ks[-1]
            if xf:                                                                     # _beam_update :195-200
                v = dec.view(K, B, -1)[:, j]
                v.copy_(v.index_select(0, pos))
            for e in (() if xf else (h, c)):                                           # _beam_update :188-194
                v = e.view(e.shape[0], K, B, -1)[:, :, j]
                v.copy_(v.index_select(1, pos))
            t_idx[:, j] = t_idx[:, j].index_select(0, pos)
    ret = {"predictions": [], "scores": []}
    for b in beams:                                                                    # _from_beam :204-217
        scores, ks = b.sort_finished(n_best)
        ret["predictions"].append([b.get_hyp(t, k)[:-1] for t, k in ks[:n_best]])
        ret["scores"].append(scores[:n_best])
    return ret
