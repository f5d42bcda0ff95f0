"""Oracle: one step of the device beam search (``pk_beam_advance`` / ``pk_beam_advance_lm``, pika_b200/csrc/beam.cu) in the
kernel's own data layout.

``advance(state at step s, word_probs [B*K, V]) -> state at step s + 1`` for every utterance of the batch, over exactly the device
buffers: scores, next_ys, prev_ks, hyp_tok / hyp_len (both parities), fin_*, fin_count, eos_top, done, not_done_total and, with an
FST, set_state / set_cost / set_n / lm_scores / err.  It is the per-utterance rule of ``oracle.decode.Beam.advance`` (pinned to the
reference by tests/test_oracle_decode.py, and to this module by tests/test_beam_step_cpu.py) plus the limits only the device has:
the finished lists hold ``cap`` entries, a partial hypothesis ``L`` tokens and a state set ``max_states`` states; all three saturate,
nothing is written past them, and a set that would overflow raises ``err``.

Float behaviour follows the kernel: the candidate score is float32 ``(word_probs + score) + lm_scale * lm_score`` (each operation
rounded), the new score ``best - lm_scale * lm_score[prev_k]``, FST costs are float64 and cast to float32 where the kernel casts.
The top-k order is value descending, then flat index (k * V + v) ascending.  ``word_probs`` is taken as given: the GPU tests feed it
``pk_log_softmax``'s output for the logits the kernel reads, so that the kernel's on-the-fly log-prob is checked bit for bit.
"""
import math

import numpy as np

EOS = -1
KILL = np.float32(-1e20)


def init_state(B, K, S, L, cap, blk, max_states=None):
    """the buffers as TransducerDecoder's workspace reset leaves them (step 0): next_ys[0] = blk, everything else zero,
    not_done_total = B.  ``max_states``: also the FST buffers."""
    i32 = lambda *s: np.zeros(s, np.int32)      # noqa: E731
    st = dict(scores=np.zeros((B, K), np.float32), next_ys=i32(S + 1, B, K), prev_ks=i32(S, B, K),
              hyp_tok=i32(2, B, K, L), hyp_len=i32(2, B, K), fin_score=np.zeros((B, cap), np.float32),
              fin_step=i32(B, cap), fin_k=i32(B, cap), fin_count=i32(B), eos_top=i32(B), done=i32(B),
              not_done_total=np.full(1, B, np.int32))
    st["next_ys"][0] = blk
    if max_states is not None:
        st.update(set_state=i32(2, B, K, max_states), set_cost=np.zeros((2, B, K, max_states), np.float64), set_n=i32(2, B, K),
                  lm_scores=np.zeros((B, K), np.float32), err=i32(1))
    return st


class Lm:
    """FST shallow fusion as pk_beam_advance_lm takes it: ``matcher`` = oracle.decode.SortedMatcher (its ``get_scores`` /
    ``final_score`` are the arc search), lm_scorer_scale, nonblk_reward."""

    def __init__(self, matcher, scale=1.0, reward=0.0):
        self.matcher, self.scale, self.reward = matcher, float(scale), float(reward)


def fusion_lm(V, seed=5):
    """A small back-off LM that reaches every branch of the FST search, as (arcs, finals, backoff_id, disambig_ids) with
    ilabel = token + 1 (token 0 = blank, so ilabel 1 is free for the back-off arcs).
      state 0: unigram, final; an arc for every token but the last (token V - 1 has no arc anywhere: its sets are empty)
      states 1-3: a back-off chain 3 -> 2 -> 1 -> 0 (depth 3), none of them final; state 2 has two arcs with the same input label
      state 4: two disambiguation arcs (to 3 and to 1), a few arcs of its own and a back-off to 0
      state 5: not final and no back-off (no final state is reachable), entered by one arc of state 4
    """
    rng = np.random.default_rng(seed)
    bo, dis = 1, [V + 1, V + 2]
    w = lambda: float(np.round(rng.uniform(0.05, 1.5), 3))                  # noqa: E731
    toks = np.arange(1, V - 1)
    some = lambda n: sorted(rng.choice(toks, size=min(n, len(toks)), replace=False).tolist())   # noqa: E731
    arcs = [[(int(t) + 1, w(), int(rng.integers(0, 5))) for t in toks]]
    finals = [0.7]
    arcs.append([(bo, w(), 0)] + [(t + 1, w(), int(rng.integers(0, 5))) for t in some(V // 3)])
    rep = int(toks[len(toks) // 2]) + 1
    arcs.append([(bo, w(), 1)] + [(t + 1, w(), int(rng.integers(0, 5))) for t in some(V // 3) if t + 1 != rep]
                + [(rep, w(), 3), (rep, w(), 4)])
    arcs.append([(bo, w(), 2)] + [(t + 1, w(), int(rng.integers(0, 5))) for t in some(V // 4)])
    arcs.append([(bo, w(), 0), (int(toks[0]) + 1, w(), 5)] + [(t + 1, w(), int(rng.integers(0, 5))) for t in some(V // 4) if t != toks[0]]
                + [(dis[0], w(), 3), (dis[1], w(), 1)])
    arcs.append([(int(t) + 1, w(), 5) for t in toks[:3]])
    finals += [math.inf, math.inf, math.inf, 1.3, math.inf]
    arcs = [sorted(a, key=lambda x: x[0]) for a in arcs]                        # stable: equal labels keep their order
    return arcs, finals, bo, dis


def stable_topk(vals, ids, k):
    """the kernel's order: value descending, then index ascending -> (values, ids) of the first k"""
    order = np.lexsort((ids, -vals.astype(np.float64)))[:k]
    return vals[order], ids[order]


def _final_min(lm, state, base):
    """min over final_score(state) of base + cost, inf when no final state is reachable (the kernel's fst_final_min)"""
    best = math.inf
    for sc in lm.matcher.final_score(state)[0]:
        best = min(best, base + sc)
    return best


def advance(st, word_probs, t_idx, num_frames, max_len, step, blk, n_best, beam_prune, lm=None):
    """-> (new state, ties [B] bool: True where the k-th and (k+1)-th candidates of an utterance are equal, i.e. where the result
    depends on the tie rule).  ``st`` is not modified.  ``word_probs`` [B*K, V] float32, ``t_idx`` [B*K], ``num_frames`` /
    ``max_len`` [B]."""
    st = {k: v.copy() for k, v in st.items()}
    B, K = st["scores"].shape
    L = st["hyp_tok"].shape[3]
    cap = st["fin_score"].shape[1]
    V = word_probs.shape[1]
    wp = np.asarray(word_probs, np.float32).reshape(B, K, V)
    po, pn = step & 1, (step & 1) ^ 1
    ties = np.zeros(B, bool)
    MS = st["set_state"].shape[3] if lm is not None else 0
    for b in range(B):
        cur_tok = st["next_ys"][step, b]
        old_hyp, old_len = st["hyp_tok"][po, b].copy(), st["hyp_len"][po, b].copy()
        # 1. which rows have children: 0 = yes, 1 = finished or a duplicate of an earlier row (V candidates at -1e20),
        #    2 = step 0 and k > 0 (no candidates)
        kill = np.zeros(K, np.int32)
        for k in range(K):
            if step > 0:
                if cur_tok[k] == EOS:
                    kill[k] = 1
                elif beam_prune and old_len[k] > 0:
                    n = old_len[k]
                    for j in range(k):
                        if cur_tok[j] != EOS and old_len[j] == n and np.array_equal(old_hyp[j, :n], old_hyp[k, :n]):
                            kill[k] = 1
                            break
            elif k > 0:
                kill[k] = 2
        lmterm = (np.float32(lm.scale) * st["lm_scores"][b]) if lm is not None else np.zeros(K, np.float32)
        # 2. candidates and top-k
        vals, ids = [], []
        for k in range(K):
            if kill[k] == 0:
                x = wp[b, k].copy()
                if step > 0:
                    x = x + st["scores"][b, k]
                    if lm is not None:
                        x = x + lmterm[k]
                vals.append(x)
            elif kill[k] == 1:
                vals.append(np.full(V, KILL, np.float32))
            else:
                continue
            ids.append(k * V + np.arange(V, dtype=np.int64))
        vals, ids = np.concatenate(vals).astype(np.float32), np.concatenate(ids)
        best, bid = stable_topk(vals, ids, K + 1)
        ties[b] = len(best) > K and best[K - 1] == best[K] or len(np.unique(best[:K])) < K
        best, bid = best[:K], bid[:K]
        # 3. new beam
        nf, len_after = int(num_frames[b]), step + 2
        fin = np.zeros(K, bool)
        for i in range(K):
            pk, y = int(bid[i] // V), int(bid[i] % V)
            sc = np.float32(best[i])
            if lm is not None:
                sc = np.float32(sc - lmterm[pk])
            st["prev_ks"][step, b, i] = pk
            fin[i] = (y == blk and int(t_idx[b * K + pk]) == nf - 1) or len_after > int(max_len[b])
            if lm is not None:
                if step > 0:
                    n_old = int(st["set_n"][po, b, pk])
                    old = list(zip(st["set_state"][po, b, pk, :n_old].tolist(), st["set_cost"][po, b, pk, :n_old].tolist()))
                else:
                    old = [(0, 0.0)]                                        # initial set {0: 0.0}
                new_s, new_c = [], []                                       # insertion-ordered set
                for state, c0 in old:
                    if y == blk:
                        if len(new_s) < MS:
                            new_s.append(state); new_c.append(c0)
                        else:
                            st["err"][0] = 1
                        continue
                    costs, nexts = lm.matcher.get_scores(state, y + 1)
                    for cost, nxt in zip(costs, nexts):
                        nc = c0 + cost
                        if nxt not in new_s:
                            if len(new_s) >= MS:
                                st["err"][0] = 1
                                continue
                            new_s.append(nxt); new_c.append(nc - lm.reward)   # first visit: nc < inf
                        else:
                            q = new_s.index(nxt)
                            if nc < new_c[q]:                               # strict <, reward off the stored value only
                                new_c[q] = nc - lm.reward
                n_new = len(new_s)
                st["set_n"][pn, b, i] = n_new
                st["set_state"][pn, b, i, :n_new] = new_s
                st["set_cost"][pn, b, i, :n_new] = new_c
                st["lm_scores"][b, i] = np.float32(-min(new_c)) if n_new else KILL
                if fin[i]:
                    # The reference takes min() over the final costs of the set, which raises when the set is empty (a label with no
                    # arc); the kernel's result there is defined: no reachable final state, score + lm_scale * (-inf).
                    fmn = min([_final_min(lm, s_, c_) for s_, c_ in zip(new_s, new_c)], default=math.inf)
                    sc = np.float32(sc + np.float32(lm.scale * -fmn))
            st["scores"][b, i] = sc
            st["next_ys"][step + 1, b, i] = EOS if fin[i] else y
        cnt = int(st["fin_count"][b])
        for i in range(K):
            if fin[i] and cnt < cap:
                st["fin_score"][b, cnt], st["fin_step"][b, cnt], st["fin_k"][b, cnt] = st["scores"][b, i], step + 1, i
                cnt += 1
        st["fin_count"][b] = cnt
        if fin[0]:
            st["eos_top"][b] = 1
        if st["eos_top"][b] and cnt >= n_best and not st["done"][b]:
            st["done"][b] = 1
            st["not_done_total"][0] -= 1
        # partial hypotheses: new[k] = finished ? old[k] : old[prev_k] + (y if y != blk), at most L tokens
        for i in range(K):
            pk, y = int(bid[i] // V), int(bid[i] % V)
            src = i if fin[i] else pk
            n = int(old_len[src])
            st["hyp_tok"][pn, b, i, :n] = old_hyp[src, :n]
            if not fin[i] and y != blk and n < L:
                st["hyp_tok"][pn, b, i, n] = y
                n += 1
            st["hyp_len"][pn, b, i] = n
    return st, ties
