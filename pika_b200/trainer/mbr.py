"""MBR (minimum Bayes risk) training batch -- the loop body of
trainer/train_transducer_mbr_bmuf_otfaug.py:93-240 on the sm_90a kernels.

  1. N-best generation with the batched device beam search (``n_best = beam_size``, ``beam_prune=False``, :79-87,113-117)
  2. one encoder forward (train mode) shared by both branches (:130-138)
  3. RNN-T branch: fused joint + loss on the reference labels, scaled by ``rnnt_scale`` (:140-161)
  4. MBR branch: path posteriors ``softmax(scores)``, edit-distance risk, ``seq_grad = prob * (dist - E[dist])``
     (:171-195); the joint is evaluated ONLY on the (t,u) nodes of each N-best alignment (:212-232) and the sparse
     ``mbr_grad`` (blank entries divided by T', :234) is back-propagated through ``log_softmax(sm_scale * out)``
  5. one backward through the encoder and the prediction net with the summed gradients.

Differences from the reference that do not change any gradient: the prediction net runs once on
[reference labels ; hypotheses] (the reference runs it twice on the same parameters), and alignment positions
beyond a hypothesis' length -- which the reference pads with node (0,0) and a zero gradient -- are skipped.
"""
import numpy as np
import torch

from .. import engine
from .. import kernels as K


def edit_distance(a, b):
    """Levenshtein distance between two int sequences (``editdistance.eval``, :188); scalar form, kept as the definition the batched
    routine is tested against."""
    la, lb = len(a), len(b)
    prev = list(range(lb + 1))
    for i in range(1, la + 1):
        cur = [i] + [0] * lb
        ai = a[i - 1]
        for j in range(1, lb + 1):
            cur[j] = min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (ai != b[j - 1]))
        prev = cur
    return prev[lb]


def edit_distance_batch(refs, hyps):
    """Levenshtein distances of P (reference, hypothesis) pairs at once: one numpy pass per reference position over a [P, Lmax + 1]
    table.  The in-row dependency ``cur[j] = min(tmp[j], cur[j-1] + 1)`` is a prefix minimum: ``cur = cummin(tmp - j) + j``.
    (The pure-Python double loop costs ~0.5 s for 64 hypotheses of 150 labels -- the reference calls a C library here.)"""
    P = len(refs)
    if P == 0:
        return np.zeros(0, np.int64)
    la = np.array([len(r) for r in refs], np.int64)
    lb = np.array([len(h) for h in hyps], np.int64)
    La, Lb = int(la.max()), int(lb.max())
    A = np.full((P, max(La, 1)), -1, np.int64)
    Bm = np.full((P, max(Lb, 1)), -2, np.int64)
    for p in range(P):
        A[p, :la[p]] = refs[p]
        Bm[p, :lb[p]] = hyps[p]
    idx = np.arange(Lb + 1, dtype=np.int64)
    prev = np.broadcast_to(idx, (P, Lb + 1)).copy()                            # row 0: distance to the empty reference prefix
    out = prev[np.arange(P), lb].copy()                                        # pairs with an empty reference
    for i in range(1, La + 1):
        tmp = np.empty_like(prev)
        tmp[:, 0] = i
        if Lb:
            sub = prev[:, :-1] + (A[:, i - 1:i] != Bm[:, :Lb])
            tmp[:, 1:] = np.minimum(prev[:, 1:] + 1, sub)
        cur = np.minimum.accumulate(tmp - idx, axis=1) + idx
        done = la == i
        if done.any():
            out[done] = cur[done, lb[done]]
        prev = cur
    return out


def _tokens(h):
    """one hypothesis (alignment incl. blanks) as an int64 array: accepts an array, a list of ints or a list of 0-d tensors"""
    if isinstance(h, np.ndarray):
        return h.astype(np.int64)
    if len(h) and torch.is_tensor(h[0]):
        return torch.stack(list(h)).cpu().numpy().astype(np.int64)
    return np.asarray(list(h), dtype=np.int64).reshape(-1)


def nbest_risk(hyps, scores, targets, ali_lens, blk):
    """host side of :171-195.  -> (hyps_nonblk, prob [bsz,beam], dist [bsz,beam], seq_grad [bsz,beam], mbr_loss)"""
    bsz, beam = len(hyps), len(hyps[0])
    sc = np.array([[float(s) for s in row] for row in scores], dtype=np.float32)
    e = np.exp(sc - sc.max(axis=1, keepdims=True))
    prob = (e / e.sum(axis=1, keepdims=True)).astype(np.float32)
    arrs = [[_tokens(h) for h in row] for row in hyps]
    nonblk = [[a[a != blk].tolist() for a in row] for row in arrs]
    refs = [[int(v) for v in targets[i][:int(ali_lens[i])]] for i in range(bsz)]
    dist = edit_distance_batch([refs[i] for i in range(bsz) for _ in range(beam)],
                               [nonblk[i][j] for i in range(bsz) for j in range(beam)]).reshape(bsz, beam).astype(np.float32)
    avg = (prob * dist).sum(axis=1, keepdims=True)
    return nonblk, prob, dist, prob * (dist - avg), float(avg.sum())


def alignment_nodes(hyps, seq_grad, Tp, U, blk):
    """The (frame, label) lattice node every alignment token sits on (:197-232) and its gradient coefficient (:234: blank entries
    divided by T'), for all hypotheses at once: token p of hypothesis (i, j) is emitted at frame #blanks-before-p and label position
    #labels-before-p.  -> (ex_idx, py_idx, tokens, coef) flat arrays in (i, j, p) order."""
    bsz, beam = len(hyps), len(hyps[0])
    U1 = U + 1
    ex, py, tk, cf = [], [], [], []
    for i in range(bsz):
        for j in range(beam):
            h = _tokens(hyps[i][j])
            isb = h == blk
            t_i = np.cumsum(isb) - isb                                          # exclusive counts
            u_i = np.cumsum(~isb) - (~isb)
            sg = float(seq_grad[i, j])
            ex.append(i * Tp + np.minimum(t_i, Tp - 1))
            py.append((i * beam + j) * U1 + np.minimum(u_i, U))
            tk.append(h)
            cf.append(np.where(isb, np.float32(sg / float(Tp)), np.float32(sg)).astype(np.float32))
    cat = lambda v, dt: np.concatenate(v).astype(dt) if v else np.zeros(0, dt)   # noqa: E731
    return cat(ex, np.int32), cat(py, np.int32), cat(tk, np.int32), cat(cf, np.float32)


def mbr_forward_backward(model, feats, target, len_batch, ali_lens, ret, blk=0, rnnt_scale=1.0, sm_scale=1.0, fastemit_lambda=0.0,
                         delay_penalty=0.0):
    """Leaves d(rnnt_scale * rnnt_loss + mbr_loss)/d(param) in every ``param.grad``.  ``fastemit_lambda`` / ``delay_penalty`` apply to
    the RNN-T branch only, as in engine.transducer_loss; the MBR loss is unchanged.
    feats [bsz,T,D] (already CMVN'd / SpecAugmented), target [bsz,Umax] int64 (padded with padding_idx),
    ret = decode_batch output with n_best == beam.  Returns (mbr_loss, rnnt_loss) as python floats / tensor."""
    dev = feats.device
    hyps, scores = ret.get("alignments") or ret["predictions"], ret["scores"]   # arrays when the decoder provides them (bulk host work)
    bsz, beam = len(hyps), len(hyps[0])
    bb = bsz * beam
    pad = model.embed.padding_idx
    V = model.fc2.weight.shape[0]
    tgt_cpu = target.cpu().numpy()
    al_cpu = ali_lens.cpu().numpy()
    nonblk, prob, dist, seq_grad, mbr_loss = nbest_risk(hyps, scores, tgt_cpu, al_cpu, blk)

    # ---- shared encoder forward; prediction net once on [reference ; hypotheses]
    enc = engine.model_encoder_forward_act(model, feats, len_batch)              # [bsz, T', H], in the autograd graph
    Tp = enc.shape[1]
    u_ref = int(target.shape[1])
    u_hyp = max(len(h) for row in nonblk for h in row)
    U = max(u_ref, u_hyp)
    y_all = torch.full((bsz + bb, U), pad, dtype=torch.long)
    y_all[:bsz, :u_ref] = target.cpu().long()
    for i in range(bsz):
        for j in range(beam):
            h = nonblk[i][j]
            if h:
                y_all[bsz + i * beam + j, :len(h)] = torch.tensor(h, dtype=torch.long)
    pred_all = engine.prednet_forward_act(model, y_all.to(dev))                  # [bsz+bb, U+1, H]
    enc_d, pred_d = enc.detach(), pred_all.detach()

    # ---- RNN-T branch (fused joint + loss, gradients scaled by rnnt_scale)
    pred_ref = pred_d[:bsz, :u_ref + 1].contiguous()
    logits, st = engine.joint_forward(enc_d, pred_ref, model)
    gs = torch.full((bsz,), float(rnnt_scale), dtype=torch.float32, device=dev)
    db2 = torch.empty(logits.shape[-1], dtype=torch.float32, device=dev)
    costs, _ = K.rnnt_loss_fwd_bwd(logits, target[:, :u_ref].int().contiguous(), len_batch.int().contiguous(),
                                   ali_lens.int().contiguous(), V=V, grad_scale=gs, dlogits=logits, colsum=db2,
                                   fastemit_lambda=fastemit_lambda, delay_penalty=delay_penalty)
    d_enc, d_pred_ref = engine.joint_backward(logits, st, model, db2=db2)
    del logits, st

    # ---- MBR branch: the joint on the alignment nodes of every hypothesis, its gradients added to the RNN-T branch's
    ex_idx, py_idx, toks, coef = alignment_nodes(hyps, seq_grad, Tp, U, blk)
    ex_idx_t, py_idx_t, tok_t = (torch.from_numpy(v).to(dev) for v in (ex_idx, py_idx, toks))
    coef_t = torch.from_numpy(coef).to(dev)
    z, st = engine.joint_forward(enc_d, pred_d[bsz:], model, nodes=(ex_idx_t, py_idx_t))
    K.ce_grad(z, tok_t, coef_t, float(sm_scale), z, V)                         # in place: z := d(mbr)/d(logits)
    d_enc_m, d_pred_h = engine.joint_backward(z, st, model, accumulate=True)

    # ---- one backward through encoder and prediction net with the summed gradients
    d_enc_tot = torch.empty_like(enc_d)
    K.add(d_enc.reshape(-1), d_enc_m.reshape(-1), d_enc_tot.reshape(-1))
    d_pred_all = torch.zeros_like(pred_d)
    d_pred_all[:bsz, :u_ref + 1] = d_pred_ref
    d_pred_all[bsz:] = d_pred_h
    torch.autograd.backward([enc, pred_all], [d_enc_tot, d_pred_all])
    return mbr_loss, costs * float(rnnt_scale)
