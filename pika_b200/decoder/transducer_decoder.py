"""Transducer beam-search decoder -- drop-in for decoder/transducer_decoder.py (reference).

Same constructor and ``decode_batch(x, x_len, max_len) -> (ret, enc_out)`` contract
(``ret = {"predictions": B x n_best lists of 0-d int64 tensors (full alignment incl. blanks, trailing EOS
stripped), "scores": B x n_best 0-d f32 tensors}``).  All per-step work runs on the GPU for the whole batch:
encoder-frame gather, masked LSTM step, factored joint, log-softmax, and one ``pk_beam_advance`` launch that
performs every utterance's score add / EOS + duplicate kill / top-k / finish rule / hypothesis update
(decoder/beam_transducer.py:82-187), optionally with on-the-fly FST shallow fusion (:135-159,167-176).

Host work per beam step is a fraction of one launch: the step chain (14 kernels) reads its step index from device
memory, two steps (one period of the state ping-pong) are captured ONCE into a CUDA graph that lives with the decoder's
workspace, and the host replays it, looking at the "utterances not done" counter every few replays; steps issued after
the last utterance finished are no-ops on the device.  The workspace (state, histories, staged weights, graph) is kept
across ``decode_batch`` calls, so the MBR trainer's per-batch N-best generation re-uses it with freshly staged weights.
The back-pointers are walked once at the end (decoder/transducer_decoder.py:204-217, decoder/beam_transducer.py:196-243).

Like the reference, every utterance keeps advancing until ALL utterances of the batch are done, so late
finishes can still enter an utterance's n-best list.
"""
import ctypes
import os

import numpy as np
import torch

from .. import engine
from .. import kernels as K
from .. import _lib
from .._lib import check, lib

_USE_GRAPH = os.environ.get("PK_DECODE_GRAPH", "1") != "0"      # 0: issue every launch of the beam loop from the host (debugging)
_POLL = 4                                                        # graph replays (= 8 beam steps) between looks at the done counter


class _Workspace:
    """Everything the beam loop touches, at fixed addresses (graph-capturable), for one (batch, beam, capacity) signature."""

    def __init__(self, dec, B, Tcap, Scap, adt, dev):
        m, Kb = dec.model, dec.beam_size
        self.B, self.Tcap, self.Scap, self.adt, self.dev = B, Tcap, Scap, adt, dev
        H = m.fc1.weight.shape[0]
        V = m.fc2.weight.shape[0]
        L = m.decoder.num_layers if dec.xf is False else 0         # transformer prediction net: no recurrent state (see _xf_states)
        E = m.embed.weight.shape[1]
        self.H, self.V, self.L, self.E = H, V, L, E
        # layer 0 reads the embedding row zero-padded to the hidden width, so that x W_ih^T + h W_hh^T of a layer is ONE GEMM launch with two
        # accumulated (A, B) pairs (pairs share the reduction extent); the padding columns of x and of the staged W_ih are zero
        self.ldx = H if (E <= H and not dec.xf) else (E + 7) // 8 * 8
        rows = self.rows = B * Kb
        i32 = lambda *s, fill=0: torch.full(s, fill, dtype=torch.int32, device=dev)     # noqa: E731
        f32 = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)                # noqa: E731
        S = Scap
        self.cap = S * Kb
        self.enc = torch.zeros(B, Tcap, H, dtype=adt, device=dev)
        self.nf, self.ml = i32(B), i32(B)
        self.next_ys, self.prev_ks = i32(S + 1, B, Kb), i32(S, B, Kb)
        self.hyp_tok, self.hyp_len = i32(2, B, Kb, S + 1), i32(2, B, Kb)
        self.fin_score = f32(B, self.cap)
        self.fin_step, self.fin_k = i32(B, self.cap), i32(B, self.cap)
        self.fin_count, self.eos_top, self.done, self.not_done = i32(B), i32(B), i32(B), i32(1)
        self.scores = f32(B, Kb)
        self.t_idx, self.t_alt = i32(rows), i32(rows)
        self.h = torch.zeros(max(L, 1), rows, H, dtype=adt, device=dev)
        self.c = f32(max(L, 1), rows, H)
        self.h_alt, self.c_alt = torch.empty_like(self.h), torch.empty_like(self.c)
        self.enc_hid = torch.empty(rows, H, dtype=adt, device=dev)
        self.x_emb = torch.zeros(rows, self.ldx, dtype=adt, device=dev)
        self.gates = f32(rows, 4 * H)
        self.pre = f32(rows, 2 * H)
        self.hj = torch.empty(rows, H, dtype=adt, device=dev)
        self.ldv = (V + 3) // 4 * 4
        self.logits = f32(rows, self.ldv)
        self.row_lse = f32(rows)
        self.step_ctx = i32(2)
        # staged weights at fixed addresses: re-filled from the live parameters at every decode_batch (the MBR trainer updates them
        # between calls), [hi] in bf16 production mode, [hi, lo] in the fp32-class parity mode
        two = adt != torch.bfloat16

        def wbuf(n, k):
            return [torch.empty(n, k, dtype=torch.bfloat16, device=dev) for _ in range(2 if two else 1)]
        self.w_ih = [wbuf(4 * H, self.ldx if l == 0 else H) for l in range(L)]
        self.w_hh = [wbuf(4 * H, H) for _ in range(L)]
        self.wx = wbuf(2 * H, 2 * H)
        self.w2 = wbuf(V, H)
        self.bsum = [f32(4 * H) for _ in range(L)]
        self.bx = f32(2 * H)
        self.b2 = f32(V)
        self.lm = None
        if dec.lm_scorer is not None:
            MS = dec.lm_max_states
            fst_struct, keep = dec.lm_scorer.device_tables(dev)
            self.lm = dict(fst=fst_struct, keep=keep, set_state=i32(2, B, Kb, MS),
                           set_cost=torch.zeros(2, B, Kb, MS, dtype=torch.float64, device=dev), set_n=i32(2, B, Kb),
                           lm_scores=f32(B, Kb), err=i32(1))
        self.graph = None
        self.kernels_per_replay = 0
        self.sig = None                     # what the captured graph baked in besides the workspace addresses

    def stage(self, dec):
        """live parameters -> the fixed staging buffers"""
        m, lstm = dec.model, dec.model.decoder

        def put(bufs, param, cols_pad=None, rows=None):
            mat = param.detach().reshape(param.shape[0], -1)
            dst = bufs if rows is None else [b[rows[0]:rows[1]] for b in bufs]
            K.cast_split(mat, dst[0], dst[1] if len(dst) > 1 else None, cols_pad=cols_pad or mat.shape[1])
        H = self.H
        for l in range(self.L):                          # (no LSTM layers with the transformer prediction net)
            put(self.w_ih[l], getattr(lstm, "weight_ih_l%d" % l), cols_pad=self.ldx if l == 0 else None)
            put(self.w_hh[l], getattr(lstm, "weight_hh_l%d" % l))
            K.add(getattr(lstm, "bias_ih_l%d" % l).detach(), getattr(lstm, "bias_hh_l%d" % l).detach(), self.bsum[l])
        put(self.wx, m.fc1.weight, rows=(0, H))
        put(self.wx, m.fc_gate.weight, rows=(H, 2 * H))
        put(self.w2, m.fc2.weight)
        self.bx[:H].copy_(m.fc1.bias.detach())
        self.bx[H:].copy_(m.fc_gate.bias.detach())
        self.b2.copy_(m.fc2.bias.detach())

    def reset(self, dec, enc, x_len, ml_list):
        B, blk = self.B, dec.blk
        Tenc = enc.shape[1]
        self.enc[:, :Tenc].copy_(enc)
        self.nf.copy_(torch.as_tensor(np.asarray([int(v) for v in x_len], np.int32)))
        self.ml.copy_(torch.as_tensor(np.asarray(ml_list, np.int32)))
        self.next_ys[0].fill_(blk)
        self.hyp_len.zero_()
        for t in (self.fin_count, self.eos_top, self.done, self.scores):
            t.zero_()
        self.not_done.fill_(B)
        self.t_idx.fill_(-1)
        self.step_ctx.copy_(torch.tensor([0, 1], dtype=torch.int32))
        if self.lm is not None:
            for k in ("set_state", "set_cost", "set_n", "lm_scores", "err"):
                self.lm[k].zero_()


class TransducerDecoder():
    def __init__(self, model, batch_size, beam_size, n_best=1, blk=0, global_scorer=None, sm_scale=1.0, lm=None, lm_scale=1.0,
                 lm_scorer=None, lm_scorer_scale=1.0, cuda=False, beam_prune=True, args=None):
        self.model, self.batch_size, self.beam_size, self.n_best, self.blk = model, batch_size, beam_size, n_best, blk
        self.global_scorer, self.sm_scale, self.cuda, self.beam_prune, self.args = global_scorer, sm_scale, cuda, beam_prune, args
        if lm is not None and lm != '':
            raise NotImplementedError("pika_b200: neural LM fusion (`lm`) is not part of the hot path; FST fusion is `lm_scorer`")
        # on-the-fly FST shallow fusion (decoder/beam_transducer.py:135-159,167-176): lm_scorer = pika_b200.decoder.sorted_matcher.SortedMatcher
        self.lm_scorer, self.lm_scorer_scale = lm_scorer, float(lm_scorer_scale)
        self.lm_max_states = 16
        # LAS rescoring hooks (decoder/transducer_decoder.py:56-62, 219-253): the rescorer networks are the caller's own modules
        # (decode_transducer.py:22-38 unpickles them); this class only scores a hypothesis with them, like the reference's
        self.las_rescorer = getattr(args, "las_rescorer", None) if args is not None else None
        self.las_rescorer_bw = getattr(args, "las_rescorer_bw", None) if args is not None else None
        if args is not None and getattr(args, "bilas_rescorer", None) is not None:
            self.bilas_rescorer = args.bilas_rescorer
        self.xf = model.decoder_type != "rnn"            # convolutional-transformer prediction net (decoder/transducer_decoder.py:117-120,151-171)
        if self.xf and lm_scorer is not None:
            raise NotImplementedError("pika_b200: FST fusion is wired to the LSTM prediction net only")
        self._ws = None
        self.last_replays = self.kernels_per_replay = 0

    # ------------------------------------------------------------------------------------------------
    def _workspace(self, B, Tenc, S, adt, dev):
        ws = self._ws
        if ws is None or ws.B != B or ws.adt != adt or ws.dev != dev or ws.Tcap < Tenc or ws.Scap < S:
            # capacities only grow, so a stream of similar batches settles on one workspace (and one captured graph)
            same = ws is not None and ws.B == B and ws.adt == adt and ws.dev == dev
            ws = self._ws = _Workspace(self, B, max(Tenc, ws.Tcap if same else 0), max(S, ws.Scap if same else 0), adt, dev)
        return ws

    def _xf_states(self, ws, par):
        """prediction-net output for every beam row from its current partial hypothesis (transformer branch,
        decoder/transducer_decoder.py:117-120,151-171).  The reference re-runs the whole history through the network for the rows that
        just emitted a label and keeps / reorders the stored output row otherwise; the network is causal and masks padding keys, so a
        row's output at its last position depends on its own history only -- recomputing every row from the hypothesis buffers
        (which ``pk_beam_advance`` already reorders) gives the same values and needs no state reorder."""
        m, rows = self.model, ws.rows
        hl = ws.hyp_len[par].reshape(rows)
        lmax = int(hl.max().item())
        pad = m.embed.padding_idx
        src = torch.full((rows, lmax + 1), pad, dtype=torch.long, device=ws.dev)
        src[:, 0] = self.blk
        if lmax > 0:
            tok = ws.hyp_tok[par].reshape(rows, -1)[:, :lmax].long()
            keep = torch.arange(lmax, device=ws.dev)[None, :] < hl[:, None]
            src[:, 1:] = torch.where(keep, tok, torch.full_like(tok, pad))
        out = engine.conv_transformer_lm_forward_act(m.decoder, src)                       # [rows, lmax + 1, H]
        return out[torch.arange(rows, device=ws.dev), hl.long()].contiguous()

    def _beam_step(self, ws, h, c, t_idx, h_out, c_out, t_out, par=None):
        """one iteration of `while not all(b.done() ...)` (decoder/transducer_decoder.py:123-186) for the whole batch;
        graph-capturable with the LSTM prediction net: no host reads, no step-dependent arguments (the kernels read the step from
        ``step_ctx``).  ``par`` (transformer prediction net only): parity of the step, selects the live hypothesis buffers."""
        m, Kb, blk = self.model, self.beam_size, self.blk
        P, st = K._P, K._stream
        H, V, L, rows = ws.H, ws.V, ws.L, ws.rows
        dt = K._dt(ws.h)
        check(lib.pk_beam_prepare(P(ws.next_ys), P(ws.step_ctx), P(t_idx), P(ws.enc), K._dt(ws.enc), ws.Tcap, H, P(ws.enc_hid),
                                  P(m.embed.weight.detach()), ws.E, P(ws.x_emb), ws.ldx, Kb, blk, rows, st()), "pk_beam_prepare")
        xin = ws.x_emb
        for l in range(L):
            if xin.shape[1] == H:
                engine.gemm_parts([engine.stage_act(xin), engine.stage_act(h[l])], [ws.w_ih[l], ws.w_hh[l]], ws.gates, bias=ws.bsum[l])
            else:
                engine.gemm_parts([engine.stage_act(xin)], [ws.w_ih[l]], ws.gates, bias=ws.bsum[l])
                engine.gemm_parts([engine.stage_act(h[l])], [ws.w_hh[l]], ws.gates, accumulate=True, k_splits=1)
            check(lib.pk_beam_lstm_cell(P(ws.gates), P(ws.next_ys), P(ws.step_ctx), blk, P(h[l]), dt, P(c[l]), rows, H, st()), "pk_beam_lstm_cell")
            xin = h[l]
        dec_hid = self._xf_states(ws, par) if self.xf else h[L - 1]
        engine.gemm_parts([engine.stage_act(ws.enc_hid), engine.stage_act(dec_hid)],
                          [[p[:, :H] for p in ws.wx], [p[:, H:] for p in ws.wx]], ws.pre, bias=ws.bx)
        check(lib.pk_beam_gate(P(ws.pre), P(ws.hj), K._dt(ws.hj), rows, H, st()), "pk_beam_gate")
        engine.gemm_parts([engine.stage_act(ws.hj)], [ws.w2], ws.logits[:, :V], bias=ws.b2)
        # log_softmax(sm_scale * logits) is not materialised: one pass leaves the row log-sum-exp, pk_beam_advance forms the log-probs
        check(lib.pk_row_lse(P(ws.logits), K._dt(ws.logits), ctypes.c_longlong(ws.ldv), P(ws.row_lse), ctypes.c_longlong(rows), V,
                             ctypes.c_float(self.sm_scale), st()), "pk_row_lse")
        common = (P(ws.logits), ws.ldv, P(ws.row_lse), ctypes.c_float(self.sm_scale), P(t_idx), P(ws.nf), P(ws.ml), P(ws.scores), P(ws.next_ys), P(ws.prev_ks), P(ws.hyp_tok), P(ws.hyp_len),
                  P(ws.fin_score), P(ws.fin_step), P(ws.fin_k), P(ws.fin_count), P(ws.eos_top), P(ws.done), P(ws.not_done), ws.B, Kb, V,
                  ws.Scap + 1, ws.cap, P(ws.step_ctx), blk, self.n_best, int(bool(self.beam_prune)))
        if ws.lm is None:
            check(lib.pk_beam_advance(*common, st()), "pk_beam_advance")
        else:
            lm = ws.lm
            check(lib.pk_beam_advance_lm(*common, ctypes.byref(lm["fst"]), ctypes.c_double(self.lm_scorer_scale),
                                         ctypes.c_double(float(getattr(self.args, "nonblk_reward", 0.0))), P(lm["set_state"]), P(lm["set_cost"]),
                                         P(lm["set_n"]), P(lm["lm_scores"]), self.lm_max_states, P(lm["err"]), st()), "pk_beam_advance_lm")
        check(lib.pk_beam_reorder(P(ws.prev_ks), P(ws.step_ctx), P(h), P(c), P(t_idx), P(h_out), P(c_out), P(t_out), dt, Kb, H, L, rows, st()),
              "pk_beam_reorder")
        check(lib.pk_beam_step_end(P(ws.step_ctx), P(ws.not_done), ws.Scap - 1, st()), "pk_beam_step_end")

    def _period(self, ws):
        """two beam steps = one period of the (h, c, t_idx) ping-pong"""
        self._beam_step(ws, ws.h, ws.c, ws.t_idx, ws.h_alt, ws.c_alt, ws.t_alt)
        self._beam_step(ws, ws.h_alt, ws.c_alt, ws.t_alt, ws.h, ws.c, ws.t_idx)

    @torch.no_grad()
    def decode_batch(self, x, x_len, max_len=None, enc_out=None):
        """``enc_out`` (extension): encoder outputs [B, T', H] computed by the caller; ``x`` is then ignored."""
        m, blk = self.model, self.blk
        dev = x.device if enc_out is None else enc_out.device
        assert dev.type == "cuda", "pika_b200 decodes on the GPU (there is no CPU fallback)"
        if enc_out is None:
            enc = engine.model_encoder_forward_act(m, x, x_len).contiguous()     # [B, T', H] (packed over x_len: LSTM encoder)
        else:
            enc = engine._to_act(enc_out)
        B, Tenc, H = enc.shape
        ml_list = [int(max_len[i]) if max_len[i] else 10000 for i in range(B)]
        S = max(ml_list) + 2
        ws = self._workspace(B, Tenc, S, enc.dtype, dev)
        ws.stage(self)
        ws.reset(self, enc, x_len, ml_list)

        if self.xf:
            return self._decode_loop_xf(ws, enc, B)
        # initial decoder state = LSTM(embed(blk)) from zeros (decoder/transducer_decoder.py:116)
        ws.x_emb.zero_()
        ws.x_emb[:, :ws.E] = m.embed.weight.detach()[blk].to(ws.adt)
        xin = ws.x_emb
        for l in range(ws.L):
            engine.gemm_parts([engine.stage_act(xin)], [ws.w_ih[l]], ws.gates, bias=ws.bsum[l])
            K.lstm_cell_fwd(ws.gates, None, None, ws.c[l], ws.h[l], None, ws.rows, H)
            xin = ws.h[l]

        max_steps = ws.Scap - 1
        sig = (m.embed.weight.data_ptr(), float(self.sm_scale), int(bool(self.beam_prune)), self.n_best, self.lm_scorer_scale,
               float(getattr(self.args, "nonblk_reward", 0.0)) if self.args is not None else 0.0)
        issued = 0
        self.last_replays = 0
        if _USE_GRAPH and ws.graph is not None and ws.sig == sig:
            period = ws.graph.replay
        else:
            # first use of this workspace: one eager period (it also performs every lazy one-time initialisation inside the library),
            # then the capture; the graph is position independent, later calls replay it from step 0
            self._period(ws)
            issued = 2
            period = lambda: self._period(ws)                                   # noqa: E731
            if _USE_GRAPH:
                graph = torch.cuda.CUDAGraph()
                l0 = _lib.launch_count()
                with torch.cuda.graph(graph):
                    self._period(ws)
                ws.graph, ws.sig, ws.kernels_per_replay = graph, sig, _lib.launch_count() - l0
                period = graph.replay
        self.kernels_per_replay = ws.kernels_per_replay
        while issued < max_steps:
            for _ in range(_POLL):
                period()
                issued += 2
                self.last_replays += 1
            if int(ws.not_done.item()) == 0:                                    # `while not all(b.done() for b in beam)`
                break
        if ws.lm is not None and int(ws.lm["err"].item()) != 0:
            raise RuntimeError("pika_b200: an FST state set outgrew lm_max_states=%d active states per beam" % self.lm_max_states)
        return self._extract(ws, enc, B)

    def _decode_loop_xf(self, ws, enc, B):
        """beam loop with the transformer prediction net: issued step by step from the host (the history length, hence every shape
        of the prediction net, changes with the step, so there is no fixed graph to replay)"""
        bufs = ((ws.t_idx, ws.t_alt), (ws.t_alt, ws.t_idx))
        for i in range(ws.Scap - 1):
            t_in, t_out = bufs[i & 1]
            self._beam_step(ws, ws.h, ws.c, t_in, ws.h, ws.c, t_out, par=i & 1)
            if int(ws.not_done.item()) == 0:                                    # `while not all(b.done() for b in beam)`
                break
        self.last_replays = 0
        return self._extract(ws, enc, B)

    # ------------------------------------------------------------------------------------------------ LAS rescoring hooks
    @staticmethod
    def _token_log_probs(proj, tgt, scale=1.0):
        """log_softmax(scale * proj) [T, 1, C] -> the log-probability of tgt[t + 1] at every step t (decoder/transducer_decoder.py:234-238)"""
        assert proj.is_cuda, "pika_b200 scores on the GPU (there is no CPU fallback)"
        logits = proj.squeeze(1).float().contiguous()
        lp = torch.empty_like(logits)
        K.log_softmax(logits, lp, logits.shape[1], scale)
        tgt_idx = tgt[1:].squeeze(-1).squeeze(-1).to(lp.device)
        return lp[torch.arange(tgt_idx.size(0), device=lp.device), tgt_idx].tolist()

    @torch.no_grad()
    def las_rescore(self, x, tgt, bw=False):
        """x [T, 1, C] encoder outputs, tgt [L, 1, 1] = SOS + hypothesis + EOS -> per-token log-probs of the (backward) LAS rescorer
        (decoder/transducer_decoder.py:219-238)"""
        net = self.las_rescorer_bw if bw else self.las_rescorer
        lens = torch.IntTensor([x.size(0)])
        outputs, _, _, _ = net(x, tgt, lens)
        return self._token_log_probs(net.dec_proj(outputs), tgt)

    @torch.no_grad()
    def bilas_rescore(self, x, tgt):
        """bidirectional LAS rescorer, logits halved before the softmax (decoder/transducer_decoder.py:240-253)"""
        lens, ali_lens = torch.IntTensor([x.size(0)]), torch.IntTensor([tgt.size(0)])
        outputs, _, _, _ = self.bilas_rescorer(x, tgt, lens, None, True, True, ali_lens)
        return self._token_log_probs(self.bilas_rescorer.dec_proj(outputs), tgt, 0.5)

    def _extract(self, ws, enc, B):
        step = int(ws.step_ctx[0].item())                                       # beam steps actually executed
        # (4) extract: sort_finished + get_hyp on the host, once
        ny, pk = ws.next_ys[:step + 1].cpu().numpy(), ws.prev_ks[:step].cpu().numpy()
        fc = ws.fin_count.cpu().numpy()
        nmax = max(int(fc.max()) if B else 0, 1)
        fs, fstep, fk = ws.fin_score[:, :nmax].cpu().numpy(), ws.fin_step[:, :nmax].cpu().numpy(), ws.fin_k[:, :nmax].cpu().numpy()
        # sort_finished (stable, like list.sort(key=-score)) per utterance, then every selected hypothesis walks its back-pointers at once
        # (BeamMergeTransducer.get_hyp): one numpy gather per beam step instead of a Python loop per token
        sel = []                                                              # (utterance, slot in the finished list)
        for b in range(B):
            order = sorted(range(int(fc[b])), key=lambda i: -fs[b, i])
            sel.extend((b, i) for i in order[:self.n_best])
        sb = np.asarray([b for b, _ in sel], np.int64)
        si = np.asarray([i for _, i in sel], np.int64)
        ln = fstep[sb, si].astype(np.int64) if len(sel) else np.zeros(0, np.int64)
        kk = fk[sb, si].astype(np.int64) if len(sel) else np.zeros(0, np.int64)
        toks = np.zeros((len(sel), int(ln.max()) if len(sel) else 0), np.int64)
        for j in range(toks.shape[1] - 1, -1, -1):
            act = ln > j
            toks[act, j] = ny[j + 1, sb[act], kk[act]]
            kk[act] = pk[j, sb[act], kk[act]]
        # "alignments" (extension): the same hypotheses as int64 arrays, for callers that post-process them in bulk (the MBR trainer)
        ret = {"predictions": [[] for _ in range(B)], "scores": [[] for _ in range(B)], "alignments": [[] for _ in range(B)]}
        for r, (b, i) in enumerate(sel):
            arr = toks[r, :max(int(ln[r]) - 1, 0)].copy()                     # strip the ending eos(-1)
            ret["alignments"][b].append(arr)
            ret["predictions"][b].append(list(torch.from_numpy(arr).unbind(0)))   # 0-d int64 tensors, like the reference's token lists
            ret["scores"][b].append(torch.tensor(float(fs[b, i]), dtype=torch.float32))
        return ret, enc.float()
