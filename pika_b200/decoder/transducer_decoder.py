"""Transducer beam-search decoder -- drop-in for decoder/transducer_decoder.py (reference).

Same constructor and ``decode_batch(x, x_len, max_len) -> (ret, enc_out)`` contract
(``ret = {"predictions": B x n_best lists of 0-d int64 tensors (full alignment incl. blanks, trailing EOS
stripped), "scores": B x n_best 0-d f32 tensors}``).  All per-step work runs on the GPU for the whole batch:
encoder-frame gather, masked LSTM step (or the transformer prediction net's incremental KV-cached step, _XfBuffers),
factored joint, log-softmax, and one ``pk_beam_advance`` launch that
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
import os

import numpy as np
import torch

from .. import engine
from .. import kernels as K
from .. import _lib
from .._lib import BeamXfState, PikaError, check, lib

_USE_GRAPH = os.environ.get("PK_DECODE_GRAPH", "1") != "0"      # 0: issue every launch of the beam loop from the host (debugging)
BEAM_SIZES = (1, 2, 4, 8, 16)                                    # the widths beam_advance_kernel is instantiated for (csrc/beam.cu)
_POLL = 4                                                        # graph replays (= 8 beam steps) between looks at the done counter


class _Workspace:
    """Everything the beam loop touches, at fixed addresses (graph-capturable), for one (batch, beam, capacity) signature."""

    def __init__(self, dec, B, Tcap, Scap, adt, dev):
        m, Kb = dec.model, dec.beam_size
        self.B, self.Tcap, self.Scap, self.adt, self.dev = B, Tcap, Scap, adt, dev
        H = m.fc1.weight.shape[0]
        V = m.fc2.weight.shape[0]
        L = m.decoder.num_layers if dec.xf is False else 0         # transformer prediction net: its state is the KV cache (_XfBuffers)
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
        self.xf = _XfBuffers(self, dec, wbuf) if dec.xf else None
        self.graph = None
        self.kernels_per_replay = 0
        self.sig = None                     # what the captured graph baked in besides the workspace addresses

    def stage(self, dec):
        """live parameters -> the fixed staging buffers"""
        m, lstm = dec.model, dec.model.decoder
        H = self.H
        for l in range(self.L):                          # (no LSTM layers with the transformer prediction net)
            _put(self.w_ih[l], getattr(lstm, "weight_ih_l%d" % l), cols_pad=self.ldx if l == 0 else None)
            _put(self.w_hh[l], getattr(lstm, "weight_hh_l%d" % l))
            K.add(getattr(lstm, "bias_ih_l%d" % l).detach(), getattr(lstm, "bias_hh_l%d" % l).detach(), self.bsum[l])
        _put(self.wx, m.fc1.weight, rows=(0, H))
        _put(self.wx, m.fc_gate.weight, rows=(H, 2 * H))
        _put(self.w2, m.fc2.weight)
        self.bx[:H].copy_(m.fc1.bias.detach())
        self.bx[H:].copy_(m.fc_gate.bias.detach())
        self.b2.copy_(m.fc2.bias.detach())
        if self.xf is not None:
            self.xf.stage(dec)

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
        if self.xf is not None:
            self.xf.slot.zero_()                # position 0 of every row is the shared SOS entry 0


class _XfBuffers:
    """Device state of the transformer prediction net's incremental beam step (pika_b200/csrc/beam_xf.cu), at fixed addresses.

    pool [1 + Scap * rows, layers, 3, d_model] (activation dtype): one entry per computed position, written once and never moved --
    per layer its K row, its V row and (layer >= 1) the layer's input, which the next positions' causal conv taps read.  Entry 0 is
    the SOS position shared by every row, entry 1 + s * rows + row the position that `row` computed at beam step s.  That is
    (1 + Scap * rows) * layers * 3 * d_model elements: 3.0 GB in bf16 at batch 64 x beam 16, 2 layers, d_model 512, Scap = T' + 102 = 477.
    slot [2, B, beam, Scap + 1] int32 maps a row's positions to entries, ping-ponged by step parity like hyp_tok and reordered by the
    back-pointers after every advance (pk_beam_xf_slots), so the rows of one utterance share their common prefix's entries."""

    def __init__(self, ws, dec, wbuf):
        pn, dev, adt = dec.model.decoder, ws.dev, ws.adt
        rows, H, S = ws.rows, ws.H, ws.Scap
        self.layers, self.D, self.heads = len(pn.transformer), pn.linear_out.weight.shape[1], pn.transformer[0].self_attn.head_count
        D, dff = self.D, pn.transformer[0].feed_forward.w_1.weight.shape[0]
        act = lambda *s: torch.zeros(*s, dtype=adt, device=dev)                         # noqa: E731
        f32 = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)               # noqa: E731
        self.n_entries = 1 + S * rows
        self.pool = torch.empty(self.n_entries, self.layers, 3, D, dtype=adt, device=dev)
        self.slot = torch.zeros(2, ws.B, dec.beam_size, S + 1, dtype=torch.int32, device=dev)
        self.ld_tap = [ws.ldx] + [D] * (self.layers - 1)                                # layer 0 reads the (padded) embedding rows
        self.taps = [act(rows, 5 * ld) for ld in self.ld_tap]
        self.cv, self.ln, self.ctx, self.h1, self.xl = (act(rows, D) for _ in range(5))
        self.qkv, self.ff, self.xo = act(rows, 3 * D), act(rows, dff), act(rows, H)
        self.mean, self.rstd = f32(rows), f32(rows)
        # staged weights, re-filled from the live parameters at every decode_batch (stage)
        n = self.layers
        self.conv_w = [wbuf(D, 5 * ld) for ld in self.ld_tap]                           # tap-major: tap k at columns [k*ld, k*ld + C)
        self.qkv_w, self.fo_w = [wbuf(3 * D, D) for _ in range(n)], [wbuf(D, D) for _ in range(n)]
        self.w1, self.w2 = [wbuf(dff, D) for _ in range(n)], [wbuf(D, dff) for _ in range(n)]
        self.conv_b, self.qkv_b, self.fo_b = [f32(D) for _ in range(n)], [f32(3 * D) for _ in range(n)], [f32(D) for _ in range(n)]
        self.b1, self.b2 = [f32(dff) for _ in range(n)], [f32(D) for _ in range(n)]
        self.ln1 = [(f32(D), f32(D)) for _ in range(n)]
        self.ln2 = [(f32(D), f32(D)) for _ in range(n)]
        self.lnf = (f32(D), f32(D))
        self.out_w, self.out_b = wbuf(H, D), f32(H)
        self.rel = [f32(*l.self_attn.relative_positions_embeddings.weight.shape) if getattr(l.self_attn, "max_relative_positions", 0) > 0
                    else None for l in pn.transformer]
        self.eps = [(l.layer_norm.eps, l.feed_forward.layer_norm.eps) for l in pn.transformer] + [pn.layer_norm.eps]
        P = K._P
        self.st, self.st_init = (BeamXfState(P(ws.next_ys), P(ws.step_ctx), P(ws.hyp_tok), P(ws.hyp_len), P(self.slot), P(self.pool),
                                             self.n_entries, dec.blk, rows, S + 1, self.layers, D, K._dt(self.pool), init)
                                 for init in (0, 1))

    def stage(self, dec):
        pn = dec.model.decoder
        for l, (conv, layer) in enumerate(zip(pn.conv, pn.transformer)):
            att, ff = layer.self_attn, layer.feed_forward
            N, C, Kw = conv.weight.shape
            taps = torch.zeros(N, Kw, self.ld_tap[l], dtype=torch.float32, device=conv.weight.device)
            taps[:, :, :C] = conv.weight.detach().permute(0, 2, 1)
            _put(self.conv_w[l], taps.view(N, -1))
            self.conv_b[l].copy_(conv.bias.detach())
            for r, lin in enumerate((att.linear_query, att.linear_keys, att.linear_values)):
                _put(self.qkv_w[l], lin.weight, rows=(r * self.D, (r + 1) * self.D))
                self.qkv_b[l][r * self.D:(r + 1) * self.D].copy_(lin.bias.detach())
            for w, b, lin in ((self.fo_w, self.fo_b, att.final_linear), (self.w1, self.b1, ff.w_1), (self.w2, self.b2, ff.w_2)):
                _put(w[l], lin.weight)
                b[l].copy_(lin.bias.detach())
            for dst, ln in ((self.ln1[l], layer.layer_norm), (self.ln2[l], ff.layer_norm)):
                dst[0].copy_(ln.weight.detach())
                dst[1].copy_(ln.bias.detach())
            if self.rel[l] is not None:
                self.rel[l].copy_(att.relative_positions_embeddings.weight.detach())
        self.lnf[0].copy_(pn.layer_norm.weight.detach())
        self.lnf[1].copy_(pn.layer_norm.bias.detach())
        _put(self.out_w, pn.linear_out.weight)
        self.out_b.copy_(pn.linear_out.bias.detach())

    def step(self, dec, h, init=False):
        """the prediction net's output at every computing row's new position -> h [rows, H] (other rows keep theirs); ``init``: the SOS
        position into entry 0 and its output into every row, ``decoder([blk])[:, -1]`` (decoder/transducer_decoder.py:117-120)"""
        st = self.st_init if init else self.st
        emb = dec.model.embed.weight.detach()
        A = engine.stage_act
        for l in range(self.layers):
            K.beam_xf_taps(st, l, emb, self.xl if l > 0 else None, self.taps[l])
            engine.gemm_parts([A(self.taps[l])], [self.conv_w[l]], self.cv, bias=self.conv_b[l], act=K.ACT_RELU)
            K.layernorm_fwd(self.cv, self.ln, self.ln1[l][0], self.ln1[l][1], self.eps[l][0], self.mean, self.rstd)
            engine.gemm_parts([A(self.ln)], [self.qkv_w[l]], self.qkv, bias=self.qkv_b[l])
            K.beam_xf_attn(st, l, self.qkv, self.heads, self.rel[l], self.ctx)
            engine.gemm_parts([A(self.ctx)], [self.fo_w[l]], self.h1, bias=self.fo_b[l], aux=self.cv, aux_mode=K.AUX_ADD)
            K.layernorm_fwd(self.h1, self.ln, self.ln2[l][0], self.ln2[l][1], self.eps[l][1], self.mean, self.rstd)
            engine.gemm_parts([A(self.ln)], [self.w1[l]], self.ff, bias=self.b1[l], act=K.ACT_RELU)
            engine.gemm_parts([A(self.ff)], [self.w2[l]], self.xl, bias=self.b2[l], aux=self.h1, aux_mode=K.AUX_ADD)
        K.layernorm_fwd(self.xl, self.ln, self.lnf[0], self.lnf[1], self.eps[-1], self.mean, self.rstd)
        engine.gemm_parts([A(self.ln)], [self.out_w], self.xo, bias=self.out_b)
        K.beam_xf_select(st, self.xo, h)


def _put(bufs, param, cols_pad=None, rows=None):
    """live parameter -> its fixed staging buffers ([hi] or [hi, lo] bf16), optionally into a row range of them"""
    mat = param.detach().reshape(param.shape[0], -1)
    dst = bufs if rows is None else [b[rows[0]:rows[1]] for b in bufs]
    K.cast_split(mat, dst[0], dst[1] if len(dst) > 1 else None, cols_pad=cols_pad or mat.shape[1])


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
        # pk_beam_advance has instances for these widths only; refuse others here, before any kernel launch
        if beam_size not in BEAM_SIZES:
            raise PikaError("pika_b200: the device beam search supports beam sizes %s (got %d)" % (", ".join(map(str, BEAM_SIZES)), beam_size))
        self.xf = model.decoder_type != "rnn"            # convolutional-transformer prediction net (decoder/transducer_decoder.py:117-120,151-171)
        if self.xf:
            heads = {l.self_attn.head_count for l in model.decoder.transformer}
            d_model = model.decoder.linear_out.weight.shape[1]
            if any(d_model != 64 * h for h in heads):
                raise PikaError("pika_b200: the transformer prediction net's beam step needs a head size of 64 (d_model %d, heads %s)"
                                % (d_model, sorted(heads)))
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

    def _beam_step(self, ws, h, c, t_idx, h_out, c_out, t_out):
        """one iteration of `while not all(b.done() ...)` (decoder/transducer_decoder.py:123-186) for the whole batch;
        graph-capturable: no host reads, no step-dependent arguments (the kernels read the step from ``step_ctx``).  With the
        transformer prediction net h[0] holds dec_states and the incremental step (_XfBuffers.step) replaces the LSTM cells."""
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
        if self.xf:
            ws.xf.step(self, h[0])
        dec_hid = h[0] if self.xf else h[L - 1]
        engine.gemm_parts([engine.stage_act(ws.enc_hid), engine.stage_act(dec_hid)],
                          [[p[:, :H] for p in ws.wx], [p[:, H:] for p in ws.wx]], ws.pre, bias=ws.bx)
        check(lib.pk_beam_gate(P(ws.pre), P(ws.hj), K._dt(ws.hj), rows, H, st()), "pk_beam_gate")
        engine.gemm_parts([engine.stage_act(ws.hj)], [ws.w2], ws.logits[:, :V], bias=ws.b2)
        # log_softmax(sm_scale * logits) is not materialised: one pass leaves the row log-sum-exp, pk_beam_advance forms the log-probs
        check(lib.pk_row_lse(P(ws.logits), K._dt(ws.logits), ws.ldv, P(ws.row_lse), rows, V, self.sm_scale, st()), "pk_row_lse")
        common = (P(ws.logits), ws.ldv, P(ws.row_lse), self.sm_scale, P(t_idx), P(ws.nf), P(ws.ml), P(ws.scores), P(ws.next_ys), P(ws.prev_ks), P(ws.hyp_tok), P(ws.hyp_len),
                  P(ws.fin_score), P(ws.fin_step), P(ws.fin_k), P(ws.fin_count), P(ws.eos_top), P(ws.done), P(ws.not_done), ws.B, Kb, V,
                  ws.Scap + 1, ws.cap, P(ws.step_ctx), blk, self.n_best, int(bool(self.beam_prune)))
        if ws.lm is None:
            check(lib.pk_beam_advance(*common, st()), "pk_beam_advance")
        else:
            lm = ws.lm
            check(lib.pk_beam_advance_lm(*common, lm["fst"], self.lm_scorer_scale,
                                         float(getattr(self.args, "nonblk_reward", 0.0)), P(lm["set_state"]), P(lm["set_cost"]),
                                         P(lm["set_n"]), P(lm["lm_scores"]), self.lm_max_states, P(lm["err"]), st()), "pk_beam_advance_lm")
        if self.xf:
            K.beam_xf_slots(ws.xf.st, ws.prev_ks, Kb)
        check(lib.pk_beam_reorder(P(ws.prev_ks), P(ws.step_ctx), P(h), P(c), P(t_idx), P(h_out), P(c_out), P(t_out), dt, Kb, H, h.shape[0], rows,
                                  st()), "pk_beam_reorder")
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
        if m.fc2.weight.shape[0] < self.beam_size:
            raise PikaError("pika_b200: the vocabulary (%d) is smaller than the beam (%d)" % (m.fc2.weight.shape[0], self.beam_size))
        if self.xf:
            # a hypothesis of up to max_len + 1 labels plus SOS; the prediction net's causal mask buffer is max_size (5000) positions long
            n = max(int(v) if v else 10000 for v in max_len) + 2
            max_size = m.decoder.mask.shape[-1]
            if n > max_size:
                raise PikaError("pika_b200: max_len allows histories of %d positions; the transformer prediction net's max_size is %d"
                                % (n, max_size))
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
            ws.xf.step(self, ws.h[0], init=True)                              # decoder([blk])[:, -1] (decoder/transducer_decoder.py:117-120)
        else:
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
