"""Forced alignment of known transcripts with an RNN-T model: token times as a CTM file, and per-utterance alignment scores.

    python -m pika_b200.decoder.align_transducer MODEL FEATS_RSPEC LABELS_RSPEC OUT_CTM --loader utt --cuda --batch_first ...

The inputs are the decoding entry point's (decode_transducer.py): a pickled model, a Kaldi feature table and label archive read by the
``utt`` loader, with the same --cmvn_stats / --cmn / --min_len handling and the same --model_lctx / --model_rctx / --model_stride frame
arithmetic.  Every utterance is aligned, the last incomplete batch included.  The best path through the RNN-T lattice
(engine.transducer_align) gives the frame t on which each label is emitted; the CTM holds one line per label

    uttid 1 start dur token      start = (model_lctx + t * model_stride) * stride * frame_shift,  dur = model_stride * stride * frame_shift

in seconds with 3 decimals (``stride`` the loader's --stride).  ``--scores FILE`` writes ``uttid T' U viterbi loglik viterbi/T'`` per
utterance: the best path's log-probability and log P(y | x).  An utterance without a finite path (under --prune_range: more labels than
frames x (prune_range - 1)) gets ``-inf`` scores and no CTM lines."""
import argparse
import importlib
import math
import sys

import torch

from .decode_transducer import add_chunk_args, apply_chunk_args, load_cmvn, prepare_batch, read_symbols_map


def build_parser():
    p = argparse.ArgumentParser(description='pika_b200 --- forced alignment with the transducer')
    p.add_argument('model', type=str, help='model used for the alignment')
    p.add_argument('input_specifier', type=str, help='rspec for input feats')
    p.add_argument('input_labels', type=str, help='rspec for the transcripts (label ids)')
    p.add_argument('output_file', type=str, help='CTM file to write')
    p.add_argument('--cmn', action="store_true", help="apply cepstrum mean normalizaiton per utterance")
    p.add_argument('--cmvn_stats', type=str, default=None, help='cmvn_stats file')
    p.add_argument('--cuda', action='store_true', help='use CUDA')
    p.add_argument('--loader', choices=['utt'], default='utt', help='loaders for inferencing')
    p.add_argument('--local_rank', type=int, default=0, help='process id when using multi-GPU')
    p.add_argument('--symbols_map', type=str, default=None, help="file mapping symbol to int (without it the CTM holds the ids)")
    p.add_argument('--min_len', type=int, default=0, help="will pad input if less than this value")
    p.add_argument('--model_lctx', type=int, default=0, help='model left context')
    p.add_argument('--model_rctx', type=int, default=0, help='model right context')
    p.add_argument('--model_stride', type=int, default=1, help='model stride, ie., subsampling in the model')
    p.add_argument('--precision', choices=['bf16', 'fp32'], default='bf16', help='activation precision of the model')
    p.add_argument('--prune_range', type=int, default=0,
                   help='align in the pruned lattice: R >= 2 label positions per frame chosen by the simple joiner (0: dense)')
    p.add_argument('--frame_shift_ms', type=float, default=10.0, help='frame shift of the features in milliseconds')
    p.add_argument('--scores', type=str, default=None, help="write 'uttid T' U viterbi loglik viterbi/T'' lines to this file")
    add_chunk_args(p)
    return p


def check_args(parser, args):
    if args.prune_range != 0 and args.prune_range < 2:
        parser.error("--prune_range must be 0 (dense) or >= 2 (got %d)" % args.prune_range)
    if args.model_stride < 1 or args.frame_shift_ms <= 0:
        parser.error("--model_stride must be >= 1 and --frame_shift_ms > 0")


def ctm_lines(uttid, frames, tokens, model_lctx, model_stride, stride, frame_shift_ms):
    """CTM lines 'uttid 1 start dur token' of one utterance: label u emitted on encoder frame frames[u]"""
    shift = stride * frame_shift_ms / 1000.0
    dur = model_stride * shift
    return ["%s 1 %.3f %.3f %s" % (uttid, (model_lctx + t * model_stride) * shift, dur, tok) for t, tok in zip(frames, tokens)]


def score_line(uttid, T, U, viterbi, loglik):
    """'uttid T' U viterbi loglik viterbi/T'' (-inf when there is no finite path)"""
    per_frame = viterbi / T if T > 0 else -math.inf
    return "%s %d %d %.4f %.4f %.6f" % (uttid, T, U, viterbi, loglik, per_frame)


def main(argv=None):
    from .. import engine
    parser = build_parser()
    args, _ = parser.parse_known_args(argv)
    loader_module = importlib.import_module('pika_b200.loader.' + args.loader + '_loader')
    loader_module.register(parser)
    args = parser.parse_args(argv)
    check_args(parser, args)
    args.input_dim = loader_module.get_inputdim(args)
    if not (args.cuda and torch.cuda.is_available()):
        sys.exit("pika_b200.decoder.align_transducer: the alignment runs on the GPU only (pass --cuda on a CUDA machine)")
    dev = torch.device("cuda", args.local_rank)
    torch.cuda.set_device(dev)
    engine.set_precision(args.precision)
    model = torch.load(args.model, map_location="cpu", weights_only=False)
    apply_chunk_args(parser, args, model)
    model.eval().to(dev)
    if args.prune_range and not hasattr(model, "simple_am_proj"):
        sys.exit("pika_b200.decoder.align_transducer: --prune_range needs a model trained with the pruned loss (simple_am_proj)")
    load_cmvn(args, dev)
    sym_map = read_symbols_map(args.symbols_map) if args.symbols_map else None
    R = args.prune_range
    scores = open(args.scores, 'w') if args.scores else None
    try:
        with open(args.output_file, 'w') as f:
            for data, target, lens, ali_lens, ids in loader_module.dataloader(args.input_labels, args.input_specifier, False, args,
                                                                               keep_tail=True, with_ids=True):
                if not args.batch_first:
                    data, target = data.transpose(0, 1), target.transpose(0, 1)
                data, tl = prepare_batch(data, lens, args, dev)
                target = target.to(dev)
                ul = torch.from_numpy(ali_lens).to(dev)
                B = len(ids)
                tl_h, ul_h = tl.tolist(), ul.tolist()
                # under --prune_range an utterance with U > T' (R - 1) has no path inside the windows: reported with -inf, not aligned
                keep = [b for b in range(B) if not R or ul_h[b] <= tl_h[b] * (R - 1)]
                frames = [[-1] * ul_h[b] for b in range(B)]
                vit, ll = [-math.inf] * B, [-math.inf] * B
                if keep:
                    idx = torch.tensor(keep, device=dev)
                    x, y, fl, lab_l = data.index_select(0, idx), target.index_select(0, idx), tl.index_select(0, idx), ul.index_select(0, idx)
                    fr, v, l = engine.transducer_align(model, x.float(), y, fl, lab_l, x_len=fl, t_out=int(fl.max()), prune_range=R)
                    fr, v, l = fr.cpu().tolist(), v.cpu().tolist(), l.cpu().tolist()
                    for i, b in enumerate(keep):
                        frames[b], vit[b], ll[b] = fr[i][:ul_h[b]], v[i], l[i]
                for b in range(B):
                    if math.isfinite(vit[b]):
                        toks = target[b, :ul_h[b]].tolist()
                        toks = [sym_map[t] for t in toks] if sym_map is not None else [str(t) for t in toks]
                        for line in ctm_lines(ids[b], frames[b], toks, args.model_lctx, args.model_stride, args.stride, args.frame_shift_ms):
                            f.write(line + "\n")
                    if scores is not None:
                        scores.write(score_line(ids[b], tl_h[b], ul_h[b], vit[b], ll[b]) + "\n")
    finally:
        if scores is not None:
            scores.close()


if __name__ == '__main__':
    main()
