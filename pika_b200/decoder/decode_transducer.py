"""Decoding entry point -- drop-in for decoder/decode_transducer.py (reference): same positional arguments and flags, same output file
format (one line per hypothesis: the mapped symbols, optionally the beam score and the rescorer token scores).

    python -m pika_b200.decoder.decode_transducer MODEL FEATS_RSPEC LABELS_RSPEC OUT --loader utt --cuda --batch_first ...

Differences forced by the environment, none in the decoding itself: feature / label tables are read by the native readers
(pika_b200/loader/kaldi_io.py) instead of PyKaldi; ``--fst_lm`` takes the LM in OpenFst text form (``fstprint``; see
sorted_matcher.read_fst_text) because reading the binary form needs PyKaldi; the model must sit on the GPU (``--cuda``): the beam
search has no CPU path.  CMVN, minimum-length padding and the frame-count arithmetic follow decoder/decode_transducer.py:54-131."""
import argparse
import importlib
import sys

import numpy as np
import torch

from ..loader.kaldi_io import read_kaldi_text_matrix
from .beam_transducer import GlobalScorer
from .sorted_matcher import SortedMatcher, read_fst_text
from .transducer_decoder import TransducerDecoder


def build_parser():
    """decoder/decode_transducer.py:183-252"""
    p = argparse.ArgumentParser(description='pika_b200 --- decoding script for the transducer')
    p.add_argument('model', type=str, help='model loaded for decoding')
    p.add_argument('input_specifier', type=str, help='rspec for input feats')
    p.add_argument('input_labels', type=str, help='rspec for dummy input labels')
    p.add_argument('output_file', type=str, help='file to write for output hypothese')
    p.add_argument('--lm', type=str, help="lm filename", default='')
    p.add_argument('--lm_scale', type=float, default=1.0, help="LM scale used in decoding")
    p.add_argument('--fst_lm', type=str, help="fst lm filename (OpenFst text form)", default='')
    p.add_argument('--fst_lm_scale', type=float, default=1.0, help="LM scale used in decoding")
    p.add_argument('--nonblk_reward', type=float, default=1.5, help="nonblk reward used in LM rescoring")
    p.add_argument('--global_lm', type=str, help="fst lm filename", default='')
    p.add_argument('--global_lm_scale', type=float, default=1.0, help="LM scale used in decoding")
    p.add_argument('--las_rescorer_model', type=str, default=None, help='LAS model used to rescore RNNT N-best')
    p.add_argument('--las_rescorer_bw_model', type=str, default=None, help='backward LAS model used to rescore RNNT N-best')
    p.add_argument('--bilas_rescorer_model', type=str, default=None, help='bidirectional LAS model used to rescore RNNT N-best')
    p.add_argument('--SOS', type=int, default=-1, help='start of seq id, valid when beyond 0')
    p.add_argument('--EOS', type=int, default=-1, help='end of seq id, valid when beyond 0')
    p.add_argument('--sm_scale', type=float, default=1.0, help="softmax scale used in decoding")
    p.add_argument('--blk', type=int, default=0, help='blank ID ')
    p.add_argument('--output_scores', action='store_true', help='output scores with hypothesis')
    p.add_argument('--cmn', action="store_true", help="apply cepstrum mean normalizaiton per utterance")
    p.add_argument('--cmvn_stats', type=str, default=None, help='cmvn_stats file')
    p.add_argument('--cuda', action='store_true', help='use CUDA')
    p.add_argument('--loader', choices=['utt'], default='utt', help='loaders for inferencing')
    p.add_argument('--beam_size', type=int, default=64, help='num of hyps for beam search')
    p.add_argument('--n_best', type=int, default=1, help='num of best hyps output after decoding finish')
    p.add_argument('--max_sent_length', type=int, default=500, help='max length limits on decoding output')
    p.add_argument('--padding_idx', type=int, default=-1, help='padding index for targets')
    p.add_argument('--local_rank', type=int, default=0, help='process id when using multi-GPU')
    p.add_argument('--symbols_map', type=str, help="file mapping symbol to int")
    p.add_argument('--disambig_ids', type=str, default='', help='comma separated disambig ids for LM fst')
    p.add_argument('--max_num_arcs', type=int, default=0, help='maximum number of arcs of LM fst')
    p.add_argument('--max_id', type=int, default=0, help='maximum i/o label id of LM fst')
    p.add_argument('--backoff_id', type=int, default=0, help='backoff label id of LM fst')
    p.add_argument('--min_len', type=int, default=0, help="will pad input if less than this value")
    p.add_argument('--model_lctx', type=int, default=0, help='model left context')
    p.add_argument('--model_rctx', type=int, default=0, help='model right context')
    p.add_argument('--model_stride', type=int, default=1, help='model stride, ie., subsampling in the model')
    add_chunk_args(p)
    return p


def add_chunk_args(p):
    """--chunk_size / --left_chunks: override the TDNN-Transformer encoder's chunk setting (DESIGN.md "Chunked attention")"""
    p.add_argument('--chunk_size', type=int, default=None,
                   help='run the encoder with self-attention limited to chunks of this many output frames; 0 = full context; '
                        'default: as trained')
    p.add_argument('--left_chunks', type=int, default=None, help='earlier chunks a frame may attend to (-1 = all); default: as trained')


def apply_chunk_args(parser, args, model):
    """sets the model encoder's chunk_size / left_chunks from the flags that were given; parser.error when they are out of range or
    the model's encoder cannot be chunked"""
    if args.chunk_size is None and args.left_chunks is None:
        return
    if (args.chunk_size is not None and args.chunk_size < 0) or (args.left_chunks is not None and args.left_chunks < -1):
        parser.error('--chunk_size must be >= 0 and --left_chunks >= -1')
    if not hasattr(model.encoder, 'chunk_masks'):
        parser.error('--chunk_size / --left_chunks apply to the TDNN-Transformer encoder only')
    if args.chunk_size is not None:
        model.encoder.chunk_size = args.chunk_size
    if args.left_chunks is not None:
        model.encoder.left_chunks = args.left_chunks


def load_cmvn(args, dev):
    """--cmvn_stats -> args.offset / args.scale [D * (lctx + 1 + rctx)] on ``dev`` (decoder/decode_transducer.py:54-71)"""
    if args.cmvn_stats:
        cmvn = read_kaldi_text_matrix(args.cmvn_stats)
        mean = cmvn[0][:-1] / cmvn[0][-1]
        var = cmvn[1][:-1] / cmvn[0][-1] - mean * mean
        if min(abs(var)) < 1.0e-20:
            sys.exit('problematic cmvn_stats, variance too small')
        rep = args.lctx + args.rctx + 1
        args.offset = torch.from_numpy(-mean).to(dev).repeat(rep)
        args.scale = torch.from_numpy(1.0 / np.sqrt(var)).to(dev).repeat(rep)


def read_symbols_map(path):
    """``symbol id`` lines -> {id: symbol} (:103-107)"""
    sym_map = {}
    with open(path, 'r', encoding='utf-8') as f:
        for line in f:
            entry = line.split(" ")
            sym_map[int(entry[1])] = entry[0]
    return sym_map


def prepare_batch(data_batch, len_batch, args, dev):
    """a loader batch -> (features, encoder output lengths): --min_len padding, --cmn / --cmvn_stats, then the model's context and
    stride (:116-134)"""
    len_batch = torch.from_numpy(len_batch).to(dev)
    if int(len_batch.max()) < args.min_len:                                                 # :116-122
        pad = data_batch[:, -1, :].unsqueeze(1).expand(-1, args.min_len - int(len_batch.max()), -1)
        data_batch = torch.cat((data_batch, pad), dim=1)
        len_batch[:] = args.min_len
    if args.cmvn_stats:                                                                     # :123-129
        if args.cmn:
            data_batch = data_batch - data_batch.mean(dim=1, keepdim=True)
        data_batch = (data_batch + args.offset.to(data_batch.dtype)) * args.scale.to(data_batch.dtype)
    len_batch = len_batch - args.model_lctx - args.model_rctx                               # :131-134
    len_batch = len_batch // args.model_stride + torch.ne(len_batch % args.model_stride, 0).int()
    return data_batch, len_batch


def main(argv=None):
    parser = build_parser()
    args, _ = parser.parse_known_args(argv)
    loader_module = importlib.import_module('pika_b200.loader.' + args.loader + '_loader')
    loader_module.register(parser)
    args = parser.parse_args(argv)
    args.input_dim = loader_module.get_inputdim(args)
    if not (args.cuda and torch.cuda.is_available()):
        sys.exit("pika_b200.decoder.decode_transducer: the beam search runs on the GPU only (pass --cuda on a CUDA machine)")
    dev = torch.device("cuda", args.local_rank)
    torch.cuda.set_device(dev)

    model = torch.load(args.model, map_location="cpu", weights_only=False)                # :19-20
    apply_chunk_args(parser, args, model)
    model.eval().to(dev)
    for name in ("las_rescorer", "las_rescorer_bw", "bilas_rescorer"):                      # :22-38
        path = getattr(args, name + "_model")
        net = None
        if path is not None:
            net = torch.load(path, map_location="cpu", weights_only=False)
            net.eval().to(dev)
        setattr(args, name, net)

    load_cmvn(args, dev)

    lm_scorer = None
    if args.fst_lm != '':                                                                   # :82-88
        disambig_ids = [int(i) for i in args.disambig_ids.split(',') if i != '']
        lm_scorer = SortedMatcher(read_fst_text(args.fst_lm), args.max_num_arcs, args.max_id, args.backoff_id, disambig_ids)

    trans_decoder = TransducerDecoder(model, batch_size=args.batch_size, beam_size=args.beam_size, n_best=args.n_best, blk=args.blk,
                                      global_scorer=GlobalScorer(), sm_scale=args.sm_scale, lm=None, lm_scale=args.lm_scale,
                                      lm_scorer=lm_scorer, lm_scorer_scale=args.fst_lm_scale, cuda=True, beam_prune=True, args=args)

    sym_map = read_symbols_map(args.symbols_map)

    with open(args.output_file, 'w') as f:
        for data_batch, _, len_batch, _ in loader_module.dataloader(args.input_labels, args.input_specifier, False, args):
            data_batch, len_batch = prepare_batch(data_batch, len_batch, args, dev)
            ret, enc_out = trans_decoder.decode_batch(data_batch.float(), len_batch, (len_batch + 100).tolist())
            hyps, scores = ret["predictions"], ret["scores"]
            for i in range(args.batch_size):                                                # :136-178
                for j in range(args.n_best):
                    nonblk_hyp = [e.item() for e in hyps[i][j] if e != args.blk]
                    las_scores = las_scores_bw = None
                    tgt = torch.LongTensor([args.SOS] + nonblk_hyp + [args.EOS]).to(dev).unsqueeze(-1).unsqueeze(-1)
                    las_in = enc_out[i].unsqueeze(1)
                    if args.las_rescorer is not None:
                        las_scores = trans_decoder.las_rescore(las_in, tgt)
                    if args.las_rescorer_bw is not None:
                        tgt_bw = torch.LongTensor([args.SOS] + nonblk_hyp[::-1] + [args.EOS]).to(dev).unsqueeze(-1).unsqueeze(-1)
                        las_scores_bw = trans_decoder.las_rescore(las_in, tgt_bw, bw=True)
                    if args.bilas_rescorer is not None:
                        las_scores = trans_decoder.bilas_rescore(las_in, tgt)
                    f.write("".join([sym_map[e] for e in nonblk_hyp]))
                    if args.output_scores:
                        f.write(" {}".format(scores[i][j]))
                        if args.las_rescorer is not None:
                            f.write(' ' + ' '.join(str(s) for s in las_scores))
                        if args.las_rescorer_bw is not None:
                            f.write(' ' + ' '.join(str(s) for s in las_scores_bw))
                        if args.bilas_rescorer is not None:
                            f.write(' ' + ' '.join(str(s) for s in las_scores + las_scores))
                    f.write("\n")
                    f.flush()


if __name__ == '__main__':
    main()
