"""MBR (minimum Bayes risk) transducer training script -- drop-in for trainer/train_transducer_mbr_bmuf_otfaug.py (reference).

Same positional arguments and flags (the parser extends the RNN-T trainer's with ``--beam_size --rnnt_scale --lm --lm_scale
--sm_scale --blk``, reference :262-397), same per-rank log / model file naming, same epoch structure (``run_one_epoch``, :39-258):
per batch, N-best generation with the batched device beam search (``n_best = beam_size``, ``beam_prune=False``), one encoder
forward shared by the RNN-T branch and the path-gathered MBR branch (``pika_b200.trainer.mbr.mbr_forward_backward``),
inf-norm clip + Nesterov SGD, BMUF block sync every ``sync_period`` batches (for EVERY loader item, empty batches included,
so that all ranks enter the collective together), a temporary model dump every 3000 synced batches (:246-250).

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 -m pika_b200.trainer.train_transducer_mbr_bmuf_otfaug \\
        transducer data.WORKER-ID.lst log.WORKER-ID out/ --cuda --init_model rnnt.model ... (flags of egs/train_transducer_mbr_bmuf_otfaug.sh)
"""
import importlib
import os
import sys

import torch

from ..decoder.beam_transducer import GlobalScorer
from ..decoder.transducer_decoder import TransducerDecoder
from ..frontend import Frontend
from ..loader.audio_bank import AudioBank
from ..loader import kaldi_io
from ..utils.logger import Logger
from ..utils.spec_augment import SpecAugment
from .. import engine
from .bmuf import BmufTrainer
from .flat import FlatParams, SgdNesterovClip, lr_at
from .mbr import mbr_forward_backward
from .step import TrainStep, chunk_for_batch, encoder_chunk, encoder_out_lens
from .train_transducer_bmuf_otfaug import apply_chunk_args, build_parser as build_rnnt_parser, check_chunk_args, check_emission_reg_args

MASTER_NODE = 0


def run_one_epoch(epoch, log_f, model, args, bmuf_trainer):
    """one epoch of MBR training (trainer/train_transducer_mbr_bmuf_otfaug.py:39-258)"""
    log_f.write('===> Epoch {} <===\n'.format(epoch))
    total = args.num_epochs * args.num_batches_per_epoch
    lr = lr_at(args.initial_lr, args.final_lr, epoch * args.num_batches_per_epoch, total)
    log_f.write('===> Start Training with learning rate {} <===\n'.format(lr))
    optimizer = SgdNesterovClip(bmuf_trainer.flat, lr, args.momentum, args.grad_clip)
    loss_logger = Logger(args.log, args.log_per_n_frames, ['MBR Loss', 'RNNT Loss'])
    spec = SpecAugment(args.max_freq_span, args.max_time_span) if args.spec_augment else None
    args.las_rescorer, args.las_rescorer_bw, args.bilas_rescorer = None, None, None
    if not hasattr(args, "nonblk_reward"):
        args.nonblk_reward = 0.0
    decoder = TransducerDecoder(model, batch_size=args.batch_size, beam_size=args.beam_size, n_best=args.beam_size, blk=args.blk,
                                global_scorer=GlobalScorer(), sm_scale=args.sm_scale, cuda=args.cuda, beam_prune=False, args=args)
    step = TrainStep(model, args, args.frontend, bmuf_trainer, optimizer, offset=args.offset, scale=args.scale, spec_augmentor=None)
    dev = torch.device("cuda", args.local_rank)
    args.epoch = epoch
    model.train()
    for num_done, (raw, target_cpu, len_cpu, ali_lens_cpu) in enumerate(args.dataloader(args.data_lst, args.rir, args.noise, args)):
        mbr_loss = rnnt_loss = 0.0
        if raw is not None:
            batch = {k: (v.to(dev, non_blocking=True) if torch.is_tensor(v) else v) for k, v in raw.items()}
            target = target_cpu.long().to(dev)
            ali_lens = ali_lens_cpu.to(dev)
            feats = step.features(batch)                                      # CMN / CMVN, no SpecAugment yet (:109-115)
            len_batch = encoder_out_lens(args.frontend.out_lens(batch["n_frames"]), args.model_lctx, args.model_rctx, args.model_stride)
            # one chunk size for the item's N-best generation and its training forward
            with encoder_chunk(model, chunk_for_batch(args, epoch * args.num_batches_per_epoch + step.num_done)):
                model.eval()                                                  # N-best generation (:117-123)
                ret, _ = decoder.decode_batch(feats, len_batch.cpu(), [int(t) + int(u) + 3 for t, u in zip(len_batch.cpu(), ali_lens_cpu)])
                model.train()
                optimizer.flat.zero_grad()
                if spec is not None:                                          # SpecAugment on the training forward only (:134-135)
                    spec.apply(feats)
                mbr, costs = mbr_forward_backward(model, feats, target, len_batch, ali_lens, ret, blk=args.blk, rnnt_scale=args.rnnt_scale,
                                                  sm_scale=args.sm_scale, fastemit_lambda=args.fastemit_lambda,
                                                  delay_penalty=args.delay_penalty)
            optimizer.step()                                                  # clip_grad_norm_(inf) + SGD(nesterov) (:236-240)
            mbr_loss, rnnt_loss = float(mbr), float(costs.sum().item())
        try:                                                                  # (:245-257) for every loader item, data or not
            if step.num_done != 0 and step.num_done % args.sync_period == 0 and step.num_done % 3000 == 0:
                with open('{}/model.{}.tmp'.format(args.output_dir, args.local_rank), 'wb') as tmp_f:
                    torch.save(model, tmp_f)
            step.end_of_item()
        except FloatingPointError:
            return float('nan')
        loss_logger.update_and_log(int(ali_lens_cpu.sum().item()), [mbr_loss, rnnt_loss])
    if bmuf_trainer.update_and_sync() != 1:
        return float('nan')
    tot_loss, tot_num = loss_logger.summarize_and_log()
    loss_tensor = torch.tensor([tot_loss, float(tot_num)], dtype=torch.float32, device=dev)
    bmuf_trainer.sum_reduce(loss_tensor)
    bmuf_trainer.broadcast(loss_tensor)
    return (loss_tensor[0] / loss_tensor[1]).item()


def build_parser():
    parser = build_rnnt_parser()
    parser.description = 'Transducer MBR training'
    parser.add_argument('--beam_size', type=int, default=8, help='beam size to generate nbest')
    parser.add_argument('--rnnt_scale', type=float, default=0.01, help='weight of the RNN-T loss next to the MBR loss')
    parser.add_argument('--lm', type=str, default='', help='LM for shallow fusion during N-best generation (not supported: FST fusion is --lm_scorer of the decoder)')
    parser.add_argument('--lm_scale', type=float, default=0.1)
    parser.add_argument('--sm_scale', type=float, default=1.0, help='softmax smoothing of the N-best generation and of the MBR branch')
    parser.add_argument('--blk', type=int, default=0)
    # defaults the reference's MBR script sets differently from its RNN-T script (trainer/train_transducer_mbr_bmuf_otfaug.py:340-420)
    parser.set_defaults(num_epochs=3, num_batches_per_epoch=100000, sync_period=5)
    return parser


def main(argv=None):
    parser = build_parser()
    args, _ = parser.parse_known_args(argv)
    loader_module = importlib.import_module('pika_b200.loader.' + args.loader + '_loader')
    loader_module.register(parser)
    args = parser.parse_args(argv)
    if args.block_sync != 'bmuf':        # inherited from the RNN-T parser; the MBR trainer runs BmufTrainer only, as the reference's
        parser.error('--block_sync %s: the MBR trainer supports only bmuf' % args.block_sync)
    if args.lm_only_scale != 0.0 or args.am_only_scale != 0.0:    # inherited from the RNN-T parser; there is no simple loss here
        parser.error('--lm_only_scale / --am_only_scale: the MBR trainer has no simple loss to smooth')
    check_emission_reg_args(parser, args)        # inherited: applied to the RNN-T branch, not to the MBR loss
    check_chunk_args(parser, args)               # inherited: the encoder of the N-best generation and of both branches
    if args.lm:
        raise NotImplementedError("pika_b200: --lm (neural LM fusion) is outside the hot path")
    args.input_dim = loader_module.get_inputdim(args)
    args.dataloader = loader_module.dataloader
    args.raw_batches = True
    world_size = int(os.environ.get('WORLD_SIZE', '1'))
    if args.local_rank is None:
        args.local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    assert args.cuda and torch.cuda.is_available(), "pika_b200 trains on the GPU (there is no CPU fallback)"
    torch.cuda.set_device(args.local_rank)
    dev = torch.device("cuda", args.local_rank)
    # on-the-fly reverberation and noise (trainer/train_transducer_bmuf_otfaug.py:272-282): banks read once, uploaded once
    args.rir = AudioBank.rir(args.rir_lst) if args.rir_lst else []
    args.noise = AudioBank.noise(args.noise_lst, args.max_len) if args.noise_lst else []
    args.data_lst = args.data_lst.replace('WORKER-ID', str(args.local_rank))
    args.log = args.log.replace('WORKER-ID', str(args.local_rank))
    log_f = open(args.log, 'w')
    args.log = log_f
    engine.set_precision(args.precision)
    engine.set_seed(args.seed + args.local_rank)
    nnet_module = importlib.import_module("pika_b200.model." + args.nnet_proto)
    torch.manual_seed(args.seed)
    if args.init_model is None:
        model = nnet_module.Net(args, args.input_dim, args.output_dim)
    else:
        model = torch.load(args.init_model, map_location=lambda storage, loc: storage, weights_only=False)
    apply_chunk_args(model, args)
    model.to(dev)
    flat = FlatParams(model)
    bmuf_trainer = BmufTrainer(MASTER_NODE, args.local_rank, world_size, model, args.block_momentum, args.block_lr, flat=flat)
    opts = loader_module.feature_options(args)
    args.frontend = Frontend(opts, args.lctx, args.rctx, dev, stride=args.stride)
    args.frontend.noise = args.noise or None
    args.frontend.rir = args.rir or None
    args.offset = args.scale = None
    if args.cmvn_stats:
        try:
            off, sc = kaldi_io.cmvn_offset_scale(args.cmvn_stats, args.lctx + args.rctx + 1)
        except ValueError as e:
            print(str(e))
            sys.exit()
        args.offset = torch.from_numpy(off).float().to(dev)
        args.scale = torch.from_numpy(sc).float().to(dev)
    for epoch in range(0, args.num_epochs):
        run_one_epoch(epoch, log_f, model, args, bmuf_trainer)
        with open('{}/model.epoch.{}.{}'.format(args.output_dir, epoch, args.local_rank), 'wb') as f:
            torch.save(model, f)
    log_f.write('Training Finished')
    log_f.flush()


if __name__ == '__main__':
    main()
