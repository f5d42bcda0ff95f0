"""Transducer training script -- drop-in for trainer/train_transducer_bmuf_otfaug.py (reference).

Same positional arguments and flags (argparse below mirrors :148-253 + the loader's ``register``), same
per-rank log / model file naming, same epoch structure (``run_one_epoch``: :32-145).  Launch exactly like the
reference recipe (one process per GPU, ``WORLD_SIZE`` / ``--local_rank`` from the launcher):

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 -m pika_b200.trainer.train_transducer_bmuf_otfaug \\
        transducer data.WORKER-ID.lst log.WORKER-ID out/ --cuda --encoder_type transformer ... (flags of egs/train_transducer_bmuf_otfaug.sh)

What runs underneath: raw-PCM loader threads -> GPU front end -> sm_90a model / loss / optimiser kernels -> BMUF over NCCL.
"""
import argparse
import importlib
import math
import os
import sys

import torch

from ..frontend import Frontend
from ..loader.audio_bank import AudioBank
from ..loader import kaldi_io
from ..utils.logger import Logger
from ..utils.spec_augment import SpecAugment
from .. import engine
from .bmuf import BlockAdamTrainer, BmufAdamTrainer, BmufTrainer
from .flat import AdamClip, FlatParams, SgdNesterovClip, lr_at
from .step import TrainStep

MASTER_NODE = 0


def run_one_epoch(epoch, model, log_f, args, bmuf_trainer, training):
    """one epoch of training (trainer/train_transducer_bmuf_otfaug.py:32-145)"""
    log_f.write('===> Epoch {} <===\n'.format(epoch))
    total_num_batches = args.num_epochs * args.num_batches_per_epoch
    lr = lr_at(args.initial_lr, args.final_lr, epoch * args.num_batches_per_epoch, total_num_batches)
    log_f.write('===Using Learning Rate {}===\n'.format(lr))
    args.epoch = epoch
    if args.block_sync == 'bmuf_adam':
        optimizer = bmuf_trainer.optim                        # one local Adam for the whole run: moments and step persist
        optimizer.reset(lr)
    else:
        optimizer = SgdNesterovClip(bmuf_trainer.flat, lr, args.momentum, args.grad_clip)
    pruned = getattr(args, 'prune_range', 0) > 0
    loss_logger = Logger(args.log, args.log_per_n_frames, ['Loss', 'Simple'] if pruned else ['Loss'])
    spec = SpecAugment(args.max_freq_span, args.max_time_span) if args.spec_augment else None
    model.train(training)
    step = TrainStep(model, args, args.frontend, bmuf_trainer, optimizer, offset=args.offset, scale=args.scale, spec_augmentor=spec)
    dev = torch.device("cuda", args.local_rank)
    for num_done, (raw, target_cpu, len_cpu, ali_lens_cpu) in enumerate(args.dataloader(args.data_lst, args.rir, args.noise, args)):
        if raw is not None:
            batch = {k: (v.to(dev, non_blocking=True) if torch.is_tensor(v) else v) for k, v in raw.items()}
            batch["target"] = target_cpu.long().to(dev)
            batch["ali_lens"] = ali_lens_cpu.to(dev)
            if training:
                try:
                    costs = step(batch)
                except FloatingPointError:
                    return float('nan')                       # BMUF returned STOP (:113-114)
                simple = step.simple_costs
            else:
                with torch.no_grad():
                    feats = step.features(batch)
                    from .step import emission_reg, encoder_out_lens, encoder_out_max, smoothing_scales
                    tl = encoder_out_lens(args.frontend.out_lens(batch["n_frames"]), args.model_lctx, args.model_rctx, args.model_stride)
                    t_out = encoder_out_max(int(batch["t_max"]), args.model_lctx, args.model_rctx, args.model_stride)
                    if pruned:
                        simple, costs = engine.transducer_loss_pruned(model, feats, batch["target"], tl, batch["ali_lens"],
                                                                      args.prune_range, args.simple_loss_scale, 1.0, x_len=tl, t_out=t_out,
                                                                      **smoothing_scales(args), **emission_reg(args))
                    else:
                        costs = engine.transducer_loss(model, feats, batch["target"], tl, batch["ali_lens"], x_len=tl, t_out=t_out,
                                                       **emission_reg(args))
            loss = float(costs.sum().item())
            simple_loss = float(simple.sum().item()) if pruned else 0.0
        else:                                                 # empty batch (:100-101)
            loss = simple_loss = 0.0
            if training:
                try:
                    step.skip()                               # still counts, still syncs (:112-123)
                except FloatingPointError:
                    return float('nan')
        labels = int(ali_lens_cpu.sum().item())
        loss_logger.update_and_log(labels, [loss, simple_loss] if pruned else [loss])
    if training and bmuf_trainer.update_and_sync() != 1:
        return float('nan')
    tot_loss, tot_num = loss_logger.summarize_and_log()
    loss_tensor = torch.tensor([tot_loss, float(tot_num)], dtype=torch.float32, device=dev)
    bmuf_trainer.sum_reduce(loss_tensor)                      # aggregate across workers (:140-145)
    bmuf_trainer.broadcast(loss_tensor)
    return (loss_tensor[0] / loss_tensor[1]).item()


def build_parser():
    parser = argparse.ArgumentParser(description='Transducer training')
    parser.add_argument('nnet_proto', type=str, help='pytorch NN proto definition filename')
    parser.add_argument('data_lst', type=str, help='list of mrk, seq, ali files for data')
    parser.add_argument('log', type=str, help='log file for the job')
    parser.add_argument('output_dir', type=str, help='path to save the final model')
    parser.add_argument('--init_model', type=str, default=None, help='initial model')
    parser.add_argument('--rir_lst', type=str, default=None, help='mrk and seq files for rir')
    parser.add_argument('--noise_lst', type=str, default=None, help='mrk and seq files for noise')
    parser.add_argument('--encoder_type', type=str, default='rnn', choices=['rnn', 'transformer'])
    parser.add_argument('--decoder_type', type=str, default='rnn', choices=['rnn', 'transformer'])
    parser.add_argument('--layers', type=int, default=-1)
    parser.add_argument('--enc_layers', type=int, default=2)
    parser.add_argument('--dec_layers', type=int, default=2)
    parser.add_argument('--max_relative_positions', type=int, default=0,
                        help='relative-position self-attention in the transformer prediction net (--decoder_type transformer): clip '
                             'distances to +-N, one table of 2N+1 rows per layer; 0 = off, the reference recipe')
    parser.add_argument('--rnn_size', type=int, default=512)
    parser.add_argument('--rnn_type', type=str, default='LSTM', choices=['LSTM'])
    parser.add_argument('--embd_dim', type=int, default=300)
    parser.add_argument('--output_dim', type=int, default=8000)
    parser.add_argument('--model_lctx', type=int, default=0)
    parser.add_argument('--model_rctx', type=int, default=0)
    parser.add_argument('--model_stride', type=int, default=1)
    parser.add_argument('--brnn', action="store_true")
    parser.add_argument('--cmn', action="store_true")
    parser.add_argument('--cmvn_stats', type=str, default=None)
    parser.add_argument('--optim', type=str, default='sgd', choices=['sgd', 'adam', 'adadelta'])
    parser.add_argument('--grad_clip', type=float, default=-1.0)
    parser.add_argument('--initial_lr', type=float, default=1.0)
    parser.add_argument('--final_lr', type=float, default=1.0)
    parser.add_argument('--momentum', type=float, default=0.9)
    parser.add_argument('--num_epochs', type=int, default=15)
    parser.add_argument('--num_batches_per_epoch', type=int, default=1000)
    parser.add_argument('--dropout', type=float, default=0.3)
    parser.add_argument('--padding_idx', type=int, default=-1)
    parser.add_argument('--loader', choices=['otf_utt'], default='otf_utt')
    parser.add_argument('--log_per_n_frames', type=int, default=1024 * 1024)
    parser.add_argument('--seed', type=int, default=777)
    parser.add_argument('--cuda', action='store_true')
    parser.add_argument('--local_rank', type=int, default=None)
    parser.add_argument('--block_momentum', type=float, default=0.9)
    parser.add_argument('--block_lr', type=float, default=1.0)
    parser.add_argument('--sync_period', type=int, default=100)
    parser.add_argument('--block_sync', choices=['bmuf', 'bmuf_adam', 'block_adam'], default='bmuf',
                        help='block trainer of trainer/bmuf.py: bmuf = BmufTrainer (Nesterov block momentum, local SGD; the '
                             'reference recipe); bmuf_adam = BmufAdamTrainer (local Adam at the scheduled learning rate, moments '
                             'averaged and filtered at every sync); block_adam = BlockAdamTrainer (local SGD, the summed block '
                             'delta applied by Adam at --block_lr)')
    parser.add_argument('--spec_augment', action='store_true')
    parser.add_argument('--max_freq_span', type=int, default=15)
    parser.add_argument('--max_time_span', type=int, default=35)
    parser.add_argument('--precision', choices=['bf16', 'fp32'], default='bf16', help='pika_b200: compute mode')
    parser.add_argument('--prune_range', type=int, default=0,
                        help='pruned RNN-T loss: train the joint over this many label positions per frame, chosen by a simple joiner '
                             '(DESIGN.md "Pruned RNN-T"); 0 = the full joint (default), otherwise >= 2.  The logged Loss is then the '
                             'pruned cost and Simple the simple joiner\'s')
    parser.add_argument('--simple_loss_scale', type=float, default=0.5,
                        help='weight of the simple joiner\'s loss in the pruned objective (the pruned loss has weight 1)')
    parser.add_argument('--prune_warmup_batches', type=int, default=0,
                        help='ramp the pruned loss weight from 0.1 to 1 and the simple loss weight from 1 to --simple_loss_scale '
                             'linearly over this many batches; 0 = off')
    parser.add_argument('--lm_only_scale', type=float, default=0.0,
                        help='pruned RNN-T (needs --prune_range): weight of the LM-only log-probs mixed into the simple joiner\'s lattice '
                             '(DESIGN.md "Pruned RNN-T"); >= 0, and with --am_only_scale < 1; not ramped by --prune_warmup_batches')
    parser.add_argument('--am_only_scale', type=float, default=0.0,
                        help='pruned RNN-T (needs --prune_range): weight of the AM-only log-probs (against the batch\'s label unigram) '
                             'mixed into the simple joiner\'s lattice; >= 0, and with --lm_only_scale < 1')
    parser.add_argument('--fastemit_lambda', type=float, default=0.0,
                        help='FastEmit (DESIGN.md "FastEmit and delay penalty"): scale the gradient of every label arc of the RNN-T '
                             'loss (the pruned loss with --prune_range) by 1 + this; the logged loss is unchanged.  >= 0, 0 = off')
    parser.add_argument('--delay_penalty', type=float, default=0.0,
                        help='delay penalty: add this x ((T-1)/2 - t) to the log-prob of every label arc emitted on frame t, in the '
                             'RNN-T loss and (with --prune_range) the simple loss too; the logged losses are the penalised ones.  '
                             '>= 0, 0 = off; not ramped by --prune_warmup_batches')
    parser.add_argument('--chunk_size', type=int, default=0,
                        help='streaming TDNN-Transformer encoder (DESIGN.md "Chunked attention"): self-attention limited to chunks of this '
                             'many encoder output frames and earlier ones; 0 = full context')
    parser.add_argument('--left_chunks', type=int, default=-1,
                        help='with --chunk_size / --dynamic_chunk_max: how many earlier chunks a frame may attend to; -1 = all')
    parser.add_argument('--dynamic_chunk_max', type=int, default=0,
                        help='per batch, full context with probability 1/2, otherwise a chunk size drawn uniformly from [1, this]; '
                             '0 = off.  Checkpoints record chunk size 0')
    return parser


def check_chunk_args(parser, args):
    """parser.error unless --chunk_size / --left_chunks / --dynamic_chunk_max are in range, consistent, and on the TDNN-Transformer"""
    C, left, M = args.chunk_size, args.left_chunks, args.dynamic_chunk_max
    if C < 0 or M < 0 or left < -1:
        parser.error('--chunk_size and --dynamic_chunk_max must be >= 0 and --left_chunks >= -1 (got %d, %d, %d)' % (C, M, left))
    if C > 0 and M > 0:
        parser.error('--chunk_size and --dynamic_chunk_max exclude each other')
    if left != -1 and C == 0 and M == 0:
        parser.error('--left_chunks needs --chunk_size or --dynamic_chunk_max')
    if args.encoder_type == 'rnn' and (C or M or left != -1):
        parser.error('--chunk_size / --left_chunks / --dynamic_chunk_max apply to the TDNN-Transformer encoder (--encoder_type transformer)')


def apply_chunk_args(model, args):
    """the encoder's static chunk setting from the flags (also for an --init_model)"""
    if hasattr(model.encoder, 'chunk_masks'):
        model.encoder.chunk_size, model.encoder.left_chunks = args.chunk_size, args.left_chunks


def check_smoothing_args(parser, args):
    """parser.error unless --lm_only_scale / --am_only_scale are both 0, or in range with --prune_range > 0"""
    lam_l, lam_a = args.lm_only_scale, args.am_only_scale
    if lam_l == 0.0 and lam_a == 0.0:
        return
    if args.prune_range <= 0:
        parser.error('--lm_only_scale / --am_only_scale smooth the simple loss of the pruned RNN-T loss: they need --prune_range > 0')
    if not (lam_l >= 0.0 and lam_a >= 0.0 and lam_l + lam_a < 1.0):
        parser.error('--lm_only_scale and --am_only_scale must be >= 0 with a sum < 1 (got %r, %r)' % (lam_l, lam_a))


def check_emission_reg_args(parser, args):
    """parser.error unless --fastemit_lambda and --delay_penalty are finite and >= 0"""
    for name in ('fastemit_lambda', 'delay_penalty'):
        v = getattr(args, name)
        if not (math.isfinite(v) and v >= 0.0):
            parser.error('--%s must be finite and >= 0 (got %r)' % (name, v))


def main(argv=None):
    parser = build_parser()
    args, _ = parser.parse_known_args(argv)
    loader_module = importlib.import_module('pika_b200.loader.' + args.loader + '_loader')
    loader_module.register(parser)
    args = parser.parse_args(argv)
    check_smoothing_args(parser, args)
    check_emission_reg_args(parser, args)
    check_chunk_args(parser, args)
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
        if args.prune_range > 0 and not hasattr(model, 'simple_am_proj'):
            from ..model.transducer import add_simple_joiner
            add_simple_joiner(model, model.fc2.weight.shape[1], model.fc2.weight.shape[0])   # drawn after the seed above
    if args.prune_range == 1 or args.prune_range < 0:
        parser.error('--prune_range must be 0 (off) or >= 2')
    apply_chunk_args(model, args)
    model.to(dev)
    flat = FlatParams(model)
    if args.block_sync == 'bmuf_adam':
        lr0 = lr_at(args.initial_lr, args.final_lr, 0, args.num_epochs * args.num_batches_per_epoch)
        bmuf_trainer = BmufAdamTrainer(MASTER_NODE, args.local_rank, world_size, model, args.block_momentum, args.block_lr,
                                       args.sync_period, AdamClip(flat, lr0, max_norm=args.grad_clip), flat=flat)
    elif args.block_sync == 'block_adam':
        bmuf_trainer = BlockAdamTrainer(MASTER_NODE, args.local_rank, world_size, model, args.block_lr, flat=flat)
    else:
        bmuf_trainer = BmufTrainer(MASTER_NODE, args.local_rank, world_size, model, args.block_momentum, args.block_lr, flat=flat)
    num_param = sum(p.numel() for p in model.parameters())
    log_f.write('*' * 60 + '\n')
    log_f.write('model proto: {}\ninput  dim: {},\toutput dim: {},\nhidden dim: {},\tnum of enc_layers: {}\n'
                'num of dec_layers: {},\trnn_type: {}\nmodel size: {} M\n'.format(args.nnet_proto, args.input_dim, args.output_dim,
                                                                                args.rnn_size, args.enc_layers, args.dec_layers,
                                                                                args.rnn_type, num_param / 1000 / 1000))
    log_f.write('*' * 60 + '\n')
    log_f.flush()
    opts = loader_module.feature_options(args)
    # opts.dither is honoured (egs/fbank.conf: dither=1): counter-based Gaussian dither in the fbank kernel; set dither=0 in the
    # feature config for bit-reproducible features (Kaldi's own RNG stream is not reproduced, DESIGN.md)
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
        run_one_epoch(epoch, model, log_f, args, bmuf_trainer, True)
        current_model = '{}/model.epoch.{}.{}'.format(args.output_dir, epoch, args.local_rank)
        with open(current_model, 'wb') as f:
            torch.save(model, f)
    log_f.write('Training Finished')
    log_f.flush()


if __name__ == '__main__':
    main()
