"""Offline (Kaldi feature archive) utterance loader -- drop-in for loader/utt_loader.py (reference), the loader the decode CLI uses
(decoder/decode_transducer.py:244 ``--loader utt``).  Same ``register`` flags, ``get_inputdim`` and ``dataloader(align_rspec,
feats_rspec, dummy, args)`` iterator of ``(data f32 [B,Tmax,D], target i64 [B,Umax], lens i32 [B], ali_lens i32 [B])``; the archives
are read by the native readers of kaldi_io.py instead of PyKaldi.  Like the reference, a trailing incomplete batch is dropped
(loader/utt_loader.py:189-228 only emits full batches) unless the caller passes ``keep_tail`` (the aligner, which must see every
utterance), and data is padded by repeating each utterance's last frame."""
import queue
from threading import Thread

import numpy as np
import torch

from .kaldi_io import read_float_matrix_table, read_int_vector_ark
from .otf_utt_loader import get_inputdim, put_thread  # noqa: F401  (same definitions as the reference's re-exports, :12)


def register(parser):
    """loader/utt_loader.py:16-43"""
    parser.add_argument('--lctx', type=int, default=10, help='left context for splice')
    parser.add_argument('--rctx', type=int, default=10, help='right context for splice')
    parser.add_argument('--max_len', type=int, default=6000, help='max length allowed to be loaded')
    parser.add_argument('--buffer_size', type=int, default=128 * 1024, help='buffer size used to shuffle data')
    parser.add_argument('--ctc_target', action='store_true', help='whether the reader is used for CTC training or not')
    parser.add_argument('--batch_first', action='store_true', help='whether 1st dim of tensor if batch or frame')
    parser.add_argument('--stride', type=int, default=1, help='strides for subsampling input (after splicing)')
    parser.add_argument('--batch_size', type=int, default=1024, help='batch size')
    parser.add_argument('--queue_size', type=int, default=8, help='queue size for threading')
    parser.add_argument('--padding_tgt', type=int, default=-1, help='padding index for targets')
    parser.add_argument('--feats_dim', type=int, default=40, help='dimension of input feature (before splicing)')
    parser.add_argument('--verbose', action='store_true', help='printing out warnings')


def splice(feats, lctx, rctx):
    """loader/otf_utt_loader.py:28-46: frame t -> frames t-lctx .. t+rctx side by side, edges repeat the first / last frame"""
    n, d = feats.shape
    idx = np.clip(np.arange(n)[:, None] + np.arange(-lctx, rctx + 1)[None, :], 0, n - 1)
    return feats[idx].reshape(n, d * (lctx + 1 + rctx)).astype(np.float32)


def utt_generator(align_rspec, feats_rspec, shuffle, args, keep_tail=False, with_ids=False):
    """loader/utt_loader.py:154-232.  ``keep_tail``: also yield the trailing incomplete batch (its first dimension is then the number of
    utterances left) instead of dropping it.  ``with_ids``: append the batch's list of utterance ids to each item."""
    if getattr(args, "ctc_target", False):
        raise NotImplementedError("pika_b200: the CTC target layout of loader/utt_loader.py:71-150 is not used by the transducer path")
    B, D = args.batch_size, get_inputdim(args)
    data_buffer = np.zeros((B, args.max_len, D), dtype=np.float32)
    target_buffer = np.zeros((B, args.max_len), dtype=np.int32)
    len_buffer, ali_len = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
    bi, tmax, umax = 0, -1, -1
    ids = []

    def emit(n_b):
        for b in range(n_b):                                   # pad data with the last valid frame, labels with padding_tgt (:193-199)
            data_buffer[b, len_buffer[b]:tmax, :] = data_buffer[b, len_buffer[b] - 1, :]
            target_buffer[b, ali_len[b]:umax] = args.padding_tgt
        data, target = data_buffer[:n_b, :tmax, :], target_buffer[:n_b, :umax]
        if not args.batch_first:
            data, target = np.transpose(data, (1, 0, 2)), np.transpose(target, (1, 0))
        data, target = torch.from_numpy(np.copy(data)), torch.from_numpy(np.copy(target)).long()
        if args.cuda:
            data, target = data.cuda(args.local_rank), target.cuda(args.local_rank)
        item = (data, target, np.copy(len_buffer[:n_b]), np.copy(ali_len[:n_b]))
        return item + (list(ids),) if with_ids else item

    for (uttid, ali), (uttid2, feats) in zip(read_int_vector_ark(align_rspec), read_float_matrix_table(feats_rspec)):
        assert uttid2 == uttid, "feature and label tables must list the same utterances in the same order (%s vs %s)" % (uttid2, uttid)
        ali = np.asarray(ali)
        n = feats.shape[0] // args.stride + int(feats.shape[0] % args.stride != 0)
        ali_len[bi] = ali.shape[0]
        data_buffer[bi, :n, :] = splice(feats, args.lctx, args.rctx)[::args.stride]
        target_buffer[bi, :ali_len[bi]] = ali
        len_buffer[bi] = n
        tmax, umax = max(tmax, n), max(umax, int(ali_len[bi]))
        ids.append(uttid)
        bi += 1
        if bi == B:
            yield emit(B)
            bi, tmax, umax = 0, -1, -1
            ids = []
    if keep_tail and bi > 0:
        yield emit(bi)
    yield None


def dataloader(align_rspec, feats_rspec, dummy_args, args, keep_tail=False, with_ids=False):
    """loader/utt_loader.py:45-68: a reader thread fills a bounded queue; iteration ends at the generator's ``None``.  ``keep_tail`` /
    ``with_ids`` as in utt_generator"""
    q = queue.Queue(args.queue_size)
    thread = Thread(target=put_thread, args=(q, utt_generator, align_rspec, feats_rspec, False, args, keep_tail, with_ids))
    thread.daemon = True
    thread.start()
    while True:
        item = q.get()
        q.task_done()
        if item is None:
            break
        yield item
    thread.join()
