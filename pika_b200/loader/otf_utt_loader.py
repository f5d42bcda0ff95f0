"""On-the-fly utterance loader -- drop-in for loader/otf_utt_loader.py (reference).

Module-level plugin API kept: ``register(parser)``, ``get_inputdim(args)``, ``dataloader(data_lst, rir, noise, args)``.
What moved: the per-utterance CPU work of the reference's producer threads (AudioSegment speed/gain
augmentation, PyKaldi fbank, splice; loader/otf_utt_loader.py:218-250) now runs on the GPU inside
``pika_b200.frontend.Frontend``.  The producer threads here only read raw int16 PCM from the ``.seq`` shards,
draw the augmentation parameters from the SAME random streams in the SAME order as the reference
(``random.randint`` for the speed rate, ``numpy.random.uniform`` for the gain target, :221-223), apply the TU
filter (:247) from the frame count the front end will produce, and assemble padded batches.

With a noise bank (``--noise_lst``) and / or an RIR bank (``--rir_lst``) each utterance also draws, in the order of the
reference's commented-out example (:224-228): ``scipy.stats.truncnorm.rvs`` for the SNR (numpy's global stream), then
``random.randint`` for the noise segment and for the noise offset, then ``random.randint`` for the RIR.  One documented
deviation: the reference's ``add_noise`` draws a float start time from a fresh, unseeded ``random.Random()``; here the offset
is an integer sample index from the module's ``random`` stream.

``dataloader`` yields, like the reference (:272-289), 4-tuples ``(data, target, lens, ali_lens)``; ``data`` is
either the reference's float feature tensor [B,Tmax,D] (``args.raw_batches`` false: features computed on the GPU
and returned as a CPU tensor) or, for the fused trainer path, a dict of raw-PCM tensors for ``TrainStep``.
End of stream = one ``None`` per worker, as in the reference.
"""
import queue
from random import randint
from threading import Thread

import numpy as np
import torch

from ..frontend import FbankOptions, Frontend, MfccOptions, noise_rir_kwargs
from . import kaldi_io


def get_inputdim(args):
    """full input dimension after splicing"""
    return args.feats_dim * (args.lctx + 1 + args.rctx)


def register(parser):
    """loader flags (same names, defaults and help strings as the reference)"""
    parser.add_argument('--lctx', type=int, default=10, help='left context for splice')
    parser.add_argument('--rctx', type=int, default=10, help='right context for splice')
    parser.add_argument('--max_len', type=int, default=6000, help='max length allowed to be loaded')
    parser.add_argument('--num_workers', type=int, default=5, help='number of workers to load/process')
    parser.add_argument('--sample_rate', type=int, default=16000, help='sample rate of waves')
    parser.add_argument('--buffer_size', type=int, default=128 * 1024, help='buffer size used to shuffle data')
    parser.add_argument('--batch_first', action='store_true', help='1st dim is batch or frame')
    parser.add_argument('--reverse_labels', action='store_true', help='reverse labels for training, eg for LAS')
    parser.add_argument('--feat_config', type=str, default=None, help='feature extraction config file')
    parser.add_argument('--feat_type', type=str, default='fbank', choices=('fbank', 'mfcc'),
                        help='Kaldi feature type that --feat_config describes (pika_b200 extension)')
    parser.add_argument('--stride', type=int, default=1, help='strides for subsampling input')
    parser.add_argument('--batch_size', type=int, default=1024, help='batch size')
    parser.add_argument('--SOS', type=int, default=-1, help='start of seq id, valid when beyond 0')
    parser.add_argument('--EOS', type=int, default=-1, help='end of seq id, valid when beyond 0')
    parser.add_argument('--queue_size', type=int, default=8, help='queue size for threading')
    parser.add_argument('--TU_limit', type=int, default=15000,
                        help='limits on the product of T (utt length) and U (label length) to avoid GPU OOM')
    parser.add_argument('--padding_tgt', type=int, default=-1, help='padding index for targets')
    parser.add_argument('--feats_dim', type=int, default=40, help='dimension of input feature (before splicing)')
    parser.add_argument('--snr_range', type=str, default='', help='comma separated SNR range in dB')
    parser.add_argument('--gain_range', type=str, default='55,10', help='comma separated negative gain range in dB')
    parser.add_argument('--speed_rate', type=str, default='0.9,1.0,1.1', help='comma separated rate for speed perturbation')
    parser.add_argument('--verbose', action='store_true', help='printing out warnings')


def snr_params(snr_range):
    """``--snr_range lo,hi`` -> (mu, sigma) of the truncated normal on [lo, hi]; empty = the reference example's 0,20 dB
    (mu 10, sigma 10, loader/otf_utt_loader.py:191-193)"""
    if not snr_range:
        lo, hi = 0.0, 20.0
    else:
        p = [float(v) for v in snr_range.split(',')]
        if len(p) != 2 or not p[1] > p[0]:
            raise ValueError("--snr_range expects 'lo,hi' with hi > lo, got %r" % snr_range)
        lo, hi = p
    return (lo + hi) / 2.0, (hi - lo) / 2.0


def draw_noise_rir(new_len, noise, rir, snr_mu_sigma):
    """the per-utterance noise / reverberation draws, after the speed and gain draws: (snr, k, off, r); None where a bank is absent.
    ``off`` is clamped at 0 for an utterance longer than the noise segment (it cannot pass the --max_len filter: the bank keeps
    only segments that cover every utterance that can)."""
    snr = k = off = r = None
    if noise:
        from scipy.stats import truncnorm
        mu, sigma = snr_mu_sigma
        snr = float(truncnorm.rvs(-1.0, 1.0, loc=mu, scale=sigma))
        k = randint(0, len(noise) - 1)
        off = randint(0, max(0, int(noise.lengths[k]) - new_len))
    if rir:
        r = randint(0, len(rir) - 1)
    return snr, k, off, r


def put_thread(q, generator, *gen_args):
    for item in generator(*gen_args):
        q.put(item)
        if item is None:
            break


def feature_options(args):
    """the feature options of ``--feat_config``, read as ``--feat_type``'s Kaldi options (FbankOptions or MfccOptions; the reference
    switches between the two by editing loader/otf_utt_loader.py:196-202).  Without a config: Kaldi's defaults with ``--feats_dim``
    mel bins (fbank) or cepstra (MFCC).  An MFCC config must have ``--feats_dim`` cepstra.  ``--sample_rate`` must be the config's
    sample frequency, as Kaldi's ComputeFeatures requires of the waveform's rate"""
    if getattr(args, "feat_type", "fbank") == "mfcc":
        opts = MfccOptions.from_config(args.feat_config) if args.feat_config else MfccOptions(num_ceps=args.feats_dim)
        if opts.num_ceps != args.feats_dim:
            raise ValueError("--feats_dim %d differs from the MFCC config's --num-ceps=%d" % (args.feats_dim, opts.num_ceps))
    else:
        opts = FbankOptions.from_config(args.feat_config) if args.feat_config else FbankOptions(num_mel_bins=args.feats_dim)
    if float(args.sample_rate) != opts.sample_frequency:
        raise ValueError("--sample_rate %s differs from the feature config's --sample-frequency=%g" % (args.sample_rate, opts.sample_frequency))
    return opts


def otf_utt_generator(data_triplets, rir, noise, args):
    """raw-PCM batches for one worker; mirrors the control flow of loader/otf_utt_loader.py:165-299"""
    geometry = feature_options(args).geometry()
    stride = args.stride
    batch_size = args.batch_size
    speed_rate = [float(r) for r in args.speed_rate.split(',')]
    gain_lo, gain_hi = [-float(g) for g in args.gain_range.split(',')]
    snr_mu_sigma = snr_params(args.snr_range) if noise else None
    pcm, tgt, meta = [], [], []
    batch_idx = 0
    for mrk_fn, seq_fn, ali_rspec in data_triplets:
        ali_reader = kaldi_io.read_int_vector_ark(ali_rspec)
        for (uttid, audio_np), (uttid1, ali) in zip(kaldi_io.iter_mrk_seq(mrk_fn, seq_fn), ali_reader):
            assert uttid == uttid1
            spr = speed_rate[randint(0, len(speed_rate) - 1)]
            target_db = np.random.uniform(gain_lo, gain_hi)
            new_len, frames = Frontend.lengths([audio_np.shape[0]], [spr], **geometry)
            draws = draw_noise_rir(new_len[0], noise, rir, snr_mu_sigma)
            ali = np.array(ali)
            if args.reverse_labels:
                ali = ali[::-1]
            if args.SOS >= 0:
                ali = np.concatenate(([args.SOS], ali))
            if args.EOS >= 0:
                ali = np.concatenate((ali, [args.EOS]))
            utt_len = frames[0] // stride + int(frames[0] % stride != 0)           # rows after the stride (:243-247)
            if utt_len > 0 and utt_len <= args.max_len and ali.shape[0] * utt_len // 3 <= args.TU_limit:
                pcm.append(audio_np)
                tgt.append(ali.astype(np.int32))
                meta.append((audio_np.shape[0], spr, target_db, new_len[0], frames[0], utt_len) + draws)
            batch_idx += 1
            if batch_idx == batch_size:
                yield assemble(pcm, tgt, meta, args, rir)
                pcm, tgt, meta, batch_idx = [], [], [], 0
    yield None


def assemble(pcm, tgt, meta, args, rir=None):
    """padded raw batch (or the reference's empty-batch tuple, loader/otf_utt_loader.py:283-287).  meta rows:
    (n_samples, rate, target_db, new_len, n_frames, utt_len[, snr, noise_idx, noise_off, rir_idx]) with n_frames the fbank frames and
    utt_len the rows after the stride; t_max and lens count rows.  The noise keys (noise_idx, noise_off, snr) and the RIR keys
    (rir_idx, and the host-side rir_max_len) are added only when those draws were made."""
    if not pcm:
        return None, None, torch.IntTensor([0]), torch.IntTensor([0])
    B = len(pcm)
    n_max = max(max(m[0] for m in meta), max(m[3] for m in meta))
    u_max = max(len(t) for t in tgt)
    pin = torch.cuda.is_available()          # page-locked staging: the trainer's non_blocking H2D copy overlaps the previous step
    pcm_t = torch.zeros(B, n_max, dtype=torch.int16, pin_memory=pin)
    target = torch.full((B, u_max), args.padding_tgt, dtype=torch.int32, pin_memory=pin)
    for i in range(B):
        pcm_t[i, :meta[i][0]] = torch.from_numpy(pcm[i].copy())
        target[i, :len(tgt[i])] = torch.from_numpy(tgt[i])
    raw = dict(pcm=pcm_t,
               n_samples=torch.tensor([m[0] for m in meta], dtype=torch.int32),
               rate=torch.tensor([m[1] for m in meta], dtype=torch.float32),
               target_db=torch.tensor([m[2] for m in meta], dtype=torch.float32),
               new_len=torch.tensor([m[3] for m in meta], dtype=torch.int32),
               n_frames=torch.tensor([m[4] for m in meta], dtype=torch.int32),
               t_max=max(m[5] for m in meta))
    if len(meta[0]) > 6 and meta[0][6] is not None:
        raw.update(noise_idx=torch.tensor([m[7] for m in meta], dtype=torch.int32),
                   noise_off=torch.tensor([m[8] for m in meta], dtype=torch.int64),
                   snr=torch.tensor([m[6] for m in meta], dtype=torch.float64))
    if len(meta[0]) > 6 and meta[0][9] is not None:
        raw.update(rir_idx=torch.tensor([m[9] for m in meta], dtype=torch.int32),
                   rir_max_len=int(max(rir.lengths[m[9]] for m in meta)))
    lens = torch.tensor([m[5] for m in meta], dtype=torch.int32)
    ali_lens = torch.tensor([len(t) for t in tgt], dtype=torch.int32)
    return raw, target, lens, ali_lens


_frontends = {}


def _frontend_for(args, device):
    key = (getattr(args, "feat_type", "fbank"), args.feat_config, args.feats_dim, args.sample_rate, args.lctx, args.rctx, args.stride,
           str(device))
    if key not in _frontends:
        opts = feature_options(args)
        if getattr(args, "no_dither", False):          # explicit opt-out (parity runs); otherwise the feature config decides
            opts.dither = 0.0
        _frontends[key] = Frontend(opts, args.lctx, args.rctx, device, stride=args.stride)
    return _frontends[key]


def raw_to_features(raw, args, device="cuda", noise=None, rir=None):
    """reference-shaped float features [B,Tmax,D] on the CPU from a raw batch (GPU front end, then D2H)"""
    fe = _frontend_for(args, device)
    if noise:
        fe.noise = noise
    if rir:
        fe.rir = rir
    dev = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in raw.items()}
    out = fe(dev["pcm"], dev["n_samples"], dev["rate"], dev["target_db"], dev["new_len"], dev["n_frames"], dev["t_max"],
             out_dtype=torch.float32, cmn=False, **noise_rir_kwargs(dev))
    return out.cpu()


def dataloader(data_lst, rir, noise, args):
    """
    Args:
        data_lst: list of mrk and seq of input audios, and label ark
        rir, noise: ``AudioBank`` (loader/audio_bank.py) for on-the-fly reverberation / noise, or empty lists for none
    """
    feature_options(args)                      # a config the front end cannot run fails here, before any worker starts
    data_triplets = kaldi_io.read_lst(data_lst)
    num_per_worker = (len(data_triplets) + args.num_workers - 1) // args.num_workers
    lst = [data_triplets[i:i + num_per_worker] for i in range(0, len(data_triplets), num_per_worker)]
    assert len(lst) == args.num_workers
    q = queue.Queue(args.queue_size)
    threads = [Thread(target=put_thread, args=(q, otf_utt_generator, lst[i], rir, noise, args)) for i in range(args.num_workers)]
    for t in threads:
        t.daemon = True
        t.start()
    num_done = 0
    raw_mode = bool(getattr(args, "raw_batches", False))
    while True:
        item = q.get()
        if item is None:
            num_done += 1
            if num_done == args.num_workers:
                break
            continue
        raw, target, lens, ali_lens = item
        if raw is None or raw_mode:
            yield raw, target, lens, ali_lens
        else:
            data = raw_to_features(raw, args, noise=noise, rir=rir)
            if not args.batch_first:
                data, target = data.transpose(0, 1).contiguous(), target.t().contiguous()
            yield data, target, lens, ali_lens
    for t in threads:
        t.join()
