"""Global CMVN statistics -- drop-in for utils/compute_global_cmvn.py (reference): same command line, same Kaldi text stats file
(` [ sum_0 .. sum_{D-1} count\\n  sumsq_0 .. sumsq_{D-1} 0 ]`, what kaldi.transform.cmvn.Cmvn.write_stats(binary=False) writes and
trainer/train_transducer_bmuf_otfaug.py:341-346 reads back).

    python -m pika_b200.utils.compute_global_cmvn DATA_LST CMVN_STATS --feat_config fbank.conf [--feat_type mfcc] [--cmn]

Every utterance of the ``.lst`` shards goes through the reference's augmentation draws (speed from {0.9, 1.0, 1.1} with
``random.randint``, gain from ``np.random.uniform(-55, -10)``, :52-55) and the GPU front end (speed / gain / Kaldi fbank kernels of
pika_b200/csrc/frontend.cu; Kaldi MFCC with ``--feat_type mfcc``), batches of ``--batch_size`` utterances at a time; sums and sums of squares accumulate in float64."""
import argparse
import sys
from random import randint

import numpy as np
import torch

from ..frontend import FbankOptions, Frontend, MfccOptions
from ..loader import kaldi_io


def write_cmvn_stats(path, s1, s2, count):
    with open(path, "w") as f:
        f.write(" [\n  %s %.10g \n  %s 0 ]\n" % (" ".join("%.10g" % v for v in s1), count, " ".join("%.10g" % v for v in s2)))


def feature_options(args):
    """the options of ``--feat_config`` as ``--feat_type``'s Kaldi options (Kaldi's defaults with ``--feat_dim`` mel bins or cepstra
    without one); ``--feat_dim`` must be the per-frame width (num-mel-bins for fbank, num-ceps for MFCC), ``--sample_rate`` the config's
    sample frequency"""
    if args.feat_type == "mfcc":
        opts = MfccOptions.from_config(args.feat_config) if args.feat_config else MfccOptions(num_ceps=args.feat_dim)
        width, name = opts.num_ceps, "num-ceps"
    else:
        opts = FbankOptions.from_config(args.feat_config) if args.feat_config else FbankOptions(num_mel_bins=args.feat_dim)
        width, name = opts.num_mel_bins, "num-mel-bins"
    if float(args.sample_rate) != opts.sample_frequency:
        raise ValueError("--sample_rate %s differs from the feature config's --sample-frequency=%g" % (args.sample_rate, opts.sample_frequency))
    if width != args.feat_dim:
        raise ValueError("--feat_dim %d must match %s=%d of the feature config" % (args.feat_dim, name, width))
    return opts


def main(argv=None):
    parser = argparse.ArgumentParser(description='global CMVN estimation')
    parser.add_argument('data_lst', type=str, help='input data_lst filename')
    parser.add_argument('cmvn_stats', type=str, help='output cmvn states filename')
    parser.add_argument('--cmn', action="store_true", help="apply cepstrum mean normalizaiton per utterance")
    parser.add_argument('--sample_rate', type=int, default=16000, help='sample rate of waves')
    parser.add_argument('--feat_config', type=str, default=None, help='feature extraction config file')
    parser.add_argument('--feat_type', type=str, default='fbank', choices=('fbank', 'mfcc'),
                        help='Kaldi feature type that --feat_config describes (pika_b200 only)')
    parser.add_argument('--feat_dim', type=int, default=80, help='feature dimension')
    parser.add_argument('--batch_size', type=int, default=64, help='utterances per GPU front-end call (pika_b200 only)')
    args, _ = parser.parse_known_args(argv)
    opts = feature_options(args)
    if not torch.cuda.is_available():
        sys.exit("pika_b200.utils.compute_global_cmvn: the front end runs on the GPU only")
    dev = torch.device("cuda", 0)
    fe = Frontend(opts, 0, 0, dev)
    speed_rate = [0.9, 1.0, 1.1]
    s1, s2, count = np.zeros(args.feat_dim), np.zeros(args.feat_dim), 0.0

    def flush(pcms, rates, gains):
        nonlocal s1, s2, count
        if not pcms:
            return
        B = len(pcms)
        ns = [len(p) for p in pcms]
        new_len, frames = Frontend.lengths(ns, rates, **opts.geometry())
        n_max, t_max = max(max(ns), max(new_len)), max(frames)
        if t_max == 0:
            return
        pcm = torch.zeros(B, n_max, dtype=torch.int16)
        for i, p in enumerate(pcms):
            pcm[i, :ns[i]] = torch.from_numpy(p.copy())
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)                      # noqa: E731
        feats = fe(pcm.to(dev), i32(ns), torch.tensor(rates, dtype=torch.float32, device=dev),
                   torch.tensor(gains, dtype=torch.float32, device=dev), i32(new_len), i32(frames), t_max, out_dtype=torch.float32, cmn=False)
        feats = feats.double()
        for i in range(B):
            f = feats[i, :frames[i]]
            if frames[i] == 0:
                continue
            if args.cmn:
                f = f - f.mean(dim=0, keepdim=True)                                         # :62-65
            s1 += f.sum(0).cpu().numpy()
            s2 += (f * f).sum(0).cpu().numpy()
            count += frames[i]

    pcms, rates, gains = [], [], []
    shards = [line.split()[:2] for line in open(args.data_lst, 'r', encoding='utf-8') if line.split()]     # mrk, seq (a label column may follow)
    for mrk_fn, seq_fn in shards:
        for _, audio in kaldi_io.iter_mrk_seq(mrk_fn, seq_fn):
            pcms.append(np.asarray(audio, dtype=np.int16))
            rates.append(speed_rate[randint(0, len(speed_rate) - 1)])                       # :52
            gains.append(float(np.random.uniform(-55, -10)))                                # :55
            if len(pcms) == args.batch_size:
                flush(pcms, rates, gains)
                pcms, rates, gains = [], [], []
    flush(pcms, rates, gains)
    write_cmvn_stats(args.cmvn_stats, s1, s2, count)


if __name__ == '__main__':
    main()
