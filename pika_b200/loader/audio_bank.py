"""Noise and room-impulse-response banks for on-the-fly augmentation (``--noise_lst`` / ``--rir_lst``).

The reference's trainer leaves these as lists of ``AudioSegment`` (trainer/train_transducer_bmuf_otfaug.py:272-282); here a
bank is one concatenated int16 array, uploaded to the device once, plus host-side offsets and lengths that the loader threads
draw against.  The list file holds one ``<mrk> <seq>`` pair per non-empty line (the utils/wav_to_seq.py layout); every entry of
every pair is one segment.  Samples are 16 kHz int16, used as float32 * 2^-15 as ``AudioSegment`` does.
"""
import logging

import numpy as np
import torch

from . import kaldi_io

RIR_MAX_LEN = 65536                 # longest RIR the GPU convolution takes (4.1 s at 16 kHz)

log = logging.getLogger(__name__)


def max_new_len(max_len):
    """longest augmented utterance (samples) whose snip-edges frame count passes the ``--max_len`` filter"""
    return 160 * int(max_len) + 399


def rms_db(samples_i16):
    """AudioSegment.rms_db (loader/audio.py:551-560) of the float32 samples of a whole int16 segment"""
    s = samples_i16.astype(np.float32)
    s *= 1.0 / 2 ** 15
    mean_square = max(1e-20, np.mean(s ** 2))
    return float(10 * np.log10(mean_square))


class AudioBank:
    """Concatenated int16 segments: ``ids``, ``offsets`` (int64), ``lengths`` (int64) and, for noise, ``rms_db`` (float64)."""

    def __init__(self, ids, segments, with_rms=False):
        self.ids = list(ids)
        self.lengths = np.array([len(s) for s in segments], dtype=np.int64)
        self.offsets = np.concatenate(([0], np.cumsum(self.lengths)[:-1])).astype(np.int64)
        self.samples = np.concatenate(segments).astype(np.int16) if segments else np.zeros(0, np.int16)
        self.rms_db = np.array([rms_db(s) for s in segments], dtype=np.float64) if with_rms else None
        self._dev = {}

    def __len__(self):
        return len(self.ids)

    @staticmethod
    def _read(lst):
        ids, segs = [], []
        with open(lst, "r", encoding="utf-8") as f:
            for line in f:
                p = line.split()
                if not p:
                    continue
                if len(p) < 2:
                    raise ValueError("%s: expected '<mrk> <seq>' per line, got %r" % (lst, line.strip()))
                for uttid, audio in kaldi_io.iter_mrk_seq(p[0], p[1]):
                    ids.append(uttid)
                    segs.append(np.asarray(audio, np.int16))
        return ids, segs

    @classmethod
    def noise(cls, lst, max_len):
        """noise bank; segments shorter than the longest utterance that can pass ``--max_len`` (``160 * max_len + 399`` samples)
        are dropped, since ``add_noise`` needs noise at least as long as the utterance (trainer/train_transducer_bmuf_otfaug.py:277-280)"""
        ids, segs = cls._read(lst)
        need = max_new_len(max_len)
        keep = [i for i, s in enumerate(segs) if len(s) >= need]
        if len(keep) < len(segs):
            log.warning("noise bank %s: dropped %d of %d segments shorter than %d samples (--max_len %d)", lst, len(segs) - len(keep),
                        len(segs), need, max_len)
        if not keep:
            raise ValueError("noise bank %s: no segment is at least %d samples long (160 * max_len + 399, --max_len %d)"
                             % (lst, need, max_len))
        return cls([ids[i] for i in keep], [segs[i] for i in keep], with_rms=True)

    @classmethod
    def rir(cls, lst):
        """RIR bank; an RIR longer than 65536 samples (or an empty one) is an error"""
        ids, segs = cls._read(lst)
        for i, s in zip(ids, segs):
            if len(s) > RIR_MAX_LEN or len(s) == 0:
                raise ValueError("RIR %s in %s has %d samples; the supported range is 1..%d" % (i, lst, len(s), RIR_MAX_LEN))
        if not segs:
            raise ValueError("RIR bank %s is empty" % lst)
        return cls(ids, segs)

    def device(self, device):
        """(samples int16, offsets int64, lengths int32, rms_db f64 or None) on ``device``, uploaded on first use"""
        key = str(device)
        if key not in self._dev:
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)  # noqa: E731
            self._dev[key] = (t(self.samples), t(self.offsets), t(self.lengths.astype(np.int32)),
                              None if self.rms_db is None else t(self.rms_db))
        return self._dev[key]
