"""numpy restatement of the reference's noise and reverberation augmentation (loader/audio.py:426-513
AudioSegment.add_noise / convolve_and_normalize) on top of oracle/frontend.py, for the parity tests of the GPU front end.

Arithmetic follows numpy's dtype rules on the reference's in-place updates: the samples keep their dtype (float32 on the
rate == 1.0 branch, float64 after speed perturbation); the scaled noise slice is float32.  The noise offset is an integer sample
index (the reference draws a float start time and rounds it).
"""
import numpy as np
from scipy import signal

from oracle import frontend as ofe


def normalize_inplace(samples, target_db, max_gain_db=300.0):
    """AudioSegment.normalize with the in-place gain of gain_db (loader/audio.py:207-215,240-262): dtype preserved"""
    gain = target_db - ofe.rms_db(samples)
    if gain > max_gain_db:
        raise ValueError("Unable to normalize segment to %f dB" % target_db)
    out = samples.copy()
    out *= 10. ** (min(max_gain_db, gain) / 20.)
    return out


def add_noise(samples, noise_i16, off, snr_db, max_gain_db=300.0):
    """AudioSegment.add_noise (loader/audio.py:467-513) with the subsegment [off, off + len(samples)) of the noise"""
    noise = ofe.to_float32(noise_i16)
    if len(noise) < off + len(samples):
        raise ValueError("noise slice [%d, %d) past the segment's %d samples" % (off, off + len(samples), len(noise)))
    gain_db = min(ofe.rms_db(samples) - ofe.rms_db(noise) - snr_db, max_gain_db)
    part = noise[off:off + len(samples)].copy()
    part *= 10. ** (gain_db / 20.)
    out = samples.copy()
    out += part
    return out


def convolve_and_normalize(samples, rir_i16):
    """AudioSegment.convolve_and_normalize (loader/audio.py:426-465): fftconvolve(.., "same"), back to the input's rms_db"""
    target_db = ofe.rms_db(samples)
    y = signal.fftconvolve(samples, ofe.to_float32(rir_i16), "same")
    return normalize_inplace(y, target_db)


def augment(pcm_i16, rate, target_db, noise=None, off=0, snr=None, rir=None):
    """loader/otf_utt_loader.py:218-230 with the example's noise and RIR stages (:224-228): speed -> gain -> noise -> RIR -> int16"""
    s = ofe.change_speed(ofe.to_float32(pcm_i16), rate)
    s = normalize_inplace(s, target_db)
    if noise is not None:
        s = add_noise(s, noise, off, np.float64(snr))
    if rir is not None:
        s = convolve_and_normalize(s, rir)
    return ofe.to_int16(s)
