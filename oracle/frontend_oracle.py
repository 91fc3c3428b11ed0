"""CPU restatement of the rows either side of the hot path (SURVEY.md section 8(f)) -- TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and the CPU arms of ``bench.py`` may import this package;
the product (``passiveradar_b200``) never does.  Each function follows the reference line by line and
calls the same NumPy/SciPy routines at the same precision, so that it can be pinned against the
reference-generated goldens under ``tests/golden/`` (``front_*``, ``cfar_*``, ``direct_*``).
"""
from __future__ import annotations

import numpy as np
import scipy.signal as signal

from .clutter_oracle import frequency_shift_oracle, xcorr_oracle


def deinterleave_iq_oracle(interleavedIQ):
    """``deinterleave_IQ`` (reference passiveRadar/signal_utils.py:19-22)."""
    interleavedIQ = np.array(interleavedIQ)
    return (interleavedIQ[0:-1:2] + 1j * interleavedIQ[1::2]).astype(np.complex64)


def resample_oracle(x, up, dn):
    """``resample`` (reference passiveRadar/signal_utils.py:15-17)."""
    return signal.resample_poly(x, up, dn, padtype='line')


def frontend_oracle(interleavedIQ, fc, Fs, phase_offset, up, dn):
    """The per-chunk chain of main.py:105-166: deinterleave -> frequency_shift -> resample."""
    return resample_oracle(frequency_shift_oracle(deinterleave_iq_oracle(interleavedIQ), fc, Fs, phase_offset), up, dn)


def resample_truth(x, up, dn, ms=None):
    """float64 statement of resample_poly(padtype='line') written out as the polyphase sum the device
    kernel evaluates (independent of SciPy's upfirdn): used to check the index arithmetic.  ``ms``: only
    these output indices (the loop is per output sample), returned in that order."""
    import math
    x = np.asarray(x, dtype=np.complex128)
    g = math.gcd(up, dn)
    up //= g
    dn //= g
    n = x.shape[0]
    max_rate = max(up, dn)
    half_len = 10 * max_rate
    h = signal.firwin(2 * half_len + 1, 1.0 / max_rate, window=('kaiser', 5.0)) * up
    n_pre_pad = dn - half_len % dn
    n_pre_remove = (half_len + n_pre_pad) // dn
    n_out = n * up // dn + bool(n * up % dn)
    hpad = np.concatenate((np.zeros(n_pre_pad), h))
    slope = (x[-1] - x[0]) / (n - 1)
    ms = range(n_out) if ms is None else ms
    out = np.zeros(len(ms), dtype=np.complex128)
    for q, m in enumerate(ms):
        T = (m + n_pre_remove) * dn
        ih, ph = divmod(T, up)
        k = np.arange(ph, hpad.shape[0], up)
        i = ih - np.arange(k.shape[0])
        xe = np.where(i < 0, x[0] + i * slope, np.where(i >= n, x[-1] + (i - n + 1) * slope, x[np.clip(i, 0, n - 1)]))
        out[q] = np.dot(hpad[k], xe)
    return out


def cfar_2d_oracle(X, fw, gw, thresh=None):
    """``CFAR_2D`` (reference passiveRadar/target_detection.py:683-703)."""
    Tfilt = np.ones((fw, fw)) / (fw ** 2 - gw ** 2)
    e1 = (fw - gw) // 2
    e2 = fw - e1 + 1
    Tfilt[e1:e2, e1:e2] = 0
    norm = X / np.mean(np.abs(X).flatten())                     # normalize(), signal_utils.py:7-9
    CR = norm / (signal.convolve2d(X, Tfilt, mode='same', boundary='wrap') + 1e-10)
    if thresh is None:
        return CR
    return CR > thresh


def direct_xambg_oracle(refChannel, srvChannel, rangeBins, freqBins, sampleRate):
    """``direct_xambg`` (reference passiveRadar/range_doppler_processing.py:93-124)."""
    if refChannel.shape != srvChannel.shape:
        raise ValueError('Input vectors must have the same length')
    CPI = refChannel.shape[0] / sampleRate
    xambg = np.zeros((freqBins, rangeBins + 1, 1), dtype=np.complex64)
    for i in range(freqBins):
        df = (i - 0.5 * freqBins) / CPI
        ref_shifted = frequency_shift_oracle(refChannel, df, sampleRate)
        xambg[i, :, 0] = xcorr_oracle(ref_shifted, srvChannel, rangeBins, 0)
    return xambg


def direct_xambg_truth(refChannel, srvChannel, rangeBins, freqBins, sampleRate):
    """float64 direct sum with the exact phase (no float32 ramp): quantifies the reference's self-noise."""
    ref = np.asarray(refChannel, dtype=np.complex128)
    srv = np.asarray(srvChannel, dtype=np.complex128)
    n = ref.shape[0]
    nn = np.arange(n, dtype=np.float64)
    out = np.zeros((freqBins, rangeBins + 1, 1), dtype=np.complex128)
    spad = np.concatenate((srv, np.zeros(rangeBins, dtype=np.complex128)))
    for i in range(freqBins):
        rs = ref * np.exp(2j * np.pi * (i - 0.5 * freqBins) * nn / n)
        for k in range(rangeBins + 1):
            lag = rangeBins - k
            out[i, k, 0] = np.dot(rs, np.conj(spad[lag:lag + n]))
    return out
