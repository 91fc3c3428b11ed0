"""Channel-offset oracle (reference passiveRadar/signal_utils.py:29-78), test infrastructure only.

* ``find_channel_offset_oracle`` / ``xcorr_oracle`` restate the reference's functions with the same SciPy calls
  (``scipy.signal.decimate``, ``numpy.pad``, ``scipy.signal.correlate``): what the reference computes, including its
  float32 arithmetic for float32 / complex64 inputs.
* ``find_channel_offset_truth`` is the float64 statement of the same thing: the odd extension in the input's own
  dtype (integers wrap, as NumPy does), then the signal widened to complex128 and filtered with decimate's sections
  -- float32-rounded for float32 / complex64 inputs, as the reference's are -- and correlated in complex128.
* ``decimate_chunked`` is a NumPy model of the device decimator: each chunk of a pass starts from a zero state
  ``warm`` samples before its own start (the first from the exact state), so tests can bound the warm-up error.
* ``fft_passes_correlate`` is a NumPy model of the device transform: radix-2 decimation in frequency in passes of
  at most 11 stages, the product X conj(Y) in bit-reversed order, and the transposed decimation-in-time inverse.
"""
from __future__ import annotations

import numpy as np
import scipy.signal as signal

PADLEN = 27


def find_channel_offset_oracle(s1, s2, nd, nl):
    B1 = signal.decimate(s1, nd)
    B2 = np.pad(signal.decimate(s2, nd), (nl, nl), 'constant')
    xc = np.abs(signal.correlate(B1, B2, mode='valid'))
    return (np.argmax(xc) - nl) * nd, xc


def xcorr_oracle(s1, s2, nlead, nlag):
    return signal.correlate(s1, np.pad(s2, (nlag, nlead), mode='constant'), mode='valid')


def decimate_sos(nd, dtype):
    """decimate's sections and sosfilt_zi for a signal of ``dtype``, as float64 arrays."""
    sos = signal.cheby1(8, 0.05, 0.8 / nd, output='sos')
    if np.dtype(dtype) in (np.float32, np.complex64):
        sos = sos.astype(np.float32)
    return sos.astype(np.float64), signal.sosfilt_zi(sos).astype(np.float64)


def odd_extension(x):
    """sosfiltfilt's odd extension of 27 samples, evaluated in the input's own dtype (integers wrap)."""
    from scipy.signal._arraytools import odd_ext
    return odd_ext(np.asarray(x), PADLEN)


def _wide(x):
    return x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)


def decimate_truth(x, nd):
    x = np.asarray(x)
    sos, zi = decimate_sos(nd, x.dtype)
    ext = _wide(odd_extension(x)) if x.dtype.kind in "iu" else odd_extension(_wide(x))
    y, _ = signal.sosfilt(sos, ext, zi=zi * ext[0])
    z, _ = signal.sosfilt(sos, y[::-1], zi=zi * y[-1])
    return z[::-1][PADLEN:-PADLEN][::nd]


def find_channel_offset_truth(s1, s2, nd, nl):
    B1 = decimate_truth(s1, nd)
    B2 = np.pad(decimate_truth(s2, nd), (nl, nl))
    xc = np.abs(signal.correlate(B1.astype(np.complex128), B2.astype(np.complex128), mode='valid', method='fft'))
    return (int(np.argmax(xc)) - nl) * nd, xc


def decimate_chunked(x, nd, chunk, warm):
    """The device decimator restated: sosfiltfilt + [::nd] with each pass cut into chunks of ``chunk`` samples."""
    x = np.asarray(x)
    sos, zi = decimate_sos(nd, x.dtype)
    ext = _wide(odd_extension(x)) if x.dtype.kind in "iu" else odd_extension(_wide(x))

    def one_pass(v):
        out = np.empty_like(v)
        for i0 in range(0, v.shape[0], chunk):
            i1 = min(i0 + chunk, v.shape[0])
            s = i0 - warm
            if s <= 0:
                y, _ = signal.sosfilt(sos, v[:i1], zi=zi * v[0])
                out[i0:i1] = y[i0:]
            else:
                out[i0:i1] = signal.sosfilt(sos, v[s:i1])[i0 - s:]
        return out

    y = one_pass(ext)
    z = one_pass(y[::-1].copy())
    return z[::-1][PADLEN:-PADLEN][::nd]


def warmup_samples(sos):
    """W of the device decimator (csrc/prcore.cu chanoff_warmup): from the largest pole radius of the sections."""
    r = 0.0
    for s in np.asarray(sos, dtype=np.float64):
        r = max(r, float(np.abs(np.roots([1.0, s[4], s[5]])).max()))
    return int(np.ceil(np.log(1e-18) / np.log(r))) + 256


def pass_plan(m):
    """(lo, nb) of each pass, top index bits first: 8 bits while more than 11 remain, then the rest."""
    out, top = [], m
    while top > 0:
        nb = top if top <= 11 else 8
        out.append((top - nb, nb))
        top -= nb
    return out


def _dif_pass(a, m, lo, nb, inverse):
    L = 1 << m
    w = np.exp((2j if inverse else -2j) * np.pi * np.arange(L // 2) / L)
    s0 = m - lo - nb
    stages = range(nb - 1, -1, -1) if inverse else range(nb)
    for r in stages:
        s = s0 + r
        h = L >> (s + 1)
        i = np.arange(L)
        top = i[(i & h) == 0]
        tw = w[(top % h) << s]
        x, y = a[top].copy(), a[top + h].copy()
        if inverse:
            t = y * tw
            a[top], a[top + h] = x + t, x - t
        else:
            a[top], a[top + h] = x + y, (x - y) * tw
    return a


def fft_passes_correlate(x, y, m):
    """L = 2^m circular correlation cc[p] = sum_j x[j + p] conj(y[j]) through the pass structure of the device."""
    L = 1 << m
    X = np.zeros(L, np.complex128)
    Y = np.zeros(L, np.complex128)
    X[:len(x)] = x
    Y[:len(y)] = y
    plan = pass_plan(m)
    for lo, nb in plan:
        _dif_pass(X, m, lo, nb, False)
        _dif_pass(Y, m, lo, nb, False)
    P = X * np.conj(Y)
    for lo, nb in reversed(plan):
        _dif_pass(P, m, lo, nb, True)
    return P / L
