"""Welch PSD and signal-preview oracle, test infrastructure only.

* ``psd_oracle`` restates ``matplotlib.mlab.psd`` (what ``plt.psd`` returns, ``freqs + Fc``) in NumPy, float64 /
  complex128: segments of NFFT at a step of NFFT - noverlap ((n - noverlap) // step of them; a signal shorter than NFFT
  zero-padded to one), times the window, ``np.fft.fft(..., n=pad_to)``, |X|^2; one-sided: bins 0 .. pad_to/2 with every
  bin but DC doubled and the pad_to/2 bin only when NFFT is odd (mlab's ``slice(1, -1)`` / ``slice(1, None)`` on NFFT);
  divided by Fs and sum |w|^2 (scale_by_freq) or by (sum |w|)^2; the mean over segments; two-sided rotated by
  pad_to // 2.  matplotlib is not a dependency, so this is what the device estimator is held to.
* ``psd_dft`` is the same definition with a direct float64 DFT (no FFT), for lengths scipy.signal.welch does not cover.
* ``preview_reference`` composes the reference's own ``deinterleave_IQ``, ``find_channel_offset``,
  ``frequency_shift``, ``resample`` and ``xcorr`` (oracle/_ref, placed there by build()) as signal_preview.py does;
  its spectra come from ``psd_oracle``, since the script's come from matplotlib.
* ``xcorr_truth`` is |xcorr(ref, srv, nlead, nlag)| in complex128.
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _segments(x, NFFT, noverlap):
    x = np.asarray(x)
    if x.shape[0] < NFFT:
        x = np.concatenate([x, np.zeros(NFFT - x.shape[0], x.dtype)])
    step = NFFT - noverlap
    nseg = (x.shape[0] - noverlap) // step
    idx = np.arange(NFFT)[None, :] + step * np.arange(nseg)[:, None]
    return x[idx]


def _finish(P, NFFT, Fs, Fc, w, pad_to, onesided, scale_by_freq):
    if onesided:
        P = P[:, :pad_to // 2 + 1].copy()
        P[:, slice(1, -1) if NFFT % 2 == 0 else slice(1, None)] *= 2.0
    if scale_by_freq:
        P = P / Fs / (np.abs(w) ** 2).sum()
    else:
        P = P / np.abs(w).sum() ** 2
    P = P.mean(axis=0)
    freqs = np.fft.fftfreq(pad_to, 1 / Fs)
    if onesided:
        freqs = freqs[:pad_to // 2 + 1]
        freqs[-1] *= -1
    else:
        freqs = np.roll(freqs, -(pad_to // 2))
        P = np.roll(P, -(pad_to // 2))
    return P, freqs + Fc


def _args(x, NFFT, Fs, Fc, window, noverlap, pad_to, sides, scale_by_freq):
    x = np.asarray(x)
    NFFT = 256 if NFFT is None else NFFT
    Fs = 2 if Fs is None else Fs
    Fc = 0 if Fc is None else Fc
    noverlap = 0 if noverlap is None else noverlap
    pad_to = NFFT if pad_to is None else pad_to
    if window is None:
        w = np.hanning(NFFT)
    elif callable(window):
        w = window(np.ones(NFFT, x.dtype))
    else:
        w = np.asarray(window)
    w = np.real(w).astype(np.float64)
    onesided = (not np.iscomplexobj(x)) if sides in (None, "default") else sides == "onesided"
    scale_by_freq = True if scale_by_freq is None else scale_by_freq
    xw = x.astype(np.complex128 if np.iscomplexobj(x) else np.float64)
    return xw, NFFT, Fs, Fc, w, noverlap, pad_to, onesided, scale_by_freq


def psd_oracle(x, NFFT=None, Fs=None, Fc=None, window=None, noverlap=None, pad_to=None, sides=None, scale_by_freq=None):
    x, NFFT, Fs, Fc, w, noverlap, pad_to, onesided, sbf = _args(x, NFFT, Fs, Fc, window, noverlap, pad_to, sides,
                                                                 scale_by_freq)
    X = np.fft.fft(_segments(x, NFFT, noverlap) * w[None, :], n=pad_to, axis=1)
    return _finish(np.abs(X) ** 2, NFFT, Fs, Fc, w, pad_to, onesided, sbf)


def psd_dft(x, NFFT=None, Fs=None, Fc=None, window=None, noverlap=None, pad_to=None, sides=None, scale_by_freq=None):
    x, NFFT, Fs, Fc, w, noverlap, pad_to, onesided, sbf = _args(x, NFFT, Fs, Fc, window, noverlap, pad_to, sides,
                                                                 scale_by_freq)
    k = np.arange(pad_to)
    E = np.exp(-2j * np.pi * np.outer(np.arange(NFFT), k) / pad_to)          # (NFFT, pad_to) direct DFT matrix
    X = (_segments(x, NFFT, noverlap) * w[None, :]) @ E
    return _finish(np.abs(X) ** 2, NFFT, Fs, Fc, w, pad_to, onesided, sbf)


def xcorr_truth(ref, srv, nlead, nlag):
    """|correlate(ref, pad(srv, (nlag, nlead)), 'valid')| in complex128 (scipy.signal.correlate's FFT path)."""
    from scipy.signal import correlate
    a = np.asarray(ref).astype(np.complex128)
    b = np.pad(np.asarray(srv).astype(np.complex128), (nlag, nlead))
    return np.abs(correlate(a, b, mode="valid", method="fft"))


def reference_signal_utils():
    """The reference's passiveRadar.signal_utils from oracle/_ref (ImportError when build() found no checkout)."""
    ref = os.path.join(HERE, "_ref")
    if not os.path.isdir(os.path.join(ref, "passiveRadar")):
        raise ImportError("oracle/_ref holds no reference modules")
    if ref not in sys.path:
        sys.path.insert(0, ref)
    from passiveRadar import signal_utils
    return signal_utils


def preview_channels(config, ref_raw, srv_raw=None, su=None):
    """signal_preview.py:28-48: the two deinterleaved channels, with the reference's deinterleave_IQ."""
    su = su or reference_signal_utils()
    icl = config["input_chunk_length"]
    if config["interleaved_input_channels"]:
        iq = su.deinterleave_IQ(ref_raw[0:icl])
        return iq[0::2], iq[1::2]
    return su.deinterleave_IQ(ref_raw[0:icl]), su.deinterleave_IQ(srv_raw[0:icl])


def preview_reference(config, ref_raw, srv_raw=None):
    """Everything signal_preview.py plots, from the reference's own functions (spectra from psd_oracle)."""
    su = reference_signal_utils()
    ref, srv = preview_channels(config, ref_raw, srv_raw, su)
    offset = su.find_channel_offset(ref, srv, 4, 50000)
    reff = su.resample(su.frequency_shift(ref, config["offset_freq"], config["input_sample_rate"]),
                       config["resamp_up"], config["resamp_dn"])
    srvv = su.resample(su.frequency_shift(srv, config["offset_freq"], config["input_sample_rate"]),
                       config["resamp_up"], config["resamp_dn"])
    xc = su.xcorr(ref, srv, 2000, 2000)
    spec = lambda s, nfft, fs, fc: psd_oracle(s, NFFT=nfft, Fs=fs, Fc=fc)
    return {"ref": ref, "srv": srv, "offset": int(offset), "ref_resampled": reff, "srv_resampled": srvv,
            "xcorr": xc,
            "input_psd": [spec(s, 8192, config["input_sample_rate"], config["input_center_freq"]) for s in (ref, srv)],
            "channel_psd": [spec(s, 2048, config["channel_bandwidth"], config["channel_freq"]) for s in (reff, srvv)]}
