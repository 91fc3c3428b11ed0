"""Oracle for the cross-ambiguity function (TEST INFRASTRUCTURE ONLY, see oracle/__init__.py).

Restates ``fast_xambg`` of the reference
(``passiveRadar/range_doppler_processing.py:12-90``):

    :46-49   shape check                       -> ``_check_pair``
    :52-55   zero-pad to ``inputLen``          -> ``_pad_to``
    :57-58   named window                      -> ``scipy.signal.get_window``
    :61      ``ndecim = int(N / freqBins)``    -> ``decimation_factor``
    :69-78   decimator taps (boxcar / flattop) -> ``decimator_taps``
    :81-86   per-lag  roll * ref * window -> decimate
    :89      FFT along Doppler + fftshift

The arithmetic lives in SciPy (unpinned by the reference's environment.yaml;
SciPy 1.18.1 / NumPy 2.3.5 here): ``signal.decimate`` with an FIR ``dlti`` is
``resample_poly(x, 1, q, window=taps)`` (scipy/signal/_signaltools.py:5344-5347)
which is ``upfirdn`` with the alignment rule of ``:4038-4091``.  The oracle
calls ``resample_poly`` directly: that skips ``dlti._as_zpk()`` (``:5322``, an
``np.roots`` of degree ``ndecim`` per range lag -- 46 s per lag at ndecim=4096)
and is bit-identical, which ``tests/test_oracle_golden.py`` proves against the
literal reference at small ``ndecim``.

Rounding points kept exactly as the reference has them: the lag product is
complex64; ``*= window`` is evaluated in complex128 and rounded back to
complex64; the block sum runs in complex128 (float64 taps) and is rounded to
complex64 on store; the Doppler FFT is ``scipy.fftpack.fft`` on complex64.
"""
from __future__ import annotations

import numpy as np
import scipy.signal as signal
from scipy.fftpack import fft as _fft_c64


def _check_pair(ref, srv):
    if ref.shape != srv.shape:
        raise ValueError('Input vectors must have the same length')


def _pad_to(x, n):
    # the reference pads only when the length differs; a longer input makes
    # np.pad raise (negative pad width) and we keep that behaviour
    if n is not None and x.shape[0] != n:
        return np.pad(x, (0, n - x.shape[0]), mode='constant')
    return x


def decimation_factor(n, freq_bins):
    return int(n / freq_bins)


def decimator_taps(ndecim, short_filt=True):
    if short_filt:
        return np.ones((ndecim + 1,))
    return signal.firwin(10 * ndecim + 1, 1. / ndecim, window='flattop')


def decimate_fir(x, q, taps, axis=-1):
    """``signal.decimate(x, q, ftype=dlti(taps, 1))`` without the zpk detour."""
    return signal.resample_poly(x, 1, q, axis=axis, window=np.asarray(taps, dtype=np.float64) / 1.0)


def decimator_alignment(ntaps, ndecim):
    """(offset c, ) such that ``out[j] = sum_m taps[m] * x[j*ndecim + c - m]``.

    From ``resample_poly`` (scipy/signal/_signaltools.py:4038-4045) with up=1.
    For ``ndecim == 1`` SciPy returns the input unchanged (``:4028-4029``), which
    is the single tap ``[1.0]`` at offset 0.
    """
    half_len = (ntaps - 1) // 2
    n_pre_pad = ndecim - half_len % ndecim
    n_pre_remove = (half_len + n_pre_pad) // ndecim
    return n_pre_remove * ndecim - n_pre_pad


def fast_xambg_oracle(refChannel, srvChannel, rangeBins, freqBins, inputLen=None,
                      window=None, shortFilt=True, lag_batch=16):
    """Range-Doppler map, shape ``(freqBins, rangeBins + 1, 1)`` complex64."""
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    _check_pair(refChannel, srvChannel)
    refChannel = _pad_to(refChannel, inputLen)
    srvChannel = _pad_to(srvChannel, inputLen)
    if isinstance(window, (tuple, str)):
        window = signal.get_window(window, inputLen)

    n = refChannel.shape[0]
    ndecim = decimation_factor(n, freqBins)
    taps = decimator_taps(ndecim, shortFilt)

    # roll(conj(srv), lag)[i] == conj(srv)[(i + d) % n] with d = -lag in [0, rangeBins]
    sconj = np.conj(srvChannel)
    reps = 1 + (rangeBins // max(n, 1))
    ring = np.concatenate([sconj] + [sconj] * reps)[: n + rangeBins]

    out = np.zeros((freqBins, rangeBins + 1, 1), dtype=np.complex64)
    for k0 in range(0, rangeBins + 1, lag_batch):
        k1 = min(rangeBins + 1, k0 + lag_batch)
        prod = np.empty((k1 - k0, n), dtype=np.result_type(sconj.dtype, refChannel.dtype))
        for k in range(k0, k1):
            d = rangeBins - k
            np.multiply(ring[d:d + n], refChannel, out=prod[k - k0])
        if window is not None:
            prod *= window          # complex128 product rounded into prod's dtype, as in the reference
        dec = decimate_fir(prod, ndecim, taps, axis=1)
        out[:, k0:k1, 0] = dec[:, 0:freqBins].T
    spec = _fft_c64(out, axis=0)
    return np.fft.fftshift(spec, axes=0)


def block_sums_truth(ref, srv, range_bins, freq_bins, window=None, short_filt=True):
    """float64 evaluation of P[j, k] (SURVEY.md section 3.2), no float32 anywhere.

    P[j,k] = sum_m taps[m] * (ref*w)[j*D + c - m] * conj(srv[(j*D + c - m + R - k) mod N])
    with terms whose product index falls outside [0, N) dropped.
    """
    ref = np.asarray(ref, dtype=np.complex128)
    srv = np.asarray(srv, dtype=np.complex128)
    n = ref.shape[0]
    d = decimation_factor(n, freq_bins)
    if d == 1:
        taps, c = np.ones(1), 0
    else:
        taps = decimator_taps(d, short_filt)
        c = decimator_alignment(taps.shape[0], d)
    x = ref if window is None else ref * np.asarray(window, dtype=np.float64)
    sconj = np.conj(srv)
    nt = taps.shape[0]
    P = np.zeros((freq_bins, range_bins + 1), dtype=np.complex128)
    boxcar = np.all(taps == 1.0)
    for k in range(range_bins + 1):
        lag = range_bins - k
        p = x * np.roll(sconj, -lag)
        if boxcar:
            cs = np.concatenate([[0.0], np.cumsum(p)])
            for j in range(freq_bins):
                hi = j * d + c
                lo = hi - (nt - 1)
                lo_c, hi_c = max(lo, 0), min(hi, n - 1)
                P[j, k] = cs[hi_c + 1] - cs[lo_c] if hi_c >= lo_c else 0.0
        else:
            for j in range(freq_bins):
                hi = j * d + c
                lo = hi - (nt - 1)
                lo_c, hi_c = max(lo, 0), min(hi, n - 1)
                if hi_c >= lo_c:
                    seg = p[lo_c:hi_c + 1]
                    w = taps[hi - hi_c: hi - lo_c + 1][::-1]
                    P[j, k] = np.dot(seg, w)
    return P


def block_sums_truth_fft(ref, srv, range_bins, freq_bins, window=None, short_filt=True, max_points=1 << 22):
    """``block_sums_truth`` evaluated with float64 FFTs, so that thousands of lags at millions of samples are affordable
    on the host.  Block j holds the nt product indices i = hi - nt + 1 .. hi (hi = j*D + c), tap taps[hi - i], and
    P[j, R - d] = sum_i taps[hi - i] x[i] conj(srv[(i + d) mod N]) for d = 0 .. R: a linear correlation of the
    weighted block (zero outside [0, N)) with the nt + R surveillance samples from its first index on, one transform of
    at least nt + R points per block (no circular alias reaches lags 0 .. R).  Blocks go ``max_points`` at a time."""
    import scipy.fft as sfft
    ref = np.asarray(ref, dtype=np.complex128)
    srv = np.asarray(srv, dtype=np.complex128)
    n = ref.shape[0]
    d = decimation_factor(n, freq_bins)
    if d == 1:
        taps, c = np.ones(1), 0
    else:
        taps = np.asarray(decimator_taps(d, short_filt), dtype=np.float64)
        c = decimator_alignment(taps.shape[0], d)
    x = ref if window is None else ref * np.asarray(window, dtype=np.float64)
    nt = taps.shape[0]
    R = range_bins
    nfft = sfft.next_fast_len(nt + R)
    t = np.arange(nt)
    ts = np.arange(nt + R)
    P = np.empty((freq_bins, R + 1), dtype=np.complex128)
    step = max(1, max_points // nfft)
    for j0 in range(0, freq_bins, step):
        js = np.arange(j0, min(freq_bins, j0 + step))
        lo = js[:, None] * d + c - (nt - 1)
        idx = lo + t[None, :]
        inside = (idx >= 0) & (idx < n)
        xb = np.where(inside, x[np.clip(idx, 0, n - 1)], 0) * taps[::-1][None, :]
        sb = srv[(lo + ts[None, :]) % n]
        corr = np.conj(sfft.ifft(np.conj(sfft.fft(xb, nfft, axis=1)) * sfft.fft(sb, nfft, axis=1), axis=1))
        P[js] = corr[:, R::-1]
    return P


def fast_xambg_truth(ref, srv, range_bins, freq_bins, input_len=None, window=None, short_filt=True, fast=False):
    """float64 truth for the whole map, same output convention as ``fast_xambg``; ``fast``: block sums by
    ``block_sums_truth_fft`` rather than the definition's loop."""
    ref = _pad_to(np.asarray(ref), input_len)
    srv = _pad_to(np.asarray(srv), input_len)
    if isinstance(window, (tuple, str)):
        window = signal.get_window(window, input_len)
    P = (block_sums_truth_fft if fast else block_sums_truth)(ref, srv, range_bins, freq_bins, window, short_filt)
    X = np.fft.fftshift(np.fft.fft(P, axis=0), axes=0)
    return X[:, :, None]


def frame_truth(ref, srv, filter_len, reg, peek, range_bins, freq_bins, window=None):
    """float64 frame: ``ls_filter_truth`` (circular LS filter), then the map of the float64 cleaned channel.  Returns
    (map [F, R+1], taps, cleaned) in complex128."""
    from .clutter_oracle import ls_filter_truth
    cleaned, taps = ls_filter_truth(ref, srv, filter_len, reg, peek)
    amb = fast_xambg_truth(np.asarray(ref, dtype=np.complex128), cleaned, range_bins, freq_bins, None, window, fast=True)
    return amb[:, :, 0], taps, cleaned


def rel_inf(a, b):
    """max|a-b| / max|b| -- the parity metric of SURVEY.md section 8d."""
    a = np.asarray(a)
    b = np.asarray(b)
    den = np.abs(b).max()
    return float(np.abs(a - b).max() / den) if den > 0 else float(np.abs(a - b).max())
