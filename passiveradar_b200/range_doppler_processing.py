"""Cross-ambiguity function on the H100 -- same call signature as the reference.

Drop-in for ``passiveRadar.range_doppler_processing.fast_xambg``
(reference ``passiveRadar/range_doppler_processing.py:12-90``).  The host side
here only mirrors the reference's argument handling (shape check ``:46-49``,
zero padding ``:52-55``, named windows ``:57-58``, decimator choice ``:69-78``);
all arithmetic runs in ``libprcore.so`` (``prc_xambg_c64``).  There is no CPU
fallback.
"""
from __future__ import annotations

import numpy as np
import scipy.signal as signal

from . import _lib


def _prepare(refChannel, srvChannel, inputLen):
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if refChannel.shape != srvChannel.shape:
        print(refChannel.shape)
        print(srvChannel.shape)
        raise ValueError('Input vectors must have the same length')
    ref = _lib.as_c64(refChannel, "refChannel")
    srv = _lib.as_c64(srvChannel, "srvChannel")
    if inputLen is not None and ref.shape[0] != inputLen:
        # np.pad raises for a negative pad width, exactly like the reference does for
        # inputs longer than inputLen
        padding = inputLen - ref.shape[0]
        ref = np.pad(ref, (0, padding), mode='constant')
        srv = np.pad(srv, (0, padding), mode='constant')
    return ref, srv


def _window_array(window, inputLen, n):
    if window is None:
        return None
    if isinstance(window, (tuple, str)):
        window = signal.get_window(window, inputLen)
    w = np.ascontiguousarray(np.asarray(window), dtype=np.float64)
    if w.shape != (n,):
        # the reference would fail inside ``channelProduct *= window`` (broadcast error)
        raise ValueError(f"operands could not be broadcast together with shapes ({n},) {w.shape}")
    return w


def fast_xambg(refChannel, srvChannel, rangeBins, freqBins, inputLen=None, window=None,
               shortFilt=True, *, device=None):
    '''Fast Cross-Ambiguity Fuction (frequency domain method), computed on the GPU.

    Args / returns exactly as the reference: ``ndarray`` of shape
    ``(freqBins, rangeBins + 1, 1)``, complex64; axis 0 is fftshift-ed Doppler,
    column ``k`` is bistatic delay ``rangeBins - k`` samples.
    '''
    ref, srv = _prepare(refChannel, srvChannel, inputLen)
    n = ref.shape[0]
    rangeBins = int(rangeBins)
    freqBins = int(freqBins)
    w = _window_array(window, inputLen, n)
    ndecim = int(n / freqBins)
    dtaps = None
    if not shortFilt and ndecim > 1:
        # flat-top decimator of the reference (:73-76); for ndecim == 1 SciPy's resample_poly
        # returns its input whatever the taps are
        dtaps = np.ascontiguousarray(signal.firwin(10 * ndecim + 1, 1. / ndecim, window='flattop'),
                                     dtype=np.float64)
    out = np.empty((freqBins, rangeBins + 1, 1), dtype=np.complex64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    st = lib.prc_xambg_c64(ref.ctypes.data, srv.ctypes.data, n, rangeBins, freqBins,
                           None if w is None else w.ctypes.data,
                           None if dtaps is None else dtaps.ctypes.data,
                           0 if dtaps is None else dtaps.shape[0],
                           out.ctypes.data, _lib.MEM_HOST, dev, None, 0)
    _lib.check(st)
    return out


def direct_xambg(refChannel, srvChannel, rangeBins, freqBins, sampleRate, *, device=None):
    ''' Direct Cross-Ambiguity Fuction (time domain method), computed on the GPU.

    Args / returns as the reference (``range_doppler_processing.py:93-124``): per Doppler bin the
    reference channel is frequency-shifted (float32 phase ramp, as ``frequency_shift`` does) and linearly
    cross-correlated with the surveillance channel; ``ndarray`` of shape ``(freqBins, rangeBins + 1, 1)``.
    '''
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if refChannel.shape != srvChannel.shape:
        raise ValueError('Input vectors must have the same length')
    ref = _lib.as_c64(refChannel, "refChannel")
    srv = _lib.as_c64(srvChannel, "srvChannel")
    rangeBins, freqBins = int(rangeBins), int(freqBins)
    out = np.empty((freqBins, rangeBins + 1, 1), dtype=np.complex64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    _lib.check(lib.prc_direct_xambg_c64(ref.ctypes.data, srv.ctypes.data, ref.shape[0], rangeBins, freqBins,
                                        float(sampleRate), out.ctypes.data, _lib.MEM_HOST, dev, None, 0))
    return out
