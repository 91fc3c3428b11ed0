"""Adaptive clutter cancellers on the H100 -- same call signatures as the reference.

Drop-ins for ``passiveRadar.clutter_removal.LS_Filter`` (reference
``passiveRadar/clutter_removal.py:6-56``) and ``NLMS_filter`` (``:189-249``), plus
``block_NLMS`` (not in the reference; DESIGN.md defines it so that ``blockLen=1``
is ``NLMS_filter``).  All arithmetic runs in ``libprcore.so``; no CPU fallback.
"""
from __future__ import annotations

import numpy as np

from . import _lib


def _pair(refChannel, srvChannel, check=True):
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if check and refChannel.shape != srvChannel.shape:
        raise ValueError('Input vectors must have the same length')
    return _lib.as_c64(refChannel, "refChannel"), _lib.as_c64(srvChannel, "srvChannel")


def LS_Filter(refChannel, srvChannel, filterLen, reg=1.0, peek=10, return_filter=False, *, device=None):
    '''Block least squares adaptive filter (direct matrix inversion semantics).

    Same parameters and returns as the reference: ``srvChannelFiltered`` (complex64) and,
    with ``return_filter=True``, the ``filterLen + peek`` taps.  The Gram matrix the
    reference forms explicitly (N x M data matrix, 2.6 GB at N=2**20, M=310) is Hermitian
    Toeplitz; the GPU computes its first column and the right-hand side as lag
    correlations, solves in float64 and applies the circular FIR.
    '''
    ref, srv = _pair(refChannel, srvChannel)
    filterLen = int(filterLen)
    peek = int(peek)
    n = ref.shape[0]
    ntaps = filterLen + peek
    out = np.empty(n, dtype=np.complex64)
    taps = np.empty(max(ntaps, 0), dtype=np.complex64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    st = lib.prc_ls_filter_c64(ref.ctypes.data, srv.ctypes.data, n, filterLen, peek, float(reg),
                               out.ctypes.data, taps.ctypes.data, _lib.MEM_HOST, dev, None, 0)
    _lib.check(st)
    if return_filter:
        return out, taps
    return out


def _nlms(refChannel, srvChannel, filterLen, mu, peek, blockLen, initialTaps, returnFilter, device):
    # NLMS_filter performs no shape check (clutter_removal.py:189-249); it indexes srv by
    # position, so only require ref to be long enough
    ref, srv = _pair(refChannel, srvChannel, check=False)
    peek = int(peek)
    init = None
    if initialTaps is not None:
        init = _lib.as_c64(initialTaps, "initialTaps")
        filterLen = init.shape[0] - peek          # clutter_removal.py:221-225
    filterLen = int(filterLen)
    n = srv.shape[0]
    if ref.shape[0] < n:
        raise IndexError(f"refChannel ({ref.shape[0]}) is shorter than srvChannel ({n})")
    ntaps = filterLen + peek
    out = np.empty(n, dtype=np.complex64)
    taps = np.empty(max(ntaps, 0), dtype=np.complex64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    st = lib.prc_nlms_c64(ref.ctypes.data, srv.ctypes.data, n, filterLen, peek, float(mu), int(blockLen),
                          None if init is None else init.ctypes.data, out.ctypes.data, taps.ctypes.data,
                          _lib.MEM_HOST, dev, None, 0)
    _lib.check(st)
    if returnFilter:
        return out, taps
    return out


def NLMS_filter(refChannel, srvChannel, filterLen, mu, peek=10, initialTaps=None, returnFilter=False,
                *, device=None):
    '''Normalized least mean square (NLMS) adaptive filter -- reference semantics, sample-serial.'''
    return _nlms(refChannel, srvChannel, filterLen, mu, peek, 1, initialTaps, returnFilter, device)


def block_NLMS(refChannel, srvChannel, filterLen, mu, peek=10, blockLen=64, initialTaps=None,
               returnFilter=False, *, device=None):
    '''Block NLMS: taps frozen inside each block of ``blockLen`` samples, the per-sample
    normalised gradients of the block are summed and applied at its end.  ``blockLen=1`` is
    ``NLMS_filter``.  Not part of the reference (see DESIGN.md).'''
    if int(blockLen) < 1:
        raise ValueError("blockLen must be >= 1")
    return _nlms(refChannel, srvChannel, filterLen, mu, peek, blockLen, initialTaps, returnFilter, device)


def LS_Filter_Toeplitz(refChannel, srvChannel, filterLen, peek=10, return_filter=False, *, device=None):
    '''Block least squares adaptive filter, Toeplitz (Levinson) formulation -- the variant ``main.py``
    runs.  Same parameters as the reference (``clutter_removal.py:109-160``); like the reference it
    returns complex128 (the GPU computes in complex64 with a float64 solve and widens the result).'''
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if refChannel.shape != srvChannel.shape:
        raise ValueError(f'Input vectors must have the same length - got {refChannel.shape} and {srvChannel.shape}')
    ref = _lib.as_c64(refChannel, "refChannel")
    srv = _lib.as_c64(srvChannel, "srvChannel")
    filterLen, peek = int(filterLen), int(peek)
    n = ref.shape[0]
    out = np.empty(n, dtype=np.complex64)
    taps = np.empty(max(filterLen + peek, 0), dtype=np.complex64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    st = lib.prc_ls_toeplitz_c64(ref.ctypes.data, srv.ctypes.data, n, filterLen, peek, out.ctypes.data,
                                 taps.ctypes.data, _lib.MEM_HOST, dev, None, 0)
    _lib.check(st)
    if return_filter:
        return out.astype(np.complex128), taps.astype(np.complex128)
    return out.astype(np.complex128)


def LS_Filter_Multiple(refChannel, srvChannel, filterLen, sampleRate, dopplerBins=[0], *, device=None):
    '''Clutter removal with the Toeplitz least squares filter applied over several Doppler bins
    (reference ``clutter_removal.py:162-187``; ``main.py:169-176`` calls it with [0, 1, -1, 2, -2]).
    All bins run back to back on the GPU; the residual never leaves the device between bins.'''
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if refChannel.shape != srvChannel.shape:
        raise ValueError(f'Input vectors must have the same length - got {refChannel.shape} and {srvChannel.shape}')
    ref = _lib.as_c64(refChannel, "refChannel")
    srv = _lib.as_c64(srvChannel, "srvChannel")
    bins = np.ascontiguousarray(list(dopplerBins), dtype=np.float64)
    if bins.shape[0] == 0:
        return srvChannel                    # the reference's loop body never runs
    n = ref.shape[0]
    out = np.empty(n, dtype=np.complex64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    st = lib.prc_ls_multiple_c64(ref.ctypes.data, srv.ctypes.data, n, int(filterLen), 10, float(sampleRate),
                                 bins.ctypes.data, bins.shape[0], out.ctypes.data, None, _lib.MEM_HOST, dev, None, 0)
    _lib.check(st)
    return out.astype(np.complex128)
