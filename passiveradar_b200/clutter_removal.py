"""Adaptive clutter cancellers on the H100 -- same call signatures as the reference.

Drop-ins for ``passiveRadar.clutter_removal.LS_Filter`` (reference
``passiveRadar/clutter_removal.py:6-56``), ``NLMS_filter`` (``:189-249``) and ``GAL_JPE``
(``:251-364``; ``gal_jpe_frames`` runs a batch of frames in one call), ``LS_Filter_SVD`` (``:58-107``;
``ls_filter_svd_frames`` likewise), plus
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
    dev = _lib.current_device(device)
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
    dev = _lib.current_device(device)
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


def _gal_args(latticeLen, delayLineLen, peek):
    latticeLen, delayLineLen, peek = int(latticeLen), int(delayLineLen), int(peek)
    if latticeLen > delayLineLen:
        raise ValueError("Delay line order must be greater than or equal to the lattice filter order")
    if latticeLen < 1:
        raise ValueError(f"latticeLen must be >= 1, got {latticeLen}")
    if peek < 0:
        raise ValueError(f"peek must be >= 0, got {peek}")
    return latticeLen, delayLineLen, peek


def GAL_JPE(refChannel, srvChannel, latticeLen, delayLineLen, mu1, mu2, peek=10, return_filter=False, *, device=None):
    '''Gradient adaptive lattice joint process estimator -- reference semantics, sample-serial.

    A lattice of ``latticeLen`` stages (gradient-adaptive reflection coefficients, step size ``mu1``,
    ballpark 1e-3) whitens the reference channel; its ``delayLineLen`` backward prediction errors (the
    stages beyond ``latticeLen`` are a plain delay line) feed an NLMS transversal filter (step size
    ``mu2``, ballpark 1e-2).  ``peek`` non-causal taps: sample n uses ``refChannel[n + peek]``.  As in the
    reference, ``mu1`` adapts itself (``min(0.999 mu1 + 1e-8 e**2, 5e-3)``).

    Returns ``srvChannelFiltered`` (complex64; the last ``peek + 1`` samples are zero) and, with
    ``return_filter=True``, the final reflection coefficients ``k`` and transversal taps ``h``
    (``delayLineLen`` complex64 values each).  Raises ``ValueError`` on a shape mismatch, on
    ``latticeLen > delayLineLen`` and on ``latticeLen < 1``.

    The inputs are rounded to complex64 first; ``mu1`` and ``mu2`` are taken as Python floats.  The reference's
    arithmetic widens to complex128 part-way through the loop when it is handed complex128 channels; this one stays
    complex64 with the reference's complex64 rounding points.  Delay lines up to 4096 taps.
    '''
    ref, srv = _pair(refChannel, srvChannel)
    latticeLen, delayLineLen, peek = _gal_args(latticeLen, delayLineLen, peek)
    n = ref.shape[0]
    out = np.empty(n, dtype=np.complex64)
    k = np.empty(delayLineLen, dtype=np.complex64)
    h = np.empty(delayLineLen, dtype=np.complex64)
    if n == 0:
        k[:] = 0
        h[:] = 0
    else:
        lib = _lib.load()
        dev = _lib.current_device(device)
        st = lib.prc_gal_jpe_frames_c64(ref.ctypes.data, srv.ctypes.data, n, 1, n, latticeLen, delayLineLen,
                                        float(mu1), float(mu2), peek, out.ctypes.data, k.ctypes.data, h.ctypes.data,
                                        _lib.MEM_HOST, dev, None, 0)
        _lib.check(st)
    if return_filter:
        return out, k, h
    return out


def gal_jpe_frames(ref_frames, srv_frames, latticeLen, delayLineLen, mu1, mu2, peek=10, return_filter=False, *,
                   device=None):
    '''``GAL_JPE`` on a batch of independent frames in one library call: row i of the 2-D host arrays
    ``ref_frames`` / ``srv_frames`` (nframes x n) is one frame.  The recurrence of a frame is serial, so a single
    frame occupies one warp (delay lines up to 256 taps) or one CTA of the GPU; a batch of frames is what fills it.

    Returns ``out`` (nframes x n complex64) and, with ``return_filter=True``, ``k`` and ``h``
    (nframes x delayLineLen complex64).  Row i equals ``GAL_JPE(ref_frames[i], srv_frames[i], ...)`` bit for bit.
    '''
    ref = np.asarray(ref_frames)
    srv = np.asarray(srv_frames)
    if ref.ndim != 2:
        raise ValueError(f"ref_frames must be two-dimensional (nframes x n), got shape {ref.shape}")
    if ref.shape != srv.shape:
        raise ValueError('Input vectors must have the same length')
    latticeLen, delayLineLen, peek = _gal_args(latticeLen, delayLineLen, peek)
    ref = np.ascontiguousarray(ref, dtype=np.complex64)
    srv = np.ascontiguousarray(srv, dtype=np.complex64)
    nframes, n = ref.shape
    out = np.zeros((nframes, n), dtype=np.complex64)
    k = np.zeros((nframes, delayLineLen), dtype=np.complex64)
    h = np.zeros((nframes, delayLineLen), dtype=np.complex64)
    if nframes > 0 and n > 0:
        lib = _lib.load()
        dev = _lib.current_device(device)
        st = lib.prc_gal_jpe_frames_c64(ref.ctypes.data, srv.ctypes.data, n, nframes, n, latticeLen, delayLineLen,
                                        float(mu1), float(mu2), peek, out.ctypes.data, k.ctypes.data, h.ctypes.data,
                                        _lib.MEM_HOST, dev, None, 0)
        _lib.check(st)
    if return_filter:
        return out, k, h
    return out


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
    dev = _lib.current_device(device)
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
    dev = _lib.current_device(device)
    st = lib.prc_ls_multiple_c64(ref.ctypes.data, srv.ctypes.data, n, int(filterLen), 10, float(sampleRate),
                                 bins.ctypes.data, bins.shape[0], out.ctypes.data, None, _lib.MEM_HOST, dev, None, 0)
    _lib.check(st)
    return out.astype(np.complex128)


def _svd_args(filterLen, peek):
    filterLen, peek = int(filterLen), int(peek)
    if filterLen < 0:
        raise ValueError(f"filterLen must be >= 0, got {filterLen}")
    if peek < 0:
        raise ValueError(f"peek must be >= 0, got {peek}")
    return filterLen, peek


def _ls_svd(ref, srv, filterLen, peek, device):
    """2-D complex64 (nframes x n) -> out (nframes x n), taps (nframes x M) complex64 and ranks (int32)."""
    nframes, n = ref.shape
    ntaps = filterLen + peek
    out = np.empty((nframes, n), dtype=np.complex64)
    taps = np.zeros((nframes, ntaps), dtype=np.complex64)
    rank = np.zeros(nframes, dtype=np.int32)
    if ntaps == 0 or nframes == 0:
        out[...] = srv
        return out, taps, rank
    if n == 0:
        return out, taps, rank
    lib = _lib.load()
    dev = _lib.current_device(device)
    st = lib.prc_ls_svd_frames_c64(ref.ctypes.data, srv.ctypes.data, n, nframes, n, filterLen, peek, out.ctypes.data,
                                   taps.ctypes.data, rank.ctypes.data, _lib.MEM_HOST, dev, None, 0)
    _lib.check(st)
    return out, taps, rank


def LS_Filter_SVD(refChannel, srvChannel, filterLen, peek=10, return_filter=False, *, device=None):
    '''Block least squares adaptive filter through the singular value decomposition -- the reference's
    ``LS_Filter_SVD`` (``clutter_removal.py:58-107``), which "doesn't get upset if the data matrix is close to
    singular": a silent, single-carrier or periodic reference channel, where ``LS_Filter(reg=0)`` raises
    ``LinAlgError`` and ``LS_Filter_Toeplitz`` fails.

    The taps are the minimum-norm least-squares solution of ``A taps = srv``, ``A[:, k] = roll(ref, k - peek)``
    (``filterLen + peek`` columns, at most 1024).  The GPU never forms ``A``: it decomposes the Hermitian Toeplitz
    Gram matrix ``A^H A`` in float64 (Householder tridiagonalisation and implicit-shift QL) and drops singular value
    ``S_k`` when ``S_k < max(1e-10, 1e-5 * S_max)``.  The reference drops ``S_k < 1e-10`` only; going through the
    Gram matrix squares the condition number, so a null direction of ``A`` shows up at ~1e-8 ``S_max`` even in
    float64, and the relative floor is what separates it (DESIGN.md section 13).  The residual
    ``srv - A @ taps`` is accumulated in float64 and rounded once.

    ``refChannel`` is rounded to complex64, as the reference's ``A`` is, and ``srvChannel`` is sent to the GPU as
    complex64.  ``srvChannelFiltered`` and, with ``return_filter=True``, the taps come back in
    ``np.result_type(np.complex64, srvChannel.dtype)`` as the reference's do; for complex128 / float64 inputs the
    result is widened, so the complex64 rounding of ``srvChannel`` is the only extra error.

    Raises ``ValueError`` on a shape mismatch or a negative ``filterLen`` / ``peek``, and
    ``np.linalg.LinAlgError("SVD did not converge")`` on non-finite input, as NumPy does.
    '''
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if refChannel.shape != srvChannel.shape:
        raise ValueError('Input vectors must have the same length')
    filterLen, peek = _svd_args(filterLen, peek)
    rt = np.result_type(np.complex64, srvChannel.dtype)
    if filterLen + peek == 0:                  # no columns: the reference subtracts nothing
        out, taps = srvChannel.astype(rt), np.zeros(0, dtype=rt)
    else:
        ref = _lib.as_c64(refChannel, "refChannel")
        srv = _lib.as_c64(srvChannel, "srvChannel")
        o, t, rank = _ls_svd(ref[None], srv[None], filterLen, peek, device)
        if rank[0] < 0:
            raise np.linalg.LinAlgError("SVD did not converge")
        out, taps = o[0].astype(rt, copy=False), t[0].astype(rt, copy=False)
    if return_filter:
        return out, taps
    return out


def ls_filter_svd_frames(ref_frames, srv_frames, filterLen, peek=10, return_filter=False, *, return_rank=False,
                         device=None):
    '''``LS_Filter_SVD`` on a batch of independent frames in one library call: row i of the 2-D host arrays
    ``ref_frames`` / ``srv_frames`` (nframes x n) is one frame.  One CTA decomposes each frame's Gram matrix, so a
    batch of frames is what fills the GPU.

    Returns ``out`` (nframes x n) and, with ``return_filter=True``, the taps (nframes x (filterLen + peek)), in
    ``np.result_type(np.complex64, srv_frames.dtype)``; row i equals ``LS_Filter_SVD(ref_frames[i], srv_frames[i],
    ...)`` bit for bit.  With ``return_rank=True`` the number of kept singular values of every frame comes last; a
    frame with non-finite input then reports -1 (its row is NaN) instead of raising ``LinAlgError``.
    '''
    ref = np.asarray(ref_frames)
    srv = np.asarray(srv_frames)
    if ref.ndim != 2:
        raise ValueError(f"ref_frames must be two-dimensional (nframes x n), got shape {ref.shape}")
    if ref.shape != srv.shape:
        raise ValueError('Input vectors must have the same length')
    filterLen, peek = _svd_args(filterLen, peek)
    rt = np.result_type(np.complex64, srv.dtype)
    out, taps, rank = _ls_svd(np.ascontiguousarray(ref, dtype=np.complex64), np.ascontiguousarray(srv, dtype=np.complex64),
                              filterLen, peek, device)
    if filterLen + peek == 0:
        out = srv.astype(rt)
    if not return_rank and (rank < 0).any():
        raise np.linalg.LinAlgError("SVD did not converge")
    res = (out.astype(rt, copy=False),)
    if return_filter:
        res += (taps.astype(rt, copy=False),)
    if return_rank:
        res += (rank,)
    return res[0] if len(res) == 1 else res
