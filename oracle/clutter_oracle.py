"""Oracle for the clutter cancellers (TEST INFRASTRUCTURE ONLY, see oracle/__init__.py).

``ls_filter_oracle``   follows ``LS_Filter``, reference
                       ``passiveRadar/clutter_removal.py:6-56``:
                       :31 lags = -peek .. filterLen-1, :34-36 A[:,k] = roll(ref, lags[k]),
                       :39 Gram A^H A, :42-45 Tikhonov solve, :51 srv - A @ taps.
                       All arithmetic stays complex64 (OpenBLAS cgemm/cgemv, LAPACK cgesv)
                       exactly as in the reference.
``nlms_filter_oracle`` follows ``NLMS_filter`` (``:189-249``, update rule ``:211-215``).
``block_nlms_oracle``  DEFINES ``block_NLMS``.  The reference has no such function
                       (``grep -rn NLMS`` finds only ``NLMS_filter`` and ``GAL_JPE``), so for
                       ``blockLen > 1`` parity is unpinned; ``blockLen == 1`` is pinned to
                       ``NLMS_filter`` by tests/test_oracle_golden.py.
``*_truth``            float64 evaluations of the same formulas.
"""
from __future__ import annotations

import numpy as np


def _same_length(ref, srv):
    if ref.shape != srv.shape:
        raise ValueError('Input vectors must have the same length')


# --------------------------------------------------------------------------- LS

def ls_filter_oracle(refChannel, srvChannel, filterLen, reg=1.0, peek=10, return_filter=False):
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    _same_length(refChannel, srvChannel)
    n = refChannel.shape[0]
    ntaps = filterLen + peek
    # column k of the data matrix is the reference delayed (circularly) by k - peek samples
    delays = np.arange(ntaps) - peek
    data = np.zeros((n, ntaps), dtype=np.complex64)
    for col, dly in enumerate(delays):
        data[:, col] = np.roll(refChannel, dly)
    data_h = data.conj().T
    gram = data_h @ data
    ridge = np.eye(ntaps, dtype=np.complex64) * reg
    taps = np.linalg.solve(gram + ridge, data_h @ srvChannel)
    cleaned = srvChannel - data @ taps
    return (cleaned, taps) if return_filter else cleaned


def ls_filter_truth(ref, srv, filter_len, reg=1.0, peek=10):
    """float64 LS_Filter via the circulant identities of SURVEY.md section 3.3.

    Gram[a,b] = c[(a-b) mod N],  c[m] = sum_i conj(ref[i]) ref[(i+m) mod N]
    rhs[a]    = x[(a-peek) mod N], x[m] = sum_i conj(ref[i]) srv[(i+m) mod N]
    Returns (cleaned, taps) in complex128.
    """
    import scipy.linalg as sla
    ref = np.asarray(ref, dtype=np.complex128)
    srv = np.asarray(srv, dtype=np.complex128)
    _same_length(ref, srv)
    n = ref.shape[0]
    m = filter_len + peek
    fr = np.fft.fft(ref)
    c = np.fft.ifft(np.conj(fr) * fr)
    x = np.fft.ifft(np.conj(fr) * np.fft.fft(srv))
    col = c[np.arange(m) % n].copy()
    row = np.conj(col)
    gram = sla.toeplitz(col, row)
    rhs = x[(np.arange(m) - peek) % n]
    taps = np.linalg.solve(gram + reg * np.eye(m), rhs)
    h = np.zeros(n, dtype=np.complex128)
    h[(np.arange(m) - peek) % n] += taps     # clutter[i] = sum_k taps[k] ref[i - (k - peek)]
    clutter = np.fft.ifft(fr * np.fft.fft(h))
    return srv - clutter, taps


# ------------------------------------------------------------------------- NLMS

def nlms_filter_oracle(refChannel, srvChannel, filterLen, mu, peek=10, initialTaps=None,
                       returnFilter=False):
    """Sample-serial NLMS in complex64, one Python iteration per sample (slow: ~8 us/sample)."""
    return block_nlms_oracle(refChannel, srvChannel, filterLen, mu, peek=peek, blockLen=1,
                             initialTaps=initialTaps, returnFilter=returnFilter)


def block_nlms_oracle(refChannel, srvChannel, filterLen, mu, peek=10, blockLen=1,
                      initialTaps=None, returnFilter=False):
    """Block NLMS.  Definition (ours; DESIGN.md "block_NLMS"):

    With M = filterLen + peek taps w and the regressor u_n[j] = ref[n + peek - j], j = 0..M-1,
    for desired-sample index n = filterLen .. N - peek - 1, processed in consecutive blocks of
    ``blockLen`` samples:

        e_n = srv[n] - w^H u_n                      (w frozen inside a block)
        w  <- w + mu * sum_{n in block} u_n conj(e_n) / (u_n^H u_n)     (at block end)

    The final block may be shorter.  out[n] = e_n, out[:filterLen] = out[N-peek:] = 0.
    ``blockLen == 1`` is exactly the recurrence of the reference's ``NLMS_filter``.
    """
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if initialTaps is None:
        w = np.zeros((filterLen + peek,), dtype=np.complex64)
    else:
        w = initialTaps
        filterLen = initialTaps.shape[0] - peek
    ntaps = filterLen + peek
    n = srvChannel.shape[0]
    out = np.zeros(srvChannel.shape, dtype=np.complex64)
    nsteps = n - filterLen - peek
    k = 0
    while k < nsteps:
        kend = min(nsteps, k + blockLen)
        grad = None
        for kk in range(k, kend):
            # u[j] = ref[ntaps + kk - j]
            u = refChannel[kk + 1: kk + ntaps + 1][::-1]
            e = srvChannel[kk + filterLen] - w.conj() @ u
            step = mu * u * e.conj() / (u.conj() @ u)
            grad = step if grad is None else grad + step
            out[filterLen + kk] = e
        w = w + grad
        k = kend
    return (out, w) if returnFilter else out


def block_nlms_truth(ref, srv, filter_len, mu, peek=10, block_len=1, initial_taps=None):
    """float64 version of ``block_nlms_oracle`` (vectorised per block). Returns (out, w)."""
    ref = np.asarray(ref, dtype=np.complex128)
    srv = np.asarray(srv, dtype=np.complex128)
    if initial_taps is None:
        w = np.zeros(filter_len + peek, dtype=np.complex128)
    else:
        w = np.asarray(initial_taps, dtype=np.complex128).copy()
        filter_len = w.shape[0] - peek
    ntaps = filter_len + peek
    n = srv.shape[0]
    out = np.zeros(n, dtype=np.complex128)
    nsteps = n - filter_len - peek
    from numpy.lib.stride_tricks import sliding_window_view
    if nsteps <= 0:
        return out, w
    win = sliding_window_view(ref, ntaps)       # win[s, t] = ref[s + t]
    for k in range(0, nsteps, block_len):
        kend = min(nsteps, k + block_len)
        # u_kk[j] = ref[kk + ntaps - j] = win[kk + 1, ntaps - 1 - j]
        U = win[k + 1: kend + 1, ::-1]          # (B, ntaps)
        e = srv[k + filter_len: kend + filter_len] - U @ np.conj(w)
        nrm = np.einsum('bj,bj->b', np.conj(U), U).real
        w = w + mu * (U * (np.conj(e) / nrm)[:, None]).sum(axis=0)
        out[k + filter_len: kend + filter_len] = e
    return out, w


# ------------------------------------------------------------------ plain-C NLMS (fast oracle)

def block_nlms_oracle_c(ref, srv, filter_len, mu, peek=10, block_len=1, initial_taps=None):
    """Same recurrence as ``block_nlms_oracle`` in plain C (oracle/nlms_oracle.c), complex float
    arithmetic; ~100x faster than the Python loop.  Returns (out, taps)."""
    import ctypes as C
    from . import build as _b
    lib = C.CDLL(_b.build())
    fn = lib.nlms_oracle_c64
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_float, C.c_int,
                   C.c_void_p, C.c_void_p, C.c_void_p]
    ref = np.ascontiguousarray(ref, dtype=np.complex64)
    srv = np.ascontiguousarray(srv, dtype=np.complex64)
    init = None
    if initial_taps is not None:
        init = np.ascontiguousarray(initial_taps, dtype=np.complex64)
        filter_len = init.shape[0] - peek
    m = filter_len + peek
    out = np.empty(srv.shape[0], dtype=np.complex64)
    taps = np.empty(m, dtype=np.complex64)
    st = fn(ref.ctypes.data, srv.ctypes.data, srv.shape[0], filter_len, peek, mu, block_len,
            None if init is None else init.ctypes.data, out.ctypes.data, taps.ctypes.data)
    if st != 0:
        raise MemoryError("nlms_oracle_c64 failed")
    return out, taps


def block_nlms_truth_c(ref, srv, filter_len, mu, peek=10, block_len=1, initial_taps=None):
    """The recurrence of ``block_nlms_oracle`` with every operation in float64 (oracle/nlms_oracle.c,
    ``nlms_truth_c128``): how far the complex64 reference is from the exact recurrence.  Returns
    (out, taps) as complex128."""
    import ctypes as C
    from . import build as _b
    lib = C.CDLL(_b.build())
    fn = lib.nlms_truth_c128
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_double, C.c_int,
                   C.c_void_p, C.c_void_p, C.c_void_p]
    ref = np.ascontiguousarray(ref, dtype=np.complex64)
    srv = np.ascontiguousarray(srv, dtype=np.complex64)
    init = None
    if initial_taps is not None:
        init = np.ascontiguousarray(initial_taps, dtype=np.complex64)
        filter_len = init.shape[0] - peek
    m = filter_len + peek
    out = np.empty(srv.shape[0], dtype=np.complex128)
    taps = np.empty(m, dtype=np.complex128)
    st = fn(ref.ctypes.data, srv.ctypes.data, srv.shape[0], filter_len, peek, float(mu), block_len,
            None if init is None else init.ctypes.data, out.ctypes.data, taps.ctypes.data)
    if st != 0:
        raise MemoryError("nlms_truth_c128 failed")
    return out, taps


# ------------------------------------------------------------ LS_Filter_Toeplitz / LS_Filter_Multiple
# (SURVEY.md section 8f rank 1: the clutter filter main.py:169-176 actually calls)

def frequency_shift_oracle(x, fc, Fs, phase_offset=0):
    """``frequency_shift`` of the reference (passiveRadar/signal_utils.py:24-27).  Note the ramp is
    ``arange(..., dtype=complex64)``: the phase is evaluated in float32, which the GPU path mirrors."""
    nn = np.arange(x.shape[0], dtype=np.complex64)
    return x * np.exp(1j * 2 * np.pi * fc * nn / Fs + 1j * phase_offset)


def xcorr_oracle(s1, s2, nlead, nlag):
    """``xcorr`` of the reference (signal_utils.py:29-32): out[m] = sum_i s1[i] conj(s2[i - m + ...])."""
    import scipy.signal as signal
    return signal.correlate(s1, np.pad(s2, (nlag, nlead), mode='constant'), mode='valid')


def ls_filter_toeplitz_oracle(refChannel, srvChannel, filterLen, peek=10, return_filter=False):
    """Follows ``LS_Filter_Toeplitz`` (passiveRadar/clutter_removal.py:109-160): :139 roll by -peek,
    :142-147 linear (zero-padded) auto/cross correlations, :150 Levinson solve (scipy solve_toeplitz,
    complex128), :153-155 linear convolution and subtraction.  Returns complex128 like the reference."""
    from scipy.linalg import solve_toeplitz
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if refChannel.shape != srvChannel.shape:
        raise ValueError(f"Input vectors must have the same length - got {refChannel.shape} and {srvChannel.shape}")
    shifted = np.roll(refChannel, -1 * peek)
    ntaps = filterLen + peek
    acorr = xcorr_oracle(shifted, shifted, 0, ntaps - 1)
    xc = xcorr_oracle(srvChannel, shifted, 0, ntaps - 1)
    taps = solve_toeplitz(acorr, xc)
    clutter = np.convolve(shifted, taps, mode='full')[0:srvChannel.shape[0]]
    cleaned = srvChannel - clutter
    return (cleaned, taps) if return_filter else cleaned


def ls_filter_multiple_oracle(refChannel, srvChannel, filterLen, sampleRate, dopplerBins=[0]):
    """Follows ``LS_Filter_Multiple`` (clutter_removal.py:162-187)."""
    cleaned = srvChannel
    for doppler in dopplerBins:
        ref_k = refChannel if doppler == 0 else frequency_shift_oracle(refChannel, doppler, sampleRate)
        cleaned = ls_filter_toeplitz_oracle(ref_k, cleaned, filterLen)
    return cleaned


def nlms_block_exact(refChannel, srvChannel, filterLen, mu, peek=10, L=32, dtype=np.complex64):
    """The NLMS recurrence of the reference evaluated L samples at a time WITHOUT changing its values
    (the statement ``nlms_block_kernel`` implements; not ``block_NLMS``, whose taps are frozen in a block).

    With the taps W at the start of a block and g(m,k) = u_m^H u_k, p_m = g(m,m):
        r_k = d_k - W^H u_k
        e_k = r_k - mu * sum_{m<k} e_m g(m,k) / p_m          (forward substitution)
        W  <- W + mu * sum_m u_m conj(e_m) / p_m
    which is the sequential recurrence (clutter_removal.py:211-215) with w_k eliminated."""
    ref = np.asarray(refChannel).astype(dtype)
    srv = np.asarray(srvChannel).astype(dtype)
    M = filterLen + peek
    n = srv.shape[0]
    nsteps = n - M
    real = np.float32 if dtype == np.complex64 else np.float64
    W = np.zeros(M, dtype)
    out = np.zeros(n, dtype)
    k0 = 0
    while k0 < nsteps:
        Lb = min(L, nsteps - k0)
        U = np.stack([ref[k + 1: k + M + 1][::-1] for k in range(k0, k0 + Lb)], axis=1)      # M x Lb, column k = u_k
        r = srv[filterLen + k0: filterLen + k0 + Lb] - W.conj() @ U
        G = U.conj().T @ U
        p = G.diagonal().real.astype(real)
        e = np.zeros(Lb, dtype)
        for m in range(Lb):
            e[m] = r[m]
            if m + 1 < Lb:
                r[m + 1:] = r[m + 1:] - dtype(mu) * e[m] * G[m, m + 1:] / p[m]
        W = (W + (U * (dtype(mu) * e.conj() / p)[None, :]).sum(axis=1)).astype(dtype)
        out[filterLen + k0: filterLen + k0 + Lb] = e
        k0 += Lb
    return out, W
