"""Front-end signal utilities on the H100 -- same call signatures as the reference.

Drop-ins for ``passiveRadar.signal_utils.deinterleave_IQ`` (reference
``passiveRadar/signal_utils.py:19-22``), ``frequency_shift`` (``:24-27``) and ``resample``
(``:15-17``), the chain ``main.py:105-166`` runs on every input chunk, plus ``frontend`` which runs
the three in one pass on the device (raw IQ in, resampled complex64 out), and the channel-offset estimator
``find_channel_offset`` (``:73-78``) with ``offset_compensation`` (``:49-71``), ``shift`` (``:34-47``) and ``xcorr``
(``:29-32``).  All arithmetic runs in
``libprcore.so``; no CPU fallback.
"""
from __future__ import annotations

import functools
import math
import operator

import numpy as np

from . import _lib


def _is_weak(v):
    """Does ``v`` stay 'weak' in the reference's expression (NumPy 2 promotion)?  Python scalars do;
    so does ``np.float64`` there, because it subclasses ``float`` and ``1j*2*np.pi*fc`` /
    ``1j*phase_offset`` are evaluated by Python's ``complex.__mul__`` before NumPy sees them.
    Arrays (what main.py passes as phase_offset) and other NumPy scalar types are strong."""
    return isinstance(v, (bool, int, float, np.float32))


def _is_weak_divisor(v):
    """``array / Fs``: here NumPy does see the scalar, and a NumPy float64 scalar is strong."""
    return isinstance(v, (bool, int, float)) and not isinstance(v, np.generic)


def _raw_iq(interleavedIQ):
    """interleaved real array -> (buffer, in_kind, n complex samples); I = x[0:-1:2], Q = x[1::2]."""
    x = np.asarray(interleavedIQ)
    if x.ndim != 1:
        raise ValueError("interleaved IQ must be one-dimensional")
    n = x.shape[0] // 2
    x = x[:2 * n]
    if x.dtype == np.int8:
        return np.ascontiguousarray(x), _lib.IQ_I8, n
    if x.dtype == np.int16:
        return np.ascontiguousarray(x), _lib.IQ_I16, n
    return np.ascontiguousarray(x, dtype=np.float32), _lib.IQ_C64, n


def _mix_mode(fc, Fs, phase_offset):
    po = np.asarray(phase_offset)
    if po.size != 1:
        raise ValueError("phase_offset must be a scalar (or a one-element array, as main.py passes)")
    if np.iscomplexobj(po):
        raise TypeError("phase_offset must be real")
    if not _is_weak(fc):
        return _lib.MIX_F64, float(po.reshape(()))
    if not _is_weak_divisor(Fs):
        return _lib.MIX_FS64, float(po.reshape(()))
    if _is_weak(phase_offset):
        return _lib.MIX_C64, float(phase_offset)
    return _lib.MIX_C128, float(po.reshape(()))


def deinterleave_IQ(interleavedIQ, *, device=None):
    '''convert interleaved IQ samples to complex64'''
    buf, kind, n = _raw_iq(interleavedIQ)
    out = np.empty(n, dtype=np.complex64)
    if n == 0:
        return out
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    _lib.check(lib.prc_iq_mix_c64(buf.ctypes.data, kind, n, _lib.MIX_NONE, 0.0, 1.0, 0.0, out.ctypes.data,
                                  _lib.MEM_HOST, dev, None, 0))
    return out


def frequency_shift(x, fc, Fs, phase_offset=0, *, device=None):
    '''frequency shift x by fc where Fs is the sample rate of x

    The reference builds the phase ramp from ``arange(..., dtype=complex64)``, i.e. in float32; the
    device kernel reproduces that rounding (it is what the reference's output actually contains).
    Returns complex64 when the reference would (complex64 ``x``, Python-scalar arguments), else
    complex128 (the device result widened).'''
    x = np.asarray(x)
    if x.ndim != 1:
        raise ValueError("x must be one-dimensional")
    mode, po = _mix_mode(fc, Fs, phase_offset)
    xin = _lib.as_c64(x, "x")
    n = xin.shape[0]
    out = np.empty(n, dtype=np.complex64)
    if n:
        lib = _lib.load()
        dev = _lib.current_device() if device is None else int(device)
        _lib.check(lib.prc_iq_mix_c64(xin.ctypes.data, _lib.IQ_C64, n, mode, float(fc), float(Fs), po,
                                      out.ctypes.data, _lib.MEM_HOST, dev, None, 0))
    narrow = mode == _lib.MIX_C64 and x.dtype in (np.complex64, np.float32, np.float16)
    return out if narrow else out.astype(np.complex128)


@functools.lru_cache(maxsize=32)
def _resample_taps(up, dn, single):
    """The low-pass resample_poly designs (scipy/signal/_signaltools.py, resample_poly), times ``up``;
    float32-rounded first when the signal is complex64 (``h = asarray(h, dtype=x.dtype)``)."""
    from scipy.signal import firwin
    max_rate = max(up, dn)
    half_len = 10 * max_rate
    h = firwin(2 * half_len + 1, 1.0 / max_rate, window=('kaiser', 5.0))
    if single:
        h = (h.astype(np.float32) * np.float32(up)).astype(np.float64)
    else:
        h = h * up
    return np.ascontiguousarray(h, dtype=np.float64)


def _reduced(up, dn):
    if up != int(up):
        raise ValueError("up must be an integer")
    if dn != int(dn):
        raise ValueError("down must be an integer")
    up, dn = int(up), int(dn)
    if up < 1 or dn < 1:
        raise ValueError('up and down must be >= 1')
    g = math.gcd(up, dn)
    return up // g, dn // g


def _run_frontend(buf, kind, n, mode, fc, Fs, po, up, dn, single, device):
    h = _resample_taps(up, dn, single)
    n_out = n * up
    n_out = n_out // dn + bool(n_out % dn)
    out = np.empty(n_out, dtype=np.complex64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    _lib.check(lib.prc_frontend_c64(buf.ctypes.data, kind, n, mode, float(fc), float(Fs), po, up, dn,
                                    h.ctypes.data, h.shape[0], out.ctypes.data, n_out, _lib.MEM_HOST, dev, None, 0))
    return out


def resample(x, up, dn, *, device=None):
    '''rational resampling by a factor of up/dn  (scipy.signal.resample_poly(x, up, dn, padtype='line'))'''
    x = np.asarray(x)
    if x.ndim != 1:
        raise ValueError("x must be one-dimensional")
    up, dn = _reduced(up, dn)
    if up == dn == 1:
        return x.copy()
    if x.shape[0] == 0:
        raise ValueError("x must not be empty")
    single = x.dtype in (np.complex64, np.float32)
    out = _run_frontend(_lib.as_c64(x, "x"), _lib.IQ_C64, x.shape[0], _lib.MIX_NONE, 0.0, 1.0, 0.0, up, dn, single, device)
    if np.iscomplexobj(x):
        return out if x.dtype == np.complex64 else out.astype(np.complex128)
    return out.real.astype(x.dtype if x.dtype.kind == 'f' else np.float64)


def frontend(interleavedIQ, fc, Fs, phase_offset, up, dn, *, device=None):
    '''``resample(frequency_shift(deinterleave_IQ(interleavedIQ), fc, Fs, phase_offset), up, dn)`` in one
    pass on the device: the raw samples cross PCIe once (2 bytes per sample for int8 IQ) and only the
    resampled complex64 block comes back.  Not a reference function; it is the composition
    ``main.py:105-166`` applies to every chunk.'''
    buf, kind, n = _raw_iq(interleavedIQ)
    if n == 0:
        raise ValueError("interleavedIQ must hold at least one I/Q pair")
    mode, po = _mix_mode(fc, Fs, phase_offset)
    up, dn = _reduced(up, dn)
    if up == dn == 1:
        out = np.empty(n, dtype=np.complex64)
        lib = _lib.load()
        dev = _lib.current_device() if device is None else int(device)
        _lib.check(lib.prc_iq_mix_c64(buf.ctypes.data, kind, n, mode, float(fc), float(Fs), po, out.ctypes.data,
                                      _lib.MEM_HOST, dev, None, 0))
        return out
    # the reference chain is complex64 end to end only with Python-scalar arguments
    return _run_frontend(buf, kind, n, mode, fc, Fs, po, up, dn, mode == _lib.MIX_C64, device)


# ---- channel offset (reference signal_utils.py:29-78) ------------------------------------------------------------
_OFFSET_DTYPES = {np.dtype(np.int8): _lib.DT_I8, np.dtype(np.uint8): _lib.DT_U8, np.dtype(np.int16): _lib.DT_I16,
                  np.dtype(np.float32): _lib.DT_F32, np.dtype(np.float64): _lib.DT_F64,
                  np.dtype(np.complex64): _lib.DT_C64, np.dtype(np.complex128): _lib.DT_C128}
_PADLEN = 27


def _offset_input(x):
    """1-D contiguous array the library accepts natively, its dtype code, and whether decimate's filter is float32
    for it.  Other numeric dtypes are widened to float64 / complex128 here, as the reference upcasts them."""
    a = np.asarray(x)
    if a.ndim != 1:
        raise ValueError("the signals must be one-dimensional")
    single = a.dtype in (np.float32, np.complex64)
    if a.dtype not in _OFFSET_DTYPES:
        a = a.astype(np.complex128 if np.iscomplexobj(a) else np.float64)
    return np.ascontiguousarray(a), _OFFSET_DTYPES[a.dtype], single


@functools.lru_cache(maxsize=64)
def _decimate_sos(nd, single):
    """scipy.signal.decimate's IIR design for factor nd (cheby1(8, 0.05, 0.8 / nd) as sections) and its
    sosfilt_zi, both float32-rounded when the signal is float32 / complex64 (``sos = asarray(sos, dtype=x.dtype)``)."""
    from scipy.signal import cheby1, sosfilt_zi
    sos = cheby1(8, 0.05, 0.8 / nd, output='sos')
    if single:
        sos = sos.astype(np.float32)
    zi = sosfilt_zi(sos)
    return np.ascontiguousarray(sos, dtype=np.float64), np.ascontiguousarray(zi, dtype=np.float64)


def _pad_width(v):
    if not isinstance(v, (int, np.integer)) or isinstance(v, bool):
        raise TypeError("`pad_width` must be of integral type.")
    if v < 0:
        raise ValueError("index can't contain negative values")
    return int(v)


def _channel_offset(s1, s2, nd, nl, device=None, want_xc=False):
    """(offset, |xc| or None) of find_channel_offset; argument errors are raised before the library loads."""
    nd = operator.index(nd)
    if nd == 0:
        raise ZeroDivisionError("float division by zero")
    if nd < 0:
        raise ValueError("Digital filter critical frequencies must be 0 < Wn < 1")
    nl = _pad_width(nl)
    a1, d1, single1 = _offset_input(s1)
    a2, d2, single2 = _offset_input(s2)
    if min(a1.shape[0], a2.shape[0]) <= _PADLEN:
        raise ValueError(f"The length of the input vector x must be greater than padlen, which is {_PADLEN}.")
    sos = np.ascontiguousarray(np.stack([_decimate_sos(nd, single1)[0], _decimate_sos(nd, single2)[0]]))
    zi = np.ascontiguousarray(np.stack([_decimate_sos(nd, single1)[1], _decimate_sos(nd, single2)[1]]))
    n1d, n2d = -(-a1.shape[0] // nd), -(-a2.shape[0] // nd)
    xc = np.empty(abs(n1d - (n2d + 2 * nl)) + 1, dtype=np.float64) if want_xc else None
    off = np.zeros(1, dtype=np.int64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    _lib.check(lib.prc_channel_offset(a1.ctypes.data, d1, a1.shape[0], a2.ctypes.data, d2, a2.shape[0], nd, nl,
                                      sos.ctypes.data, zi.ctypes.data, off.ctypes.data,
                                      None if xc is None else xc.ctypes.data, _lib.MEM_HOST, dev, None, 0))
    return off[0], xc


def find_channel_offset(s1, s2, nd, nl, *, device=None):
    '''use cross-correlation to find channel offset in samples

    ``(argmax|correlate(decimate(s1, nd), pad(decimate(s2, nd), (nl, nl)), 'valid')| - nl) * nd`` as a NumPy integer,
    computed on the device in float64 / complex128 (scipy.signal.decimate's Chebyshev filter, zero phase).'''
    return _channel_offset(s1, s2, nd, nl, device)[0]


def shift(x, n):
    '''shift x by n samples, pad with zeros'''
    if n == 0:
        return x
    e = np.empty_like(x)
    k = min(abs(n), len(x))
    if n > 0:
        e[:k] = 0
        e[k:] = x[:len(x) - k]
    else:
        e[len(x) - k:] = 0
        e[:len(x) - k] = x[k:]
    return e


def offset_compensation(x1, x2, ns, ndec, nlag=2000, *, device=None):
    '''Find and correct a constant time offset between two signals using a cross-correlation

    The offset is found on the first ``ns`` samples (find_channel_offset(x1[:ns], x2[:ns], ndec, nlag)); returns x2
    shifted by it with zeros at the edges, or x2 itself when the offset is 0.'''
    os_ = find_channel_offset(x1[0:int(ns)], x2[0:int(ns)], ndec, nlag, device=device)
    return x2 if os_ == 0 else shift(x2, os_)


def xcorr(s1, s2, nlead, nlag, *, device=None):
    ''' cross-correlate s1 and s2 with sample offsets from -1*nlag to nlead

    correlate(s1, pad(s2, (nlag, nlead)), 'valid') in complex128 / float64 on the device, returned in the dtype the
    reference returns (integer results rounded, and wrapped to the input's width, as SciPy does).'''
    nlag, nlead = _pad_width(nlag), _pad_width(nlead)
    a1, d1, _ = _offset_input(s1)
    a2, d2, _ = _offset_input(s2)
    if a1.shape[0] == 0 or a2.shape[0] == 0:
        raise ValueError("xcorr needs non-empty signals")
    rt = np.result_type(np.asarray(s1), np.asarray(s2))
    cplx = np.iscomplexobj(a1) or np.iscomplexobj(a2)
    out = np.empty(abs(a1.shape[0] - (a2.shape[0] + nlag + nlead)) + 1, dtype=np.complex128 if cplx else np.float64)
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    _lib.check(lib.prc_xcorr(a1.ctypes.data, d1, a1.shape[0], a2.ctypes.data, d2, a2.shape[0], nlead, nlag,
                             out.ctypes.data, _lib.MEM_HOST, dev, None, 0))
    if rt.kind in "iu":
        return np.around(out).astype(np.int64).astype(rt)
    return out.astype(rt, copy=False)
