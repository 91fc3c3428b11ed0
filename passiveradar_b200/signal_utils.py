"""Front-end signal utilities on the H100 -- same call signatures as the reference.

Drop-ins for ``passiveRadar.signal_utils.deinterleave_IQ`` (reference
``passiveRadar/signal_utils.py:19-22``), ``frequency_shift`` (``:24-27``) and ``resample``
(``:15-17``), the chain ``main.py:105-166`` runs on every input chunk, plus ``frontend`` which runs
the three in one pass on the device (raw IQ in, resampled complex64 out).  All arithmetic runs in
``libprcore.so``; no CPU fallback.
"""
from __future__ import annotations

import functools
import math

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
