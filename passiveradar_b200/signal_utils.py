"""Front-end signal utilities on the H100 -- same call signatures as the reference.

Drop-ins for ``passiveRadar.signal_utils.deinterleave_IQ`` (reference
``passiveRadar/signal_utils.py:19-22``), ``frequency_shift`` (``:24-27``) and ``resample``
(``:15-17``), the chain ``main.py:105-166`` runs on every input chunk, plus ``frontend`` which runs
the three in one pass on the device (raw IQ in, resampled complex64 out), and the channel-offset estimator
``find_channel_offset`` (``:73-78``) with ``offset_compensation`` (``:49-71``), ``shift`` (``:34-47``) and ``xcorr``
(``:29-32``), and ``decimate`` (``:11-13``), ``channel_preprocessing`` (``:80-85``) and ``normalize`` (``:7-9``).  All
arithmetic runs in ``libprcore.so``; no CPU fallback.
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


def _raw_sources(interleaved, ref_raw, srv_raw):
    """The raw sources of a run: the one stream of an interleaved configuration, or ref_raw and srv_raw."""
    if interleaved:
        if srv_raw is not None:
            raise ValueError("interleaved_input_channels is True: pass the one interleaved source only")
        return (ref_raw,)
    if srv_raw is None:
        raise ValueError("interleaved_input_channels is False: pass ref_raw and srv_raw")
    return ref_raw, srv_raw


def _raw_iq_kind(name, t, tdev):
    """The PRC_IQ_* kind of a raw interleaved IQ source tensor, which must be one-dimensional and contiguous on tdev."""
    import torch
    if not isinstance(t, torch.Tensor) or t.device != tdev:
        raise ValueError(f"{name} must be a tensor on {tdev}")
    if t.dim() != 1 or not t.is_contiguous():
        raise ValueError(f"{name} must be one-dimensional and contiguous")
    kind = _lib.IQ_KINDS.get(_lib.np_dtype(t.dtype))
    if kind is None:
        raise TypeError(f"{name} must be int8, int16 or float32 raw IQ, got {t.dtype}")
    return kind


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
    dev = _lib.current_device(device)
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
        dev = _lib.current_device(device)
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
    dev = _lib.current_device(device)
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
        dev = _lib.current_device(device)
        _lib.check(lib.prc_iq_mix_c64(buf.ctypes.data, kind, n, mode, float(fc), float(Fs), po, out.ctypes.data,
                                      _lib.MEM_HOST, dev, None, 0))
        return out
    # the reference chain is complex64 end to end only with Python-scalar arguments
    return _run_frontend(buf, kind, n, mode, fc, Fs, po, up, dn, mode == _lib.MIX_C64, device)


# ---- channel offset (reference signal_utils.py:29-78) ------------------------------------------------------------
_PADLEN = 27


def _offset_input(x):
    """1-D contiguous array the library accepts natively, its dtype code, and whether decimate's filter is float32
    for it.  Other numeric dtypes are widened to float64 / complex128 here, as the reference upcasts them."""
    a = np.asarray(x)
    if a.ndim != 1:
        raise ValueError("the signals must be one-dimensional")
    single = a.dtype in (np.float32, np.complex64)
    if a.dtype not in _lib.DT_CODES:
        a = a.astype(np.complex128 if np.iscomplexobj(a) else np.float64)
    return np.ascontiguousarray(a), _lib.DT_CODES[a.dtype], single


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


def _offset_sections(nd, single1, single2):
    """prc_channel_offset's sos and zi arguments: decimate's sections and sosfilt_zi for each of the two signals
    (float32-rounded for a float32 / complex64 one), stacked."""
    (sos1, zi1), (sos2, zi2) = _decimate_sos(nd, single1), _decimate_sos(nd, single2)
    return np.ascontiguousarray(np.stack([sos1, sos2])), np.ascontiguousarray(np.stack([zi1, zi2]))


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
    sos, zi = _offset_sections(nd, single1, single2)
    n1d, n2d = -(-a1.shape[0] // nd), -(-a2.shape[0] // nd)
    xc = np.empty(abs(n1d - (n2d + 2 * nl)) + 1, dtype=np.float64) if want_xc else None
    off = np.zeros(1, dtype=np.int64)
    lib = _lib.load()
    dev = _lib.current_device(device)
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
    dev = _lib.current_device(device)
    _lib.check(lib.prc_xcorr(a1.ctypes.data, d1, a1.shape[0], a2.ctypes.data, d2, a2.shape[0], nlead, nlag,
                             out.ctypes.data, _lib.MEM_HOST, dev, None, 0))
    if rt.kind in "iu":
        return np.around(out).astype(np.int64).astype(rt)
    return out.astype(rt, copy=False)


# ---- decimate, channel_preprocessing, normalize (reference signal_utils.py:7-13, :80-85) ---------------------------
def _device_of(torch, device):
    if not torch.cuda.is_available():
        raise _lib.PrcoreError(_lib.PRC_E_CUDA, "no CUDA device available; libprcore has no CPU fallback")
    return torch.device("cuda", _lib.current_device(device))


@functools.lru_cache(maxsize=32)
def _decimate_taps(q, single):
    """decimate's FIR design, firwin(20q + 1, 1/q, window='hamming'), float32-rounded when the result is float32 or
    complex64 (``b = np.asarray(b, dtype=result_type)`` in scipy.signal.decimate)."""
    from scipy.signal import firwin
    b = firwin(20 * q + 1, 1.0 / q, window='hamming')
    if single:
        b = b.astype(np.float32).astype(np.float64)
    return np.ascontiguousarray(b, dtype=np.float64)


def _decimation_factor(q):
    """scipy.signal.decimate's argument errors for q, raised before the library is loaded."""
    q = operator.index(q)
    if q == 0:
        raise ZeroDivisionError("float division by zero")
    if q < 2:
        raise ValueError("Invalid cutoff frequency: frequencies must be greater than 0 and less than fs/2.")
    return q


def _decimate_dtype(dt):
    """scipy.signal.decimate's result dtype: x's own when inexact, float64 for integers, bools and float16."""
    dt = np.dtype(dt)
    if dt in (np.dtype(np.longdouble), np.dtype(np.clongdouble)) and dt not in _lib.DT_CODES:
        raise TypeError("No matching signature found")
    if dt.kind == "c":
        return dt
    if dt.kind not in "biuf":
        raise TypeError(f"decimate takes numeric arrays, got {dt}")
    return dt if dt == np.float32 else np.dtype(np.float64)


def _run_decimate(torch, rows, src, n, mode, fc, Fs, po, q, single, out_dtype, tdev):
    """One prc_decimate_rows call on the current torch stream: rows (k, n) contiguous on tdev -> (k, ceil(n/q))."""
    k = rows.shape[0]
    out = torch.empty(k, -(-n // q), dtype=_lib.torch_dtype(out_dtype), device=tdev)
    taps = _decimate_taps(q, single)
    lib = _lib.load()
    _lib.forked(tdev, lambda st: lib.prc_decimate_rows(rows.data_ptr(), src, n, k, n, mode, float(fc), float(Fs), po,
                                                       taps.ctypes.data, q, out.data_ptr(), out.shape[1], tdev.index, st,
                                                       _lib.FLAG_ASYNC))
    return out


def decimate(x, q, *, device=None):
    '''decimate x by a factor of q

    ``scipy.signal.decimate(x, q, 20*q, ftype='fir', axis=0)`` on the device: the zero-phase FIR decimator with 20q+1
    Hamming taps along axis 0 of an array of any shape, in SciPy's dtype (x's own when inexact, float64 otherwise;
    float32 taps and sums for float32 and complex64, float64 for the rest).  A NumPy (or array-like) x gives NumPy; a
    CUDA tensor gives a tensor on its device, ordered on the current torch stream.'''
    import torch
    q = _decimation_factor(q)
    is_t = isinstance(x, torch.Tensor)
    if is_t:
        if not x.is_cuda:
            raise ValueError("a tensor input must be a CUDA tensor; pass host data as a NumPy array")
        ndt = _lib.np_dtype(x.dtype)
        if ndt is None:
            raise TypeError(f"decimate takes numeric tensors, got {x.dtype}")
        shape, rd = tuple(x.shape), _decimate_dtype(ndt)
    else:
        x = np.asarray(x)
        shape, rd = x.shape, _decimate_dtype(x.dtype)
    if len(shape) == 0:
        raise IndexError("tuple index out of range")
    n = shape[0]
    k = int(np.prod(shape[1:], dtype=np.int64))
    nout = -(-n // q)
    if n == 0 or k == 0:
        if is_t:
            return torch.empty((nout,) + shape[1:], dtype=_lib.torch_dtype(rd), device=x.device)
        return np.empty((nout,) + shape[1:], dtype=rd)
    single = rd in (np.float32, np.complex64)
    if is_t:
        t = x if ndt in _lib.DT_CODES else x.to(torch.float64)
        rows = t.reshape(n, k).T.contiguous()
        out = _run_decimate(torch, rows, _lib.DT_CODES[_lib.np_dtype(rows.dtype)], n, _lib.MIX_NONE, 0.0, 1.0, 0.0,
                            q, single, rd, x.device)
        return out.T.reshape((nout,) + shape[1:])
    a = x if x.dtype in _lib.DT_CODES else x.astype(rd)
    tdev = _device_of(torch, device)
    rows = torch.from_numpy(np.ascontiguousarray(a.reshape(n, k).T)).to(tdev)
    out = _run_decimate(torch, rows, _lib.DT_CODES[a.dtype], n, _lib.MIX_NONE, 0.0, 1.0, 0.0, q, single, rd, tdev)
    return np.ascontiguousarray(out.cpu().numpy().T).reshape((nout,) + shape[1:])


def channel_preprocessing(sig, dec, fc, Fs, *, device=None):
    '''deinterleave IQ samples, tune to channel frequency and decimate

    ``decimate(frequency_shift(deinterleave_IQ(sig), fc, Fs), dec)`` in one pass on the device: the raw int8, int16 or
    float32 I/Q is deinterleaved (I = sig[0:-1:2], Q = sig[1::2]) and mixed as it is staged, so the tuned signal is never
    stored.  complex64 when the reference's is (Python-scalar fc and Fs), complex128 otherwise.  A CUDA tensor of raw
    samples gives a tensor on its device, ordered on the current torch stream.'''
    import torch
    q = _decimation_factor(dec)
    mode, po = _mix_mode(fc, Fs, 0)
    rd = np.dtype(np.complex64) if mode == _lib.MIX_C64 else np.dtype(np.complex128)
    if isinstance(sig, torch.Tensor):
        if not sig.is_cuda:
            raise ValueError("a tensor input must be a CUDA tensor; pass host data as a NumPy array")
        if sig.dim() != 1:
            raise ValueError("interleaved IQ must be one-dimensional")
        n = sig.shape[0] // 2
        t = sig[:2 * n]
        if _lib.np_dtype(t.dtype) not in _lib.IQ_KINDS:
            t = t.to(torch.float32)
        if n == 0:
            return torch.empty(0, dtype=_lib.torch_dtype(rd), device=sig.device)
        raw, kind, tdev = t.contiguous(), _lib.IQ_KINDS[_lib.np_dtype(t.dtype)], sig.device
    else:
        buf, kind, n = _raw_iq(sig)
        if n == 0:
            return np.empty(0, dtype=rd)
        tdev = _device_of(torch, device)
        raw = torch.from_numpy(buf).to(tdev)
    out = _run_decimate(torch, raw.view(1, -1), _lib.DEC_RAW + kind, n, mode, fc, Fs, po, q, mode == _lib.MIX_C64, rd,
                        tdev)[0]
    return out if isinstance(sig, torch.Tensor) else out.cpu().numpy()


_NORM_OUT = {np.dtype(np.float32): np.dtype(np.float32), np.dtype(np.complex64): np.dtype(np.complex64),
             np.dtype(np.complex128): np.dtype(np.complex128)}


def normalize(x, *, device=None):
    '''normalize ndarray to unit mean

    ``x / np.mean(np.abs(x).flatten())`` on the device for int8, uint8, int16, float32, float64, complex64 and
    complex128 x of any shape, in NumPy's result dtype (float64 for the integers).  The mean is summed in float64 in a
    fixed order.  An all-zero x gives NaN, an empty x an empty result.  A CUDA tensor gives a tensor on its device,
    ordered on the current torch stream.'''
    import torch
    is_t = isinstance(x, torch.Tensor)
    if is_t:
        if not x.is_cuda:
            raise ValueError("a tensor input must be a CUDA tensor; pass host data as a NumPy array")
        dt = _lib.np_dtype(x.dtype)
    else:
        x = np.asarray(x)
        dt = x.dtype
    if dt not in _lib.DT_CODES:
        raise TypeError(f"normalize takes int8, uint8, int16, float32, float64, complex64 or complex128, got {dt}")
    rd = _NORM_OUT.get(dt, np.dtype(np.float64))
    shape = tuple(x.shape)
    n = int(np.prod(shape, dtype=np.int64))
    if n == 0:
        if is_t:
            return torch.empty(shape, dtype=_lib.torch_dtype(rd), device=x.device)
        return np.empty(shape, dtype=rd)
    if is_t:
        src, tdev = x.contiguous(), x.device
    else:
        tdev = _device_of(torch, device)
        src = torch.from_numpy(np.ascontiguousarray(x).reshape(-1)).to(tdev)
    out = torch.empty(shape, dtype=_lib.torch_dtype(rd), device=tdev)
    lib = _lib.load()
    _lib.forked(tdev, lambda st: lib.prc_normalize(src.data_ptr(), _lib.DT_CODES[dt], n, out.data_ptr(), tdev.index, st,
                                                   _lib.FLAG_ASYNC))
    return out if is_t else out.cpu().numpy()
