"""Welch power spectral density on the H100, with ``matplotlib.mlab.psd``'s definition, and signal_preview.py's chain.

``psd`` returns what ``plt.psd`` returns (``Axes.psd`` without its plotting arguments): ``(Pxx, freqs)``, float64, from
``prc_psd_frames`` (``csrc/spectrum.cuh``), which computes in float64 / complex128 whatever the input dtype.
``psd_frames`` runs the same estimator on a stack of frames in one call; a row of the result is bit-identical to ``psd``
of that row.  ``SignalPreview`` runs everything the reference's ``signal_preview.py`` plots, on the device, without
plotting.

Limits of the device transform: ``pad_to`` (``NFFT`` by default) is a power of two in [16, 8192]; only
``detrend=None`` (mlab's ``detrend_none``) is supported.
"""
from __future__ import annotations

import math
import operator

import numpy as np

from . import _lib
from .signal_utils import _decimate_sos, _mix_mode, _resample_taps

MIN_PAD_TO, MAX_PAD_TO = 16, 8192
_DTYPES = {np.dtype(np.float32): _lib.DT_F32, np.dtype(np.float64): _lib.DT_F64,
           np.dtype(np.complex64): _lib.DT_C64, np.dtype(np.complex128): _lib.DT_C128}


def _torch():
    import torch
    return torch


def _host_dtype(dt):
    """The dtype a host array is handed to the device in: the four native ones as they are, other complex types as
    complex128, everything else (integers, bools, float16) widened to float64 as NumPy widens them for mlab."""
    dt = np.dtype(dt)
    if dt in _DTYPES:
        return dt
    return np.dtype(np.complex128) if dt.kind == "c" else np.dtype(np.float64)


def _plan(dtype, NFFT, Fs, Fc, detrend, window, noverlap, pad_to, sides, scale_by_freq):
    """mlab's defaults and checks -> (nfft, noverlap, pad_to, window float64, scale, onesided, freqs)."""
    NFFT = 256 if NFFT is None else operator.index(NFFT)
    Fs = 2 if Fs is None else Fs
    Fc = 0 if Fc is None else Fc
    noverlap = 0 if noverlap is None else operator.index(noverlap)
    if detrend is not None and not (isinstance(detrend, str) and detrend == "none") and \
            getattr(detrend, "__name__", None) != "detrend_none":
        raise NotImplementedError(f"detrend={detrend!r} is not supported: the device estimator implements "
                                  "detrend=None ('none', mlab.detrend_none) only")
    if noverlap >= NFFT:
        raise ValueError("noverlap must be less than NFFT")
    if noverlap < 0:
        raise ValueError(f"noverlap={noverlap} must not be negative")
    pad_to = NFFT if pad_to is None else operator.index(pad_to)
    if pad_to < NFFT:
        raise ValueError(f"pad_to={pad_to} must not be smaller than NFFT={NFFT}")
    if pad_to < MIN_PAD_TO or pad_to > MAX_PAD_TO or pad_to & (pad_to - 1):
        raise ValueError(f"pad_to={pad_to}: the device transform takes powers of two in [{MIN_PAD_TO}, {MAX_PAD_TO}]")
    if sides is None or sides == "default":
        onesided = np.dtype(dtype).kind != "c"
    elif sides in ("onesided", "twosided"):
        onesided = sides == "onesided"
    else:
        raise ValueError(f"{sides!r} is not a valid value for sides; supported values are 'default', 'onesided', "
                         "'twosided'")
    if window is None:
        w = np.hanning(NFFT)                                  # mlab.window_hanning
    elif callable(window):
        w = window(np.ones(NFFT, np.dtype(dtype)))            # mlab evaluates it on ones of x's dtype
    else:
        w = window
    w = np.asarray(w)
    if w.ndim != 1 or w.shape[0] != NFFT:
        raise ValueError("The window length must match the data's first dimension")
    if np.iscomplexobj(w):
        if np.any(w.imag != 0):
            raise ValueError("the window must be real")
        w = w.real
    w = np.ascontiguousarray(w, dtype=np.float64)
    if scale_by_freq is None or scale_by_freq:
        scale = 1.0 / (float(Fs) * float((np.abs(w) ** 2).sum()))
    else:
        scale = 1.0 / float(np.abs(w).sum()) ** 2
    freqs = np.fft.fftfreq(pad_to, 1 / Fs)
    if onesided:
        freqs = freqs[:pad_to // 2 + 1]
        freqs[-1] *= -1
    else:
        freqs = np.roll(freqs, -(pad_to // 2))
    return NFFT, noverlap, pad_to, w, scale, onesided, freqs + Fc


def _run(lib, dev, x, dtype_code, n, nframes, row_stride, plan, out, stream):
    """One prc_psd_frames call on device tensors (x: nframes rows of n samples, row_stride elements apart)."""
    nfft, noverlap, pad_to, w_dev, scale, onesided = plan
    _lib.check(lib.prc_psd_frames(x.data_ptr(), dtype_code, n, nframes, row_stride, nfft, noverlap, pad_to,
                                  w_dev.data_ptr(), scale, int(onesided), out.data_ptr(), out.stride(0), dev,
                                  stream.cuda_stream, _lib.FLAG_ASYNC))


def _device_rows(torch, frames, device):
    """A CUDA tensor, or a host array (staged with torch), as (tensor of rows with unit element stride, dtype code, host?)."""
    if isinstance(frames, torch.Tensor):
        if not frames.is_cuda:
            raise ValueError("a tensor input must be a CUDA tensor; pass host data as a NumPy array")
        t = frames
        tdt = {torch.complex64: np.complex64, torch.complex128: np.complex128, torch.float32: np.float32,
               torch.float64: np.float64}.get(t.dtype)
        if tdt is None:
            t = t.to(torch.complex128 if t.is_complex() else torch.float64)
            tdt = np.complex128 if t.is_complex() else np.float64
        if t.dim() >= 1 and t.shape[-1] > 0 and t.stride(-1) != 1:
            t = t.contiguous()
        return t, _DTYPES[np.dtype(tdt)], False
    if not torch.cuda.is_available():
        raise _lib.PrcoreError(_lib.PRC_E_CUDA, "psd needs a CUDA device (no CPU fallback)")
    a = np.asarray(frames)
    a = np.ascontiguousarray(a, dtype=_host_dtype(a.dtype))
    dev = _lib.current_device() if device is None else int(device)
    return torch.from_numpy(a).to(torch.device("cuda", dev)), _DTYPES[a.dtype], True


def _psd_rows(frames, NFFT, Fs, Fc, detrend, window, noverlap, pad_to, sides, scale_by_freq, device, ndim):
    torch = _torch()
    if isinstance(frames, torch.Tensor):
        dtype = {torch.complex64: np.complex64, torch.complex128: np.complex128, torch.float32: np.float32}.get(
            frames.dtype, np.complex128 if frames.is_complex() else np.float64)
        shape = tuple(frames.shape)
    else:
        a = np.asarray(frames)
        dtype, shape = a.dtype, a.shape
    if len(shape) != ndim:
        raise ValueError(f"x must be {'one' if ndim == 1 else 'two'}-dimensional, got shape {shape}")
    if shape[-1] == 0 or (ndim == 2 and shape[0] == 0):
        raise ValueError("x must not be empty")
    nfft, noverlap, pad_to, w, scale, onesided, freqs = _plan(dtype, NFFT, Fs, Fc, detrend, window, noverlap, pad_to,
                                                              sides, scale_by_freq)
    t, code, host = _device_rows(torch, frames, device)
    tdev = t.device
    rows = t.view(1, -1) if ndim == 1 else t
    lib = _lib.load()
    cur = torch.cuda.current_stream(tdev)
    side = torch.cuda.Stream(device=tdev)
    w_dev = torch.from_numpy(w).to(tdev)
    out = torch.empty(rows.shape[0], pad_to // 2 + 1 if onesided else pad_to, dtype=torch.float64, device=tdev)
    side.wait_stream(cur)
    _run(lib, tdev.index, rows, code, rows.shape[1], rows.shape[0], rows.stride(0) if rows.shape[0] > 1 else rows.shape[1],
         (nfft, noverlap, pad_to, w_dev, scale, onesided), out, side)
    cur.wait_stream(side)
    out = out[0] if ndim == 1 else out
    if host:
        return out.cpu().numpy(), freqs
    return out, torch.from_numpy(freqs).to(tdev)


def psd(x, NFFT=None, Fs=None, Fc=None, detrend=None, window=None, noverlap=None, pad_to=None, sides=None,
        scale_by_freq=None, *, device=None):
    """``(Pxx, freqs)`` of ``plt.psd(x, ...)`` (``matplotlib.mlab.psd``, ``freqs + Fc``), computed on the device.

    Defaults as mlab's: ``NFFT`` 256, ``Fs`` 2, ``Fc`` 0, ``noverlap`` 0, ``pad_to`` = ``NFFT``, ``window`` the Hanning
    window (``np.hanning(NFFT)``; an array of ``NFFT`` real values, or a callable applied to ``np.ones(NFFT)``),
    ``sides`` two-sided for complex ``x`` and one-sided for real ``x``, ``scale_by_freq`` True (``1 / (Fs sum w^2)``;
    False: ``1 / (sum |w|)^2``).  A NumPy (or array-like) ``x`` gives NumPy results; a CUDA tensor gives tensors on
    its device, ordered on the current torch stream.  ``Pxx`` is float64.  ``device`` picks the GPU for host input."""
    return _psd_rows(x, NFFT, Fs, Fc, detrend, window, noverlap, pad_to, sides, scale_by_freq, device, 1)


def psd_frames(frames, NFFT, Fs=2, Fc=0, detrend=None, window=None, noverlap=None, pad_to=None, sides=None,
               scale_by_freq=None, *, device=None):
    """``psd`` of every row of a ``(B, n)`` stack in one ``prc_psd_frames`` call: ``(Pxx (B, nbins), freqs)``.

    ``frames`` is an ndarray or a CUDA tensor with any row stride (its elements contiguous within a row).  Row ``b``
    of ``Pxx`` is bit-identical to ``psd(frames[b], ...)``: the estimator splits a frame's segments over CTAs by the
    frame's geometry alone and sums their partial spectra in a fixed order."""
    return _psd_rows(frames, NFFT, Fs, Fc, detrend, window, noverlap, pad_to, sides, scale_by_freq, device, 2)


# ---- signal_preview.py (reference signal_preview.py:24-82) -----------------------------------------------------------
PREVIEW_NFFT_INPUT = 8192            # signal_preview.py:52-55
PREVIEW_NFFT_CHANNEL = 2048          # signal_preview.py:68-71
PREVIEW_OFFSET_ND, PREVIEW_OFFSET_NL = 4, 50000          # find_channel_offset(ref, srv, 4, 50000)
PREVIEW_XCORR_LAGS = 2000            # xcorr(ref, srv, 2000, 2000)
_IQ_KINDS = {np.dtype(np.int8): _lib.IQ_I8, np.dtype(np.int16): _lib.IQ_I16, np.dtype(np.float32): _lib.IQ_C64}


class SignalPreview:
    """What ``signal_preview.py`` computes and plots, on one device, without plotting::

        pre = SignalPreview.from_config(config)     # the dict the reference's getConfiguration returns
        r = pre.run(ref_raw, srv_raw)               # or pre.run(data) when interleaved_input_channels is True

    ``r`` holds ``offset`` (find_channel_offset(ref, srv, 4, 50000)), ``input_freqs`` / ``input_psd`` (plt.psd of both
    channels at NFFT 8192, ``input_sample_rate``, ``input_center_freq``; rows ref, srv), ``channel_freqs`` /
    ``channel_psd`` (plt.psd of both shifted and resampled channels at NFFT 2048, ``channel_bandwidth``,
    ``channel_freq``), ``xcorr_lags`` and ``xcorr_abs`` (|xcorr(ref, srv, 2000, 2000)| in float64).

    Inputs are the raw interleaved IQ (int8, int16 or float32) of which the script reads ``[0:input_chunk_length]``:
    one source per channel, or with ``interleaved_input_channels`` one source whose complex samples alternate between
    the channels (ref = ``[0::2]``, srv = ``[1::2]``, so the two may differ in length by one sample).

    The reference's quirks are kept: the channel spectrum is scaled and labelled with ``channel_bandwidth`` although
    the resampled channel runs at ``IF_sample_rate``; the offset is estimated with nd = 4 here, but nd = 1 in main.py.
    ``xcorr_lags`` are ``arange(len(xcorr_abs)) - 2000``: the script's ``arange(-2000, 2001)`` when the channels have
    the same length (with one sample fewer in srv, the correlation has 4000 lags, which the script cannot plot).

    The device chain runs on one stream and synchronises once: ``prc_iq_mix_c64`` (deinterleave), ``prc_psd_frames``
    (both channels in one call when their lengths agree), ``prc_frontend_c64`` (frequency_shift with phase offset 0, then
    resample), ``prc_psd_frames``, ``prc_channel_offset`` and ``prc_xcorr``, then ``abs`` on the device."""

    def __init__(self, config, *, device=None):
        self.icl = int(config["input_chunk_length"])
        self.fs = config["input_sample_rate"]
        self.fc = config["input_center_freq"]
        self.fo = config["offset_freq"]
        self.up, self.dn = int(config["resamp_up"]), int(config["resamp_dn"])
        self.bw = config["channel_bandwidth"]
        self.ch_fc = config["channel_freq"]
        self.interleaved = bool(config["interleaved_input_channels"])
        self.device = device
        g = math.gcd(self.up, self.dn)
        self.up_r, self.dn_r = self.up // g, self.dn // g
        self.mix_mode, self.phase = _mix_mode(self.fo, self.fs, 0)      # frequency_shift(x, offset_freq, fs)
        self.taps = _resample_taps(self.up_r, self.dn_r, self.mix_mode == _lib.MIX_C64)

    @classmethod
    def from_config(cls, config, **kw):
        """From the dict ``passiveRadar.config.getConfiguration`` returns."""
        return cls(config, **kw)

    # ------------------------------------------------------------------ geometry (no device)
    def geometry(self, n_raw):
        """Lengths the chain gives raw sources of ``n_raw`` elements (the shorter of the two when separate)."""
        n = min(int(n_raw), self.icl) // 2
        n_ref, n_srv = ((n + 1) // 2, n // 2) if self.interleaved else (n, n)
        rs = lambda k: k if self.up_r == self.dn_r else -(-k * self.up_r // self.dn_r)
        nx = abs(n_ref - (n_srv + 2 * PREVIEW_XCORR_LAGS)) + 1
        return {"n_ref": n_ref, "n_srv": n_srv, "n_ref_resampled": rs(n_ref), "n_srv_resampled": rs(n_srv),
                "xcorr_lags": np.arange(nx) - PREVIEW_XCORR_LAGS,
                "input_freqs": _plan(np.complex64, PREVIEW_NFFT_INPUT, self.fs, self.fc, None, None, None, None, None,
                                     None)[-1],
                "channel_freqs": _plan(np.complex64, PREVIEW_NFFT_CHANNEL, self.bw, self.ch_fc, None, None, None, None,
                                       None, None)[-1]}

    # ------------------------------------------------------------------ device chain
    def _setup(self, tdev=None):
        torch = _torch()
        if not torch.cuda.is_available():
            raise _lib.PrcoreError(_lib.PRC_E_CUDA, "SignalPreview needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        if tdev is None:
            tdev = torch.device("cuda", _lib.current_device() if self.device is None else int(self.device))
        self.tdev = tdev
        self.dev = tdev.index
        self.stream = torch.cuda.Stream(device=tdev)

    def _check_raw(self, name, t):
        torch = _torch()
        if not isinstance(t, torch.Tensor) or t.device != self.tdev:
            raise ValueError(f"{name} must be a tensor on {self.tdev}")
        if t.dim() != 1 or not t.is_contiguous():
            raise ValueError(f"{name} must be one-dimensional and contiguous")
        dt = {torch.int8: np.int8, torch.int16: np.int16, torch.float32: np.float32}.get(t.dtype)
        if dt is None:
            raise TypeError(f"{name} must be int8, int16 or float32 raw IQ, got {t.dtype}")
        return _IQ_KINDS[np.dtype(dt)]

    def _deinterleave(self, raw, kind, out):
        n = raw.shape[0] // 2
        _lib.check(self.lib.prc_iq_mix_c64(raw.data_ptr(), kind, n, _lib.MIX_NONE, 0.0, 1.0, 0.0, out.data_ptr(),
                                           _lib.MEM_DEVICE, self.dev, self.stream.cuda_stream, _lib.FLAG_ASYNC))

    def _psd(self, rows, n, nfft, Fs, out):
        """plt.psd's spectrum of rows (a (k, >= n) complex64 tensor) at NFFT nfft, scaled with Fs, into out."""
        w = self._window(nfft)
        scale = 1.0 / (float(Fs) * float((w[1] ** 2).sum()))
        _lib.check(self.lib.prc_psd_frames(rows.data_ptr(), _lib.DT_C64, n, rows.shape[0], rows.stride(0), nfft, 0,
                                           nfft, w[0].data_ptr(), scale, 0, out.data_ptr(), out.stride(0), self.dev,
                                           self.stream.cuda_stream, _lib.FLAG_ASYNC))

    def _window(self, nfft):
        cache = self.__dict__.setdefault("_windows", {})
        if (nfft, self.dev) not in cache:
            w = np.hanning(nfft)
            cache[(nfft, self.dev)] = (_torch().from_numpy(w).to(self.tdev), w)
        return cache[(nfft, self.dev)]

    def _spectra(self, chans, lens, nfft, Fs, out):
        if lens[0] == lens[1]:
            self._psd(chans, lens[0], nfft, Fs, out)
        else:
            for q in range(2):
                self._psd(chans[q:q + 1], lens[q], nfft, Fs, out[q:q + 1])

    def _chain(self, ref_raw, srv_raw):
        torch = _torch()
        if self.interleaved:
            if srv_raw is not None:
                raise ValueError("interleaved_input_channels is True: pass the one interleaved source only")
            k = self._check_raw("data", ref_raw)
            data = ref_raw[:self.icl]
            iq = torch.empty(data.shape[0] // 2, dtype=torch.complex64, device=self.tdev)
            self._deinterleave(data, k, iq)
            n_ref, n_srv = (iq.shape[0] + 1) // 2, iq.shape[0] // 2
            chans = torch.zeros(2, n_ref, dtype=torch.complex64, device=self.tdev)
            chans[0].copy_(iq[0::2])
            chans[1, :n_srv].copy_(iq[1::2])
        else:
            if srv_raw is None:
                raise ValueError("interleaved_input_channels is False: pass ref_raw and srv_raw")
            kinds = [self._check_raw("ref_raw", ref_raw), self._check_raw("srv_raw", srv_raw)]
            raws = [ref_raw[:self.icl], srv_raw[:self.icl]]
            n_ref, n_srv = raws[0].shape[0] // 2, raws[1].shape[0] // 2
            chans = torch.zeros(2, max(n_ref, n_srv), dtype=torch.complex64, device=self.tdev)
            for q in range(2):
                self._deinterleave(raws[q], kinds[q], chans[q])
        lens = (n_ref, n_srv)
        if min(lens) < 1:
            raise ValueError("the sources hold no complex sample in [0:input_chunk_length]")
        input_psd = torch.empty(2, PREVIEW_NFFT_INPUT, dtype=torch.float64, device=self.tdev)
        self._spectra(chans, lens, PREVIEW_NFFT_INPUT, self.fs, input_psd)
        rs = [n if self.up_r == self.dn_r else -(-n * self.up_r // self.dn_r) for n in lens]
        res = torch.zeros(2, max(rs), dtype=torch.complex64, device=self.tdev)
        for q in range(2):
            if self.up_r == self.dn_r:              # resample(x, 1, 1) returns x: the shift alone
                _lib.check(self.lib.prc_iq_mix_c64(chans[q].data_ptr(), _lib.IQ_C64, lens[q], self.mix_mode,
                                                   float(self.fo), float(self.fs), self.phase, res[q].data_ptr(),
                                                   _lib.MEM_DEVICE, self.dev, self.stream.cuda_stream, _lib.FLAG_ASYNC))
            else:
                _lib.check(self.lib.prc_frontend_c64(chans[q].data_ptr(), _lib.IQ_C64, lens[q], self.mix_mode,
                                                     float(self.fo), float(self.fs), self.phase, self.up_r, self.dn_r,
                                                     self.taps.ctypes.data, self.taps.shape[0], res[q].data_ptr(),
                                                     res.shape[1], _lib.MEM_DEVICE, self.dev, self.stream.cuda_stream,
                                                     _lib.FLAG_ASYNC))
        channel_psd = torch.empty(2, PREVIEW_NFFT_CHANNEL, dtype=torch.float64, device=self.tdev)
        self._spectra(res, rs, PREVIEW_NFFT_CHANNEL, self.bw, channel_psd)
        sos, zi = _decimate_sos(PREVIEW_OFFSET_ND, True)           # decimate's sections for complex64 signals
        sos2, zi2 = np.ascontiguousarray(np.stack([sos, sos])), np.ascontiguousarray(np.stack([zi, zi]))
        off = torch.zeros(1, dtype=torch.int64, device=self.tdev)
        _lib.check(self.lib.prc_channel_offset(chans[0].data_ptr(), _lib.DT_C64, n_ref, chans[1].data_ptr(),
                                               _lib.DT_C64, n_srv, PREVIEW_OFFSET_ND, PREVIEW_OFFSET_NL,
                                               sos2.ctypes.data, zi2.ctypes.data, off.data_ptr(), None,
                                               _lib.MEM_DEVICE, self.dev, self.stream.cuda_stream, _lib.FLAG_ASYNC))
        L = PREVIEW_XCORR_LAGS
        xc = torch.empty(abs(n_ref - (n_srv + 2 * L)) + 1, dtype=torch.complex128, device=self.tdev)
        _lib.check(self.lib.prc_xcorr(chans[0].data_ptr(), _lib.DT_C64, n_ref, chans[1].data_ptr(), _lib.DT_C64, n_srv,
                                      L, L, xc.data_ptr(), _lib.MEM_DEVICE, self.dev, self.stream.cuda_stream,
                                      _lib.FLAG_ASYNC))
        return {"offset": off, "input_psd": input_psd, "channel_psd": channel_psd, "xcorr_abs": xc.abs()}

    def run_device(self, ref_raw, srv_raw=None):
        """CUDA tensors of raw interleaved IQ -> the preview's results as tensors on their device (``offset`` an int).
        Work is forked from, and joined back into, the current torch stream."""
        torch = _torch()
        self._setup(ref_raw.device if isinstance(ref_raw, torch.Tensor) and ref_raw.is_cuda else None)
        cur = torch.cuda.current_stream(self.tdev)
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            r = self._chain(ref_raw, srv_raw)
        cur.wait_stream(self.stream)
        for v in r.values():
            v.record_stream(cur)                                  # the caller's stream uses them from here on
        r["offset"] = int(r["offset"].item())                     # the one synchronisation
        g = self.geometry(self.icl)
        r["input_freqs"] = torch.from_numpy(g["input_freqs"]).to(self.tdev)
        r["channel_freqs"] = torch.from_numpy(g["channel_freqs"]).to(self.tdev)
        r["xcorr_lags"] = torch.arange(r["xcorr_abs"].shape[0], device=self.tdev) - PREVIEW_XCORR_LAGS
        return r

    def run(self, ref_raw, srv_raw=None):
        """Host sources (ndarray, np.memmap, h5py dataset; int8, int16 or float32 raw interleaved IQ) -> the preview's
        results as NumPy arrays (``offset`` an int).  Only ``[0:input_chunk_length]`` of each source is read."""
        torch = _torch()
        self._setup()

        def stage(src):
            a = np.ascontiguousarray(np.asarray(src[0:self.icl]))
            if a.dtype not in _IQ_KINDS:
                raise TypeError(f"raw IQ must be int8, int16 or float32, got {a.dtype}")
            return torch.from_numpy(a).to(self.tdev)

        r = self.run_device(stage(ref_raw), None if srv_raw is None else stage(srv_raw))
        return {k: (v if isinstance(v, int) else v.cpu().numpy()) for k, v in r.items()}
