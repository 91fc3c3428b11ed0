"""The frame chain of the reference's ``range_doppler_plot.py`` (lines 45-85) on the H100: ``persistence`` with the
reference's call signature (``passiveRadar/plotting_tools.py:9-30``), its batched form ``persistence_frames``, and
``RenderPipeline``: CFAR_2D of every frame, persistence, orientation and the per-frame colour limits, with the maps
kept on the device.  Colour mapping and video encoding (matplotlib) stay with the caller.  No CPU fallback."""
from __future__ import annotations

import numpy as np

from . import _lib

PERCENTILES = (35.0, 99.0)        # range_doppler_plot.py: vmin = percentile 35, vmax = 1.5 * percentile 99
VMAX_SCALE = 1.5
MAX_CFAR_FRAMES = 65535           # frames of one prc_cfar2d_frames call
_KERNEL_FLOATS = (np.dtype(np.float32), np.dtype(np.float64))


def _is_tensor(x):
    try:
        import torch
    except ImportError:
        return False
    return isinstance(x, torch.Tensor)


def _decay_plan(x_dtype, decay, n):
    """The reference's weights decay**i, i < n, as Python computes them, and the precision NumPy 2 gives
    ``X[:, :, j] * decay**i``: (weights as float64, product dtype).  Integer products are formed in float64."""
    if isinstance(decay, (complex, np.complexfloating)):
        raise TypeError("decay must be real")
    w = [decay ** i for i in range(n)]
    prod = np.result_type(x_dtype, w[0] if n else decay)
    if prod.kind == "c":
        raise TypeError("decay must be real")
    if prod.kind != "f":
        prod = np.dtype(np.float64)
    if prod not in _KERNEL_FLOATS:
        raise TypeError(f"X * decay**i is formed in {prod} here; persistence forms float32 or float64 products only")
    return np.array([float(v) for v in w], dtype=np.float64), prod


def _stack_dtype(x):
    """The NumPy dtype of a stack (ndarray or tensor).  Float stacks other than float32 and float64 are refused: the
    kernel reads and multiplies float32 or float64, so a float16 or long-double stack could not be reproduced."""
    if _is_tensor(x):
        try:
            dtype = np.dtype(str(x.dtype).replace("torch.", ""))
        except TypeError:
            raise TypeError(f"unsupported stack dtype {x.dtype}") from None
    else:
        dtype = np.dtype(x.dtype)
    if dtype.kind == "c":
        raise TypeError("persistence expects a real frame stack (the reference is called with CFAR output)")
    if dtype.kind not in "biuf":
        raise TypeError(f"unsupported stack dtype {dtype}")
    if dtype.kind == "f" and dtype not in _KERNEL_FLOATS:
        raise TypeError(f"unsupported stack dtype {dtype}: persistence reads float32 or float64 stacks (or integers)")
    return dtype


def _launch_persistence(x, rows, cols, n_carry, nframes, hold, w, prod, out, device, stream, mem):
    """x holds float32 or float64 frames (n_carry + nframes of them, compact); out: nframes float64 frames."""
    flags = _lib.FLAG_ASYNC if mem == _lib.MEM_DEVICE else 0
    if prod == np.float32:
        flags |= _lib.FLAG_PROD_F32
    if np.dtype(x.dtype if isinstance(x, np.ndarray) else _np_dtype(x)) == np.float64:
        flags |= _lib.FLAG_MAP_F64
    _lib.check(_lib.load().prc_persistence_frames(_lib.ptr(x), rows, cols, nframes, rows * cols, n_carry, hold,
                                                  w.ctypes.data, _lib.ptr(out), mem, device, stream, flags))


def _stream_arg(torch, device):
    """The current torch stream as the library's ``stream`` argument.  torch's default stream is CUDA's legacy default
    stream, whose handle is 0; the library would take 0 for "my own stream", so it is passed as cudaStreamLegacy."""
    return torch.cuda.current_stream(device).cuda_stream or 1       # 1 == cudaStreamLegacy


def _np_dtype(t):
    import torch
    return {torch.float32: np.float32, torch.float64: np.float64}[t.dtype]


def _cfar_choice(cfar, os_rank, fw, gw):
    """The pipelines' cfar / os_rank options -> (cfar, k): k is the ordered-statistic rank, None for CFAR_2D."""
    if cfar not in ("ca", "os"):
        raise ValueError(f"cfar must be 'ca' (CFAR_2D) or 'os' (OS_CFAR_2D), got {cfar!r}")
    if cfar == "ca":
        if os_rank is not None:
            raise ValueError("os_rank applies to cfar='os' only")
        return cfar, None
    from .target_detection import os_rank as rank, os_window_cells
    if not (1 <= fw <= 64) or gw < 0 or fw * fw == gw * gw:
        raise ValueError(f"fw={fw} gw={gw}: OS_CFAR_2D needs 1 <= fw <= 64, gw >= 0 and fw != gw")
    n = os_window_cells(fw, gw)
    k = rank(fw, gw, os_rank)
    if not 1 <= k <= n:
        raise ValueError(f"os_rank={k} outside [1, N = {n}], the cells of the fw={fw} gw={gw} window")
    return cfar, k


def _cfar_frames_into(lib, cfar, k, maps_d, cf, fw, gw, dev, stream):
    """The float64 CR of every map of maps_d (T compact complex64 / float32 device maps) into cf (T maps): CFAR_2D
    (prc_cfar2d_frames) or, with cfar == "os", the ordered-statistic CFAR of rank k (prc_os_cfar2d_frames)."""
    import torch
    T, F, R1 = maps_d.shape
    cells = F * R1
    flags = _lib.FLAG_ASYNC | _lib.FLAG_CR_F64 | (_lib.FLAG_ABS_C64 if maps_d.dtype == torch.complex64 else 0)
    for t0 in range(0, T, MAX_CFAR_FRAMES):
        nb = min(MAX_CFAR_FRAMES, T - t0)
        if cfar == "os":
            _lib.check(lib.prc_os_cfar2d_frames(maps_d[t0].data_ptr(), F, R1, nb, cells, fw, gw, k,
                                                cf[t0].data_ptr(), cells, dev, stream, flags))
        else:
            _lib.check(lib.prc_cfar2d_frames(maps_d[t0].data_ptr(), F, R1, nb, cells, fw, gw,
                                             cf[t0].data_ptr(), cells, _lib.MEM_DEVICE, dev, stream, flags))


def _frames_for(prod, dtype):
    """The dtype the kernel reads a stack in: float32 when the products are float32 (exact for every dtype that
    promotes to them), else the stack's own float dtype, float64 for integers."""
    if prod == np.float32:
        return np.dtype(np.float32)
    return np.dtype(dtype) if np.dtype(dtype).kind == "f" else np.dtype(np.float64)


def _persist(frames, n_carry, hold, decay, device):
    """frames: (n_carry + T, rows, cols) numpy array or CUDA tensor -> (T, rows, cols) float64 of the same kind."""
    total, rows, cols = frames.shape
    T = total - n_carry
    if _is_tensor(frames):
        import torch
        if not frames.is_cuda:
            frames = frames.numpy()
        else:
            src = _stack_dtype(frames)
            w, prod = _decay_plan(src, decay, min(hold, total))
            want = _frames_for(prod, src)
            x = frames.to({np.float32: torch.float32, np.float64: torch.float64}[want.type]).contiguous()
            out = torch.empty((T, rows, cols), dtype=torch.float64, device=frames.device)
            if T:
                dev = frames.device.index if device is None else int(device)
                stream = _stream_arg(torch, frames.device)
                _launch_persistence(x, rows, cols, n_carry, T, hold, w, prod, out, dev, stream, _lib.MEM_DEVICE)
            return out
    src = _stack_dtype(frames)
    w, prod = _decay_plan(src, decay, min(hold, total))
    x = np.ascontiguousarray(frames, dtype=_frames_for(prod, src))
    out = np.empty((T, rows, cols), dtype=np.float64)
    if T:
        dev = _lib.current_device() if device is None else int(device)
        _launch_persistence(x, rows, cols, n_carry, T, hold, w, prod, out, dev, None, _lib.MEM_HOST)
    return out


def persistence(X, k, hold, decay, *, device=None):
    '''Add persistence (digital phosphor) effect along the time axis of a sequence of range-doppler maps

    Parameters:
        X: Input frame stack (NxMxL matrix): numpy array, or a CUDA tensor (the result is then a CUDA tensor)
        k: index of frame to acquire
        hold: number of samples to persist
        decay: frame decay rate (should be less than 1)

    Returns:
        frame: (NxM float64 matrix) frame k of the original stack with persistence effect.  Only the min(k+1, hold)
        frames it sums are copied; the sums and their rounding are the reference's.'''
    tensor = _is_tensor(X) and X.is_cuda
    if not tensor:
        X = np.asarray(X)
    if X.ndim != 3:
        raise ValueError(f"X must be a three-dimensional (N, M, L) frame stack, got {X.ndim} dimensions")
    _stack_dtype(X)
    k, hold = int(k), int(hold)
    N, M, L = X.shape
    n = min(k + 1, hold)
    if n <= 0:                                   # the reference's loop runs no iteration
        if tensor:
            import torch
            return torch.zeros((N, M), dtype=torch.float64, device=X.device)
        return np.zeros((N, M))
    if k >= L:
        raise IndexError(f"index {k} is out of bounds for axis 2 with size {L}")
    if tensor:
        frames = X[:, :, k - n + 1:k + 1].permute(2, 0, 1)
    else:
        frames = np.moveaxis(X[:, :, k - n + 1:k + 1], 2, 0)
    return _persist(frames, n - 1, hold, decay, device)[0]


def persistence_frames(stack, hold, decay, *, device=None):
    """persistence(stack.transpose(1, 2, 0), k, hold, decay) for every k in one launch: stack is a (T, rows, cols)
    numpy array or CUDA tensor; returns (T, rows, cols) float64 of the same kind."""
    tensor = _is_tensor(stack) and stack.is_cuda
    if not tensor:
        stack = np.asarray(stack)
    if stack.ndim != 3:
        raise ValueError(f"stack must be three-dimensional (T, rows, cols), got {stack.ndim} dimensions")
    hold = int(hold)
    if hold <= 0:
        _stack_dtype(stack)
        if tensor:
            import torch
            return torch.zeros(tuple(stack.shape), dtype=torch.float64, device=stack.device)
        return np.zeros(stack.shape)
    return _persist(stack, 0, hold, decay, device)


class RenderPipeline:
    """range_doppler_plot.py:45-85 on the device: for every frame kk of a map stack,
    ``CF = CFAR_2D(|map|, fw, gw)`` (float64), ``data = fliplr(persistence(CF, kk, hold, decay).T)``,
    ``vmin = percentile(data, 35)``, ``vmax = 1.5 * percentile(data, 99)``.

    ``run_device`` takes (T, F, R+1) complex64 or float32 CUDA tensors (``RecordingPipeline.run_device`` /
    ``FramePipeline.run_device`` output) and carries the last hold - 1 CFAR frames to the next call, so a stack cut
    into batches of any size renders bit-identically to one call; ``reset()`` starts a new sequence.  ``run`` takes
    main.py's host layout (F, R+1, nframes).

    ``cfar="os"`` replaces CFAR_2D by the ordered-statistic CFAR on the same window (``OS_CFAR_2D``): the k-th smallest
    window cell, k = ``os_rank`` or ceil(3N / 4), is the noise estimate instead of the window mean."""

    def __init__(self, fw=18, gw=4, hold=20, decay=0.90, *, device=None, batch=64, cfar="ca", os_rank=None):
        self.fw, self.gw, self.hold, self.decay = int(fw), int(gw), int(hold), decay
        self.cfar, self.os_rank = _cfar_choice(cfar, os_rank, self.fw, self.gw)
        if self.hold < 1:
            raise ValueError("hold must be >= 1")
        if int(batch) < 1:
            raise ValueError("batch must be >= 1")
        self.batch = int(batch)
        self.device = device
        # CF is float64 in the reference (np.zeros(xambg.shape)): the products are float64 whatever decay's type
        self.weights, _ = _decay_plan(np.float64, decay, self.hold)
        self._carry = None
        self._q = np.array(PERCENTILES, dtype=np.float64)
        self._scale = np.array([1.0, VMAX_SCALE], dtype=np.float64)
        if not (1 <= self.fw <= 64) or self.gw < 0 or self.fw * self.fw == self.gw * self.gw:
            raise ValueError(f"fw={fw} gw={gw}: CFAR_2D needs 1 <= fw <= 64, gw >= 0 and fw != gw")

    def reset(self):
        """Start a new sequence: the next frame is frame 0 of the persistence."""
        self._carry = None

    def run_device(self, maps_d):
        """maps_d: (T, F, R+1) complex64 or float32 CUDA tensor; either way its magnitude is what is rendered, as
        range_doppler_plot.py renders np.abs(xambg).  Returns device tensors data (T, R+1, F) float64 and
        limits (T, 2) = [vmin, vmax], ordered on the current torch stream."""
        import torch
        if not (_is_tensor(maps_d) and maps_d.is_cuda and maps_d.dim() == 3):
            raise TypeError("maps_d must be a (T, F, R+1) CUDA tensor")
        if maps_d.dtype not in (torch.complex64, torch.float32):
            raise TypeError(f"maps_d must be complex64 or float32, got {maps_d.dtype}")
        T, F, R1 = maps_d.shape
        dev = maps_d.device.index if self.device is None else int(self.device)
        if self._carry is not None and tuple(self._carry.shape[1:]) != (F, R1):
            raise ValueError(f"maps of shape {(F, R1)} continue a sequence of {tuple(self._carry.shape[1:])} maps; "
                             "call reset() first")
        data = torch.empty((T, R1, F), dtype=torch.float64, device=maps_d.device)
        limits = torch.empty((T, 2), dtype=torch.float64, device=maps_d.device)
        if T == 0:
            return data, limits
        lib = _lib.load()
        # range_doppler_plot.py takes np.abs of the stack before CFAR_2D, and the CFAR kernel keeps the sign of a real
        # cell in its numerator: a float32 map is made |map| first (exact, and a no-op on magnitudes)
        maps_d = (maps_d.abs() if maps_d.dtype == torch.float32 else maps_d).contiguous()
        stream = _stream_arg(torch, maps_d.device)
        nc = 0 if self._carry is None else self._carry.shape[0]
        cf = torch.empty((nc + T, F, R1), dtype=torch.float64, device=maps_d.device)
        if nc:
            cf[:nc] = self._carry
        cells = F * R1
        _cfar_frames_into(lib, self.cfar, self.os_rank, maps_d, cf[nc:], self.fw, self.gw, dev, stream)
        _lib.check(lib.prc_persistence_frames(cf.data_ptr(), F, R1, T, cells, nc, self.hold, self.weights.ctypes.data,
                                              data.data_ptr(), _lib.MEM_DEVICE, dev, stream,
                                              _lib.FLAG_ASYNC | _lib.FLAG_MAP_F64 | _lib.FLAG_ORIENT))
        _lib.check(lib.prc_percentiles_frames(data.data_ptr(), cells, T, cells, self._q.ctypes.data,
                                              self._scale.ctypes.data, 2, limits.data_ptr(), _lib.MEM_DEVICE, dev,
                                              stream, _lib.FLAG_ASYNC))
        keep = min(nc + T, self.hold - 1)
        self._carry = cf[nc + T - keep:].clone() if keep else None
        return data, limits

    def run(self, stack):
        """stack: main.py's (F, R+1, nframes) maps on the host, complex64 or already np.abs-ed float32 / float64
        (CFAR_2D reads float32, as the drop-in does).  Starts a new sequence and streams it through in batches.
        Returns host arrays data (nframes, R+1, F) float64 and limits (nframes, 2)."""
        import torch
        stack = np.asarray(stack)
        if stack.ndim != 3:
            raise ValueError(f"stack must be (F, R+1, nframes), got {stack.ndim} dimensions")
        if stack.dtype.kind == "c":
            dt = np.complex64
        elif stack.dtype.kind in "biuf":
            dt = np.float32
        else:
            raise TypeError(f"unsupported stack dtype {stack.dtype}")
        F, R1, N = stack.shape
        dev = _lib.current_device() if self.device is None else int(self.device)
        tdev = torch.device("cuda", dev)
        self.reset()
        data = np.empty((N, R1, F), dtype=np.float64)
        limits = np.empty((N, 2), dtype=np.float64)
        with torch.cuda.device(tdev):
            for b0 in range(0, N, self.batch):
                b1 = min(N, b0 + self.batch)
                maps = torch.from_numpy(np.ascontiguousarray(np.moveaxis(stack[:, :, b0:b1], 2, 0), dtype=dt))
                d, lim = self.run_device(maps.to(tdev))
                data[b0:b1] = d.cpu().numpy()
                limits[b0:b1] = lim.cpu().numpy()
        return data, limits
