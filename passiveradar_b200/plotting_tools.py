"""The frame chain of the reference's ``range_doppler_plot.py`` (lines 45-85) on the H100: ``persistence`` with the
reference's call signature (``passiveRadar/plotting_tools.py:9-30``), its batched form ``persistence_frames``, and
``RenderPipeline``: CFAR_2D of every frame, persistence, orientation and the per-frame colour limits, with the maps
kept on the device.  Colour mapping and video encoding (matplotlib) stay with the caller.  No CPU fallback."""
from __future__ import annotations

import numpy as np

from . import _lib
from .target_detection import _cfar_frames_into, os_rank, os_window_cells

PERCENTILES = (35.0, 99.0)        # range_doppler_plot.py: vmin = percentile 35, vmax = 1.5 * percentile 99
VMAX_SCALE = 1.5
_KERNEL_FLOATS = (np.dtype(np.float32), np.dtype(np.float64))


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
    dtype = x.dtype if isinstance(x, np.ndarray) else _lib.np_dtype(x.dtype)
    if dtype is None:
        raise TypeError(f"unsupported stack dtype {x.dtype}")
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
    if (x.dtype if isinstance(x, np.ndarray) else _lib.np_dtype(x.dtype)) == np.float64:
        flags |= _lib.FLAG_MAP_F64
    _lib.check(_lib.load().prc_persistence_frames(_lib.ptr(x), rows, cols, nframes, rows * cols, n_carry, hold,
                                                  w.ctypes.data, _lib.ptr(out), mem, device, stream, flags))


def _cfar_choice(cfar, rank, fw, gw):
    """The pipelines' cfar / os_rank options -> (cfar, k): k is the ordered-statistic rank, None for CFAR_2D."""
    if cfar not in ("ca", "os"):
        raise ValueError(f"cfar must be 'ca' (CFAR_2D) or 'os' (OS_CFAR_2D), got {cfar!r}")
    if cfar == "ca":
        if rank is not None:
            raise ValueError("os_rank applies to cfar='os' only")
        return cfar, None
    if not (1 <= fw <= 64) or gw < 0 or fw * fw == gw * gw:
        raise ValueError(f"fw={fw} gw={gw}: OS_CFAR_2D needs 1 <= fw <= 64, gw >= 0 and fw != gw")
    n = os_window_cells(fw, gw)
    k = os_rank(fw, gw, rank)
    if not 1 <= k <= n:
        raise ValueError(f"os_rank={k} outside [1, N = {n}], the cells of the fw={fw} gw={gw} window")
    return cfar, k


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
    if _lib.is_cuda_tensor(frames):
        import torch
        src = _stack_dtype(frames)
        w, prod = _decay_plan(src, decay, min(hold, total))
        x = frames.to(_lib.torch_dtype(_frames_for(prod, src))).contiguous()
        out = torch.empty((T, rows, cols), dtype=torch.float64, device=frames.device)
        if T:
            dev = frames.device.index if device is None else int(device)
            _launch_persistence(x, rows, cols, n_carry, T, hold, w, prod, out, dev, _lib.stream_arg(frames.device),
                                _lib.MEM_DEVICE)
        return out
    src = _stack_dtype(frames)
    w, prod = _decay_plan(src, decay, min(hold, total))
    x = np.ascontiguousarray(frames, dtype=_frames_for(prod, src))
    out = np.empty((T, rows, cols), dtype=np.float64)
    if T:
        _launch_persistence(x, rows, cols, n_carry, T, hold, w, prod, out, _lib.current_device(device), None,
                            _lib.MEM_HOST)
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
    tensor = _lib.is_cuda_tensor(X)
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
    tensor = _lib.is_cuda_tensor(stack)
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

    def _check(self, maps_d):
        """(T, F, R+1) of a map stack ``run_device`` takes that continues the sequence."""
        import torch
        if not (_lib.is_cuda_tensor(maps_d) and maps_d.dim() == 3):
            raise TypeError("maps_d must be a (T, F, R+1) CUDA tensor")
        if maps_d.dtype not in (torch.complex64, torch.float32):
            raise TypeError(f"maps_d must be complex64 or float32, got {maps_d.dtype}")
        T, F, R1 = maps_d.shape
        if self._carry is not None and tuple(self._carry.shape[1:]) != (F, R1):
            raise ValueError(f"maps of shape {(F, R1)} continue a sequence of {tuple(self._carry.shape[1:])} maps; "
                             "call reset() first")
        return T, F, R1

    def _cf(self, maps_d, dev):
        """The CFAR stage: (cf, nc), the float64 CR of maps_d's T maps after the nc CR frames carried from earlier
        calls, a (nc + T, F, R+1) device tensor."""
        import torch
        T, F, R1 = maps_d.shape
        # range_doppler_plot.py takes np.abs of the stack before CFAR_2D, and the CFAR kernel keeps the sign of a real
        # cell in its numerator: a float32 map is made |map| first (exact, and a no-op on magnitudes)
        maps_d = (maps_d.abs() if maps_d.dtype == torch.float32 else maps_d).contiguous()
        nc = 0 if self._carry is None else self._carry.shape[0]
        cf = torch.empty((nc + T, F, R1), dtype=torch.float64, device=maps_d.device)
        if nc:
            cf[:nc] = self._carry
        _cfar_frames_into(maps_d, cf[nc:], self.fw, self.gw, self.os_rank, dev)
        return cf, nc

    def _phosphor(self, cf, nc, dev):
        """The phosphor stage: data (T, R+1, F) and limits (T, 2) of the last T frames of the CFAR stage's cf, whose
        last hold - 1 frames are carried to the next call."""
        import torch
        lib = _lib.load()
        total, F, R1 = cf.shape
        T, cells = total - nc, F * R1
        stream = _lib.stream_arg(cf.device)
        data = torch.empty((T, R1, F), dtype=torch.float64, device=cf.device)
        limits = torch.empty((T, 2), dtype=torch.float64, device=cf.device)
        _lib.check(lib.prc_persistence_frames(cf.data_ptr(), F, R1, T, cells, nc, self.hold, self.weights.ctypes.data,
                                              data.data_ptr(), _lib.MEM_DEVICE, dev, stream,
                                              _lib.FLAG_ASYNC | _lib.FLAG_MAP_F64 | _lib.FLAG_ORIENT))
        _lib.check(lib.prc_percentiles_frames(data.data_ptr(), cells, T, cells, self._q.ctypes.data,
                                              self._scale.ctypes.data, 2, limits.data_ptr(), _lib.MEM_DEVICE, dev,
                                              stream, _lib.FLAG_ASYNC))
        keep = min(total, self.hold - 1)
        self._carry = cf[total - keep:].clone() if keep else None
        return data, limits

    def run_device(self, maps_d):
        """maps_d: (T, F, R+1) complex64 or float32 CUDA tensor; either way its magnitude is what is rendered, as
        range_doppler_plot.py renders np.abs(xambg).  Returns device tensors data (T, R+1, F) float64 and
        limits (T, 2) = [vmin, vmax], ordered on the current torch stream."""
        import torch
        T, F, R1 = self._check(maps_d)
        if T == 0:
            return (maps_d.new_empty((0, R1, F), dtype=torch.float64),
                    maps_d.new_empty((0, 2), dtype=torch.float64))
        dev = maps_d.device.index if self.device is None else int(self.device)
        return self._phosphor(*self._cf(maps_d, dev), dev)

    def run(self, stack):
        """stack: main.py's (F, R+1, nframes) maps on the host, complex64 or already np.abs-ed float32 / float64
        (CFAR_2D reads float32, as the drop-in does).  Starts a new sequence and streams it through in batches.
        Returns host arrays data (nframes, R+1, F) float64 and limits (nframes, 2)."""
        self.reset()
        parts = [[t.cpu().numpy() for t in self.run_device(maps)]
                 for maps in _host_batches(stack, "stack", "stack", self.device, self.batch)]
        data, limits = (np.concatenate(p) for p in zip(*parts))
        return data, limits


def _host_batches(stack, name, what, device, batch):
    """Device batches of at most ``batch`` maps, frames first, of main.py's (F, R+1, nframes) host maps: complex maps
    as complex64, real ones as float32 (as the drop-in CFAR_2D reads them).  An empty stack gives one empty batch.
    Each batch's device is current while it is used."""
    import torch
    stack = np.asarray(stack)
    if stack.ndim != 3:
        raise ValueError(f"{name} must be (F, R+1, nframes), got {stack.ndim} dimensions")
    if stack.dtype.kind == "c":
        dt = np.complex64
    elif stack.dtype.kind in "biuf":
        dt = np.float32
    else:
        raise TypeError(f"unsupported {what} dtype {stack.dtype}")
    tdev = torch.device("cuda", _lib.current_device(device))
    with torch.cuda.device(tdev):
        for b0 in range(0, max(stack.shape[2], 1), batch):
            maps = np.ascontiguousarray(np.moveaxis(stack[:, :, b0:b0 + batch], 2, 0), dtype=dt)
            yield torch.from_numpy(maps).to(tdev)
