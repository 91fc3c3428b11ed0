"""Frame pipeline: streams of CPI frames through  LS_Filter -> fast_xambg  on one H100.

The reference processes one dask chunk per task on a thread pool (``main.py:169-194``); with ``overlap_cpi`` on, the
shipped setting, a CPI frame is a chunk plus a quarter CPI of each neighbour (``passiveradar_b200.recording`` builds
those frames).  This pipeline takes frames that are already whole.  On the GPU the same independence is used differently: a
``FramePipeline`` owns ``nslots`` CUDA streams, each with its own device buffers and
libprcore workspace, and issues batch ``b`` of ``batch`` frames on slot ``b % nslots`` through
``prc_frames_c64`` (one launch of each kernel per batch).  Host->device copies, the kernels of
neighbouring batches and device->host copies of the maps overlap; the one-CTA-per-frame Toeplitz
solves of a batch run side by side and hide behind the other slots' kernels.  torch is used for device memory, pinned host memory, streams and events only.

    pipe = FramePipeline(n=2**20, range_bins=300, freq_bins=256)      # LS filterLen = range_bins
    maps = pipe.run_host(ref_frames, srv_frames)      # (nframes, F, R+1, 1) complex64, host
    pipe.run_device(ref_d, srv_d, maps_d)             # everything resident in HBM
"""
from __future__ import annotations

import numpy as np
import scipy.signal as signal

from . import _lib


def _torch():
    import torch
    return torch


def pinned_empty(shape, dtype=np.complex64):
    """Host ndarray backed by page-locked memory (so copies to the GPU are truly async).  The array owns its
    memory: it is released when the last reference to the array goes away."""
    torch = _torch()
    tdt = {np.dtype(np.complex64): torch.complex64, np.dtype(np.float32): torch.float32,
           np.dtype(np.float64): torch.float64}[np.dtype(dtype)]
    t = torch.empty(tuple(shape) if not isinstance(shape, int) else (shape,), dtype=tdt, pin_memory=True)
    return t.numpy()          # the ndarray keeps the tensor (its base object) alive


class FramePipeline:
    """``nslots`` CUDA streams, each taking ``batch`` frames per library call (``prc_frames_c64``): one launch of each
    kernel covers the whole batch, the Toeplitz solves of a batch run side by side, and neighbouring slots overlap
    their copies and kernels."""

    def __init__(self, n, range_bins, freq_bins, filter_len=None, reg=1.0, peek=10,
                 window=("kaiser", 5.0), device=None, nslots=4, batch=16):
        torch = _torch()
        if not torch.cuda.is_available():
            raise _lib.PrcoreError(_lib.PRC_E_CUDA, "FramePipeline needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.n = int(n)
        self.R = int(range_bins)
        self.F = int(freq_bins)
        self.filter_len = self.R if filter_len is None else int(filter_len)
        self.peek = int(peek)
        self.reg = float(reg)
        self.device = _lib.current_device() if device is None else int(device)
        self.tdev = torch.device("cuda", self.device)
        self.nslots = max(1, int(nslots))
        self.batch = max(1, int(batch))
        if isinstance(window, (tuple, str)):
            window = signal.get_window(window, self.n)
        self.window = None
        if window is not None:
            w = np.ascontiguousarray(window, dtype=np.float64)
            if w.shape != (self.n,):
                raise ValueError(f"window must have shape ({self.n},)")
            self.window = torch.from_numpy(w.astype(np.float32)).to(self.tdev)
        with torch.cuda.device(self.tdev):
            self.streams = [torch.cuda.Stream(device=self.tdev) for _ in range(self.nslots)]
            self.done = [torch.cuda.Event() for _ in range(self.nslots)]
        self._host_bufs = None            # device staging of run_host, allocated on first use
        self.map_bytes = self.F * (self.R + 1) * 8
        self.frame_bytes = 2 * self.n * 8

    # ------------------------------------------------------------------ one batch, device pointers
    def _enqueue(self, ref_ptr, srv_ptr, nf, stride, map_ptr, stream, taps_ptr=None, cleaned_ptr=None):
        flags = _lib.FLAG_ASYNC | (_lib.FLAG_WINDOW_F32 if self.window is not None else 0)
        st = self.lib.prc_frames_c64(ref_ptr, srv_ptr, self.n, nf, stride, self.filter_len, self.peek, self.reg,
                                     self.R, self.F,
                                     None if self.window is None else self.window.data_ptr(),
                                     map_ptr, taps_ptr, cleaned_ptr, _lib.MEM_DEVICE, self.device,
                                     stream.cuda_stream, flags)
        _lib.check(st)

    def ls_status(self, slot, nf):
        """Toeplitz-solve status of the last batch issued on ``slot`` (synchronises that stream): array of nf ints,
        0 = ok, 1 = normal equations not positive definite (the synchronous LS_Filter raises LinAlgError then)."""
        import ctypes as C
        st = (C.c_int * nf)()
        _lib.check(self.lib.prc_ls_status(self.device, self.streams[slot].cuda_stream, st, nf))
        return np.frombuffer(st, dtype=np.int32).copy()

    def _raise_on_singular(self, issued):
        for slot, first, nf in issued:
            bad = np.nonzero(self.ls_status(slot, nf))[0]
            if bad.size:
                raise np.linalg.LinAlgError(
                    f"LS normal equations are not positive definite (singular Gram matrix) in frame {first + int(bad[0])}")

    def run_device(self, ref_d, srv_d, maps_d, check=False):
        """ref_d, srv_d: (nframes, n) complex64 CUDA tensors (rows may be strided); maps_d: (nframes, F, R+1) complex64.
        Work is forked from, and joined back into, the current torch stream.  ``check=True`` synchronises and raises
        ``LinAlgError`` for a frame whose normal equations were singular; otherwise the caller may query
        :meth:`ls_status`."""
        torch = _torch()
        nf = ref_d.shape[0]
        stride = ref_d.stride(0) if nf > 1 else self.n
        if nf > 1 and srv_d.stride(0) != stride:
            raise ValueError("ref_d and srv_d must have the same frame stride")
        if ref_d.stride(-1) != 1 or srv_d.stride(-1) != 1 or not maps_d.is_contiguous():
            raise ValueError("frames must be contiguous along the sample axis and maps_d must be contiguous")
        if maps_d.shape[0] < nf or tuple(maps_d.shape[1:3]) != (self.F, self.R + 1):
            raise ValueError(f"maps_d must have shape (>= {nf}, {self.F}, {self.R + 1})")
        cur = torch.cuda.current_stream(self.tdev)
        fork = torch.cuda.Event()
        fork.record(cur)
        nb = -(-nf // self.batch)
        used = min(self.nslots, nb)
        for s in self.streams[:used]:
            s.wait_event(fork)
        issued = {}
        for b in range(nb):
            k = b % self.nslots
            i0 = b * self.batch
            m = min(self.batch, nf - i0)
            self._enqueue(ref_d[i0].data_ptr(), srv_d[i0].data_ptr(), m, stride, maps_d[i0].data_ptr(), self.streams[k])
            issued[k] = (k, i0, m)
        for k in range(used):
            self.done[k].record(self.streams[k])
            cur.wait_event(self.done[k])
        if check:
            self._raise_on_singular(issued.values())
        return maps_d

    def run_host(self, ref_frames, srv_frames, out=None):
        """ref_frames, srv_frames: (nframes, n) complex64 host arrays (pinned for full overlap).
        Returns (nframes, F, R+1, 1) complex64 host array; synchronises before returning and raises ``LinAlgError``
        if a frame's normal equations were singular (as the synchronous ``LS_Filter`` does).  Pass a preallocated
        (ideally pinned) ``out`` when streaming: without it a new pinned array is allocated per call."""
        torch = _torch()
        ref_frames = np.asarray(ref_frames)
        srv_frames = np.asarray(srv_frames)
        if ref_frames.shape != srv_frames.shape:
            raise ValueError('Input vectors must have the same length')
        if ref_frames.ndim != 2 or ref_frames.shape[1] != self.n:
            raise ValueError(f"expected frames of shape (nframes, {self.n})")
        if ref_frames.dtype != np.complex64 or srv_frames.dtype != np.complex64:
            raise TypeError("frames must be complex64")
        nf = ref_frames.shape[0]
        if out is None:
            out = pinned_empty((nf, self.F, self.R + 1, 1))
        if self._host_bufs is None:
            with torch.cuda.device(self.tdev):
                mk = lambda *shape: torch.empty(shape, dtype=torch.complex64, device=self.tdev)
                self._host_bufs = [(mk(self.batch, self.n), mk(self.batch, self.n), mk(self.batch, self.F, self.R + 1))
                                   for _ in range(self.nslots)]
        tref = torch.from_numpy(ref_frames)
        tsrv = torch.from_numpy(srv_frames)
        tout = torch.from_numpy(out.reshape(nf, self.F, self.R + 1))
        nb = -(-nf // self.batch)
        last = {}
        for b in range(nb):
            k = b % self.nslots
            i0 = b * self.batch
            m = min(self.batch, nf - i0)
            s = self.streams[k]
            rd, sd, md = self._host_bufs[k]
            if k in last:
                # the slot's status words are overwritten by its next batch: look at them first (this waits for the
                # batch issued nslots batches ago, which the copies below have to wait for anyway)
                self._raise_on_singular([last[k]])
            with torch.cuda.stream(s):
                # slot buffers are reused in stream order: the copies below wait for batch b - nslots
                rd[:m].copy_(tref[i0:i0 + m], non_blocking=True)
                sd[:m].copy_(tsrv[i0:i0 + m], non_blocking=True)
                self._enqueue(rd.data_ptr(), sd.data_ptr(), m, self.n, md.data_ptr(), s)
                tout[i0:i0 + m].copy_(md[:m], non_blocking=True)
            last[k] = (k, i0, m)
        self._raise_on_singular(last.values())          # synchronises every used stream
        for s in self.streams:
            s.synchronize()
        return out

    def process(self, ref, srv):
        """One frame, host arrays in, (F, R+1, 1) map out (convenience; synchronous)."""
        ref = _lib.as_c64(ref, "refChannel")
        srv = _lib.as_c64(srv, "srvChannel")
        return self.run_host(ref[None, :], srv[None, :])[0]
