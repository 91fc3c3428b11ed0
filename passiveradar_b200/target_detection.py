"""Target detection on the H100 -- ``CFAR_2D`` with the reference's call signature
(``passiveRadar/target_detection.py:683-703``).  No CPU fallback."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib


def CFAR_2D(X, fw, gw, thresh=None, *, device=None):
    '''constant false alarm rate target detection

    Parameters:
        fw: CFAR kernel width
        gw: number of guard cells
        thresh: detection threshold

    Returns:
        X with CFAR filter applied (float64 like the reference; bool array when ``thresh`` is given)'''
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError("X must be two-dimensional")
    if np.iscomplexobj(X):
        raise TypeError("CFAR_2D expects a real map (the reference is called with np.abs(xambg))")
    x = np.ascontiguousarray(X, dtype=np.float32)
    rows, cols = x.shape
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    if thresh is None:
        cr = np.empty((rows, cols), dtype=np.float32)
        _lib.check(lib.prc_cfar2d_f32(x.ctypes.data, rows, cols, int(fw), int(gw), None, cr.ctypes.data, None,
                                      _lib.MEM_HOST, dev, None, 0))
        return cr.astype(np.float64)
    t = C.c_float(float(thresh))
    det = np.empty((rows, cols), dtype=np.uint8)
    _lib.check(lib.prc_cfar2d_f32(x.ctypes.data, rows, cols, int(fw), int(gw), C.addressof(t), None, det.ctypes.data,
                                  _lib.MEM_HOST, dev, None, 0))
    return det.astype(bool)


# ---------------------------------------------------------------------------------------------- ordered-statistic CFAR
MAX_OS_FRAMES = 65535          # frames of one prc_os_cfar2d_frames call


def os_window_cells(fw, gw):
    """N, the cells of CFAR_2D's window (fw x fw minus the reference's guard hole, NumPy slice rules)."""
    T = np.ones((fw, fw), dtype=np.int64)
    e1 = (fw - gw) // 2
    e2 = fw - e1 + 1
    T[e1:e2, e1:e2] = 0
    return int(T.sum())


def os_rank(fw, gw, k=None):
    """The rank OS_CFAR_2D uses: k, or ceil(3N / 4) when k is None.  Out-of-range windows and ranks are left for the
    library to refuse with its message."""
    if k is not None:
        return int(k)
    fw, gw = int(fw), int(gw)
    if not (1 <= fw <= 64 and gw >= 0):
        return 1
    return -(-3 * os_window_cells(fw, gw) // 4)


def _os_launch(x, rows, cols, nframes, fw, gw, k, out, flags, dev, stream):
    """prc_os_cfar2d_frames over device tensors x (nframes compact float32 / complex64 maps) -> out (float64)."""
    lib = _lib.load()
    cells = rows * cols
    for t0 in range(0, nframes, MAX_OS_FRAMES):
        nb = min(MAX_OS_FRAMES, nframes - t0)
        _lib.check(lib.prc_os_cfar2d_frames(x[t0].data_ptr(), rows, cols, nb, cells, fw, gw, k, out[t0].data_ptr(),
                                            cells, dev, stream, flags))


def OS_CFAR_2D(X, fw, gw, k=None, thresh=None, *, device=None):
    '''ordered-statistic constant false alarm rate target detection (Rohling) on CFAR_2D's window

    Parameters:
        fw: CFAR kernel width
        gw: number of guard cells
        k: rank of the noise estimate among the N window cells, 1 <= k <= N (default ceil(3N / 4))
        thresh: detection threshold

    Returns:
        (X / mean|X|) / (k-th smallest window cell + 1e-10) as float64; bool array when ``thresh`` is given'''
    import torch
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError("X must be two-dimensional")
    if np.iscomplexobj(X):
        raise TypeError("OS_CFAR_2D expects a real map (the reference is called with np.abs(xambg))")
    x = np.ascontiguousarray(X, dtype=np.float32)
    rows, cols = x.shape
    fw, gw = int(fw), int(gw)
    dev = _lib.current_device() if device is None else int(device)
    tdev = torch.device("cuda", dev)
    xd = torch.from_numpy(x).to(tdev)[None]
    cr = torch.empty((1, rows, cols), dtype=torch.float64, device=tdev)
    with torch.cuda.device(tdev):
        _os_launch(xd, rows, cols, 1, fw, gw, os_rank(fw, gw, k), cr, _lib.FLAG_CR_F64, dev,
                   torch.cuda.current_stream(tdev).cuda_stream or 1)
    out = cr[0].cpu().numpy()
    return out if thresh is None else out > thresh


def os_cfar_frames(stack, fw, gw, k=None, *, device=None):
    '''OS_CFAR_2D of every frame of a (T, rows, cols) float32 or complex64 stack (complex maps: their magnitude) in one
    launch per 65 535 frames.  A host array gives a host float64 CR stack; a CUDA tensor gives a float64 CUDA tensor,
    ordered on the current torch stream.  Frame b's CR is bit-identical to a one-frame call on it.'''
    import torch
    host = not (hasattr(stack, "is_cuda") and stack.is_cuda)
    if host:
        a = np.asarray(stack)
        if a.dtype not in (np.float32, np.complex64):
            raise TypeError(f"stack must be float32 or complex64, got {a.dtype}")
        dev = _lib.current_device() if device is None else int(device)
        t = torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", dev))
    else:
        if stack.dtype not in (torch.float32, torch.complex64):
            raise TypeError(f"stack must be float32 or complex64, got {stack.dtype}")
        t = stack.contiguous()
        dev = t.device.index if device is None else int(device)
    if t.dim() != 3:
        raise ValueError(f"stack must be three-dimensional (T, rows, cols), got {t.dim()} dimensions")
    T, rows, cols = t.shape
    fw, gw = int(fw), int(gw)
    out = torch.empty((T, rows, cols), dtype=torch.float64, device=t.device)
    flags = _lib.FLAG_ASYNC | _lib.FLAG_CR_F64 | (_lib.FLAG_ABS_C64 if t.dtype == torch.complex64 else 0)
    if T:
        with torch.cuda.device(t.device):
            _os_launch(t, rows, cols, T, fw, gw, os_rank(fw, gw, k), out, flags, dev,
                       torch.cuda.current_stream(t.device).cuda_stream or 1)
    return out.cpu().numpy() if host else out


# ---------------------------------------------------------------------------------------------- Kalman trackers
# The reference's record dtypes (target_detection.py:9-17, :151-162, :530-537) with np.float -> float64 and
# np.int -> int64 (the aliases NumPy >= 1.24 removed).  Packed, every field 8 bytes: the C structs prc_kalman,
# prc_track and prc_track_simple of include/prcore.h have the same bytes.
kalman_filter_dtype = np.dtype([
    ('x', np.float64, (4,)),
    ('P', np.float64, (4, 4)),
    ('F1', np.float64, (4, 4)),
    ('F2', np.float64, (4, 4)),
    ('Q', np.float64, (4, 4)),
    ('H', np.float64, (2, 4)),
    ('R', np.float64, (2, 2)),
    ('S', np.float64, (2, 2))])

target_track_dtype = np.dtype([
    ('status', np.int64),                     # 0 free, 1 preliminary, 2 confirmed
    ('lifetime', np.int64),
    ('measurement', np.float64, (2,)),
    ('estimate', np.float64, (2,)),
    ('measurement_history', np.float64, (20,)),
    ('kalman_state', kalman_filter_dtype)])

target_track_dtype_simple = np.dtype([
    ('lock_mode', np.float64, (4,)),
    ('measurement', np.float64, (2,)),
    ('measurement_idx', np.int64, (2,)),
    ('estimate', np.float64, (2,)),
    ('range_extent', np.float64),
    ('doppler_extent', np.float64),
    ('kalman_state', kalman_filter_dtype)])

MAX_TRACKS = 64            # largest N_TRACKS of the multi-target tracker kernel


def _real_maps(a, name):
    """float32 / float64 maps as they are, other real dtypes as float64; complex maps are refused."""
    if np.iscomplexobj(a):
        raise TypeError(f"{name} must be real (the reference tracks CFAR_2D output, not complex maps)")
    if a.dtype not in (np.float32, np.float64):
        if a.dtype.kind not in "fiub":
            raise TypeError(f"{name} must be a real numeric array, got {a.dtype}")
        a = a.astype(np.float64)
    return a


def _extent(frame_extent):
    fe = list(frame_extent)
    if len(fe) != 2:
        raise ValueError("frame_extent must be [doppler_extent, range_extent]")
    return float(fe[0]), float(fe[1])


def _is_tensor(x):
    return hasattr(x, "data_ptr") and hasattr(x, "is_cuda")


def _frames_layout(maps, name):
    """(S, T, rows, cols) numpy array or CUDA tensor -> (array, S, T, rows, cols, seq_stride, frame_stride, f64)."""
    if _is_tensor(maps):
        if not maps.is_cuda:
            maps = maps.numpy()
        else:
            import torch
            if maps.dim() != 4:
                raise ValueError(f"{name} must have shape (S, T, rows, cols)")
            if maps.dtype not in (torch.float32, torch.float64):
                raise TypeError(f"{name} must be a float32 or float64 CUDA tensor")
            S, T, rows, cols = maps.shape
            if maps.stride(3) != 1 or maps.stride(2) != cols:
                raise ValueError(f"{name} frames must be contiguous (row-major rows x cols)")
            return maps, S, T, rows, cols, maps.stride(0), maps.stride(1), maps.dtype == torch.float64
    a = _real_maps(np.asarray(maps), name)
    if a.ndim != 4:
        raise ValueError(f"{name} must have shape (S, T, rows, cols)")
    a = np.ascontiguousarray(a)
    S, T, rows, cols = a.shape
    return a, S, T, rows, cols, T * rows * cols, rows * cols, a.dtype == np.float64


def _initial_state(initial_state, dtype, shape):
    """initial_state of a *_frames tracker: None, or records of the tracker's dtype and shape (S, ...)."""
    if initial_state is None:
        return None
    a = np.asarray(initial_state)
    if a.dtype != dtype:
        raise TypeError(f"initial_state must be an array of {dtype}, got {a.dtype}")
    if a.shape != shape:
        raise ValueError(f"initial_state must have shape {shape}, got {a.shape}")
    return a


def _launch(fn, maps, S, T, rows, cols, ss, fs, f64, args, out_dtype, out_shape, device, initial_state=None):
    """Run a tracker entry point on host arrays or on a CUDA tensor (on the tensor's current stream).  With
    initial_state every sequence continues from its records (PRC_FLAG_TRACK_RESUME) instead of starting fresh."""
    lib = _lib.load()
    flags = _lib.FLAG_MAP_F64 if f64 else 0
    hist = np.zeros(out_shape, dtype=out_dtype)
    if initial_state is not None:
        hist[:, 0] = initial_state
        flags |= _lib.FLAG_TRACK_RESUME
    if _is_tensor(maps):
        import torch
        dev = maps.device.index if device is None else int(device)
        if initial_state is not None:
            hd = torch.from_numpy(hist.view(np.uint8).reshape(-1)).to(maps.device)
        else:
            hd = torch.empty(hist.nbytes, dtype=torch.uint8, device=maps.device)
        stream = torch.cuda.current_stream(maps.device).cuda_stream
        _lib.check(getattr(lib, fn)(maps.data_ptr(), rows, cols, S, T, ss, fs, *args, hd.data_ptr(),
                                    _lib.MEM_DEVICE, dev, stream, flags))
        hist.view(np.uint8).reshape(-1)[:] = hd.cpu().numpy()
        return hist
    dev = _lib.current_device() if device is None else int(device)
    _lib.check(getattr(lib, fn)(maps.ctypes.data, rows, cols, S, T, ss, fs, *args, hist.ctypes.data,
                                _lib.MEM_HOST, dev, None, flags))
    return hist


def get_measurements(dataFrame, p, frame_extent, *, device=None):
    ''' extract a list of candidate measurements from a range-doppler map frame
    (reference target_detection.py:164-229)

    Parameters:
        dataFrame:      2D range-Doppler map (rows = Doppler bins, cols = range bins)
        p:              ignored, as in the reference, which always takes the 99.8th percentile
        frame_extent:   [doppler_extent (Hz), range_extent (km)]
    Returns:
        (3, M) float64 array of candidate range, Doppler and strength, strongest first; equal strengths in
        descending position of the transformed frame (DESIGN.md section 11)
    '''
    x = np.asarray(dataFrame)
    if x.ndim != 2:
        raise ValueError("dataFrame must be two-dimensional")
    x = np.ascontiguousarray(_real_maps(x, "dataFrame"))
    dext, rext = _extent(frame_extent)
    rows, cols = x.shape
    n = rows * cols
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    counts = np.zeros(1, dtype=np.int32)
    meas = np.empty((3, n), dtype=np.float64)
    _lib.check(lib.prc_get_measurements_frames(x.ctypes.data, rows, cols, 1, 1, n, n, dext, rext, n,
                                               counts.ctypes.data, meas.ctypes.data, _lib.MEM_HOST, dev, None,
                                               _lib.FLAG_MAP_F64 if x.dtype == np.float64 else 0))
    return np.ascontiguousarray(meas[:, :int(counts[0])])


def _frames_last(data, name):
    a = np.asarray(data)
    if a.ndim != 3:
        raise ValueError(f"{name} must be three-dimensional (rows, cols, Nframes)")
    a = _real_maps(a, name)
    return np.ascontiguousarray(np.moveaxis(a, 2, 0))[None]     # (1, Nframes, rows, cols)


def multitarget_tracker(data, frame_extent, N_TRACKS, *, device=None):
    ''' Radar target tracker for multiple targets (reference target_detection.py:455-526).

    Parameters:
        data:           (rows, cols, Nframes) stack of range-Doppler maps, frames on the last axis
        frame_extent:   [doppler_extent (Hz), range_extent (km)]
        N_TRACKS:       number of tracks, 0 .. MAX_TRACKS
    Returns:
        history:        (Nframes, N_TRACKS) array of target_track_dtype
    '''
    a = np.asarray(data)
    if a.ndim != 3:
        raise ValueError("data must be three-dimensional (rows, cols, Nframes)")
    _real_maps(a[:0], "data")
    _extent(frame_extent)
    n_tracks = int(N_TRACKS)
    if n_tracks < 0:
        raise ValueError("N_TRACKS must be >= 0")
    if n_tracks == 0 or a.shape[2] == 0:
        return np.zeros((a.shape[2], n_tracks), dtype=target_track_dtype)
    return multitarget_tracker_frames(_frames_last(a, "data"), frame_extent, n_tracks, device=device)[0]


def multitarget_tracker_frames(maps, frame_extent, n_tracks, *, initial_state=None, device=None):
    '''multitarget_tracker on S independent sequences in one call.  maps: (S, T, rows, cols) numpy array or CUDA
    tensor (float32 / float64; a tensor's sequences may be strided).  Returns an (S, T, n_tracks) target_track_dtype
    array.  initial_state: an (S, n_tracks) target_track_dtype array -- normally history[:, -1] of an earlier call --
    that each sequence continues from instead of starting with every track free; cutting a sequence anywhere and
    continuing it this way gives the same records as one call.'''
    dext, rext = _extent(frame_extent)
    n_tracks = int(n_tracks)
    if n_tracks < 0:
        raise ValueError("n_tracks must be >= 0")
    m, S, T, rows, cols, ss, fs, f64 = _frames_layout(maps, "maps")
    init = _initial_state(initial_state, target_track_dtype, (S, n_tracks))
    if n_tracks == 0 or S == 0 or T == 0:
        return np.zeros((S, T, n_tracks), dtype=target_track_dtype)
    return _launch("prc_multitarget_track_frames", m, S, T, rows, cols, ss, fs, f64, (dext, rext, n_tracks),
                   target_track_dtype, (S, T, n_tracks), device, init)


def simple_target_tracker(data, rangeExtent, dopplerExtent, *, device=None):
    ''' Single-target tracker (reference target_detection.py:539-681).

    Parameters:
        data:           (rows, cols, Nframes) stack of range-Doppler maps, frames on the last axis
        rangeExtent:    km
        dopplerExtent:  Hz
    Returns:
        (Nframes,) array of target_track_dtype_simple
    '''
    a = np.asarray(data)
    if a.ndim != 3:
        raise ValueError("data must be three-dimensional (rows, cols, Nframes)")
    _real_maps(a[:0], "data")
    if a.shape[2] == 0:
        return np.zeros((0,), dtype=target_track_dtype_simple)
    return simple_tracker_frames(_frames_last(a, "data"), rangeExtent, dopplerExtent, device=device)[0]


def simple_tracker_frames(maps, range_extent, doppler_extent, *, initial_state=None, device=None):
    '''simple_target_tracker on S independent sequences in one call.  maps: (S, T, rows, cols) numpy array or CUDA
    tensor.  Returns an (S, T) target_track_dtype_simple array.  initial_state: an (S,) target_track_dtype_simple
    array -- normally history[:, -1] of an earlier call -- that each sequence continues from instead of the
    tracker's initial record; the record's own range_extent / doppler_extent stay in use.'''
    rext, dext = float(range_extent), float(doppler_extent)
    m, S, T, rows, cols, ss, fs, f64 = _frames_layout(maps, "maps")
    init = _initial_state(initial_state, target_track_dtype_simple, (S,))
    if S == 0 or T == 0:
        return np.zeros((S, T), dtype=target_track_dtype_simple)
    return _launch("prc_simple_track_frames", m, S, T, rows, cols, ss, fs, f64, (rext, dext),
                   target_track_dtype_simple, (S, T), device, init)


def cfar_track(maps_d, fw, gw, frame_extent, n_tracks, *, device=None):
    '''The reference tracker scripts' chain on the device: CFAR_2D(|map|, fw, gw) of every frame, then
    multitarget_tracker.  maps_d: (T, F, R+1) complex64 CUDA tensor (FramePipeline.run_device output); the maps are
    never copied to the host.  Returns the (T, n_tracks) target_track_dtype history.'''
    import torch
    if not (_is_tensor(maps_d) and maps_d.is_cuda and maps_d.dtype == torch.complex64 and maps_d.dim() == 3):
        raise TypeError("maps_d must be a (T, F, R+1) complex64 CUDA tensor")
    dext, rext = _extent(frame_extent)
    n_tracks = int(n_tracks)
    if n_tracks < 0:
        raise ValueError("n_tracks must be >= 0")
    T, F, R1 = maps_d.shape
    if n_tracks == 0 or T == 0:
        return np.zeros((T, n_tracks), dtype=target_track_dtype)
    maps_d = maps_d.contiguous()
    lib = _lib.load()
    dev = maps_d.device.index if device is None else int(device)
    cf = torch.empty((1, T, F, R1), dtype=torch.float32, device=maps_d.device)
    stream = torch.cuda.current_stream(maps_d.device).cuda_stream
    for t in range(T):
        _lib.check(lib.prc_cfar2d_f32(maps_d[t].data_ptr(), F, R1, int(fw), int(gw), None, cf[0, t].data_ptr(), None,
                                      _lib.MEM_DEVICE, dev, stream, _lib.FLAG_ABS_C64 | _lib.FLAG_ASYNC))
    return _launch("prc_multitarget_track_frames", cf, 1, T, F, R1, T * F * R1, F * R1, False,
                   (dext, rext, n_tracks), target_track_dtype, (1, T, n_tracks), dev)[0]


# ---------------------------------------------------------------------------------------------- tracker scripts' chain
_MULTI_WORDS = target_track_dtype.itemsize // 8           # a record as 8-byte words: status is word 0, estimate 4-5
_SIMPLE_WORDS = target_track_dtype_simple.itemsize // 8   # lock_mode is words 0-3, estimate 8-9


class TrackerPipeline:
    """The chain of the reference's tracker scripts (multitarget_kalman_tracker.py / simple_kalman_tracker.py) on the
    device, for a stream of maps:

        CF[:, :, i] = CFAR_2D(|xambg[:, :, i]|, fw, gw)                     (float64 stack, one launch per batch)
        history = multitarget_tracker(CF, [max_doppler, max_range], n_tracks)  or
                  simple_target_tracker(CF, max_range, max_doppler)
        the scripts' masks of the estimates, and with render=True
        data = fliplr(persistence(CF, kk, hold, decay).T), [percentile(data, 35), 1.5 * percentile(data, 99)]

    The trackers read the float64 CF itself, as the scripts do.  ``run_device`` carries the last tracker records
    (continued with PRC_FLAG_TRACK_RESUME) and the last hold - 1 CF frames to the next call, so a stack cut into
    batches of any size, one map per call included, gives the same bytes as one call; ``reset()`` starts a new
    sequence.  ``run`` takes the scripts' host layout (F, R+1, nframes).  Plotting stays with the caller.

    ``cfar="os"`` replaces CFAR_2D by the ordered-statistic CFAR on the same window (``OS_CFAR_2D``, rank ``os_rank``
    or ceil(3N / 4)); the trackers and the phosphor frames then read its CR."""

    def __init__(self, max_range, max_doppler, *, tracker="multi", n_tracks=10, fw=18, gw=4, hold=20, decay=0.90,
                 render=True, batch=64, device=None, cfar="ca", os_rank=None):
        from .plotting_tools import _cfar_choice, _decay_plan
        if tracker not in ("multi", "simple"):
            raise ValueError(f"tracker must be 'multi' or 'simple', got {tracker!r}")
        self.tracker = tracker
        self.max_range, self.max_doppler = float(max_range), float(max_doppler)
        self.n_tracks = int(n_tracks) if tracker == "multi" else 1
        if not 0 <= self.n_tracks <= MAX_TRACKS:
            raise ValueError(f"n_tracks={n_tracks} outside [0, {MAX_TRACKS}]")
        self.fw, self.gw, self.hold, self.decay = int(fw), int(gw), int(hold), decay
        if not (1 <= self.fw <= 64) or self.gw < 0 or self.fw * self.fw == self.gw * self.gw:
            raise ValueError(f"fw={fw} gw={gw}: CFAR_2D needs 1 <= fw <= 64, gw >= 0 and fw != gw")
        self.cfar, self.os_rank = _cfar_choice(cfar, os_rank, self.fw, self.gw)
        if self.hold < 1:
            raise ValueError("hold must be >= 1")
        if int(batch) < 1:
            raise ValueError("batch must be >= 1")
        self.render, self.batch, self.device = bool(render), int(batch), device
        # CF is float64 in the scripts (np.zeros(xambg.shape)): the products are float64 whatever decay's type
        self.weights, _ = _decay_plan(np.float64, decay, self.hold)
        self.dtype = target_track_dtype if tracker == "multi" else target_track_dtype_simple
        self.reset()

    @classmethod
    def from_config(cls, config, tracker="multi", **kw):
        """From the dict ``passiveRadar.config.getConfiguration`` returns: its max_range_actual and
        max_doppler_actual are the extents the scripts pass their tracker."""
        missing = [k for k in ("max_range_actual", "max_doppler_actual") if k not in config]
        if missing:
            raise ValueError(f"config lacks {missing} (getConfiguration derives them)")
        return cls(config["max_range_actual"], config["max_doppler_actual"], tracker=tracker, **kw)

    def reset(self):
        """Start a new sequence: the next map is frame 0 of the tracker and of the persistence."""
        self._shape = None
        self._state = None          # the last frame's tracker records (uint8 device tensor)
        self._carry = None          # the last hold - 1 CF frames

    def records(self, history, T=None):
        """The ``history`` bytes of ``run_device`` (T maps) as the tracker's NumPy records: (T, n_tracks)
        target_track_dtype for the multi-target tracker, (T,) target_track_dtype_simple for the simple one.  T may be
        left out unless n_tracks is 0."""
        raw = history.cpu().numpy() if _is_tensor(history) else np.asarray(history, dtype=np.uint8)
        a = np.frombuffer(raw.tobytes(), dtype=self.dtype).copy()
        return a.reshape(-1 if T is None else T, self.n_tracks) if self.tracker == "multi" else a

    def run_device(self, maps_d):
        """maps_d: (T, F, R+1) complex64 or float32 CUDA tensor (``RecordingPipeline.run_device`` output); either way
        its magnitude is tracked, as the scripts track np.abs(xambg).  Returns a dict of device tensors, ordered on
        the current torch stream:

        * ``cf``: the (T, F, R+1) float64 CFAR_2D maps the tracker and the phosphor frames read;
        * ``history``: the tracker records as raw bytes (``records()`` turns them into NumPy records);
        * multi-target tracker: ``track_range``, ``track_doppler`` (T, n_tracks) float64 estimates, NaN where the
          track is not confirmed (status != 2);
        * simple tracker: ``estimate_locked``, ``estimate_unlocked`` (T, 2) estimates, NaN in the rows where
          lock_mode[:, 0] is set / not set;
        * with render=True: ``data`` (T, R+1, F) float64 and ``limits`` (T, 2) = [vmin, vmax], as
          ``RenderPipeline.run_device`` gives them."""
        import torch
        from .plotting_tools import PERCENTILES, VMAX_SCALE, _cfar_frames_into, _stream_arg
        if not (_is_tensor(maps_d) and maps_d.is_cuda and maps_d.dim() == 3):
            raise TypeError("maps_d must be a (T, F, R+1) CUDA tensor")
        if maps_d.dtype not in (torch.complex64, torch.float32):
            raise TypeError(f"maps_d must be complex64 or float32, got {maps_d.dtype}")
        T, F, R1 = maps_d.shape
        if self._shape is not None and self._shape != (F, R1):
            raise ValueError(f"maps of shape {(F, R1)} continue a sequence of {self._shape} maps; call reset() first")
        if F * R1 > 1 << 19:
            raise ValueError(f"a {F} x {R1} map exceeds the trackers' maximum of {1 << 19} cells")
        tdev = maps_d.device
        dev = tdev.index if self.device is None else int(self.device)
        N, rec = self.n_tracks, self.dtype.itemsize * self.n_tracks
        out = {"history": torch.empty(T * rec, dtype=torch.uint8, device=tdev)}
        if T == 0:
            out["cf"] = torch.empty((0, F, R1), dtype=torch.float64, device=tdev)
            if self.render:
                out["data"] = torch.empty((0, R1, F), dtype=torch.float64, device=tdev)
                out["limits"] = torch.empty((0, 2), dtype=torch.float64, device=tdev)
            return self._masks(out, 0, torch)
        lib = _lib.load()
        # the scripts take np.abs of the stack before CFAR_2D, and the CFAR kernel keeps the sign of a real cell in its
        # numerator: a float32 map is made |map| first (exact, and a no-op on magnitudes)
        maps_d = (maps_d.abs() if maps_d.dtype == torch.float32 else maps_d).contiguous()
        stream = _stream_arg(torch, tdev)
        nc = 0 if self._carry is None else self._carry.shape[0]
        cells = F * R1
        cf = torch.empty((nc + T, F, R1), dtype=torch.float64, device=tdev)
        if nc:
            cf[:nc] = self._carry
        _cfar_frames_into(lib, self.cfar, self.os_rank, maps_d, cf[nc:], self.fw, self.gw, dev, stream)
        hist = out["history"]
        flags = _lib.FLAG_ASYNC | _lib.FLAG_MAP_F64
        if self._state is not None:
            hist[:rec] = self._state
            flags |= _lib.FLAG_TRACK_RESUME
        if self.tracker == "multi":
            if N:
                _lib.check(lib.prc_multitarget_track_frames(cf[nc].data_ptr(), F, R1, 1, T, T * cells, cells,
                                                            self.max_doppler, self.max_range, N, hist.data_ptr(),
                                                            _lib.MEM_DEVICE, dev, stream, flags))
        else:
            _lib.check(lib.prc_simple_track_frames(cf[nc].data_ptr(), F, R1, 1, T, T * cells, cells, self.max_range,
                                                   self.max_doppler, hist.data_ptr(), _lib.MEM_DEVICE, dev, stream,
                                                   flags))
        if self.render:
            data = torch.empty((T, R1, F), dtype=torch.float64, device=tdev)
            limits = torch.empty((T, 2), dtype=torch.float64, device=tdev)
            q = np.array(PERCENTILES, dtype=np.float64)
            scale = np.array([1.0, VMAX_SCALE], dtype=np.float64)
            _lib.check(lib.prc_persistence_frames(cf.data_ptr(), F, R1, T, cells, nc, self.hold,
                                                  self.weights.ctypes.data, data.data_ptr(), _lib.MEM_DEVICE, dev,
                                                  stream, _lib.FLAG_ASYNC | _lib.FLAG_MAP_F64 | _lib.FLAG_ORIENT))
            _lib.check(lib.prc_percentiles_frames(data.data_ptr(), cells, T, cells, q.ctypes.data, scale.ctypes.data,
                                                  2, limits.data_ptr(), _lib.MEM_DEVICE, dev, stream, _lib.FLAG_ASYNC))
            out["data"], out["limits"] = data, limits
            keep = min(nc + T, self.hold - 1)
            self._carry = cf[nc + T - keep:].clone() if keep else None
        self._shape = (F, R1)
        self._state = hist[(T - 1) * rec:].clone() if rec else None
        out["cf"] = cf[nc:]
        return self._masks(out, T, torch)

    def _masks(self, out, T, torch):
        """The scripts' masks of the estimates, from the history bytes."""
        hist = out["history"]
        dev = hist.device
        nan = torch.tensor(float("nan"), dtype=torch.float64, device=dev)
        if self.tracker == "multi":
            # multitarget_kalman_tracker.py:66-75: estimate[..., 0] / [..., 1], NaN where status != 2
            w = hist.view(torch.float64).view(T, self.n_tracks, _MULTI_WORDS)
            unconfirmed = hist.view(torch.int64).view(T, self.n_tracks, _MULTI_WORDS)[:, :, 0] != 2
            out["track_range"] = torch.where(unconfirmed, nan, w[:, :, 4])
            out["track_doppler"] = torch.where(unconfirmed, nan, w[:, :, 5])
        else:
            # simple_kalman_tracker.py:63-73: unlocked = lock_mode[:, 0].astype(bool)
            w = hist.view(torch.float64).view(T, _SIMPLE_WORDS)
            unlocked = (w[:, 0] != 0)[:, None]
            out["estimate_locked"] = torch.where(unlocked, nan, w[:, 8:10])
            out["estimate_unlocked"] = torch.where(~unlocked, nan, w[:, 8:10])
        return out

    def run(self, xambg):
        """xambg: the scripts' (F, R+1, nframes) maps on the host, complex64 or already np.abs-ed float32 / float64
        (CFAR_2D reads float32, as the drop-in does).  Starts a new sequence and streams it through in batches.
        Returns host arrays: ``history`` exactly as multitarget_tracker / simple_target_tracker return it, the masked
        estimates and, with render=True, ``data`` (nframes, R+1, F) and ``limits`` (nframes, 2)."""
        import torch
        xambg = np.asarray(xambg)
        if xambg.ndim != 3:
            raise ValueError(f"xambg must be (F, R+1, nframes), got {xambg.ndim} dimensions")
        if xambg.dtype.kind == "c":
            dt = np.complex64
        elif xambg.dtype.kind in "biuf":
            dt = np.float32
        else:
            raise TypeError(f"unsupported map dtype {xambg.dtype}")
        N = xambg.shape[2]
        dev = _lib.current_device() if self.device is None else int(self.device)
        tdev = torch.device("cuda", dev)
        self.reset()
        parts = []
        with torch.cuda.device(tdev):
            for b0 in range(0, max(N, 1), self.batch):      # an empty stack still gives empty outputs
                b1 = min(N, b0 + self.batch)
                maps = torch.from_numpy(np.ascontiguousarray(np.moveaxis(xambg[:, :, b0:b1], 2, 0), dtype=dt))
                got = self.run_device(maps.to(tdev))
                del got["cf"]
                parts.append({k: v.cpu().numpy() for k, v in got.items()})
        res = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
        res["history"] = self.records(res["history"], N)
        return res
