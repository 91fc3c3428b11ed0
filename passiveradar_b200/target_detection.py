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


def _launch(fn, maps, S, T, rows, cols, ss, fs, f64, args, out_dtype, out_shape, device):
    """Run a tracker entry point on host arrays or on a CUDA tensor (on the tensor's current stream)."""
    lib = _lib.load()
    flags = _lib.FLAG_MAP_F64 if f64 else 0
    hist = np.zeros(out_shape, dtype=out_dtype)
    if _is_tensor(maps):
        import torch
        dev = maps.device.index if device is None else int(device)
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


def multitarget_tracker_frames(maps, frame_extent, n_tracks, *, device=None):
    '''multitarget_tracker on S independent sequences in one call.  maps: (S, T, rows, cols) numpy array or CUDA
    tensor (float32 / float64; a tensor's sequences may be strided).  Returns an (S, T, n_tracks) target_track_dtype
    array.'''
    dext, rext = _extent(frame_extent)
    n_tracks = int(n_tracks)
    if n_tracks < 0:
        raise ValueError("n_tracks must be >= 0")
    m, S, T, rows, cols, ss, fs, f64 = _frames_layout(maps, "maps")
    if n_tracks == 0 or S == 0 or T == 0:
        return np.zeros((S, T, n_tracks), dtype=target_track_dtype)
    return _launch("prc_multitarget_track_frames", m, S, T, rows, cols, ss, fs, f64, (dext, rext, n_tracks),
                   target_track_dtype, (S, T, n_tracks), device)


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


def simple_tracker_frames(maps, range_extent, doppler_extent, *, device=None):
    '''simple_target_tracker on S independent sequences in one call.  maps: (S, T, rows, cols) numpy array or CUDA
    tensor.  Returns an (S, T) target_track_dtype_simple array.'''
    rext, dext = float(range_extent), float(doppler_extent)
    m, S, T, rows, cols, ss, fs, f64 = _frames_layout(maps, "maps")
    if S == 0 or T == 0:
        return np.zeros((S, T), dtype=target_track_dtype_simple)
    return _launch("prc_simple_track_frames", m, S, T, rows, cols, ss, fs, f64, (rext, dext),
                   target_track_dtype_simple, (S, T), device)


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
