"""ctypes binding of libprcore.so (C ABI: include/prcore.h).

The library is the ONLY compute path of this package: if it is missing, cannot
be built, or finds no CUDA device, every operator raises -- there is no CPU
fallback (the numpy oracle under ``oracle/`` is test infrastructure and is never
imported from here).
"""
from __future__ import annotations

import ctypes as C
import os
import sys
import threading

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PRC_LIBRARY") or os.path.join(_PKG, "libprcore.so")     # PRC_LIBRARY: A/B builds during development

PRC_OK = 0
PRC_E_INVALID = -1
PRC_E_CUDA = -2
PRC_E_SINGULAR = -3
PRC_E_NOMEM = -4
MEM_HOST = 0
MEM_DEVICE = 1
FLAG_ASYNC = 1
FLAG_WINDOW_F32 = 2
FLAG_ABS_C64 = 4
FLAG_MAP_F64 = 8
FLAG_CR_F64 = 16
FLAG_PROD_F32 = 32
FLAG_ORIENT = 64
FLAG_TRACK_RESUME = 128
FLAG_CHANNEL_PAIR = 256
IQ_C64, IQ_I8, IQ_I16 = 0, 1, 2
MIX_NONE, MIX_C64, MIX_C128, MIX_F64, MIX_FS64 = 0, 1, 2, 3, 4
DT_I8, DT_U8, DT_I16, DT_F32, DT_F64, DT_C64, DT_C128 = 0, 1, 2, 3, 4, 5, 6
DEC_RAW = 16

# every symbol include/prcore.h declares: name -> (restype, argtypes)
_c64p = C.c_void_p
SIGNATURES = {
    "prc_version": (C.c_int, []),
    "prc_last_error": (C.c_char_p, []),
    "prc_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "prc_init": (C.c_int, [C.c_int]),
    "prc_shutdown": (None, []),
    "prc_sync": (C.c_int, [C.c_int, C.c_void_p]),
    "prc_launch_count": (C.c_uint64, []),
    "prc_profile_enable": (C.c_int, [C.c_int]),
    "prc_profile_collect": (C.c_int, []),
    "prc_profile_kernels": (C.c_int, []),
    "prc_profile_read": (C.c_int, [C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    "prc_profile_reset": (C.c_int, []),
    "prc_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_uint64]),
    "prc_host_free": (C.c_int, [C.c_void_p]),
    "prc_host_register": (C.c_int, [C.c_void_p, C.c_uint64]),
    "prc_host_unregister": (C.c_int, [C.c_void_p]),
    "prc_xambg_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                C.c_int64, _c64p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_ls_filter_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int, C.c_float, _c64p, _c64p,
                                    C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_ls_toeplitz_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int, _c64p, _c64p,
                                      C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_ls_multiple_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_int,
                                      _c64p, _c64p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_ls_multiple_frames_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_double, C.c_void_p,
                                             C.c_int, _c64p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_nlms_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_int, _c64p,
                               _c64p, _c64p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_frame_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                                C.c_void_p, _c64p, _c64p, _c64p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_frames_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                                 C.c_void_p, _c64p, _c64p, _c64p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_nlms_frames_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_int,
                                      _c64p, _c64p, _c64p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_xambg_frames_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p, _c64p,
                                       C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_gal_jpe_frames_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_double,
                                         C.c_double, C.c_int, _c64p, _c64p, _c64p, C.c_int, C.c_int, C.c_void_p,
                                         C.c_uint]),
    "prc_ls_svd_frames_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int, _c64p, _c64p,
                                        C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_frames_multi_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int,
                                       C.c_float, C.c_int, C.c_int, C.c_void_p, _c64p, _c64p, C.c_int, C.c_void_p,
                                       C.c_uint]),
    "prc_ls_status": (C.c_int,[C.c_int, C.c_void_p, C.POINTER(C.c_int), C.c_int]),
    "prc_set_option": (C.c_int, [C.c_char_p, C.c_int]),
    "prc_get_option": (C.c_int, [C.c_char_p, C.POINTER(C.c_int)]),
    "prc_direct_xambg_c64": (C.c_int, [_c64p, _c64p, C.c_int64, C.c_int, C.c_int, C.c_double, _c64p,
                                       C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_iq_mix_c64": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_double, C.c_double, C.c_double,
                                 _c64p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_resample_out_len": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int64)]),
    "prc_frontend_c64": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_double, C.c_double, C.c_double,
                                   C.c_int, C.c_int, C.c_void_p, C.c_int, _c64p, C.c_int64,
                                   C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_frontend_chunks_c64": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_double,
                                          C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, _c64p,
                                          C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_cfar2d_f32": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_cfar2d_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                    C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_os_cfar2d_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int,
                                       C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_uint]),
    "prc_persistence_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_percentiles_frames": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_get_measurements_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64,
                                              C.c_double, C.c_double, C.c_int64, C.c_void_p, C.c_void_p,
                                              C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_multitarget_track_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64,
                                               C.c_double, C.c_double, C.c_int, C.c_void_p,
                                               C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_simple_track_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64,
                                          C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_channel_offset": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                     C.c_uint]),
    "prc_xcorr": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int64,
                            C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint]),
    "prc_psd_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int,
                                 C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                 C.c_uint]),
    "prc_decimate_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int, C.c_double, C.c_double,
                                    C.c_double, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                    C.c_uint]),
    "prc_normalize": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_uint]),
}


# the tracker records of include/prcore.h (byte for byte the reference's NumPy dtypes)
class PrcKalman(C.Structure):
    _fields_ = [("x", C.c_double * 4), ("P", C.c_double * 16), ("F1", C.c_double * 16), ("F2", C.c_double * 16),
                ("Q", C.c_double * 16), ("H", C.c_double * 8), ("R", C.c_double * 4), ("S", C.c_double * 4)]


class PrcTrack(C.Structure):
    _fields_ = [("status", C.c_int64), ("lifetime", C.c_int64), ("measurement", C.c_double * 2),
                ("estimate", C.c_double * 2), ("measurement_history", C.c_double * 20), ("kalman_state", PrcKalman)]


class PrcTrackSimple(C.Structure):
    _fields_ = [("lock_mode", C.c_double * 4), ("measurement", C.c_double * 2), ("measurement_idx", C.c_int64 * 2),
                ("estimate", C.c_double * 2), ("range_extent", C.c_double), ("doppler_extent", C.c_double),
                ("kalman_state", PrcKalman)]

_lib = None
_lock = threading.Lock()


class PrcoreError(RuntimeError):
    """A libprcore call returned a non-zero status."""

    def __init__(self, code, message):
        super().__init__(f"libprcore error {code}: {message}")
        self.code = code


def load(build_if_missing: bool = True):
    """Load (building first if the .so is absent and nvcc exists) and type the library."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if build_if_missing and not os.environ.get("PRC_LIBRARY"):
            # rebuild when the library is missing OR older than any source/header (a stale .so after an edit is
            # the worst kind of bug); a no-op when up to date.  Without nvcc an existing library is used as is
            # (the GPU box receives the library built here).
            from . import build as _build
            try:
                _build.build(force=False)
            except RuntimeError:
                if not os.path.exists(LIB_PATH):
                    raise
        if not os.path.exists(LIB_PATH):
            raise OSError(f"{LIB_PATH} not found")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(status: int):
    if status == PRC_OK:
        return
    msg = load().prc_last_error().decode("utf-8", "replace")
    if status == PRC_E_SINGULAR:
        raise np.linalg.LinAlgError(msg or "Singular matrix")
    if status == PRC_E_NOMEM:
        raise MemoryError(msg)
    raise PrcoreError(status, msg)


def set_option(name: str, value: int):
    """Run-time switch of the library (include/prcore.h: "fft", "fft_min_n", "frame_onepass").

    ``get_option`` also reads "fft_ctas_ls", "fft_ctas_fir" and "fft_ctas_frame": CTAs per SM of the FFT-domain LS
    and FIR kernels at L = 2048 and of the one-pass frame kernel on the current device, which their one-wave grids are
    sized from.  Those names are read-only: setting one raises PrcoreError."""
    check(load().prc_set_option(name.encode(), int(value)))


def get_option(name: str) -> int:
    v = C.c_int(0)
    check(load().prc_get_option(name.encode(), C.byref(v)))
    return v.value


def device_count() -> int:
    n = C.c_int(0)
    st = load().prc_device_count(C.byref(n))
    return n.value if st == PRC_OK else 0


def launch_count() -> int:
    return int(load().prc_launch_count())


def profile(enable: bool):
    check(load().prc_profile_enable(1 if enable else 0))


def profile_reset():
    check(load().prc_profile_reset())


def profile_read():
    """{kernel name: (total_ms, launches)} accumulated since the last reset (synchronises)."""
    lib = load()
    check(lib.prc_profile_collect())
    out = {}
    for i in range(lib.prc_profile_kernels()):
        name = C.c_char_p()
        ms = C.c_double()
        cnt = C.c_uint64()
        check(lib.prc_profile_read(i, C.byref(name), C.byref(ms), C.byref(cnt)))
        out[name.value.decode()] = (ms.value, int(cnt.value))
    return out


def current_device(device=None) -> int:
    """Device used by the drop-in operators: ``device`` when given, else PRC_DEVICE, else LOCAL_RANK (torchrun), else 0."""
    if device is not None:
        return int(device)
    for key in ("PRC_DEVICE", "LOCAL_RANK"):
        v = os.environ.get(key)
        if v not in (None, ""):
            return int(v)
    return 0


# ---------------------------------------------------------------------------------------------- torch <-> library
# NumPy dtype -> the PRC_DT_* code of an input the library reads natively, and -> the PRC_IQ_* kind of raw IQ
DT_CODES = {np.dtype(np.int8): DT_I8, np.dtype(np.uint8): DT_U8, np.dtype(np.int16): DT_I16,
            np.dtype(np.float32): DT_F32, np.dtype(np.float64): DT_F64,
            np.dtype(np.complex64): DT_C64, np.dtype(np.complex128): DT_C128}
IQ_KINDS = {np.dtype(np.int8): IQ_I8, np.dtype(np.int16): IQ_I16, np.dtype(np.float32): IQ_C64}


def np_dtype(torch_dtype):
    """The NumPy dtype of a torch dtype; None for the ones NumPy has no name for (bfloat16, complex32, ...)."""
    try:
        return np.dtype(str(torch_dtype).removeprefix("torch."))
    except TypeError:
        return None


def torch_dtype(dtype):
    """The torch dtype of a NumPy dtype."""
    import torch
    return getattr(torch, np.dtype(dtype).name)


def is_cuda_tensor(x) -> bool:
    """Is ``x`` a torch tensor on a CUDA device?  Without torch imported, nothing is."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(x, torch.Tensor) and x.is_cuda


def stream_arg(device):
    """The current torch stream of ``device`` as the library's ``stream`` argument.  torch's default stream is CUDA's
    legacy default stream, whose handle is 0; the library takes 0 for "my own stream", which is non-blocking and so
    not ordered after work queued on torch's, so the default stream is passed as cudaStreamLegacy."""
    import torch
    return torch.cuda.current_stream(device).cuda_stream or 1       # 1 == cudaStreamLegacy


def forked(device, call):
    """Run ``call(stream)``, one library call that returns a status, on a side stream forked from, and joined back
    into, the current torch stream of ``device``."""
    import torch
    cur = torch.cuda.current_stream(device)
    side = torch.cuda.Stream(device=device)
    side.wait_stream(cur)
    check(call(side.cuda_stream))
    cur.wait_stream(side)


def ptr(a) -> int:
    """Address of a numpy array (host) or of a torch CUDA tensor (device)."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()


def as_c64(x, name="input"):
    """1-D C-contiguous complex64 view/copy of an array-like (complex128 is rounded, as
    main.py:186-194 effectively does when it declares dtype=complex64)."""
    a = np.asarray(x)
    if a.ndim != 1:
        raise ValueError(f"{name} must be one-dimensional, got shape {a.shape}")
    return np.ascontiguousarray(a, dtype=np.complex64)
