"""Host operands are staged through one path (prcore_host.h: stage_in / unstage): a host call on frames laid out wider than
a frame gives the bits of the same call on device copies, and writes nothing into the caller's padding."""
import numpy as np
import pytest

from passiveradar_b200 import _lib

pytestmark = pytest.mark.gpu

HOST, DEV = _lib.MEM_HOST, _lib.MEM_DEVICE
SENTINEL = {np.complex64: np.complex64(1234.5 - 77j), np.float64: -4321.25, np.int32: -7, np.uint8: 0xA5}


def _c64(rng, *shape):
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)


def _out(shape, dtype):
    return np.full(shape, SENTINEL[dtype], dtype)


def _host_and_device(entry, inputs, outputs, args):
    """`entry` on host arrays and on device copies of the same arrays; args({name: pointer}) gives the arguments before
    mem_kind.  Returns the outputs of both calls."""
    import torch
    lib = _lib.load()
    dev = torch.device("cuda", _lib.current_device())
    host = {k: v.copy() for k, v in {**inputs, **outputs}.items()}
    _lib.check(getattr(lib, entry)(*args({k: a.ctypes.data for k, a in host.items()}), HOST, _lib.current_device(),
                                   None, 0))
    d = {k: torch.from_numpy(v).to(dev) for k, v in {**inputs, **outputs}.items()}
    torch.cuda.synchronize()
    _lib.check(getattr(lib, entry)(*args({k: t.data_ptr() for k, t in d.items()}), DEV, _lib.current_device(), None, 0))
    return {k: host[k] for k in outputs}, {k: d[k].cpu().numpy() for k in outputs}


def _same(host, device):
    for k in host:
        assert host[k].tobytes() == device[k].tobytes(), k


def test_nlms_frames():
    rng = np.random.default_rng(11)
    n, nf, pad, M = 2048, 3, 40, 18
    inputs = {"ref": _c64(rng, nf, n + pad), "srv": _c64(rng, nf, n + pad)}
    outputs = {"out": _out((nf, n + pad), np.complex64), "taps": _out((nf, M), np.complex64)}
    h, d = _host_and_device("prc_nlms_frames_c64", inputs, outputs,
                            lambda p: (p["ref"], p["srv"], n, nf, n + pad, 16, 2, 0.1, 1, None, p["out"], p["taps"]))
    _same(h, d)
    assert (h["out"][:, n:] == SENTINEL[np.complex64]).all()


def test_xambg_frames():
    rng = np.random.default_rng(12)
    n, nf, pad, R, F = 4096, 3, 24, 15, 32
    inputs = {"ref": _c64(rng, nf, n + pad), "srv": _c64(rng, nf, n + pad)}
    outputs = {"out": _out((nf, F, R + 1), np.complex64)}
    h, d = _host_and_device("prc_xambg_frames_c64", inputs, outputs,
                            lambda p: (p["ref"], p["srv"], n, nf, n + pad, R, F, None, p["out"]))
    _same(h, d)


def test_ls_svd_frames():
    rng = np.random.default_rng(13)
    n, nf, pad, L, peek = 1024, 3, 8, 6, 2
    inputs = {"ref": _c64(rng, nf, n + pad), "srv": _c64(rng, nf, n + pad)}
    outputs = {"out": _out((nf, n + pad), np.complex64), "taps": _out((nf, L + peek), np.complex64),
               "rank": _out((nf,), np.int32)}
    h, d = _host_and_device("prc_ls_svd_frames_c64", inputs, outputs,
                            lambda p: (p["ref"], p["srv"], n, nf, n + pad, L, peek, p["out"], p["taps"], p["rank"]))
    _same(h, d)
    assert (h["out"][:, n:] == SENTINEL[np.complex64]).all()


def test_persistence_frames():
    rng = np.random.default_rng(14)
    rows, cols, nf, pad = 16, 24, 5, 16
    w = np.array([1.0, 0.9, 0.81])                 # host memory whatever mem_kind
    inputs = {"x": rng.random((nf, rows * cols + pad), dtype=np.float32)}
    outputs = {"out": _out((nf, rows * cols), np.float64)}
    h, d = _host_and_device("prc_persistence_frames", inputs, outputs,
                            lambda p: (p["x"], rows, cols, nf, rows * cols + pad, 0, 3, w.ctypes.data, p["out"]))
    _same(h, d)


def test_percentiles_frames():
    rng = np.random.default_rng(15)
    n, nf, pad = 1000, 4, 10
    q = np.array([35.0, 99.0])
    inputs = {"x": rng.standard_normal((nf, n + pad))}
    outputs = {"out": _out((nf, 2), np.float64)}
    h, d = _host_and_device("prc_percentiles_frames", inputs, outputs,
                            lambda p: (p["x"], n, nf, n + pad, q.ctypes.data, None, 2, p["out"]))
    _same(h, d)


def test_simple_tracker_frames():
    import ctypes as C
    rng = np.random.default_rng(16)
    rows, cols, nseq, nf = 64, 101, 2, 3
    fs = rows * cols + 16
    ss = nf * fs + 32
    inputs = {"maps": rng.random(nseq * ss, dtype=np.float32)}
    outputs = {"hist": _out(nseq * nf * C.sizeof(_lib.PrcTrackSimple), np.uint8)}
    h, d = _host_and_device("prc_simple_track_frames", inputs, outputs,
                            lambda p: (p["maps"], rows, cols, nseq, nf, ss, fs, 200.0, 256.0, p["hist"]))
    _same(h, d)


def test_frames_taps_refusal_writes_nothing():
    """Host taps of a batch come from the FFT-domain path only; off it (n below fft_min_n) the call is refused before
    any copy or launch, so the caller's maps keep what they held."""
    rng = np.random.default_rng(17)
    lib = _lib.load()
    n, nf, R, F, M = 2048, 2, 8, 16, 10
    ref, srv = _c64(rng, nf, n), _c64(rng, nf, n)
    maps = _out((nf, F, R + 1), np.complex64)
    taps = _out((nf, M), np.complex64)
    before = _lib.launch_count()
    st = lib.prc_frames_c64(ref.ctypes.data, srv.ctypes.data, n, nf, n, 8, 2, 0.0, R, F, None, maps.ctypes.data,
                            taps.ctypes.data, None, HOST, _lib.current_device(), None, 0)
    assert st == _lib.PRC_E_INVALID
    assert "taps_out with host pointers and nframes > 1 needs the FFT-domain path" in lib.prc_last_error().decode()
    assert (maps == SENTINEL[np.complex64]).all() and (taps == SENTINEL[np.complex64]).all()
    assert _lib.launch_count() == before
