"""Kalman target trackers (reference passiveRadar/target_detection.py:164-681): the NumPy oracle against the reference's
own outputs, the drop-in's dtypes, signatures and argument checks (no GPU needed), and the sm_90a kernels against the
goldens and the oracle (GPU)."""
import ctypes as C
import hashlib
import inspect
import json
import os
import sys
import threading

import numpy as np
import pytest

import _golden as G
import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200 import target_detection as tdm

MEAS = ["track_meas_256x301", "track_meas_64x101"]
MULTI = ["track_multi_small_n10", "track_multi_small_n1", "track_multi_small_n32", "track_multi_256x301"]
SIMPLE = ["track_simple_256x301"]
MULTI_DISCRETE = ["status", "lifetime", "measurement_history", "measurement"]
SIMPLE_DISCRETE = ["lock_mode", "measurement", "measurement_idx"]
EXTENT = [256.0, 200.0]


def _maps(g):
    """The golden's (T, rows, cols) float32 maps, regenerated and checked against the recorded sha256."""
    tg = int(g["n_targets"]) if int(g["n_targets"]) >= 0 else [tuple(r) for r in g["targets"]]
    maps = synth.track_maps(int(g["seed"]), int(g["rows"]), int(g["cols"]), int(g["T"]), tg)
    assert hashlib.sha256(maps.tobytes()).hexdigest() == str(g["maps_sha256"]), "synth.track_maps drifted"
    return maps


def _data(g):
    return np.moveaxis(_maps(g), 0, 2).astype(np.float64)


def _rel(a, b):
    d = float(np.abs(b).max())
    if d == 0.0:
        return float(np.abs(a).max())
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / d)


def _floats_multi(h):
    k = h["kalman_state"]
    return {"estimate": h["estimate"], "x": k["x"], "P": k["P"], "S": k["S"]}


def assert_multi_close(got, want, tol):
    for f in MULTI_DISCRETE:
        assert np.array_equal(got[f], want[f]), f
    for f, a in _floats_multi(got).items():
        assert _rel(a, _floats_multi(want)[f]) <= tol, f


def assert_simple_close(got, want, tol):
    for f in SIMPLE_DISCRETE:
        assert np.array_equal(got[f], want[f]), f
    for f, a in _floats_multi(got).items():
        assert _rel(a, _floats_multi(want)[f]) <= tol, f


# ------------------------------------------------------------------ CPU: oracle, goldens, wrapper contract
@pytest.mark.parametrize("name", MEAS + MULTI + SIMPLE)
def test_oracle_matches_reference_golden(name):
    from oracle import track_oracle as O
    g = G.load(name)
    data = _data(g)
    ext = list(g["extent"])
    if str(g["kind"]) == "meas":
        got = O.get_measurements(data[:, :, 0], 99.8, ext)
        assert np.array_equal(got, g["meas"])
    elif str(g["kind"]) == "multi":
        assert_multi_close(O.multitarget_tracker(data, ext, int(g["n_tracks"])), g["history"], 1e-12)
    else:
        assert_simple_close(O.simple_target_tracker(data, ext[1], ext[0]), g["history"], 1e-12)


@pytest.mark.parametrize("name", MEAS + MULTI + SIMPLE)
def test_track_golden_is_what_the_reference_produces(name):
    with open(os.path.join(G.GOLDEN_DIR, "track_reference_digests.json")) as f:
        want = json.load(f)[name]
    committed = G.load(name)
    assert set(want) == set(committed) - {"seconds"}
    for key, digest in want.items():
        a = np.ascontiguousarray(committed[key])
        hsh = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
        hsh.update(a.tobytes())
        assert hsh.hexdigest() == digest, f"{name}[{key}] differs from the reference's output"


def test_goldens_exercise_promote_kill_and_the_edge_gate():
    st = G.load("track_multi_small_n10")["history"]["status"]
    assert ((st[:-1] == 1) & (st[1:] == 2)).any(), "a preliminary track is promoted"
    assert ((st[:-1] == 2) & (st[1:] == 0)).any() or ((st[:-1] == 1) & (st[1:] == 0)).any(), "a track is killed"
    assert (st == 2).sum() > 100, "confirmed tracks go through the Mahalanobis gate"
    idx = G.load("track_simple_256x301")["history"]["measurement_idx"]
    assert ((idx[:-1, 0] < 24) & (idx[1:, 0] == 0)).any(), "a gate near the range edge wraps and is empty"


def test_dtypes_equal_the_reference():
    ref_multi = G.load("track_multi_small_n1")["history"].dtype
    ref_simple = G.load("track_simple_256x301")["history"].dtype
    assert tdm.target_track_dtype == ref_multi and tdm.target_track_dtype.descr == ref_multi.descr
    assert tdm.target_track_dtype_simple == ref_simple and tdm.target_track_dtype_simple.descr == ref_simple.descr
    assert tdm.kalman_filter_dtype == ref_multi["kalman_state"]
    assert (tdm.kalman_filter_dtype.itemsize, tdm.target_track_dtype.itemsize,
            tdm.target_track_dtype_simple.itemsize) == (672, 880, 768)
    assert (C.sizeof(_lib.PrcKalman), C.sizeof(_lib.PrcTrack), C.sizeof(_lib.PrcTrackSimple)) == (672, 880, 768)
    for st, dt in ((_lib.PrcTrack, tdm.target_track_dtype), (_lib.PrcTrackSimple, tdm.target_track_dtype_simple)):
        assert [f[0] for f in st._fields_] == list(dt.names)
        assert [getattr(st, f).offset for f in dt.names] == [dt.fields[f][1] for f in dt.names]


def test_signatures_match_reference():
    def names(f):
        return [p for p in inspect.signature(f).parameters if p != "device"]
    assert names(prb.get_measurements) == ["dataFrame", "p", "frame_extent"]
    assert names(prb.multitarget_tracker) == ["data", "frame_extent", "N_TRACKS"]
    assert names(prb.simple_target_tracker) == ["data", "rangeExtent", "dopplerExtent"]
    for f in (prb.get_measurements, prb.multitarget_tracker, prb.simple_target_tracker, prb.multitarget_tracker_frames,
              prb.simple_tracker_frames, prb.cfar_track):
        assert inspect.signature(f).parameters["device"].kind is inspect.Parameter.KEYWORD_ONLY


def test_argument_errors_raise_before_touching_the_gpu(monkeypatch):
    def no_library(*a, **k):
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "load", no_library)
    m3 = np.zeros((16, 20, 3))
    with pytest.raises(ValueError):
        prb.multitarget_tracker(m3[:, :, 0], EXTENT, 4)
    with pytest.raises(ValueError):
        prb.multitarget_tracker(m3, [1.0], 4)
    with pytest.raises(ValueError):
        prb.multitarget_tracker(m3, EXTENT, -1)
    with pytest.raises(TypeError):
        prb.multitarget_tracker(m3.astype(np.complex64), EXTENT, 4)
    with pytest.raises(ValueError):
        prb.simple_target_tracker(m3[:, :, 0], 200.0, 256.0)
    with pytest.raises(TypeError):
        prb.simple_target_tracker(m3.astype(np.complex128), 200.0, 256.0)
    with pytest.raises(ValueError):
        prb.get_measurements(m3, 99.8, EXTENT)
    with pytest.raises(TypeError):
        prb.get_measurements(m3[:, :, 0].astype(np.complex64), 99.8, EXTENT)
    with pytest.raises(ValueError):
        prb.get_measurements(m3[:, :, 0], 99.8, [1.0, 2.0, 3.0])
    with pytest.raises(ValueError):
        prb.multitarget_tracker_frames(m3, EXTENT, 4)
    h = prb.multitarget_tracker(m3, EXTENT, 0)
    assert h.shape == (3, 0) and h.dtype == tdm.target_track_dtype


def test_no_cpu_fallback_without_a_device():
    if _lib.device_count() > 0:
        pytest.skip("a CUDA device is present")
    m = np.ones((32, 40, 2), np.float32)
    with pytest.raises(_lib.PrcoreError):
        prb.multitarget_tracker(m, EXTENT, 4)
    with pytest.raises(_lib.PrcoreError):
        prb.simple_target_tracker(m, 200.0, 256.0)
    with pytest.raises(_lib.PrcoreError):
        prb.get_measurements(m[:, :, 0], 99.8, EXTENT)


def test_c_abi_names_its_limits():
    lib = _lib.load()
    m = np.zeros(64 * 101, np.float32)
    hist = np.zeros(65, tdm.target_track_dtype)
    st = lib.prc_multitarget_track_frames(m.ctypes.data, 64, 101, 1, 1, 0, 0, 256.0, 200.0, 65, hist.ctypes.data,
                                          _lib.MEM_HOST, 0, None, 0)
    assert st == _lib.PRC_E_INVALID and "64" in lib.prc_last_error().decode()
    st = lib.prc_multitarget_track_frames(m.ctypes.data, 1024, 1024, 1, 1, 0, 0, 256.0, 200.0, 4, hist.ctypes.data,
                                          _lib.MEM_HOST, 0, None, 0)
    assert st == _lib.PRC_E_INVALID and "524288" in lib.prc_last_error().decode()


def test_install_replaces_the_trackers_of_a_reference_package(tmp_path, monkeypatch):
    pkg = tmp_path / "fakeTrack"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    (pkg / "range_doppler_processing.py").write_text("def fast_xambg(*a, **k):\n    return 'cpu'\n")
    (pkg / "clutter_removal.py").write_text("def LS_Filter(*a, **k):\n    return 'cpu'\n")
    (pkg / "signal_utils.py").write_text("def resample(*a, **k):\n    return 'cpu'\n")
    (pkg / "target_detection.py").write_text(
        "def CFAR_2D(*a, **k):\n    return 'cpu'\n"
        "def get_measurements(*a, **k):\n    return 'cpu'\n"
        "def multitarget_tracker(*a, **k):\n    return 'cpu'\n"
        "def simple_target_tracker(*a, **k):\n    return 'cpu'\n"
        "def kalman_update(*a, **k):\n    return 'untouched'\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    try:
        replaced = prb.install("fakeTrack")
        import fakeTrack.target_detection as td
        for name in ("get_measurements", "multitarget_tracker", "simple_target_tracker"):
            assert f"fakeTrack.target_detection.{name}" in replaced
            assert getattr(td, name) is getattr(prb, name)
        assert td.kalman_update() == "untouched"
    finally:
        for m in [k for k in sys.modules if k.startswith("fakeTrack")]:
            del sys.modules[m]


def test_pairwise_mean_twin_equals_numpy_bitwise():
    from oracle import track_oracle as O
    rng = np.random.default_rng(7)
    sizes = list(range(1, 300)) + [511, 1024, 1031, 6464, 77056, 77056 + 13]
    for n in sizes:
        x = rng.rayleigh(1.0, n) * 10.0 ** rng.uniform(-3, 3, n)
        assert O.pairwise_mean_twin(x) == np.mean(np.abs(x).flatten()), n
    x = rng.rayleigh(1.0, (256, 301)).astype(np.float32).astype(np.float64)
    assert O.pairwise_mean_twin(x) == np.mean(np.abs(x).flatten())


def test_track_kernels_build_for_sm90a_without_spills():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    text = open(log).read()
    blocks = [blk for blk in text.split("Compiling entry function")[1:] if "track_" in blk.split("\n")[0]]
    assert len(blocks) == 9, "six measurement, one multi-target and two simple-tracker instantiations"
    for blk in blocks:
        assert "'sm_90a'" in blk.split("\n")[0]
        assert "0 bytes spill stores, 0 bytes spill loads" in blk


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", MEAS)
def test_get_measurements_matches_golden_bitwise(name):
    g = G.load(name)
    got = prb.get_measurements(_data(g)[:, :, 0], 99.8, list(g["extent"]))
    assert got.dtype == np.float64 and got.shape == g["meas"].shape
    assert np.array_equal(got, g["meas"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", MULTI)
def test_multitarget_tracker_matches_golden(name):
    g = G.load(name)
    got = prb.multitarget_tracker(_data(g), list(g["extent"]), int(g["n_tracks"]))
    assert got.dtype == tdm.target_track_dtype and got.shape == g["history"].shape
    assert_multi_close(got, g["history"], 1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SIMPLE)
def test_simple_target_tracker_matches_golden(name):
    g = G.load(name)
    ext = list(g["extent"])
    got = prb.simple_target_tracker(_data(g), ext[1], ext[0])
    assert got.dtype == tdm.target_track_dtype_simple and got.shape == g["history"].shape
    assert_simple_close(got, g["history"], 1e-9)
    assert np.array_equal(got["range_extent"], g["history"]["range_extent"])


@pytest.mark.gpu
def test_reference_script_length_run_matches_oracle():
    """The reference scripts' num_frames = 1200 frames of config-2 maps (256 x 301), N_TRACKS = 10; the simple tracker
    on the same maps."""
    from oracle import track_oracle as O
    maps = synth.track_maps(2024, 256, 301, 1200, 10)
    data = np.moveaxis(maps, 0, 2)
    got = prb.multitarget_tracker(data, EXTENT, 10)
    want = O.multitarget_tracker(data, EXTENT, 10)
    assert_multi_close(got, want, 1e-9)
    assert_simple_close(prb.simple_target_tracker(data, 200.0, 256.0), O.simple_target_tracker(data, 200.0, 256.0), 1e-9)


@pytest.mark.gpu
def test_float32_equals_float64_and_frame_layouts_agree():
    maps = synth.track_maps(31, 64, 101, 60, 4)
    data32 = np.moveaxis(maps, 0, 2)
    h32 = prb.multitarget_tracker(data32, EXTENT, 8)
    h64 = prb.multitarget_tracker(data32.astype(np.float64), EXTENT, 8)
    assert h32.tobytes() == h64.tobytes()
    hf = prb.multitarget_tracker_frames(maps[None], EXTENT, 8)[0]
    assert hf.tobytes() == h32.tobytes()
    s32 = prb.simple_target_tracker(data32, 200.0, 256.0)
    assert s32.tobytes() == prb.simple_target_tracker(data32.astype(np.float64), 200.0, 256.0).tobytes()
    assert s32.tobytes() == prb.simple_tracker_frames(maps[None], 200.0, 256.0)[0].tobytes()
    hi = prb.multitarget_tracker(data32.astype(np.int64), EXTENT, 8)       # other real dtypes: as float64
    assert hi.tobytes() == prb.multitarget_tracker(data32.astype(np.int64).astype(np.float64), EXTENT, 8).tobytes()
    m = prb.get_measurements(data32[:, :, 3], 99.8, EXTENT)
    assert np.array_equal(m, prb.get_measurements(data32[:, :, 3].astype(np.float64), 99.8, EXTENT))


@pytest.mark.gpu
def test_strided_batch_filling_the_gpu_is_bit_identical_to_single_sequences():
    import torch
    nsm = torch.cuda.get_device_properties(_lib.current_device()).multi_processor_count
    S, T, rows, cols = 2 * nsm, 12, 64, 101
    dev = torch.device("cuda", _lib.current_device())
    base = torch.full((S, T + 3, rows, cols), float("nan"), dtype=torch.float32, device=dev)
    host = np.stack([synth.track_maps(500 + s, rows, cols, T, 3) for s in range(S)])
    base[:, :T] = torch.from_numpy(host).to(dev)
    maps = base[:, :T]                                   # seq_stride = (T + 3) * rows * cols
    hm = prb.multitarget_tracker_frames(maps, EXTENT, 6)
    hs = prb.simple_tracker_frames(maps, 200.0, 256.0)
    for s in range(S):
        assert hm[s].tobytes() == prb.multitarget_tracker_frames(host[s:s + 1], EXTENT, 6)[0].tobytes(), s
        assert hs[s].tobytes() == prb.simple_tracker_frames(host[s:s + 1], 200.0, 256.0)[0].tobytes(), s


def _degenerate_frames():
    rng = np.random.default_rng(9)
    zero = np.zeros((64, 101))
    const = np.full((64, 101), 3.25)
    onehot = np.zeros((64, 101))
    onehot[20, 40] = 7.0
    sparse = np.zeros((64, 101))                          # > 99.8 % zeros: every cell ties at the threshold 0
    sparse[rng.integers(0, 64, 9), rng.integers(8, 93, 9)] = rng.uniform(1, 5, 9)
    noisy = rng.rayleigh(1.0, (64, 101))
    return [zero, const, onehot, sparse, noisy]


@pytest.mark.gpu
def test_degenerate_maps_follow_the_tie_rule():
    from oracle import track_oracle as O
    frames = _degenerate_frames()
    for k, fr in enumerate(frames):
        got = prb.get_measurements(fr, 99.8, EXTENT)
        want = O.get_measurements(fr, 99.8, EXTENT)
        assert got.shape == want.shape and np.array_equal(got, want), k
    assert prb.get_measurements(frames[1], 99.8, EXTENT).shape[1] > 4000        # a constant map: every unzeroed cell
    data = np.stack(frames * 4, axis=2)                   # each degenerate frame several times in one sequence
    for n in (1, 10, tdm.MAX_TRACKS):
        assert_multi_close(prb.multitarget_tracker(data, EXTENT, n), O.multitarget_tracker(data, EXTENT, n), 1e-9)
    assert_simple_close(prb.simple_target_tracker(data, 200.0, 256.0), O.simple_target_tracker(data, 200.0, 256.0), 1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(64, 16), (64, 12), (6, 101), (4, 101), (1, 40), (100, 120)])
def test_small_maps_match_oracle(rows, cols):
    """cols <= 16 zeroes every range row; rows < 8 wraps the Doppler band's start; rows < 250 for the simple tracker."""
    from oracle import track_oracle as O
    maps = synth.track_maps(77 + rows + cols, rows, cols, 30, 3)
    data = np.moveaxis(maps, 0, 2)
    for t in (0, 7):
        assert np.array_equal(prb.get_measurements(data[:, :, t], 99.8, EXTENT), O.get_measurements(data[:, :, t], 99.8, EXTENT))
    assert_multi_close(prb.multitarget_tracker(data, EXTENT, 5), O.multitarget_tracker(data, EXTENT, 5), 1e-9)
    assert_simple_close(prb.simple_target_tracker(data, 200.0, 256.0), O.simple_target_tracker(data, 200.0, 256.0), 1e-9)


@pytest.mark.gpu
def test_candidates_run_out_before_the_free_tracks():
    from oracle import track_oracle as O
    maps = synth.track_maps(5, 64, 101, 20, 2)            # ~13 candidates per frame, 64 tracks
    data = np.moveaxis(maps, 0, 2)
    got = prb.multitarget_tracker(data, EXTENT, 64)
    assert_multi_close(got, O.multitarget_tracker(data, EXTENT, 64), 1e-9)
    assert (got["status"][0] == 0).sum() > 40


def _run_pipeline_maps(T):
    import torch
    from passiveradar_b200.frames import FramePipeline
    n, R, F = 1 << 15, 100, 64
    pipe = FramePipeline(n, R, F)
    frames = [synth.make_frame(n, "P1", frame=60 + i) for i in range(T)]
    dev = pipe.tdev
    ref = torch.from_numpy(np.stack([f[0] for f in frames]).view(np.float32)).to(dev).view(torch.complex64)
    srv = torch.from_numpy(np.stack([f[1] for f in frames]).view(np.float32)).to(dev).view(torch.complex64)
    maps_d = torch.empty((T, F, R + 1), dtype=torch.complex64, device=dev)
    pipe.run_device(ref, srv, maps_d)
    torch.cuda.current_stream(dev).synchronize()
    return maps_d


@pytest.mark.gpu
def test_cfar_track_equals_tracker_on_downloaded_cfar_maps():
    maps_d = _run_pipeline_maps(12)
    got = prb.cfar_track(maps_d, 18, 4, EXTENT, 6)
    host = maps_d.cpu().numpy()
    lib = _lib.load()
    cf = np.empty(host.shape, np.float32)
    for t in range(host.shape[0]):
        _lib.check(lib.prc_cfar2d_f32(np.ascontiguousarray(host[t]).ctypes.data, host.shape[1], host.shape[2], 18, 4,
                                      None, cf[t].ctypes.data, None, _lib.MEM_HOST, _lib.current_device(), None,
                                      _lib.FLAG_ABS_C64))
    want = prb.multitarget_tracker(np.moveaxis(cf, 0, 2).astype(np.float64), EXTENT, 6)
    assert got.tobytes() == want.tobytes()


@pytest.mark.gpu
def test_device_pointers_async_on_caller_stream():
    import torch
    maps = np.stack([synth.track_maps(700 + s, 64, 101, 25, 4) for s in range(3)])
    want = prb.multitarget_tracker_frames(maps, EXTENT, 7)
    wants = prb.simple_tracker_frames(maps, 200.0, 256.0)
    dev = torch.device("cuda", _lib.current_device())
    s = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(s):
        dm = torch.from_numpy(maps).to(dev)
        dh = torch.empty(want.nbytes, dtype=torch.uint8, device=dev)
        dhs = torch.empty(wants.nbytes, dtype=torch.uint8, device=dev)
        dc = torch.empty(3 * 25, dtype=torch.int32, device=dev)
        dmeas = torch.empty(3 * 25 * 3 * 64 * 101, dtype=torch.float64, device=dev)
    lib = _lib.load()
    n = 64 * 101
    args = (dm.data_ptr(), 64, 101, 3, 25, 25 * n, n)
    _lib.check(lib.prc_multitarget_track_frames(*args, 256.0, 200.0, 7, dh.data_ptr(), _lib.MEM_DEVICE,
                                                _lib.current_device(), C.c_void_p(s.cuda_stream), _lib.FLAG_ASYNC))
    _lib.check(lib.prc_simple_track_frames(*args, 200.0, 256.0, dhs.data_ptr(), _lib.MEM_DEVICE,
                                           _lib.current_device(), C.c_void_p(s.cuda_stream), _lib.FLAG_ASYNC))
    _lib.check(lib.prc_get_measurements_frames(*args, 256.0, 200.0, n, dc.data_ptr(), dmeas.data_ptr(),
                                               _lib.MEM_DEVICE, _lib.current_device(), C.c_void_p(s.cuda_stream),
                                               _lib.FLAG_ASYNC))
    s.synchronize()
    assert dh.cpu().numpy().tobytes() == want.tobytes()
    assert dhs.cpu().numpy().tobytes() == wants.tobytes()
    counts = dc.cpu().numpy()
    meas = dmeas.cpu().numpy().reshape(3, 25, 3, n)
    for q in (0, 11, 24):
        m = prb.get_measurements(maps[2, q], 99.8, EXTENT)
        assert counts[2 * 25 + q] == m.shape[1] and np.array_equal(meas[2, q][:, :m.shape[1]], m)


@pytest.mark.gpu
def test_concurrent_threads_give_serial_results():
    jobs = [np.moveaxis(synth.track_maps(900 + i, 64 + 8 * i, 101, 30, 3), 0, 2) for i in range(8)]
    serial = [(prb.multitarget_tracker(d, EXTENT, 5), prb.simple_target_tracker(d, 200.0, 256.0)) for d in jobs]
    results = [None] * len(jobs)
    errors = []

    def run(i):
        try:
            results[i] = (prb.multitarget_tracker(jobs[i], EXTENT, 5), prb.simple_target_tracker(jobs[i], 200.0, 256.0))
        except Exception as exc:           # pragma: no cover - reported below
            errors.append(exc)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for a, b in zip(results, serial):
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
