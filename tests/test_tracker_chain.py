"""The tracker scripts' chain (multitarget_kalman_tracker.py / simple_kalman_tracker.py) on the device: the trackers'
resume mode (PRC_FLAG_TRACK_RESUME) and TrackerPipeline.  The flag, the build, the refusals and the scripts' masks
need no GPU; resume against one call, the stages against the oracles, the reference golden, batch invariance and the
recording chain do."""
import ctypes as C
import hashlib
import json
import os
import re

import numpy as np
import pytest

import _golden as G
import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200 import target_detection as tdm
from passiveradar_b200.target_detection import TrackerPipeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXTENT = [256.0, 200.0]                  # [max_doppler, max_range]
MULTI_DISCRETE = ["status", "lifetime", "measurement_history", "measurement"]
SIMPLE_DISCRETE = ["lock_mode", "measurement", "measurement_idx"]
MULTI_REC, SIMPLE_REC = tdm.target_track_dtype.itemsize, tdm.target_track_dtype_simple.itemsize


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    d = float(np.abs(b).max())
    return float(np.abs(a - b).max()) / (d if d else 1.0)


def _floats(h):
    k = h["kalman_state"]
    return {"estimate": h["estimate"], "x": k["x"], "P": k["P"], "S": k["S"]}


def assert_records_close(got, want, discrete, tol=1e-9):
    assert got.dtype == want.dtype and got.shape == want.shape
    for f in discrete:
        assert np.array_equal(got[f], want[f]), f
    for f, a in _floats(got).items():
        assert _rel(a, _floats(want)[f]) <= tol, f


def _same_nan(a, b):
    """Equal arrays with NaN in the same places."""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    return a[~np.isnan(a)], b[~np.isnan(b)]


def _complex_maps(seed, rows, cols, T, targets=4):
    """(T, rows, cols) complex64: tracker maps as magnitudes, seeded phases (as make_tracker_chain_golden.py)."""
    rng = np.random.default_rng(seed)
    mag = synth.track_maps(seed, rows, cols, T, targets)
    return (mag * np.exp(1j * rng.uniform(0, 2 * np.pi, mag.shape))).astype(np.complex64)


def _script_masks_multi(h):
    """multitarget_kalman_tracker.py:66-75, as written."""
    tracker_status = h['status']
    idx = np.nonzero(tracker_status != 2)
    tracker_range = np.squeeze(h['estimate'][:, :, 0]).copy()
    tracker_doppler = np.squeeze(h['estimate'][:, :, 1]).copy()
    tracker_range[idx] = np.nan
    tracker_doppler[idx] = np.nan
    return tracker_range, tracker_doppler


def _script_masks_simple(h):
    """simple_kalman_tracker.py:212-222, as written."""
    estimate = h['estimate']
    unlocked = h['lock_mode'][:, 0].astype(bool)
    locked_est = estimate.copy()
    locked_est[unlocked, 0] = np.nan
    locked_est[unlocked, 1] = np.nan
    unlocked_est = estimate.copy()
    unlocked_est[~unlocked, 0] = np.nan
    unlocked_est[~unlocked, 1] = np.nan
    return locked_est, unlocked_est


# ------------------------------------------------------------------ CPU
def test_resume_flag_is_declared_in_the_header_and_the_binding():
    with open(os.path.join(ROOT, "include", "prcore.h")) as f:
        src = f.read()
    m = re.search(r"^#define PRC_FLAG_TRACK_RESUME\s+(\d+)u", src, re.M)
    assert m and int(m.group(1)) == 128 == _lib.FLAG_TRACK_RESUME
    flags = [int(v) for v in re.findall(r"^#define PRC_FLAG_\w+\s+(\d+)u", src, re.M)]
    assert len(set(flags)) == len(flags) and all(v & (v - 1) == 0 for v in flags), "one bit per flag"


def test_tracker_kernels_still_build_as_nine_spill_free_sm90a_entries():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    text = open(log).read()
    blocks = [blk for blk in text.split("Compiling entry function")[1:] if "track_" in blk.split("\n")[0]]
    assert len(blocks) == 9
    for blk in blocks:
        assert "'sm_90a'" in blk.split("\n")[0]
        assert "0 bytes spill stores, 0 bytes spill loads" in blk


def test_refusals_before_any_launch(monkeypatch):
    before = _lib.launch_count()

    def no_library(*a, **k):
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "load", no_library)
    bad = [dict(tracker="kalman"), dict(n_tracks=65), dict(n_tracks=-1), dict(fw=0), dict(fw=65), dict(fw=4, gw=4),
           dict(gw=-1), dict(hold=0), dict(batch=0)]
    for kw in bad:
        with pytest.raises(ValueError):
            TrackerPipeline(200.0, 256.0, **kw)
    with pytest.raises(TypeError):
        TrackerPipeline(200.0, 256.0, decay=0.9j)
    with pytest.raises(ValueError, match="max_range_actual"):
        TrackerPipeline.from_config({"max_doppler_actual": 256.0})
    with pytest.raises(ValueError):
        TrackerPipeline.from_config({"max_range_actual": 200.0, "max_doppler_actual": 256.0}, tracker="both")
    pipe = TrackerPipeline.from_config({"max_range_actual": 200.0, "max_doppler_actual": 256.0}, tracker="simple")
    assert (pipe.max_range, pipe.max_doppler, pipe.tracker) == (200.0, 256.0, "simple")
    with pytest.raises(TypeError):
        pipe.run_device(np.zeros((2, 8, 9), np.complex64))               # host arrays go through run()
    with pytest.raises(ValueError):
        pipe.run(np.zeros((8, 9)))
    with pytest.raises(TypeError):
        pipe.run(np.zeros((8, 9, 2), dtype="U1"))
    maps = np.zeros((2, 3, 16, 20), np.float32)
    with pytest.raises(TypeError):
        prb.multitarget_tracker_frames(maps, EXTENT, 4, initial_state=np.zeros((2, 4)))
    with pytest.raises(ValueError):
        prb.multitarget_tracker_frames(maps, EXTENT, 4, initial_state=np.zeros((2, 3), tdm.target_track_dtype))
    with pytest.raises(ValueError):
        prb.simple_tracker_frames(maps, 200.0, 256.0, initial_state=np.zeros((1,), tdm.target_track_dtype_simple))
    with pytest.raises(TypeError):
        prb.simple_tracker_frames(maps, 200.0, 256.0, initial_state=np.zeros((2,), tdm.target_track_dtype))
    monkeypatch.undo()
    assert _lib.launch_count() == before


def test_reference_named_drop_ins_keep_their_signatures():
    import inspect
    names = lambda f: [p for p in inspect.signature(f).parameters if p != "device"]
    assert names(prb.multitarget_tracker) == ["data", "frame_extent", "N_TRACKS"]
    assert names(prb.simple_target_tracker) == ["data", "rangeExtent", "dopplerExtent"]
    for f in (prb.multitarget_tracker_frames, prb.simple_tracker_frames):
        p = inspect.signature(f).parameters["initial_state"]
        assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is None


def _hand_made_multi(T=7, N=5):
    rng = np.random.default_rng(3)
    h = np.zeros((T, N), tdm.target_track_dtype)
    h["status"] = rng.integers(0, 3, (T, N))
    h["status"][0, 0] = 3                                          # only 2 is "confirmed"
    h["estimate"] = rng.standard_normal((T, N, 2)) * 100
    h["estimate"][1, 1] = [-0.0, np.inf]
    h["lifetime"] = rng.integers(1, 50, (T, N))
    return h


def _hand_made_simple(T=9):
    rng = np.random.default_rng(4)
    h = np.zeros((T,), tdm.target_track_dtype_simple)
    h["lock_mode"][:, 0] = [1.0, 0.0, -0.0, np.nan, 0.5, 0.0, 1.0, -2.0, 0.0][:T]
    h["lock_mode"][:, 2] = 1.0 - h["lock_mode"][:, 0]
    h["estimate"] = rng.standard_normal((T, 2)) * 50
    h["measurement_idx"] = rng.integers(-5, 5, (T, 2))
    return h


def test_masks_match_the_scripts_lines_on_hand_made_records():
    import torch
    h = _hand_made_multi()
    pipe = TrackerPipeline(200.0, 256.0, n_tracks=h.shape[1], render=False)
    got = pipe._masks({"history": torch.from_numpy(h.view(np.uint8).reshape(-1).copy())}, h.shape[0], torch)
    want_r, want_d = _script_masks_multi(h)
    for k, w in (("track_range", want_r), ("track_doppler", want_d)):
        g = got[k].numpy()
        assert g.dtype == np.float64
        a, b = _same_nan(g, w)
        assert a.tobytes() == b.tobytes(), k
    assert pipe.records(got["history"]).tobytes() == h.tobytes()
    s = _hand_made_simple()
    pipe = TrackerPipeline(200.0, 256.0, tracker="simple", render=False)
    got = pipe._masks({"history": torch.from_numpy(s.view(np.uint8).reshape(-1).copy())}, s.shape[0], torch)
    for k, w in zip(("estimate_locked", "estimate_unlocked"), _script_masks_simple(s)):
        a, b = _same_nan(got[k].numpy(), w)
        assert a.tobytes() == b.tobytes(), k
    assert pipe.records(got["history"]).tobytes() == s.tobytes()


def test_committed_golden_is_what_the_reference_produces():
    with open(os.path.join(G.GOLDEN_DIR, "tracker_chain_reference_digests.json")) as f:
        want = json.load(f)["tracker_chain"]
    committed = G.load("tracker_chain")
    assert set(want) == set(committed)
    for key, digest in want.items():
        a = np.ascontiguousarray(committed[key])
        hsh = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
        hsh.update(a.tobytes())
        assert hsh.hexdigest() == digest, f"tracker_chain[{key}] differs from the reference's output"
    st = committed["multi_history"]["status"]
    assert (st == 2).any() and (st == 0).any(), "the golden has confirmed tracks and free ones"
    lm = committed["simple_history"]["lock_mode"][:, 0]
    assert (lm == 0).any() and (lm != 0).any(), "the golden has locked and unlocked frames"


# ------------------------------------------------------------------ GPU: resume
_CUTS_N = 10                             # tracks of the multi-target tracker in the resume cases


def _call(tracker, maps_ptr, rows, cols, S, T, ss, hist_ptr, mem, stream=None, flags=0, f64=False):
    lib = _lib.load()
    n = rows * cols
    flags |= _lib.FLAG_MAP_F64 if f64 else 0
    if tracker == "multi":
        st = lib.prc_multitarget_track_frames(maps_ptr, rows, cols, S, T, ss, n, EXTENT[0], EXTENT[1], _CUTS_N,
                                              hist_ptr, mem, _lib.current_device(), stream, flags)
    else:
        st = lib.prc_simple_track_frames(maps_ptr, rows, cols, S, T, ss, n, EXTENT[1], EXTENT[0], hist_ptr, mem,
                                         _lib.current_device(), stream, flags)
    _lib.check(st)


def _cuts(whole, tracker, T, rng):
    """Random cuts plus the ones the records call for: right after tracks become confirmed (and at the frame they do),
    and at a frame where free tracks ran out of candidates (or, for the simple tracker, where the lock changes)."""
    cuts = set(int(c) for c in rng.integers(1, T, 5))
    if tracker == "multi":
        st = whole["status"]                                   # (S, T, N)
        conf = np.nonzero(((st[:, :-1] == 1) & (st[:, 1:] == 2)).any(axis=(0, 2)))[0] + 1
        out = np.nonzero(((st[:, :-1] == 0) & (st[:, 1:] == 0)).any(axis=(0, 2)))[0] + 1
        assert conf.size and out.size, "the sequence confirms tracks and runs out of candidates"
        cuts |= {int(conf[0]), int(conf[0]) + 1, int(out[0]), int(out[-1])}
    else:
        lm = whole["lock_mode"][..., 0]
        change = np.nonzero((lm[:, :-1] != lm[:, 1:]).any(axis=0))[0] + 1
        assert change.size, "the simple tracker locks and unlocks"
        cuts |= {int(change[0]), int(change[-1])}
    return sorted(c for c in cuts if 0 < c < T)


@pytest.mark.gpu
@pytest.mark.parametrize("tracker", ["multi", "simple"])
@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("mem", ["host", "device"])
def test_resume_at_any_cut_is_byte_identical_to_one_call(tracker, f64, mem):
    import torch
    S, T, rows, cols, pad = 2, 1200, 64, 101, 3
    n = rows * cols
    dt, esz = (np.float64, 8) if f64 else (np.float32, 4)
    base = np.full((S, T + pad, rows, cols), np.nan, dt)          # strided: seq_stride = (T + pad) * n
    for s in range(S):
        base[s, :T] = synth.track_maps(41 + s, rows, cols, T, 6)
    ss = (T + pad) * n
    rec, dtype = (MULTI_REC * _CUTS_N, tdm.target_track_dtype) if tracker == "multi" else \
        (SIMPLE_REC, tdm.target_track_dtype_simple)
    shape = (lambda t: (S, t, _CUTS_N)) if tracker == "multi" else (lambda t: (S, t))
    if mem == "device":
        dev = torch.device("cuda", _lib.current_device())
        maps_d = torch.from_numpy(base).to(dev)
        ptr = maps_d.data_ptr()

        def run(t0, t1, init):
            h = np.zeros(shape(t1 - t0), dtype)
            if init is not None:
                h[:, 0] = init
            hd = torch.from_numpy(h.view(np.uint8).reshape(-1).copy()).to(dev)
            _call(tracker, ptr + t0 * n * esz, rows, cols, S, t1 - t0, ss, hd.data_ptr(), _lib.MEM_DEVICE,
                  flags=0 if init is None else _lib.FLAG_TRACK_RESUME, f64=f64)
            return np.frombuffer(hd.cpu().numpy().tobytes(), dtype).reshape(shape(t1 - t0))
    else:
        def run(t0, t1, init):
            h = np.zeros(shape(t1 - t0), dtype)
            if init is not None:
                h[:, 0] = init
            _call(tracker, base.ctypes.data + t0 * n * esz, rows, cols, S, t1 - t0, ss, h.ctypes.data,
                  _lib.MEM_HOST, flags=0 if init is None else _lib.FLAG_TRACK_RESUME, f64=f64)
            return h
    whole = run(0, T, None)
    want = (prb.multitarget_tracker_frames(base[:, :T], EXTENT, _CUTS_N) if tracker == "multi"
            else prb.simple_tracker_frames(base[:, :T], EXTENT[1], EXTENT[0]))
    assert whole.tobytes() == want.tobytes()
    cuts = _cuts(whole, tracker, T, np.random.default_rng(7 + f64))
    parts, state = [], None
    for t0, t1 in zip([0] + cuts, cuts + [T]):
        h = run(t0, t1, state)
        parts.append(h)
        state = h[:, -1].copy()
    got = np.concatenate(parts, axis=1)
    assert got.tobytes() == whole.tobytes(), f"cuts {cuts}"
    # one frame per call from the last cut on
    state, tail = whole[:, cuts[-1] - 1].copy(), []
    for t in range(cuts[-1], min(T, cuts[-1] + 12)):
        tail.append(run(t, t + 1, state))
        state = tail[-1][:, -1].copy()
    assert np.concatenate(tail, axis=1).tobytes() == whole[:, cuts[-1]:cuts[-1] + len(tail)].tobytes()


@pytest.mark.gpu
def test_initial_state_of_the_python_wrappers_continues_a_sequence():
    import torch
    maps = np.stack([synth.track_maps(60 + s, 64, 101, 90, 5) for s in range(3)])
    for name, fn, args in (("multi", prb.multitarget_tracker_frames, (EXTENT, 12)),
                           ("simple", prb.simple_tracker_frames, (EXTENT[1], EXTENT[0]))):
        whole = fn(maps, *args)
        a = fn(maps[:, :37], *args)
        b = fn(maps[:, 37:], *args, initial_state=a[:, -1])
        assert np.concatenate([a, b], axis=1).tobytes() == whole.tobytes(), name
        dm = torch.from_numpy(maps).cuda()
        bd = fn(dm[:, 37:], *args, initial_state=a[:, -1])
        assert bd.tobytes() == b.tobytes(), name
    # the simple tracker keeps the record's own extents
    s0 = prb.simple_tracker_frames(maps[:, :5], 150.0, 100.0)
    s1 = prb.simple_tracker_frames(maps[:, 5:9], 999.0, 999.0, initial_state=s0[:, -1])
    assert (s1["range_extent"] == 150.0).all() and (s1["doppler_extent"] == 100.0).all()
    assert s1.tobytes() == prb.simple_tracker_frames(maps[:, :9], 150.0, 100.0)[:, 5:].tobytes()


@pytest.mark.gpu
def test_resume_on_a_caller_stream_async():
    import torch
    maps = np.stack([synth.track_maps(700 + s, 64, 101, 25, 4) for s in range(3)])
    want = prb.multitarget_tracker_frames(maps, EXTENT, 7)
    wants = prb.simple_tracker_frames(maps, 200.0, 256.0)
    dev = torch.device("cuda", _lib.current_device())
    s = torch.cuda.Stream(device=dev)
    n, cut = 64 * 101, 11
    with torch.cuda.stream(s):
        dm = torch.from_numpy(maps).to(dev)
        dh = torch.empty(want.nbytes, dtype=torch.uint8, device=dev)
        dhs = torch.empty(wants.nbytes, dtype=torch.uint8, device=dev)
    lib = _lib.load()
    stream = C.c_void_p(s.cuda_stream)
    d = _lib.current_device()
    # frames [0, cut) into rows [0, cut) of a (3, 25) history whose sequences are 25 frames apart ...
    _lib.check(lib.prc_multitarget_track_frames(dm.data_ptr(), 64, 101, 3, cut, 25 * n, n, 256.0, 200.0, 7,
                                                dh.data_ptr(), _lib.MEM_DEVICE, d, stream, _lib.FLAG_ASYNC))
    _lib.check(lib.prc_simple_track_frames(dm.data_ptr(), 64, 101, 3, cut, 25 * n, n, 200.0, 256.0, dhs.data_ptr(),
                                           _lib.MEM_DEVICE, d, stream, _lib.FLAG_ASYNC))
    s.synchronize()
    first_m = np.frombuffer(dh[:3 * cut * 7 * MULTI_REC].cpu().numpy().tobytes(), tdm.target_track_dtype).reshape(3, cut, 7)
    first_s = np.frombuffer(dhs[:3 * cut * SIMPLE_REC].cpu().numpy().tobytes(), tdm.target_track_dtype_simple).reshape(3, cut)
    # ... then the rest, resumed from the last records, queued on the same stream without a synchronise
    rest = 25 - cut
    with torch.cuda.stream(s):
        hm = torch.zeros((3, rest, 7 * MULTI_REC), dtype=torch.uint8, device=dev)
        hs = torch.zeros((3, rest, SIMPLE_REC), dtype=torch.uint8, device=dev)
        hm[:, 0] = torch.from_numpy(first_m[:, -1].copy().view(np.uint8).reshape(3, -1)).to(dev)
        hs[:, 0] = torch.from_numpy(first_s[:, -1].copy().view(np.uint8).reshape(3, -1)).to(dev)
    flags = _lib.FLAG_ASYNC | _lib.FLAG_TRACK_RESUME
    _lib.check(lib.prc_multitarget_track_frames(dm[:, cut].data_ptr(), 64, 101, 3, rest, 25 * n, n, 256.0, 200.0, 7,
                                                hm.data_ptr(), _lib.MEM_DEVICE, d, stream, flags))
    _lib.check(lib.prc_simple_track_frames(dm[:, cut].data_ptr(), 64, 101, 3, rest, 25 * n, n, 200.0, 256.0,
                                           hs.data_ptr(), _lib.MEM_DEVICE, d, stream, flags))
    s.synchronize()
    got_m = np.frombuffer(hm.cpu().numpy().tobytes(), tdm.target_track_dtype).reshape(3, rest, 7)
    got_s = np.frombuffer(hs.cpu().numpy().tobytes(), tdm.target_track_dtype_simple).reshape(3, rest)
    assert np.concatenate([first_m, got_m], axis=1).tobytes() == want.tobytes()
    assert np.concatenate([first_s, got_s], axis=1).tobytes() == wants.tobytes()


# ------------------------------------------------------------------ GPU: TrackerPipeline
def _host(out):
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(256, 301), (1024, 176)])
def test_stages_match_the_oracles_and_render_pipeline(rows, cols):
    import torch
    from oracle import plot_oracle as po
    from oracle import track_oracle as O
    T = 40
    maps = _complex_maps(61, rows, cols, T, 8)
    md = torch.from_numpy(maps).cuda()
    rd, rl = (t.cpu().numpy() for t in prb.RenderPipeline().run_device(md))
    cf_want = po.cfar_stack_oracle(np.moveaxis(maps, 0, 2))
    for tracker in ("multi", "simple"):
        got = _host(TrackerPipeline(EXTENT[1], EXTENT[0], tracker=tracker).run_device(md))
        cf = got["cf"]
        assert cf.shape == (T, rows, cols) and cf.dtype == np.float64
        assert _rel(np.moveaxis(cf, 0, 2), cf_want) <= 1e-6
        np.testing.assert_array_equal(got["data"], rd)
        np.testing.assert_array_equal(got["limits"], rl)
        data = np.moveaxis(cf, 0, 2)
        pipe = TrackerPipeline(EXTENT[1], EXTENT[0], tracker=tracker)
        h = pipe.records(got["history"])
        if tracker == "multi":
            want = O.multitarget_tracker(data, EXTENT, 10)
            assert_records_close(h, want, MULTI_DISCRETE)
            for k, w in zip(("track_range", "track_doppler"), _script_masks_multi(h)):
                a, b = _same_nan(got[k], w)
                assert a.tobytes() == b.tobytes(), k
        else:
            want = O.simple_target_tracker(data, EXTENT[1], EXTENT[0])
            assert_records_close(h, want, SIMPLE_DISCRETE)
            for k, w in zip(("estimate_locked", "estimate_unlocked"), _script_masks_simple(h)):
                a, b = _same_nan(got[k], w)
                assert a.tobytes() == b.tobytes(), k


@pytest.mark.gpu
def test_pipeline_matches_the_reference_golden():
    g = G.load("tracker_chain")
    maps = _complex_maps(int(g["seed"]), int(g["rows"]), int(g["cols"]), int(g["T"]), int(g["targets"]))
    assert hashlib.sha256(maps.tobytes()).hexdigest() == str(g["maps_sha256"])
    xambg = np.moveaxis(maps, 0, 2)
    kw = dict(n_tracks=int(g["n_tracks"]), fw=int(g["fw"]), gw=int(g["gw"]), hold=int(g["hold"]),
              decay=float(g["decay"]), batch=16)
    cfg = {"max_range_actual": float(g["max_range"]), "max_doppler_actual": float(g["max_doppler"])}
    m = TrackerPipeline.from_config(cfg, tracker="multi", **kw).run(xambg)
    s = TrackerPipeline.from_config(cfg, tracker="simple", **kw).run(xambg)
    assert m["history"].dtype == tdm.target_track_dtype and m["history"].shape == g["multi_history"].shape
    assert s["history"].dtype == tdm.target_track_dtype_simple and s["history"].shape == g["simple_history"].shape
    assert_records_close(m["history"], g["multi_history"], MULTI_DISCRETE)
    assert_records_close(s["history"], g["simple_history"], SIMPLE_DISCRETE)
    assert np.array_equal(s["history"]["range_extent"], g["simple_history"]["range_extent"])
    for res, keys in ((m, ("track_range", "track_doppler")), (s, ("estimate_locked", "estimate_unlocked"))):
        for k in keys:
            a, b = _same_nan(res[k], g[k])
            assert _rel(a, b) <= 1e-9, k
    for res in (m, s):
        assert _rel(res["limits"], g["limits"]) <= 1e-6
        assert _rel(res["data"][g["data_frames"]], g["data"]) <= 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("tracker", ["multi", "simple"])
def test_batches_of_any_size_give_the_same_bytes_and_reset_starts_over(tracker):
    import torch
    T = 130
    md = torch.from_numpy(_complex_maps(5, 64, 101, T, 6)).cuda()
    pipe = TrackerPipeline(EXTENT[1], EXTENT[0], tracker=tracker, hold=20)
    whole = _host(pipe.run_device(md))
    for b in (1, 7, 64):
        pipe.reset()
        parts = [_host(pipe.run_device(md[t0:t0 + b])) for t0 in range(0, T, b)]
        for k, v in whole.items():
            got = np.concatenate([p[k] for p in parts])
            assert got.tobytes() == v.tobytes(), (b, k)
    pipe.reset()
    again = _host(pipe.run_device(md))
    assert all(again[k].tobytes() == v.tobytes() for k, v in whole.items())
    # without reset() the pipeline continues: the second pass differs from a fresh start
    cont = _host(pipe.run_device(md))
    assert cont["history"].tobytes() != whole["history"].tobytes()
    with pytest.raises(ValueError, match="reset"):
        pipe.run_device(md[:, :32])
    # the host entry point: the same result, as NumPy records
    res = TrackerPipeline(EXTENT[1], EXTENT[0], tracker=tracker, batch=9).run(md.cpu().numpy().transpose(1, 2, 0))
    assert res["history"].tobytes() == whole["history"].tobytes()
    assert set(res) == set(whole) - {"cf"}
    for k in set(res) - {"history"}:
        assert res[k].tobytes() == whole[k].tobytes(), k
    # render=False leaves the tracker's outputs as they are
    bare = _host(TrackerPipeline(EXTENT[1], EXTENT[0], tracker=tracker, render=False).run_device(md))
    assert "data" not in bare and bare["history"].tobytes() == whole["history"].tobytes()
    empty = TrackerPipeline(EXTENT[1], EXTENT[0], tracker=tracker).run(np.zeros((64, 101, 0), np.complex64))
    assert empty["history"].shape[0] == 0 and empty["data"].shape == (0, 101, 64)


@pytest.mark.gpu
def test_recording_maps_streamed_batch_by_batch_equal_one_call():
    import torch
    from passiveradar_b200.recording import RecordingPipeline
    fast = dict(synth.RECORDING_CONFIGS["fast"])
    fast["max_range_actual"] = fast["num_range_cells"] * fast["range_cell_width"]                   # config.py:50
    fast["max_doppler_actual"] = fast["num_doppler_cells"] * fast["doppler_cell_width"] / 2         # config.py:58
    ref, srv, _, _ = synth.recording_for(fast, 12, seed=5)
    rmaps = RecordingPipeline.from_config(fast, batch=4).run_device(torch.from_numpy(ref).cuda(),
                                                                    torch.from_numpy(srv).cuda(), offset=7)
    assert rmaps.is_cuda and rmaps.shape[0] >= 10
    for tracker in ("multi", "simple"):
        whole = _host(TrackerPipeline.from_config(fast, tracker=tracker, fw=8, gw=2, hold=4).run_device(rmaps))
        pipe = TrackerPipeline.from_config(fast, tracker=tracker, fw=8, gw=2, hold=4)
        parts = [_host(pipe.run_device(rmaps[t0:t0 + 3])) for t0 in range(0, rmaps.shape[0], 3)]
        for k, v in whole.items():
            assert np.concatenate([p[k] for p in parts]).tobytes() == v.tobytes(), (tracker, k)
        rd, rl = (t.cpu().numpy() for t in prb.RenderPipeline(fw=8, gw=2, hold=4).run_device(rmaps))
        np.testing.assert_array_equal(whole["data"], rd)
        np.testing.assert_array_equal(whole["limits"], rl)
