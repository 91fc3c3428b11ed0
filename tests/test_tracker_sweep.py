"""The Kalman trackers (csrc/track.cuh, planned by prcore_detect.cu) against oracle/track_oracle.py where their
planner and kernels branch: maps up to the 524 288-cell limit (candidate slots of 2048 and 4096, the largest
summation trees), the multi-target tracker's frame chunks, candidate counts either side of the slot, truncated
measurement buffers, the percentile's k / k + 1 tie boundary, signed maps with -0.0 cells, and degenerate extents.

The CPU tests hold a Python twin of the planner (trk_stage, trk_smem and the frame chunking of
prc_multitarget_track_frames) to the sources' constants, and check that every GPU case sits in the regime its name
says: a case that drifts off its edge fails instead of passing vacuously.  Discrete fields are compared exactly,
continuous ones to 1e-9 relative."""
import functools
import math
import os
import re

import numpy as np
import pytest

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200 import target_detection as tdm
from oracle import track_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "passiveradar_b200", "csrc")
EXTENT = [256.0, 200.0]
TOL = 1e-9


# ------------------------------------------------------------------ the planner's constants, read from the sources
def _const(fname, name):
    """A constexpr integer of the sources: a literal, a product or a shift of two literals."""
    with open(os.path.join(CSRC, fname)) as f:
        src = f.read()
    m = re.search(rf"constexpr [\w ]+ {name} = (\d+)u?(?:\s*(<<|\*)\s*(\d+)u?)?;", src)
    assert m, f"{name} not found in {fname}"
    a = int(m.group(1))
    if m.group(2) == "<<":
        return a << int(m.group(3))
    if m.group(2) == "*":
        return a * int(m.group(3))
    return a


MAX_CELLS = _const("track.cuh", "TRK_MAX_CELLS")
MAX_CAP = _const("track.cuh", "TRK_MAX_CAP")
SLOT_BUDGET = _const("prcore_detect.cu", "TRK_SLOT_BUDGET")
SMEM_LIMIT = _const("prcore_host.h", "SMEM_LIMIT")


# ------------------------------------------------------------------ planner twin
@functools.lru_cache(maxsize=None)
def _nodes(length):
    """Nodes of NumPy's pairwise-summation tree over `length` elements (trk_plan)."""
    if length <= 128:
        return 1
    h = length // 2 - (length // 2) % 8
    return 1 + _nodes(h) + _nodes(length - h)


def _py_slice(start, stop, length):
    lo, hi, _ = slice(start, stop).indices(length)
    return lo, max(lo, hi)


def plan(rows, cols):
    """trk_stage and trk_smem for a rows x cols map."""
    n = rows * cols
    v = float(n - 1) * (99.8 / 100.0)
    k = math.floor(v)
    dlo, dhi = _py_slice(rows // 2 - 4, rows // 2 + 4, rows)
    want = max(256, 2 * (n - 1 - k) + 64)
    cap = 256
    while cap < want and cap < MAX_CAP:
        cap <<= 1
    nnodes = _nodes(n)
    nv = (nnodes * 8 + 15) & ~15
    return dict(n=n, k=k, g=v - k, dlo=dlo, dhi=dhi, n_unbanded=max(0, cols - 16) * (rows - (dhi - dlo)), cap=cap,
                nnodes=nnodes, smem_mean=nv, smem=nv + cap * 12)


def chunks(rows, cols, nseq, nframes):
    """(frames per launch, launches) of prc_multitarget_track_frames: the candidate slots of one launch stay under
    TRK_SLOT_BUDGET."""
    slot = 3 * plan(rows, cols)["cap"] * 8
    fc = max(1, min(nframes, SLOT_BUDGET // (slot * nseq)))
    return fc, -(-nframes // fc)


def order_stats(frame):
    """(M, thr, le, k, g) of the oracle's view of one map: le counts the cells at or below order statistic k, so
    statistic k + 1 equals statistic k exactly when le >= k + 2 (the kernel's test)."""
    y = O.measurement_frame(frame)
    p = plan(*np.shape(frame))
    thr = np.percentile(y, 99.8)
    a = np.partition(y.ravel(), p["k"])[p["k"]]
    return int((y >= thr).sum()), float(thr), int((y <= a).sum()), p["k"], p["g"]


# ------------------------------------------------------------------ map builders
def _unbanded(rows, cols):
    """Map-order flat indices of the cells outside the zeroed range rows and Doppler columns."""
    p = plan(rows, cols)
    r = np.arange(rows)[:, None]
    c = np.arange(cols)[None, :]
    j = rows - 1 - r
    ok = (c >= 8) & (c < cols - 8) & ~((j >= p["dlo"]) & (j < p["dhi"]))
    return np.flatnonzero(ok.ravel())


PLATEAU = 10.0
LEVELS = ((13.0, 1), (12.0, 3), (11.0, 2))        # (value, cells) above the plateau


def plateau_map(rows, cols, m, levels=(), seed=0, dtype=np.float32):
    """A background below 1 with exactly m cells at or above PLATEAU in the unbanded region: the levels' cells and
    m - sum(levels) cells tied at PLATEAU, where the threshold lands."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.05, 1.0, rows * cols)
    cells = rng.choice(_unbanded(rows, cols), m, replace=False)
    at = 0
    for v, cnt in levels:
        x[cells[at:at + cnt]] = v
        at += cnt
    x[cells[at:]] = PLATEAU
    return x.reshape(rows, cols).astype(dtype)


def boundary_map(rows, cols, le_side, seed=0, mid=3):
    """Three levels above a background below 1: `mid` cells at 5 and U cells at 9, with U = n - 1 - k (order
    statistic k is the last 5: le = k + 1) or U = n - 2 - k (statistics k and k + 1 are both 5: le = k + 2)."""
    p = plan(rows, cols)
    up = p["n"] - 1 - p["k"] if le_side == 1 else p["n"] - 2 - p["k"]
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.05, 1.0, rows * cols)
    cells = rng.choice(_unbanded(rows, cols), up + mid, replace=False)
    x[cells[:up]] = 9.0
    x[cells[up:]] = 5.0
    return x.reshape(rows, cols)


def quantized_map(rows, cols, seed=0):
    """Rayleigh(1) rounded down to 8 levels (0 .. 7 at a step of 1 / 1.68): the top two levels hold about 0.17 % of
    the cells, so the threshold lands on level 5 and every cell of that level (about 1 %) is a candidate."""
    rng = np.random.default_rng(seed)
    return np.minimum(np.floor(rng.rayleigh(1.0, (rows, cols)) * 1.68), 7.0).astype(np.float32)


def nonpositive_map(rows, cols, seed=0):
    """No positive cell, -0.0 scattered among negative ones: the percentile is 0 and every zero cell -- the +0 bands
    and the -0 cells -- is a candidate tied at strength 0."""
    rng = np.random.default_rng(seed)
    x = -rng.rayleigh(1.0, (rows, cols))
    x.ravel()[rng.choice(rows * cols, rows * cols // 2, replace=False)] = -0.0
    return x


def signed_maps(seed, rows, cols, T):
    """track_maps with random signs and -0.0 cells: scattered, at the transformed frame's first cell and at the first
    cell outside its bands (where the simple tracker's argmax lands on a frame without a positive cell)."""
    rng = np.random.default_rng(seed)
    x = synth.track_maps(seed, rows, cols, T, 5).astype(np.float64)
    x *= np.where(rng.random(x.shape) < 0.5, -1.0, 1.0)
    x.reshape(T, -1)[:, rng.choice(rows * cols, rows * cols // 50, replace=False)] = -0.0
    p = plan(rows, cols)
    j0 = 0 if p["dlo"] > 0 else p["dhi"]
    x[:, rows - 1, 0] = -0.0                             # transformed (0, 0)
    x[:, rows - 1 - j0, 8] = -0.0                        # transformed (8, j0)
    return x


# ------------------------------------------------------------------ the named GPU cases
CAP_SHAPES = {256: (64, 101), 512: (256, 301), 1024: (1024, 176), 2048: (512, 512), 4096: (512, 1024)}
WORST_SMEM = (114704, 496002)                            # (bytes, cells) of the largest dynamic shared memory
WORST_SHAPE = (6, 82667)
LARGE_SHAPES = [(512, 1024), (1024, 512), (2048, 256), (512, 512), (1024, 176), WORST_SHAPE]
CHUNK = dict(rows=512, cols=1024, nseq=128, nframes=50, fc=21, launches=3, n_tracks=8)
CHUNK_C2 = dict(rows=256, cols=301, nseq=8000, nframes=5, fc=2, launches=3, n_tracks=2)
PCT_SHAPES = {"g_low": (64, 101), "g_high": (256, 301), "g_zero": (73, 137)}
EXTENTS = [[0.0, 0.0], [5e-324, 5e-324], [-256.0, -200.0], [1e300, 1e300]]


def slot_frames(cap):
    """(name, map, M) of the slot-boundary frames at the shape whose slot holds cap candidates."""
    rows, cols = CAP_SHAPES[cap]
    out = []
    for d in (-1, 0, 1):
        out.append((f"plateau_{d:+d}", plateau_map(rows, cols, cap + d, (), seed=cap + d + 1), cap + d))
        out.append((f"levels_{d:+d}", plateau_map(rows, cols, cap + d, LEVELS, seed=cap + d + 7), cap + d))
    x = quantized_map(rows, cols, seed=cap)
    out.append(("quantized", x, order_stats(x)[0]))
    return out


def pct_frames(shape_name, seed=0):
    rows, cols = PCT_SHAPES[shape_name]
    return [boundary_map(rows, cols, side, seed=seed + side) for side in (1, 2)]


# ------------------------------------------------------------------ comparisons
def _close(a, b, scale=0.0):
    """Relative error of a against b over b's finite entries, relative to the larger of max |b| and `scale`;
    non-finite entries must agree exactly."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    fin = np.isfinite(b)
    assert np.array_equal(np.isfinite(a), fin)
    assert np.array_equal(a[~fin], b[~fin], equal_nan=True)
    if not fin.any():
        return 0.0
    d = max(float(np.abs(b[fin]).max()), scale)
    e = float(np.abs(a[fin] - b[fin]).max())
    return e if d == 0.0 else e / d


def _floats(h):
    k = h["kalman_state"]
    return {"estimate": h["estimate"], "x": k["x"], "P": k["P"], "S": k["S"]}


def _assert_floats(got, want):
    """The Kalman fields to TOL relative.  The estimate H x is held to the scale of x: with zero extents every
    measurement is 0, the estimate is round-off of order 1e-19 and only its error against x means anything."""
    fin = want["kalman_state"]["x"][np.isfinite(want["kalman_state"]["x"])]
    x_scale = float(np.abs(fin).max()) if fin.size else 0.0
    for f, a in _floats(got).items():
        assert _close(a, _floats(want)[f], x_scale if f == "estimate" else 0.0) <= TOL, f


def assert_multi(got, want):
    assert got.shape == want.shape
    for f in ("status", "lifetime", "measurement_history", "measurement"):
        assert np.array_equal(got[f], want[f]), f
    _assert_floats(got, want)


def assert_simple(got, want):
    assert got.shape == want.shape
    for f in ("lock_mode", "measurement", "measurement_idx"):
        assert np.array_equal(got[f], want[f]), f
    _assert_floats(got, want)


def measurements_abi(frames, capacity, extent=EXTENT, f64=False, meas=True):
    """prc_get_measurements_frames on an (S, T, rows, cols) host stack: (counts (S, T), meas (S, T, 3, capacity),
    the NaN canary after meas)."""
    x = np.ascontiguousarray(frames, dtype=np.float64 if f64 else np.float32)
    S, T, rows, cols = x.shape
    counts = np.full(S * T, -7, np.int32)
    size = S * T * 3 * capacity
    buf = np.full(size + 16, np.nan)
    lib = _lib.load()
    _lib.check(lib.prc_get_measurements_frames(x.ctypes.data, rows, cols, S, T, T * rows * cols, rows * cols,
                                               float(extent[0]), float(extent[1]), capacity, counts.ctypes.data,
                                               buf.ctypes.data if meas else None, _lib.MEM_HOST,
                                               _lib.current_device(), None, _lib.FLAG_MAP_F64 if f64 else 0))
    return counts.reshape(S, T), buf[:size].reshape(S, T, 3, capacity), buf[size:]


def _check_multi(data, n_tracks, extent=EXTENT):
    assert_multi(prb.multitarget_tracker(data, extent, n_tracks), O.multitarget_tracker(data, extent, n_tracks))


def _check_simple(data, extent=EXTENT):
    assert_simple(prb.simple_target_tracker(data, extent[1], extent[0]),
                  O.simple_target_tracker(data, extent[1], extent[0]))


# ================================================================== CPU: the twin and the cases' placement
def test_constants_are_read_from_the_sources():
    assert MAX_CELLS == 1 << 19 and MAX_CAP == 4096
    assert SLOT_BUDGET == 256 << 20 and SMEM_LIMIT == 200 * 1024
    with open(os.path.join(CSRC, "track.cuh")) as f:
        src = f.read()
    assert "le >= p.k + 2" in src, "the order-statistic step the percentile cases straddle"


def test_twin_agrees_with_the_oracle_and_numpy():
    rng = np.random.default_rng(3)
    for n in list(range(1, 300)) + [6464, 77056, 180224, 262144, WORST_SMEM[1], MAX_CELLS]:
        assert _nodes(n) == len(O.pairwise_plan(n)[0]), n
    for rows, cols in [(64, 101), (256, 301), (73, 137), (5, 200), (1, 40), (9, 33)]:
        p = plan(rows, cols)
        y = rng.rayleigh(1.0, rows * cols)
        s = np.sort(y)
        b = s[min(p["k"] + 1, p["n"] - 1)]
        a = s[p["k"]]
        lerp = b - (b - a) * (1 - p["g"]) if p["g"] >= 0.5 else a + (b - a) * p["g"]
        assert np.percentile(y, 99.8) == lerp, (rows, cols)
        band = np.ones(rows, bool)
        band[slice(rows // 2 - 4, rows // 2 + 4)] = False
        assert p["n_unbanded"] == max(0, cols - 16) * int(band.sum()) == _unbanded(rows, cols).size
    assert {c: plan(*s)["cap"] for c, s in CAP_SHAPES.items()} == {c: c for c in CAP_SHAPES}


def test_shared_memory_fits_every_map_size():
    """trk_smem <= SMEM_LIMIT for every n up to TRK_MAX_CELLS; the worst size is pinned so a change to the tree or
    to the cap rule is noticed."""
    worst = (0, 0, 0)
    for n in range(1, MAX_CELLS + 1):
        p = plan(1, n)
        assert p["smem"] <= SMEM_LIMIT, n
        if p["smem"] > worst[0]:
            worst = (p["smem"], n, p["cap"])
    assert worst == WORST_SMEM + (MAX_CAP,)
    assert WORST_SHAPE[0] * WORST_SHAPE[1] == WORST_SMEM[1] and plan(*WORST_SHAPE)["smem"] == WORST_SMEM[0]


def test_large_shapes_reach_the_largest_slots_and_trees():
    caps = {s: plan(*s)["cap"] for s in LARGE_SHAPES}
    assert caps == {(512, 1024): 4096, (1024, 512): 4096, (2048, 256): 4096, (512, 512): 2048, (1024, 176): 1024,
                    WORST_SHAPE: 4096}
    assert all(r * c <= MAX_CELLS for r, c in LARGE_SHAPES) and (512 * 1024) == MAX_CELLS
    assert plan(512, 1024)["nnodes"] == 8191 and plan(512, 1024)["smem"] > 100 * 1024
    assert min(r * c for r, c in LARGE_SHAPES) > 180223    # all above the largest map of the other tests


def test_chunk_cases_split_into_launches():
    for case in (CHUNK, CHUNK_C2):
        fc, launches = chunks(case["rows"], case["cols"], case["nseq"], case["nframes"])
        assert (fc, launches) == (case["fc"], case["launches"]) and launches > 1
        assert chunks(case["rows"], case["cols"], 1, case["nframes"]) == (case["nframes"], 1)   # one sequence: one launch
    # config 2 chunks by sequence count alone: its few frames fit one launch at a few hundred sequences
    assert chunks(256, 301, 300, CHUNK_C2["nframes"])[1] == 1


@pytest.mark.parametrize("cap", sorted(CAP_SHAPES))
def test_slot_cases_straddle_the_slot(cap):
    """Plateau maps give exactly M = cap - 1, cap, cap + 1 candidates (with the threshold on the plateau), and the
    quantized map's threshold lands on a tie level far larger than one cell."""
    rows, cols = CAP_SHAPES[cap]
    p = plan(rows, cols)
    assert p["cap"] == cap
    for name, x, m in slot_frames(cap):
        M, thr, le, k, _ = order_stats(x)
        assert M == m, name
        y = O.measurement_frame(x)
        if name != "quantized":
            assert m in (cap - 1, cap, cap + 1)
            assert thr == float(np.float32(PLATEAU)) / O.pairwise_mean_twin(x), name
            assert (y == thr).sum() == m - (sum(c for _, c in LEVELS) if name.startswith("levels") else 0)
        else:
            ties = int((y == thr).sum())
            levels = np.unique(y[y >= thr]).size
            assert ties > 30 and levels == 3, (ties, levels)
            assert (M > cap) == (cap >= 512), (M, cap)        # the level-by-level path at every slot but the smallest
        assert O.get_measurements(x, 99.8, EXTENT).shape[1] == m


@pytest.mark.parametrize("shape_name", sorted(PCT_SHAPES))
def test_percentile_cases_straddle_the_order_statistic_step(shape_name):
    rows, cols = PCT_SHAPES[shape_name]
    g = plan(rows, cols)["g"]
    assert {"g_low": 0 < g < 0.5, "g_high": g >= 0.5, "g_zero": g == 0.0}[shape_name], g
    for side, x in zip((1, 2), pct_frames(shape_name)):
        M, thr, le, k, g = order_stats(x)
        assert le == k + side and (le >= k + 2) == (side == 2)
        mean = O.pairwise_mean_twin(x)
        lo, hi = 5.0 / mean, 9.0 / mean
        up = rows * cols - 1 - k if side == 1 else rows * cols - 2 - k
        if side == 1 and g > 0:
            assert lo < thr < hi and M == up, (thr, lo, hi, M, up)
        else:                                   # statistic k + 1 is 5 too (le = k + 2), or g = 0: the mid ties pass
            assert thr == lo and M == up + 3
        assert M <= plan(rows, cols)["cap"]


def test_truncation_and_signed_zero_cases():
    a, b, a2, b2 = _truncation_frames()
    cap = plan(64, 101)["cap"]
    assert max(order_stats(a)[0], order_stats(a2)[0]) <= cap < min(order_stats(b)[0], order_stats(b2)[0])
    for x in _nonpositive_frames():
        M, thr, _, _, _ = order_stats(x)
        y = O.measurement_frame(x)
        assert thr == 0.0 and M == (y == 0).sum() <= plan(*x.shape)["cap"]
        assert (np.signbit(y) & (y == 0)).sum() >= 4, "-0 candidates tie with the +0 bands"


def test_extent_cases_reach_numpys_zero_step():
    """[5e-324, 5e-324] makes linspace's step round to 0 with a non-zero span: NumPy's k / div * delta branch."""
    rows, cols = 64, 101
    assert (0.0 - 5e-324) / (cols - 1) == 0.0 and (5e-324 - -5e-324) / (rows - 1) == 0.0
    r = np.linspace(5e-324, 0, cols)
    assert r[0] == 5e-324 and r[-2] == 0.0 and len(set(r.tolist())) == 2
    assert np.linspace(0.0, 0.0, cols).tolist() == [0.0] * cols


# ------------------------------------------------------------------ shared inputs
def _truncation_frames():
    """Two frames sorted in the slot and two emitted level by level, 64 x 101 float64: with and without levels above
    the tie at the threshold."""
    return (plateau_map(64, 101, 200, LEVELS, seed=31, dtype=np.float64),
            plateau_map(64, 101, 300, LEVELS, seed=32, dtype=np.float64),
            plateau_map(64, 101, 180, (), seed=33, dtype=np.float64),
            plateau_map(64, 101, 257, (), seed=34, dtype=np.float64))


def _nonpositive_frames():
    return [nonpositive_map(12, 20, seed=s) for s in range(3)] + [nonpositive_map(10, 24, seed=9)]


# ================================================================== GPU
@pytest.mark.gpu
@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
@pytest.mark.parametrize("rows,cols", LARGE_SHAPES)
def test_large_maps_match_oracle(rows, cols, f64):
    """Maps above 180 224 cells up to the 524 288-cell limit: slots of 1024, 2048 and 4096 candidates, trees of up to
    8191 nodes, the worst shared-memory size; get_measurements, both multi-target widths and the simple tracker."""
    T = 30
    maps = synth.track_maps(rows * 7 + cols, rows, cols, T, 6)
    data = np.moveaxis(maps, 0, 2)
    if f64:                                              # values a float32 map cannot hold
        rng = np.random.default_rng(rows + cols)
        data = data.astype(np.float64) * (1.0 + 1e-9 * rng.random(data.shape))
    for t in (0, 13, T - 1):
        got = prb.get_measurements(data[:, :, t], 99.8, EXTENT)
        want = O.get_measurements(data[:, :, t], 99.8, EXTENT)
        assert got.shape == want.shape and np.array_equal(got, want), t
    for n_tracks in (10, tdm.MAX_TRACKS):
        _check_multi(data, n_tracks)
    _check_simple(data)


def _scrolling_maps(case, seed, dev):
    """(S, T, rows, cols) float32 view into one scrolling buffer: frames one row apart, sequences 7.5 rows (or one
    row) apart, so S x T large maps need a few MB."""
    import torch
    rows, cols, S, T = case["rows"], case["cols"], case["nseq"], case["nframes"]
    fs = cols
    ss = 7 * cols + cols // 2 if cols > 512 else cols
    size = (S - 1) * ss + (T - 1) * fs + rows * cols
    tall = synth.track_maps(seed, -(-size // cols), cols, 1, max(8, size // (rows * cols) * 12))[0].ravel()[:size]
    buf = torch.from_numpy(np.ascontiguousarray(tall)).to(dev)
    return torch.as_strided(buf, (S, T, rows, cols), (ss, fs, cols, 1))


def _profiled(fn):
    _lib.profile(True)
    try:
        _lib.profile_reset()
        out = fn()
        prof = _lib.profile_read()
    finally:
        _lib.profile(False)
    return out, prof


def _chunked_run(case, samples, oracle_seqs):
    import torch
    dev = torch.device("cuda", _lib.current_device())
    maps = _scrolling_maps(case, 4242 + case["nseq"], dev)
    assert maps.stride(2) == case["cols"] and maps.stride(3) == 1 and maps.untyped_storage().nbytes() < 12 << 20
    nt = case["n_tracks"]
    fc, launches = chunks(case["rows"], case["cols"], case["nseq"], case["nframes"])
    hist, prof = _profiled(lambda: prb.multitarget_tracker_frames(maps, EXTENT, nt))
    assert prof["track_meas"][1] == launches and prof["track_multi"][1] == launches, prof
    for s in samples:                                    # one sequence never chunks
        one, p1 = _profiled(lambda: prb.multitarget_tracker_frames(maps[s:s + 1], EXTENT, nt))
        assert p1["track_multi"][1] == 1
        assert one[0].tobytes() == hist[s].tobytes(), s
    for s in oracle_seqs:
        data = np.moveaxis(maps[s].cpu().numpy(), 0, 2)
        assert_multi(hist[s], O.multitarget_tracker(data, EXTENT, nt))
    # resumed: every sequence continues from its last records over the same frames again
    init = hist[:, -1].copy()
    res, prof = _profiled(lambda: prb.multitarget_tracker_frames(maps, EXTENT, nt, initial_state=init))
    assert prof["track_multi"][1] == launches
    assert (res["lifetime"][:, 0] > 1).any(), "the records resumed"
    for s in samples:
        one = prb.multitarget_tracker_frames(maps[s:s + 1], EXTENT, nt, initial_state=init[s:s + 1])
        assert one[0].tobytes() == res[s].tobytes(), s
    return hist


@pytest.mark.gpu
def test_chunked_frames_equal_single_sequences_and_the_oracle():
    """128 sequences x 50 frames of 512 x 1024 maps: 21 frames per launch, 3 launches with f0 = 0, 21, 42."""
    S = CHUNK["nseq"]
    _chunked_run(CHUNK, samples=[0, 1, 63, S - 2, S - 1], oracle_seqs=[0, S - 1])


@pytest.mark.gpu
def test_config2_chunks_by_sequence_count():
    """8000 sequences x 5 frames of 256 x 301 maps: 2 frames per launch, 3 launches."""
    S = CHUNK_C2["nseq"]
    _chunked_run(CHUNK_C2, samples=[0, 1, S // 2, S - 1], oracle_seqs=[1, S - 2])


@pytest.mark.gpu
@pytest.mark.parametrize("cap", sorted(CAP_SHAPES))
def test_slot_boundary_matches_oracle(cap):
    """M = cap - 1 and cap sort in the slot; M = cap + 1 and the quantized map's tie level go level by level in
    get_measurements and are enumerated from the map by the tracker (LIST = false)."""
    rows, cols = CAP_SHAPES[cap]
    frames = slot_frames(cap)
    stack = np.stack([x for _, x, _ in frames])[None]
    want = [O.get_measurements(x, 99.8, EXTENT) for _, x, _ in frames]
    capacity = max(w.shape[1] for w in want) + 1
    counts, meas, canary = measurements_abi(stack, capacity)
    assert counts[0].tolist() == [m for _, _, m in frames]
    assert {m for _, _, m in frames} >= {cap - 1, cap, cap + 1}
    for t, (name, _, m) in enumerate(frames):
        assert np.array_equal(meas[0, t, :, :m], want[t]), name
    assert np.isnan(canary).all()
    # short sequences mixing ordinary, slot-sorted and map-enumerated frames
    ordinary = synth.track_maps(cap, rows, cols, 3, 4)
    by = {name: x for name, x, _ in frames}
    seq = [ordinary[0], by["plateau_-1"], by["levels_+1"], ordinary[1], by["quantized"], by["levels_+0"],
           by["plateau_+1"], ordinary[2]]
    data = np.stack(seq, axis=2).astype(np.float32)
    for n_tracks in (10, tdm.MAX_TRACKS):
        _check_multi(data, n_tracks)
    _check_simple(data)


@pytest.mark.gpu
def test_truncated_measurement_buffers():
    """meas_capacity of 0 (no buffer), 1, M - 1, M and M + 1 for a slot-sorted and a level-by-level frame: counts stay
    exact, each frame's first min(M, capacity) columns are the oracle's and nothing is written past the buffer."""
    a, b, a2, b2 = _truncation_frames()
    stack = np.stack([np.stack([a, b]), np.stack([b2, a2])])
    want = [[O.get_measurements(x, 99.8, EXTENT) for x in row] for row in stack]
    ms = sorted({w.shape[1] for row in want for w in row})
    caps = sorted({0, 1} | {m + d for m in ms for d in (-1, 0, 1)})
    for capacity in caps:
        counts, meas, canary = measurements_abi(stack, capacity, f64=True, meas=capacity > 0)
        assert counts.tolist() == [[w.shape[1] for w in row] for row in want], capacity
        for s in range(2):
            for t in range(2):
                m = min(want[s][t].shape[1], capacity)
                assert np.array_equal(meas[s, t, :, :m], want[s][t][:, :m]), (capacity, s, t)
        assert np.isnan(canary).all(), capacity


@pytest.mark.gpu
@pytest.mark.parametrize("shape_name", sorted(PCT_SHAPES))
def test_percentile_boundary_matches_oracle(shape_name):
    """Two-level maps with le = k + 1 (statistic k + 1 is the upper level) and le = k + 2 (it equals statistic k),
    at g < 0.5, g >= 0.5 and g = 0."""
    rows, cols = PCT_SHAPES[shape_name]
    frames = pct_frames(shape_name) + pct_frames(shape_name, seed=10)
    for x in frames:
        got = prb.get_measurements(x, 99.8, EXTENT)
        assert np.array_equal(got, O.get_measurements(x, 99.8, EXTENT))
        assert got.shape[1] == order_stats(x)[0]
    ordinary = synth.track_maps(rows + cols, rows, cols, 2, 3).astype(np.float64)
    data = np.stack([ordinary[0]] + frames + [ordinary[1]], axis=2)
    for n_tracks in (4, 16):
        _check_multi(data, n_tracks)
    _check_simple(data)


@pytest.mark.gpu
def test_signed_maps_and_negative_zero():
    """Rayleigh maps with random signs and -0.0 cells (rows >= 260: the simple tracker's whole zero band is inside),
    and maps without a positive cell, where -0 and +0 candidates tie at the threshold and must interleave by
    position."""
    data = np.moveaxis(signed_maps(17, 288, 301, 20), 0, 2)
    for t in (0, 9):
        assert np.array_equal(prb.get_measurements(data[:, :, t], 99.8, EXTENT),
                              O.get_measurements(data[:, :, t], 99.8, EXTENT))
    for n_tracks in (10, 32):
        _check_multi(data, n_tracks)
    _check_simple(data)
    for x in _nonpositive_frames():
        assert np.array_equal(prb.get_measurements(x, 99.8, EXTENT), O.get_measurements(x, 99.8, EXTENT))
        assert np.array_equal(prb.get_measurements(x.astype(np.float32), 99.8, EXTENT),
                              O.get_measurements(x.astype(np.float32), 99.8, EXTENT))
    small = np.stack(_nonpositive_frames()[:3] * 2, axis=2)
    for n_tracks in (1, 5):
        _check_multi(small, n_tracks)
    _check_simple(small)


@pytest.mark.gpu
@pytest.mark.parametrize("extent", EXTENTS, ids=["zero", "subnormal", "negative", "huge"])
def test_degenerate_extents_match_oracle(extent):
    """Zero, subnormal (linspace's step rounds to 0 over a non-zero span), negative and near-overflow extents."""
    maps = synth.track_maps(55, 96, 101, 25, 4)
    data = np.moveaxis(maps, 0, 2)
    for t in (0, 11):
        got = prb.get_measurements(data[:, :, t], 99.8, extent)
        assert np.array_equal(got, O.get_measurements(data[:, :, t], 99.8, extent)), t
    for n_tracks in (10, tdm.MAX_TRACKS):
        got = prb.multitarget_tracker(data, extent, n_tracks)
        assert_multi(got, O.multitarget_tracker(data, extent, n_tracks))
        if extent == [0.0, 0.0]:            # every candidate at (0, 0): one track takes the whole list each frame
            assert ((got["status"] != 0).sum(axis=1) == 1).all()
    _check_simple(data, extent)
