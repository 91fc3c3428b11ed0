"""Frame chain of range_doppler_plot.py:45-85 (passiveradar_b200.plotting_tools): the ABI, the launch coverage, the
build, the golden provenance, a NumPy statement of the persistence rounding and the refusals (no GPU needed); the
batched CFAR against per-frame CFAR_2D calls, persistence against the reference's goldens, the percentiles against
np.percentile and RenderPipeline against the oracle chain (GPU)."""
import hashlib
import json
import os
import re
import sys
import threading

import numpy as np
import pytest

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200.plotting_tools import RenderPipeline, persistence, persistence_frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DETECT = os.path.join(ROOT, "passiveradar_b200", "csrc", "detect.cuh")
RENDER = os.path.join(ROOT, "passiveradar_b200", "csrc", "render.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden")
ENTRIES = ("prc_cfar2d_frames", "prc_persistence_frames", "prc_percentiles_frames")
DECAYS = {"py0.9": 0.9, "f32_0.9": np.float32(0.9), "f64_0.9": np.float64(0.9), "py0.0": 0.0, "py1.0": 1.0,
          "py1.5": 1.5}
HOLDS = (1, 2, 20, 30)


@pytest.fixture(scope="module")
def pgold():
    with np.load(os.path.join(GOLDEN, "render_persistence.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def cgold():
    with np.load(os.path.join(GOLDEN, "render_chain.npz")) as z:
        return {k: z[k] for k in z.files}


def _same(a, b):
    """Equal values, NaN where the other is NaN, and the same sign on zeros (NaN payloads are not compared)."""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    np.testing.assert_array_equal(a, b)
    ok = ~np.isnan(b)
    np.testing.assert_array_equal(np.signbit(a[ok]), np.signbit(b[ok]))


# ------------------------------------------------------------------ CPU
def test_abi_entries_are_declared():
    header = open(os.path.join(ROOT, "include", "prcore.h")).read()
    for name in ENTRIES:
        assert name in _lib.SIGNATURES
        assert re.search(rf"\bint {name}\(", header)
    for flag, value in (("PRC_FLAG_CR_F64", 16), ("PRC_FLAG_PROD_F32", 32), ("PRC_FLAG_ORIENT", 64)):
        assert re.search(rf"#define {flag}\s+{value}u", header)
    assert (_lib.FLAG_CR_F64, _lib.FLAG_PROD_F32, _lib.FLAG_ORIENT) == (16, 32, 64)
    assert prb.persistence is persistence and prb.RenderPipeline is RenderPipeline
    assert prb.persistence_frames is persistence_frames


# every launch in detect.cuh and render.cuh -> the GPU tests that reach it (a test of this file, or
# "tests/<file>::<test>")
FE, RS = "tests/test_gpu_frontend.py::", "tests/test_rows_sweep.py::"
COVERAGE = {
    "cfar_frames_abssum_kernel": ["test_cfar_frames_bit_identical_to_per_frame_calls", "test_chain_matches_oracle",
                                  FE + "test_cfar_matches_reference_golden",
                                  RS + "test_cfar_map_contents_match_oracle"],       # real maps and |x| of complex maps
    "cfar_frames_kernel": ["test_cfar_frames_bit_identical_to_per_frame_calls", "test_chain_matches_oracle",
                           FE + "test_cfar_matches_reference_golden",
                           RS + "test_cfar_fw_gw_grid_matches_oracle",      # fw = 1 .. 64, gw below, at and above fw
                           RS + "test_cfar_map_sizes_match_oracle",         # 1 x 1 .. 2048 x 301, smaller than tile and fw
                           RS + "test_cfar_map_contents_match_oracle",      # signed, float64, complex, zero plateaus
                           RS + "test_cfar_row_limit"],                     # the tallest map, 524 280 rows
    "pst_kernel": ["test_persistence_matches_reference_goldens", "test_chain_matches_oracle"],
    "pct_kernel": ["test_percentiles_bit_identical_to_numpy", "test_chain_matches_oracle"],
}


def _is_gpu_test(test_id):
    path, _, name = test_id.rpartition("::")
    src = open(os.path.join(ROOT, path) if path else os.path.abspath(__file__)).read()
    i = src.index(f"\ndef {name}(")
    decorators = src[src.rindex("\n\n", 0, i):i]
    return "@pytest.mark.gpu" in decorators or re.search(r"^pytestmark = pytest\.mark\.gpu$", src, re.M) is not None


def test_every_cfar_and_render_launch_has_a_covering_gpu_test():
    src = open(DETECT).read() + open(RENDER).read()
    sites = {m.group(1) + (m.group(2) or "") for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", src)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    for tests in COVERAGE.values():
        for t in tests:
            assert _is_gpu_test(t), f"{t} is not a GPU test"


def test_cfar_and_render_kernels_build_for_sm90a_without_spills():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    blocks = [blk for blk in open(log).read().split("Compiling entry function")[1:]
              if "3prc3rdr" in blk.split("\n")[0] or "cfar_frames" in blk.split("\n")[0]]
    assert len(blocks) == 4, "cfar abssum, cfar, persistence, percentile"
    for blk in blocks:
        assert "'sm_90a'" in blk.split("\n")[0]
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in blk


def _digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("name", ["render_persistence", "render_chain"])
def test_committed_render_golden_is_what_the_reference_produces(name):
    with open(os.path.join(GOLDEN, "render_reference_digests.json")) as f:
        want = json.load(f)[name]
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        assert set(z.files) == set(want)
        for k in want:
            assert _digest(z[k]) == want[k], f"{name}[{k}] differs from the reference's output"


def _persistence_statement(X, k, hold, decay):
    """The kernel's rounding order in NumPy: +0.0, then one rounded product and one rounded sum per term, the
    product in float32 when NumPy 2 promotes X * decay**i to float32."""
    w = [decay ** i for i in range(max(0, min(k + 1, hold)))]
    s = np.zeros(X.shape[:2])
    for i, wi in enumerate(w):
        prod = np.result_type(X.dtype, wi)
        with np.errstate(invalid="ignore", over="ignore"):
            if prod == np.float32:
                p = (X[:, :, k - i].astype(np.float32) * np.float32(wi)).astype(np.float64)
            else:
                p = X[:, :, k - i].astype(np.float64) * np.float64(wi)
            s = s + p
    return s


def test_numpy_statement_of_the_rounding_equals_the_golden(pgold):
    for tag in ("f64", "f32"):
        X = pgold[f"stack_{tag}"]
        for dname, decay in DECAYS.items():
            for hold in HOLDS:
                want = pgold[f"out_{tag}_{dname}_h{hold}"]
                got = np.stack([_persistence_statement(X, k, hold, decay) for k in range(X.shape[2])])
                _same(got, want)
        # a float32 stack with a Python-float decay really has float32 products: a float64 product differs
        if tag == "f32":
            wide = np.stack([sum((X[:, :, k - i].astype(np.float64) * 0.9 ** i for i in range(min(k + 1, 20))),
                                 np.zeros(X.shape[:2])) for k in range(X.shape[2])])
            with np.errstate(invalid="ignore"):
                assert not np.array_equal(wide, pgold["out_f32_py0.9_h20"], equal_nan=True)


def test_refusals_before_any_launch():
    before = _lib.launch_count()
    X = np.ones((4, 5, 6))
    with pytest.raises(IndexError, match="out of bounds"):
        persistence(X, 6, 3, 0.9)
    with pytest.raises(TypeError, match="real"):
        persistence(X.astype(np.complex64), 1, 3, 0.9)
    with pytest.raises(ValueError, match="three-dimensional"):
        persistence(np.ones((4, 5)), 0, 3, 0.9)
    with pytest.raises(ValueError, match="three-dimensional"):
        persistence_frames(np.ones((4, 5)), 3, 0.9)
    # the reference reads no frame: zeros, whatever k
    for k, hold in ((-1, 20), (-2, 20), (3, 0), (9, 0), (9, -2)):
        z = persistence(X, k, hold, 0.9)
        assert z.dtype == np.float64 and z.shape == (4, 5) and not z.any()
    with pytest.raises(ValueError, match="hold"):
        RenderPipeline(hold=0)
    lib = _lib.load()
    buf = np.zeros(64)
    w = np.ones(4)
    q = np.array([35.0, 99.0])
    checks = [
        (lambda: lib.prc_persistence_frames(buf.ctypes.data, 2, 2, 1, 4, 0, 0, w.ctypes.data, buf.ctypes.data, 0, 0, None, 0),
         "hold=0 must be >= 1"),
        (lambda: lib.prc_persistence_frames(buf.ctypes.data, 2, 2, 1, 4, 3, 3, w.ctypes.data, buf.ctypes.data, 0, 0, None, 0),
         "n_carry=3 outside [0, hold - 1 = 2]"),
        (lambda: lib.prc_persistence_frames(buf.ctypes.data, 2, 2, 1, 4, 0, 2, w.ctypes.data, buf.ctypes.data, 0, 0, None,
                                    _lib.FLAG_MAP_F64 | _lib.FLAG_PROD_F32), "float32 products need a float32 stack"),
        (lambda: lib.prc_persistence_frames(buf.ctypes.data, 524289, 2, 1, 4, 0, 2, w.ctypes.data, buf.ctypes.data, 0, 0, None,
                                    0), "persistence maximum of 524280 rows"),
        (lambda: lib.prc_percentiles_frames(buf.ctypes.data, 8, 1, 8, q.ctypes.data, None, 5, buf.ctypes.data, 0, 0, None, 0),
         "nq=5 outside [1, 4]"),
        (lambda: lib.prc_percentiles_frames(buf.ctypes.data, 0, 1, 8, q.ctypes.data, None, 2, buf.ctypes.data, 0, 0, None, 0),
         "n=0 outside"),
        (lambda: lib.prc_percentiles_frames(buf.ctypes.data, 2 ** 31 - 512, 1, 2 ** 31 - 512, q.ctypes.data, None, 2,
                                            buf.ctypes.data, 0, 0, None, 0), "n=2147483136 outside [1, 2147483135]"),
        (lambda: lib.prc_percentiles_frames(buf.ctypes.data, 8, 1, 8, np.array([101.0]).ctypes.data, None, 1, buf.ctypes.data,
                                    0, 0, None, 0), "q[0]=101 outside [0, 100]"),
        (lambda: lib.prc_cfar2d_frames(buf.ctypes.data, 4, 4, 1, 16, 65, 4, buf.ctypes.data, 16, 0, 0, None, 0),
         "fw=65 outside [1, 64]"),
        (lambda: lib.prc_cfar2d_frames(buf.ctypes.data, 524281, 4, 1, 16, 18, 4, buf.ctypes.data, 16, 0, 0, None, 0),
         "rows=524281 exceed the CFAR maximum of 524280 rows"),
        (lambda: lib.prc_cfar2d_frames(buf.ctypes.data, 4, 4, 65536, 16, 18, 4, buf.ctypes.data, 16, 0, 0, None, 0),
         "nframes=65536 outside [0, 65535]"),
        (lambda: lib.prc_cfar2d_frames(buf.ctypes.data, 4, 4, 2, 15, 18, 4, buf.ctypes.data, 16, 0, 0, None, 0),
         "frame_stride=15"),
    ]
    for call, msg in checks:
        assert call() == _lib.PRC_E_INVALID
        assert msg in lib.prc_last_error().decode(), (msg, lib.prc_last_error())
    assert _lib.launch_count() == before


def test_float_stacks_the_kernel_cannot_reproduce_are_refused():
    """float16 and long-double stacks (and decays that make the products so) are refused before any launch: the
    kernel reads and multiplies float32 or float64 only."""
    import torch
    from passiveradar_b200.plotting_tools import _stack_dtype
    before = _lib.launch_count()
    for dt in (np.float16, np.longdouble):
        X = np.ones((3, 4, 5), dtype=dt)
        with pytest.raises(TypeError, match="unsupported stack dtype"):
            persistence(X, 2, 3, 0.9)
        with pytest.raises(TypeError, match="unsupported stack dtype"):
            persistence(X, -1, 3, 0.9)
        with pytest.raises(TypeError, match="unsupported stack dtype"):
            persistence_frames(np.moveaxis(X, 2, 0), 3, 0.9)
    for t in (torch.float16, torch.bfloat16):
        with pytest.raises(TypeError, match="unsupported stack dtype"):
            _stack_dtype(torch.ones((3, 4, 5), dtype=t))
    with pytest.raises(TypeError, match="float32 or float64 products"):
        persistence(np.ones((3, 4, 5), np.float32), 2, 3, np.longdouble(0.9))
    with pytest.raises(TypeError, match="float32 or float64 products"):
        persistence(np.ones((3, 4, 5), np.int8), 2, 3, np.float16(0.9))
    assert _stack_dtype(torch.ones(2, dtype=torch.int16)) == np.int16
    assert _lib.launch_count() == before


def test_install_replaces_plotting_persistence(tmp_path, monkeypatch):
    pkg = tmp_path / "fakeref_render"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    (pkg / "range_doppler_processing.py").write_text("def fast_xambg(*a):\n    pass\n")
    (pkg / "clutter_removal.py").write_text("def LS_Filter(*a):\n    pass\n")
    (pkg / "plotting_tools.py").write_text("def persistence(X, k, hold, decay):\n    return 'reference'\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    replaced = prb.install("fakeref_render")
    import fakeref_render.plotting_tools as pt
    assert "fakeref_render.plotting_tools.persistence" in replaced
    assert pt.persistence is persistence
    for m in [m for m in sys.modules if m.startswith("fakeref_render")]:
        del sys.modules[m]


# ------------------------------------------------------------------ GPU
def _cfar_frames(x, rows, cols, T, stride, fw, gw, out, out_stride, flags, mem, stream=None):
    return _lib.load().prc_cfar2d_frames(_lib.ptr(x), rows, cols, T, stride, fw, gw, _lib.ptr(out), out_stride, mem, 0,
                                         stream, flags)


@pytest.mark.gpu
def test_cfar_frames_bit_identical_to_per_frame_calls():
    import torch
    lib = _lib.load()
    rng = np.random.default_rng(7)
    for rows, cols in ((1, 1), (7, 5), (64, 101), (256, 301), (1024, 176)):
        for fw, gw in ((1, 0), (3, 2), (18, 4), (64, 10)):
            for cplx in (False, True):
                T, pad = 3, 5
                cells = rows * cols
                if cplx:
                    x = (rng.standard_normal((T, cells + pad)) + 1j * rng.standard_normal((T, cells + pad))).astype(np.complex64)
                else:
                    x = rng.standard_normal((T, cells + pad)).astype(np.float32)
                flag = _lib.FLAG_ABS_C64 if cplx else 0
                want = np.empty((T, cells), np.float32)
                for b in range(T):
                    fr = np.ascontiguousarray(x[b, :cells])
                    _lib.check(lib.prc_cfar2d_f32(fr.ctypes.data, rows, cols, fw, gw, None, want[b].ctypes.data, None,
                                                  _lib.MEM_HOST, 0, None, flag))
                got32 = np.full((T, cells + 2), np.nan, np.float32)
                _lib.check(_cfar_frames(x, rows, cols, T, cells + pad, fw, gw, got32, cells + 2, flag, _lib.MEM_HOST))
                np.testing.assert_array_equal(got32[:, :cells].view(np.uint32), want.view(np.uint32),
                                              err_msg=f"{rows}x{cols} fw={fw} gw={gw} complex={cplx}")
                assert np.isnan(got32[:, cells:]).all()
                # float64 CR on device pointers and a caller stream: its float32 rounding is the float32 CR
                s = torch.cuda.Stream()
                xd = torch.from_numpy(x).cuda()
                got64 = torch.empty((T, cells), dtype=torch.float64, device="cuda")
                with torch.cuda.stream(s):
                    _lib.check(_cfar_frames(xd, rows, cols, T, cells + pad, fw, gw, got64, cells,
                                            flag | _lib.FLAG_CR_F64 | _lib.FLAG_ASYNC, _lib.MEM_DEVICE, s.cuda_stream))
                s.synchronize()
                g64 = got64.cpu().numpy()
                np.testing.assert_array_equal(g64.astype(np.float32).view(np.uint32), want.view(np.uint32))


@pytest.mark.gpu
def test_persistence_matches_reference_goldens(pgold):
    import torch
    for tag in ("f64", "f32"):
        X = pgold[f"stack_{tag}"]
        L = X.shape[2]
        stack = np.ascontiguousarray(np.moveaxis(X, 2, 0))
        stream = torch.cuda.Stream()
        for dname, decay in DECAYS.items():
            for hold in HOLDS:
                want = pgold[f"out_{tag}_{dname}_h{hold}"]
                for k in range(L):
                    _same(persistence(X, k, hold, decay), want[k])
                _same(persistence_frames(stack, hold, decay), want)
                with torch.cuda.stream(stream):
                    Xd, Sd = torch.from_numpy(X).cuda(), torch.from_numpy(stack).cuda()
                    got_k = [persistence(Xd, k, hold, decay) for k in (0, L // 2, L - 1)]
                    got_f = persistence_frames(Sd, hold, decay)
                    host = [g.cpu().numpy() for g in got_k] + [got_f.cpu().numpy()]
                for g, k in zip(host[:3], (0, L // 2, L - 1)):
                    _same(g, want[k])
                _same(host[3], want)
        for edge, (k, hold) in (("km1", (-1, 20)), ("km2", (-2, 20)), ("h0", (5, 0))):
            _same(persistence(X, k, hold, 0.9), pgold[f"edge_{tag}_{edge}"])


def _percentiles(frames, q, scale=None, device=False):
    import torch
    frames = np.ascontiguousarray(frames, dtype=np.float64)
    T, n = frames.shape
    q = np.asarray(q, dtype=np.float64)
    sc = None if scale is None else np.asarray(scale, dtype=np.float64)
    if device:
        xd = torch.from_numpy(frames).cuda()
        out = torch.empty((T, q.size), dtype=torch.float64, device="cuda")
        _lib.check(_lib.load().prc_percentiles_frames(xd.data_ptr(), n, T, n, q.ctypes.data,
                                                      None if sc is None else sc.ctypes.data, q.size, out.data_ptr(),
                                                      _lib.MEM_DEVICE, 0, None, 0))
        return out.cpu().numpy()
    out = np.empty((T, q.size))
    _lib.check(_lib.load().prc_percentiles_frames(frames.ctypes.data, n, T, n, q.ctypes.data,
                                                  None if sc is None else sc.ctypes.data, q.size, out.ctypes.data,
                                                  _lib.MEM_HOST, 0, None, 0))
    return out


@pytest.mark.gpu
def test_percentiles_bit_identical_to_numpy():
    rng = np.random.default_rng(3)
    cases = {
        "random": rng.standard_normal((5, 77003)),
        "tied": rng.integers(0, 5, (4, 1000)).astype(np.float64),
        "constant": np.full((2, 513), 2.5),
        "n1": rng.standard_normal((3, 1)),
        "n2": rng.standard_normal((3, 2)),
        "positive_maps": np.abs(rng.standard_normal((3, 301 * 256))) * 1e3,
    }
    special = rng.standard_normal((6, 400))
    special[0, 17] = np.nan
    special[1, 3] = np.inf
    special[2, 9] = -np.inf
    special[3, [1, 5]] = [np.inf, -np.inf]
    special[4, :] = np.inf
    special[5, :200] = -np.inf
    cases["special"] = special
    cases["one_inf"] = np.array([[np.inf], [-np.inf], [np.nan]])
    for qs in ([35, 99], [0, 100, 50, 99.9], [12.5]):
        for name, frames in cases.items():
            with np.errstate(invalid="ignore"):
                want = np.stack([np.percentile(f, qs) for f in frames]).reshape(frames.shape[0], len(qs))
            for dev in (False, True):
                got = _percentiles(frames, qs, device=dev)
                _same(got, want)
    # the colour limits: vmax = 1.5 * percentile 99
    f = cases["positive_maps"]
    got = _percentiles(f, [35, 99], [1.0, 1.5])
    want = np.array([[np.percentile(x, 35), 1.5 * np.percentile(x, 99)] for x in f])
    _same(got, want)


def _complex_maps(seed, rows, cols, T):
    rng = np.random.default_rng(seed + 1000)
    mag = synth.track_maps(seed, rows, cols, T, 4)
    return (mag * np.exp(1j * rng.uniform(0, 2 * np.pi, mag.shape))).astype(np.complex64)   # (T, rows, cols)


def _rel(a, b):
    return float(np.max(np.abs(a - b) / np.abs(b)))


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(256, 301), (1024, 176)])
def test_chain_matches_oracle(rows, cols):
    import torch
    from oracle import plot_oracle as po
    maps = _complex_maps(61, rows, cols, 60)
    data, lim = RenderPipeline().run_device(torch.from_numpy(maps).cuda())
    data, lim = data.cpu().numpy(), lim.cpu().numpy()
    want_d, want_l = po.render_oracle(np.moveaxis(maps, 0, 2))
    e_d, e_l = _rel(data, want_d), _rel(lim, want_l)
    print(f"[render] {rows}x{cols}: data {e_d:.2e}, limits {e_l:.2e}")
    assert data.shape == (60, cols, rows) and lim.shape == (60, 2)
    assert e_d <= 1e-6 and e_l <= 1e-6


@pytest.mark.gpu
def test_chain_matches_reference_golden(cgold):
    c = cgold
    maps = synth.track_maps(int(c["seed"]), int(c["rows"]), int(c["cols"]), int(c["T"]), int(c["targets"]))
    assert hashlib.sha256(maps.tobytes()).hexdigest() == str(c["maps_sha256"])
    data, lim = RenderPipeline(int(c["fw"]), int(c["gw"]), int(c["hold"]), float(c["decay"])).run(np.moveaxis(maps, 0, 2))
    assert _rel(data, c["data"]) <= 1e-6
    assert _rel(lim[:, 0], c["vmin"]) <= 1e-6 and _rel(lim[:, 1], c["vmax"]) <= 1e-6


@pytest.mark.gpu
def test_batches_host_run_and_recording_chain_bit_identical():
    import torch
    from passiveradar_b200.recording import RecordingPipeline
    T = 30
    maps = _complex_maps(5, 64, 101, T)
    md = torch.from_numpy(maps).cuda()
    pipe = RenderPipeline()
    d1, l1 = (t.cpu().numpy() for t in pipe.run_device(md))
    for b in (1, 7, T):
        pipe.reset()
        parts = [pipe.run_device(md[t0:t0 + b]) for t0 in range(0, T, b)]
        np.testing.assert_array_equal(np.concatenate([p[0].cpu().numpy() for p in parts]), d1)
        np.testing.assert_array_equal(np.concatenate([p[1].cpu().numpy() for p in parts]), l1)
    d2, l2 = RenderPipeline(batch=4).run(np.moveaxis(maps, 0, 2))
    np.testing.assert_array_equal(d2, d1)
    np.testing.assert_array_equal(l2, l1)
    d3, l3 = RenderPipeline(batch=8).run(np.abs(np.moveaxis(maps, 0, 2)))           # already np.abs-ed
    assert _rel(d3, d1) <= 1e-6 and _rel(l3, l1) <= 1e-6
    # chained from the recording pipeline: the maps stay on the device
    fast = synth.RECORDING_CONFIGS["fast"]
    ref, srv, _, _ = synth.recording_for(fast, 6, seed=5)
    rp = RecordingPipeline.from_config(fast, batch=3)
    rmaps = rp.run_device(torch.from_numpy(ref).cuda(), torch.from_numpy(srv).cuda(), offset=7)
    assert rmaps.is_cuda
    rd, rl = RenderPipeline(fw=8, gw=2, hold=4).run_device(rmaps)
    assert rd.is_cuda and rl.is_cuda
    hd, hl = RenderPipeline(fw=8, gw=2, hold=4).run(rmaps.cpu().numpy().transpose(1, 2, 0))
    np.testing.assert_array_equal(rd.cpu().numpy(), hd)
    np.testing.assert_array_equal(rl.cpu().numpy(), hl)


@pytest.mark.gpu
def test_cuda_float16_stacks_refused_and_signed_float32_maps_rendered_as_magnitudes():
    import torch
    before = _lib.launch_count()
    for t in (torch.float16, torch.bfloat16):
        X = torch.ones((3, 4, 5), dtype=t, device="cuda")
        with pytest.raises(TypeError, match="unsupported stack dtype"):
            persistence(X, 2, 3, 0.9)
        with pytest.raises(TypeError, match="unsupported stack dtype"):
            persistence_frames(X, 3, 0.9)
    assert _lib.launch_count() == before
    rng = np.random.default_rng(21)
    signed = rng.standard_normal((9, 48, 70)).astype(np.float32)
    got = [t.cpu().numpy() for t in RenderPipeline(hold=4).run_device(torch.from_numpy(signed).cuda())]
    want = [t.cpu().numpy() for t in RenderPipeline(hold=4).run_device(torch.from_numpy(np.abs(signed)).cuda())]
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])


@pytest.mark.gpu
def test_concurrent_threads_bit_identical():
    import torch
    maps = _complex_maps(9, 128, 151, 25)
    want = [t.cpu().numpy() for t in RenderPipeline().run_device(torch.from_numpy(maps).cuda())]
    results, errors = [None] * 8, []

    def work(i):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                md = torch.from_numpy(maps).cuda()
                pipe = RenderPipeline()
                parts = [pipe.run_device(md[t0:t0 + 5 + i]) for t0 in range(0, 25, 5 + i)]
                results[i] = [torch.cat([p[j] for p in parts]).cpu().numpy() for j in (0, 1)]
        except Exception as exc:           # surfaced below
            errors.append(exc)

    threads = [threading.Thread(target=work, args=(i,)) for i in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for r in results:
        np.testing.assert_array_equal(r[0], want[0])
        np.testing.assert_array_equal(r[1], want[1])
