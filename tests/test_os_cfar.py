"""Ordered-statistic CFAR (OS_CFAR_2D, os_cfar_frames, prc_os_cfar2d_frames, csrc/oscfar.cuh): the float64 oracle
against scipy's rank filter and CFAR_2D's window sums, the ABI, the refusals, the launch coverage and the build (no GPU
needed); the kernel against the oracle bit for bit and within tolerance, batching, the masking case that motivates the
detector, and the render and tracker chains with cfar="os" (GPU)."""
import math
import os
import re

import numpy as np
import pytest
from scipy import ndimage, signal

import passiveradar_b200 as prb
from oracle import frontend_oracle as fo
from oracle import os_cfar_oracle as oo
from passiveradar_b200 import _lib
from passiveradar_b200.plotting_tools import RenderPipeline
from passiveradar_b200.target_detection import OS_CFAR_2D, TrackerPipeline, os_cfar_frames, os_window_cells

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OSCFAR = os.path.join(ROOT, "passiveradar_b200", "csrc", "oscfar.cuh")
OS_PARAMS = "x rows cols nframes frame_stride fw gw k cr_out cr_stride device stream flags"


def _grid(fws, extra=2):
    """(fw, gw, N) for gw below, at and above fw, the pairs with fw^2 = gw^2 left out (CFAR_2D refuses them)."""
    out = []
    for fw in fws:
        for gw in sorted(set(range(0, fw + extra + 1)) | {2 * fw, 3 * fw + 1}):
            if fw * fw != gw * gw:
                out.append((fw, gw, oo.window_cells(fw, gw)))
    return out


def _ranks(n):
    return sorted({1, oo.default_rank(n), n})


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("shape", [(1, 1), (2, 7), (5, 3), (9, 11)])
def test_oracle_equals_scipy_rank_filter(shape):
    rng = np.random.default_rng(sum(shape))
    X = rng.integers(-50, 50, shape).astype(np.float64)
    rows_checked = 0
    for fw, gw, n in _grid((1, 2, 3, 4, 5, 7, 8, 18)):
        if n == 0:
            continue
        fp = oo.tfilt(fw, gw)[::-1, ::-1] != 0
        for k in _ranks(n):
            want = ndimage.rank_filter(X, k - 1, footprint=fp, mode="wrap", origin=0)
            np.testing.assert_array_equal(oo.os_statistic(X, fw, gw, k), want, err_msg=f"fw={fw} gw={gw} k={k}")
            rows_checked += 1
    assert rows_checked > 150


def test_oracle_window_is_cfar_2d_window():
    rng = np.random.default_rng(4)
    for shape in ((1, 1), (5, 3), (40, 37)):
        X = rng.standard_normal(shape)
        for fw, gw, n in _grid((1, 3, 7, 8, 18)):
            if n == 0:
                continue
            W = oo.os_window(X, fw, gw)
            assert W.shape == shape + (n,) and n == os_window_cells(fw, gw)
            den = signal.convolve2d(X, oo.tfilt(fw, gw) / (fw ** 2 - gw ** 2), mode="same", boundary="wrap")
            np.testing.assert_allclose(W.sum(axis=2) / (fw ** 2 - gw ** 2), den, rtol=1e-12, atol=1e-12)
            # and cfar_2d_oracle's CR is num / (that denominator + 1e-10)
            cr = fo.cfar_2d_oracle(X, fw, gw)
            norm = X / np.mean(np.abs(X))
            np.testing.assert_allclose(cr, norm / (W.sum(axis=2) / (fw ** 2 - gw ** 2) + 1e-10), rtol=1e-9)


def test_defaults_and_window_counts():
    assert oo.window_cells(18, 4) == os_window_cells(18, 4) == 299
    assert oo.default_rank(299) == 225 == prb.target_detection.os_rank(18, 4)
    assert os_window_cells(3, 2) == 0 and os_window_cells(1, 0) == 0


def test_abi_entry_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "prcore.h")).read()
    m = re.search(r"\bint prc_os_cfar2d_frames\(([^)]*)\);", header)
    assert m, "prc_os_cfar2d_frames is not declared"
    params = [p.strip().split()[-1].lstrip("*") for p in m.group(1).split(",")]
    assert " ".join(params) == "x rows cols nframes frame_stride fw gw k cr_out cr_stride device stream flags"
    assert "mem_kind" not in params                         # device pointers only
    assert len(_lib.SIGNATURES["prc_os_cfar2d_frames"][1]) == len(params)
    assert hasattr(_lib.load(), "prc_os_cfar2d_frames")
    assert prb.OS_CFAR_2D is OS_CFAR_2D and prb.os_cfar_frames is os_cfar_frames
    assert {"OS_CFAR_2D", "os_cfar_frames"} <= set(prb.__all__)


def _os_call(**kw):
    buf = np.zeros(64)
    args = dict(x=buf.ctypes.data, rows=4, cols=4, nframes=1, frame_stride=16, fw=18, gw=4, k=225,
                cr_out=buf.ctypes.data, cr_stride=16, device=0, stream=None, flags=0)
    args.update(kw)
    return _lib.load().prc_os_cfar2d_frames(*[args[p] for p in OS_PARAMS.split()])


def test_refusals_before_any_launch():
    lib = _lib.load()
    before = _lib.launch_count()
    checks = [
        (dict(x=None), "x and cr_out must not be NULL"),
        (dict(cr_out=None), "x and cr_out must not be NULL"),
        (dict(fw=65), "fw=65 outside [1, 64]"),
        (dict(fw=0), "fw=0 outside [1, 64]"),
        (dict(fw=4, gw=4), "fw=4 gw=4: fw^2 - gw^2 must not be 0"),
        (dict(gw=-1), "gw=-1: fw^2 - gw^2 must not be 0"),
        (dict(rows=0), "rows=0 cols=4 invalid"),
        (dict(rows=524281), "rows=524281 exceed the CFAR maximum of 524280 rows"),
        (dict(nframes=65536), "nframes=65536 outside [0, 65535]"),
        (dict(nframes=-1), "nframes=-1 outside [0, 65535]"),
        (dict(nframes=2, frame_stride=15), "frame_stride=15"),
        (dict(nframes=2, cr_stride=15), "cr_stride=15"),
        (dict(k=0), "k=0 outside [1, N = 299]"),
        (dict(k=300), "k=300 outside [1, N = 299]"),
        (dict(fw=64, gw=10, k=4096 - 121 + 1), "k=3976 outside [1, N = 3975]"),
    ]
    # every window whose guard hole covers it (N = 0) is refused, whatever k
    for fw, gw, n in _grid(range(1, 65)):
        if n == 0:
            checks.append((dict(fw=fw, gw=gw, k=1), f"fw={fw} gw={gw}: the guard hole covers the whole window"))
    assert sum(1 for c in checks if "guard hole" in c[1]) >= 64
    for kw, msg in checks:
        assert _os_call(**kw) == _lib.PRC_E_INVALID, kw
        assert msg in lib.prc_last_error().decode(), (kw, msg, lib.prc_last_error())
    assert _lib.launch_count() == before


def test_python_argument_checks():
    before = _lib.launch_count()
    with pytest.raises(ValueError, match="two-dimensional"):
        OS_CFAR_2D(np.ones((2, 3, 4)), 18, 4)
    with pytest.raises(TypeError, match="real map"):
        OS_CFAR_2D(np.ones((4, 4), np.complex64), 18, 4)
    with pytest.raises(TypeError, match="float32 or complex64"):
        os_cfar_frames(np.ones((2, 4, 4)), 18, 4)
    for cls, args in ((RenderPipeline, ()), (TrackerPipeline, (100.0, 200.0))):
        with pytest.raises(ValueError, match="cfar must be"):
            cls(*args, cfar="go")
        with pytest.raises(ValueError, match="os_rank applies to cfar='os' only"):
            cls(*args, os_rank=3)
        with pytest.raises(ValueError, match=r"os_rank=300 outside \[1, N = 299\]"):
            cls(*args, cfar="os", os_rank=300)
        with pytest.raises(ValueError, match=r"os_rank=0 outside"):
            cls(*args, cfar="os", os_rank=0)
        with pytest.raises(ValueError, match="needs 1 <= fw <= 64, gw >= 0 and fw != gw"):
            cls(*args, fw=3, gw=3, cfar="os")
        with pytest.raises(ValueError, match=r"os_rank=1 outside \[1, N = 0\]"):
            cls(*args, fw=3, gw=2, cfar="os", os_rank=1)
        assert (cls(*args, cfar="os").os_rank, cls(*args, cfar="os", os_rank=7).os_rank) == (225, 7)
        assert cls(*args).cfar == "ca" and cls(*args).os_rank is None
    assert _lib.launch_count() == before


# every launch in oscfar.cuh -> the GPU tests of this file that reach it
COVERAGE = {
    "cfar_frames_abssum_kernel": ["test_integer_maps_bit_identical_to_oracle", "test_tolerances_and_float32_rounding"],
    "os_select_kernel": ["test_integer_maps_bit_identical_to_oracle",        # fw 3 .. 64, every gw, k = 1, default, N
                         "test_map_sizes_bit_identical_to_oracle",           # 1 x 1 .. 2048 x 301, 524 280 x 4
                         "test_tolerances_and_float32_rounding",             # float32, complex64, float32 CR
                         "test_batched_frames_bit_identical_to_single_calls",
                         "test_strong_neighbour_does_not_mask_the_weak_cell",
                         "test_chains_with_os_cfar"],
}


def _is_gpu_test(name):
    src = open(os.path.abspath(__file__)).read()
    i = src.index(f"\ndef {name}(")
    return "@pytest.mark.gpu" in src[src.rindex("\n\n", 0, i):i]


def test_every_oscfar_launch_has_a_covering_gpu_test():
    src = re.sub(r"//[^\n]*", "", open(OSCFAR).read())
    sites = {m.group(1) for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", src)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    for tests in COVERAGE.values():
        for t in tests:
            assert _is_gpu_test(t), f"{t} is not a GPU test"


def test_os_kernel_builds_for_sm90a_without_spills():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    blocks = [blk for blk in open(log).read().split("Compiling entry function")[1:]
              if "os_select_kernel" in blk.split("\n")[0]]
    assert len(blocks) == 1
    blk = blocks[0]
    assert "'sm_90a'" in blk.split("\n")[0]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in blk
    regs = int(re.search(r"Used (\d+) registers", blk).group(1))
    assert regs <= 64, f"os_select_kernel uses {regs} registers: 256-thread CTAs would lose residency"


# ------------------------------------------------------------------ GPU
def _device_cr(x, fw, gw, k, flags=_lib.FLAG_CR_F64, out_dtype=None):
    """One prc_os_cfar2d_frames call on a (T, rows, cols) float32 / complex64 host stack, through device tensors."""
    import torch
    x = np.ascontiguousarray(x)
    T, rows, cols = x.shape
    if x.dtype == np.complex64:
        flags |= _lib.FLAG_ABS_C64
    xd = torch.from_numpy(x).cuda()
    odt = out_dtype or (torch.float64 if flags & _lib.FLAG_CR_F64 else torch.float32)
    out = torch.empty((T, rows, cols), dtype=odt, device="cuda")
    _lib.check(_lib.load().prc_os_cfar2d_frames(xd.data_ptr(), rows, cols, T, rows * cols, fw, gw, k, out.data_ptr(),
                                                rows * cols, 0, None, flags))
    return out.cpu().numpy()


def _int_map(rng, shape):
    return rng.integers(-1000, 1001, shape).astype(np.float32)


def _bits(a):
    return np.asarray(a).view(np.uint64 if np.asarray(a).dtype == np.float64 else np.uint32)


@pytest.mark.gpu
def test_integer_maps_bit_identical_to_oracle():
    """Integer-valued maps (many ties; sum|X| exact in any order): the float64 CR equals the oracle bit for bit for
    every (fw, gw) of the grid with N >= 1 and k = 1, ceil(3N / 4), N, on a map larger than the tile and one smaller
    than the window."""
    rng = np.random.default_rng(11)
    maps = {"23x37": _int_map(rng, (23, 37)), "5x3": _int_map(rng, (5, 3))}
    maps["ties"] = rng.integers(-3, 4, (19, 40)).astype(np.float32)
    cases = 0
    for fw, gw, n in _grid((3, 8, 18, 33, 64)):
        if n == 0:
            continue
        for name, X in maps.items():
            if name == "ties" and fw not in (8, 33):
                continue
            for k in _ranks(n):
                got = _device_cr(X[None], fw, gw, k)[0]
                want = oo.os_cfar_2d_oracle(X, fw, gw, k)
                np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=f"{name} fw={fw} gw={gw} k={k}")
                cases += 1
    assert cases > 800


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,fw,gw", [(1, 1, 18, 4), (1, 1, 3, 1), (5, 3, 64, 10), (256, 301, 18, 4),
                                             (256, 301, 64, 10), (1024, 176, 33, 7), (1024, 176, 18, 4),
                                             (2048, 301, 18, 4), (524280, 4, 8, 2)])
def test_map_sizes_bit_identical_to_oracle(rows, cols, fw, gw):
    rng = np.random.default_rng(rows * 7 + cols)
    X = _int_map(rng, (rows, cols))
    n = oo.window_cells(fw, gw)
    for k in _ranks(n):
        got = _device_cr(X[None], fw, gw, k)[0]
        want = oo.os_cfar_2d_oracle(X, fw, gw, k)
        np.testing.assert_array_equal(_bits(got), _bits(want), err_msg=f"{rows}x{cols} fw={fw} gw={gw} k={k}")


@pytest.mark.gpu
def test_tolerances_and_float32_rounding():
    rng = np.random.default_rng(5)
    worst = 0.0
    for rows, cols, fw, gw in ((256, 301, 18, 4), (64, 101, 8, 2), (7, 5, 33, 6)):
        n = oo.window_cells(fw, gw)
        for k in _ranks(n):
            X = rng.exponential(1.0, (rows, cols)).astype(np.float32)
            got = _device_cr(X[None], fw, gw, k)[0]
            want = oo.os_cfar_2d_oracle(X, fw, gw, k)
            assert np.max(np.abs(got - want) / np.abs(want)) <= 1e-13, (rows, cols, fw, gw, k)
            # without PRC_FLAG_CR_F64: the float32 rounding of the float64 CR, bit for bit
            got32 = _device_cr(X[None], fw, gw, k, flags=0)[0]
            np.testing.assert_array_equal(_bits(got32), _bits(got.astype(np.float32)))
            Z = (rng.standard_normal((rows, cols)) + 1j * rng.standard_normal((rows, cols))).astype(np.complex64)
            gotc = _device_cr(Z[None], fw, gw, k)[0]
            # np.abs and the device's hypotf differ in the last ulps of num and of T (2.8e-7 seen at 256 x 301, k = 1)
            wantc = oo.os_cfar_2d_oracle(np.abs(Z), fw, gw, k)
            worst = max(worst, np.max(np.abs(gotc - wantc) / np.abs(wantc)))
            assert np.max(np.abs(gotc - wantc) / np.abs(wantc)) <= 4 * 2.0 ** -23, (rows, cols, fw, gw, k)
            gotc32 = _device_cr(Z[None], fw, gw, k, flags=0)[0]
            np.testing.assert_array_equal(_bits(gotc32), _bits(gotc.astype(np.float32)))
    print(f"[os-cfar] complex64 maps: worst relative difference from the oracle on np.abs {worst:.3e}")
    # OS_CFAR_2D: host map in, float64 CR (or CR > thresh) out
    X = rng.exponential(1.0, (64, 101)).astype(np.float32)
    cr = OS_CFAR_2D(X, 18, 4)
    np.testing.assert_array_equal(_bits(cr), _bits(_device_cr(X[None], 18, 4, 225)[0]))
    np.testing.assert_array_equal(OS_CFAR_2D(X, 18, 4, 100, thresh=1.5), _device_cr(X[None], 18, 4, 100)[0] > 1.5)


@pytest.mark.gpu
def test_batched_frames_bit_identical_to_single_calls():
    import torch
    lib = _lib.load()
    rng = np.random.default_rng(8)
    for rows, cols, fw, gw, cplx in ((1, 1, 3, 1, False), (37, 29, 18, 4, True), (256, 301, 18, 4, False),
                                     (100, 70, 64, 3, True)):
        T, pad, opad = 4, 7, 3
        cells = rows * cols
        shape = (T, cells + pad)
        if cplx:
            x = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)
        else:
            x = rng.exponential(1.0, shape).astype(np.float32)
        k = oo.default_rank(oo.window_cells(fw, gw))
        flags = _lib.FLAG_CR_F64 | (_lib.FLAG_ABS_C64 if cplx else 0)
        xd = torch.from_numpy(x).cuda()
        out = torch.full((T, cells + opad), float("nan"), dtype=torch.float64, device="cuda")
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            _lib.check(lib.prc_os_cfar2d_frames(xd.data_ptr(), rows, cols, T, cells + pad, fw, gw, k, out.data_ptr(),
                                                cells + opad, 0, s.cuda_stream, flags | _lib.FLAG_ASYNC))
        s.synchronize()
        got = out.cpu().numpy()
        assert np.isnan(got[:, cells:]).all()
        for b in range(T):
            one = _device_cr(x[b, :cells].reshape(1, rows, cols), fw, gw, k)[0].reshape(-1)
            np.testing.assert_array_equal(_bits(got[b, :cells]), _bits(one), err_msg=f"{rows}x{cols} frame {b}")
        # os_cfar_frames: host stack and CUDA tensor give the same bytes
        stack = np.ascontiguousarray(x[:, :cells].reshape(T, rows, cols))
        h = os_cfar_frames(stack, fw, gw)
        d = os_cfar_frames(torch.from_numpy(stack).cuda(), fw, gw)
        assert d.is_cuda and d.dtype == torch.float64
        np.testing.assert_array_equal(_bits(h), _bits(got[:, :cells].reshape(T, rows, cols)))
        np.testing.assert_array_equal(_bits(d.cpu().numpy()), _bits(h))


@pytest.mark.gpu
def test_strong_neighbour_does_not_mask_the_weak_cell():
    """A 1000 cell five columns from a 10 cell, inside the weak cell's window and outside its guard hole: the OS
    estimate stays at the background, while CFAR_2D's window mean is lifted to (298 + 1000) / 308."""
    X = np.ones((256, 301), np.float32)
    X[100, 150] = 10.0
    X[100, 155] = 1000.0
    fw, gw = 18, 4
    W = oo.os_window(X, fw, gw, 100, 101)[0, 150]
    assert 1000.0 in W and 10.0 not in W             # the strong cell is in the window, the weak one in its hole
    inv_mean = X.size / np.abs(X.astype(np.float64)).sum()
    os_cr = OS_CFAR_2D(X, fw, gw)[100, 150]
    assert os_cr == 10.0 * inv_mean / (1.0 + 1e-10)
    ca_cr = prb.CFAR_2D(X, fw, gw)[100, 150]
    np.testing.assert_allclose(ca_cr, 10.0 * inv_mean / ((298.0 + 1000.0) / 308.0), rtol=1e-6)
    print(f"[os-cfar] weak cell: OS CR {os_cr:.4f}, CA CR {ca_cr:.4f}, ratio {os_cr / ca_cr:.3f}")
    assert 4.1 < os_cr / ca_cr < 4.3


@pytest.mark.gpu
def test_chains_with_os_cfar():
    import torch
    from passiveradar_b200 import synth
    lib = _lib.load()
    T, F, R1 = 23, 64, 101
    rng = np.random.default_rng(31)
    mag = synth.track_maps(17, F, R1, T, 4)
    maps = (mag * np.exp(1j * rng.uniform(0, 2 * np.pi, mag.shape))).astype(np.complex64)     # (T, F, R+1)
    md = torch.from_numpy(maps).cuda()
    want_cf = os_cfar_frames(md, 18, 4).cpu().numpy()
    # the OS CR is not CFAR_2D's
    assert not np.array_equal(want_cf, TrackerPipeline(300.0, 250.0).run_device(md)["cf"].cpu().numpy())
    for k in (None, 40):
        want_cf_k = want_cf if k is None else os_cfar_frames(md, 18, 4, k).cpu().numpy()
        tp = TrackerPipeline(300.0, 250.0, cfar="os", os_rank=k)
        one = tp.run_device(md)
        np.testing.assert_array_equal(_bits(one["cf"].cpu().numpy()), _bits(want_cf_k))
        # RenderPipeline: persistence and percentiles of that stack
        cfd = torch.from_numpy(want_cf_k).cuda()
        data = torch.empty((T, R1, F), dtype=torch.float64, device="cuda")
        lim = torch.empty((T, 2), dtype=torch.float64, device="cuda")
        rp = RenderPipeline(cfar="os", os_rank=k)
        _lib.check(lib.prc_persistence_frames(cfd.data_ptr(), F, R1, T, F * R1, 0, rp.hold, rp.weights.ctypes.data,
                                              data.data_ptr(), _lib.MEM_DEVICE, 0, None,
                                              _lib.FLAG_MAP_F64 | _lib.FLAG_ORIENT))
        q, sc = np.array([35.0, 99.0]), np.array([1.0, 1.5])
        _lib.check(lib.prc_percentiles_frames(data.data_ptr(), F * R1, T, F * R1, q.ctypes.data, sc.ctypes.data, 2,
                                              lim.data_ptr(), _lib.MEM_DEVICE, 0, None, 0))
        d1, l1 = (t.cpu().numpy() for t in rp.run_device(md))
        np.testing.assert_array_equal(_bits(d1), _bits(data.cpu().numpy()))
        np.testing.assert_array_equal(_bits(l1), _bits(lim.cpu().numpy()))
        np.testing.assert_array_equal(_bits(one["data"].cpu().numpy()), _bits(d1))
        # batches of 1, 7 and the whole stack give the same bytes; run equals run_device
        for b in (1, 7, T):
            rp.reset()
            tp.reset()
            rparts = [rp.run_device(md[t0:t0 + b]) for t0 in range(0, T, b)]
            tparts = [tp.run_device(md[t0:t0 + b]) for t0 in range(0, T, b)]
            np.testing.assert_array_equal(np.concatenate([p[0].cpu().numpy() for p in rparts]), d1)
            np.testing.assert_array_equal(np.concatenate([p[1].cpu().numpy() for p in rparts]), l1)
            for key in ("cf", "history", "data", "limits"):
                np.testing.assert_array_equal(np.concatenate([p[key].cpu().numpy() for p in tparts]),
                                              one[key].cpu().numpy(), err_msg=f"{key}, batch {b}")
        d2, l2 = RenderPipeline(cfar="os", os_rank=k, batch=5).run(np.moveaxis(maps, 0, 2))
        np.testing.assert_array_equal(d2, d1)
        np.testing.assert_array_equal(l2, l1)
        host = TrackerPipeline(300.0, 250.0, cfar="os", os_rank=k, batch=6).run(np.moveaxis(maps, 0, 2))
        np.testing.assert_array_equal(host["history"], tp.records(one["history"], T))
        np.testing.assert_array_equal(host["data"], d1)
    # the default path keeps CFAR_2D's bytes
    ca = RenderPipeline().run_device(md)[0].cpu().numpy()
    np.testing.assert_array_equal(ca, RenderPipeline(cfar="ca").run_device(md)[0].cpu().numpy())
    assert math.isfinite(float(np.max(ca)))
