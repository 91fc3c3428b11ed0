"""Sweeps of the rows either side of the hot path (DESIGN.md section 9) against float64 truths and the reference's
own arithmetic: CFAR_2D over its (fw, gw) grid, map sizes, map contents and thresholds; resample over a ratio grid,
CTA boundaries, short inputs and its shared-memory limit; frequency_shift and the fused frontend past 2^24 samples and
in every mix mode; direct_xambg at R >= n, one or an odd number of Doppler bins, and its lag limit; device pointers on
a caller stream; concurrent threads.

Criteria (SURVEY.md 8d): E = max|gpu - x| / max|x| <= 1e-5.  Where the reference is itself complex64 arithmetic,
GPU-vs-truth <= 1e-5 and GPU-vs-reference <= 1e-5 + 1.2 x (reference-vs-truth).  Figures go to
$PRC_PARITY_DIR/parity.json (conftest.record_parity).

The one CPU test states cfar_frames_kernel's summation order in NumPy, with the accumulator type read from
csrc/detect.cuh, and holds it to the float64 oracle on non-negative and signed maps."""
import ctypes as C
import math
import os
import re
import threading

import numpy as np
import pytest

from conftest import record_parity
import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200 import signal_utils as psu
from oracle import frontend_oracle as FO
from oracle.clutter_oracle import frequency_shift_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DETECT = os.path.join(ROOT, "passiveradar_b200", "csrc", "detect.cuh")
TOL = 1e-5
CELL_TOL = 1e-4        # per cell, as tests/test_gpu_frontend.py holds the CFAR goldens


def rel(a, b, den):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / den)


def two_sided(gpu, ref, truth, den):
    """(GPU-vs-truth, GPU-vs-reference, reference-vs-truth), each over ``den``."""
    return rel(gpu, truth, den), rel(gpu, ref, den), rel(ref, truth, den)


# ------------------------------------------------------------------ maps
def rayleigh(rows, cols, seed):
    return np.random.default_rng(seed).rayleigh(1.0, size=(rows, cols)).astype(np.float32)


def clutter_ridge(rows, cols, seed):
    """Rayleigh background with a 55 dB zero-Doppler ridge falling off in range, as |xambg| of an unfiltered channel."""
    x = rayleigh(rows, cols, seed)
    x[rows // 2] *= np.float32(10 ** (55 / 20)) * np.exp(-np.arange(cols) / 40.0).astype(np.float32)
    return x


def zero_plateaus(rows, cols, seed):
    """Rayleigh with exact-zero blocks and a few targets, like the maps the trackers see after masking."""
    x = rayleigh(rows, cols, seed)
    x[rows // 4: rows // 2, : cols // 3] = 0
    x[:, cols - cols // 5:] = 0
    x[rows // 3, cols // 2] = 30.0
    return x


def signed(rows, cols, seed):
    return np.random.default_rng(seed).standard_normal((rows, cols)).astype(np.float32)


def cfar_cells(gpu, want):
    """(rel-inf, worst per-cell relative error); a cell the oracle gives as 0 must be 0."""
    z = want == 0
    assert np.all(gpu[z] == 0)
    nz = ~z
    cell = float(np.max(np.abs(gpu[nz] - want[nz]) / np.abs(want[nz]))) if nz.any() else 0.0
    return rel(gpu, want, np.abs(want).max()), cell


# ------------------------------------------------------------------ CPU: the kernel's summation order
def _acc_dtype():
    """The accumulator cfar_frames_kernel declares for its window sums."""
    src = open(DETECT).read()
    kern = src[src.index("cfar_frames_kernel("):src.index("// ---- launches")]
    acc = re.search(r"\b(float|double) acc = ", kern).group(1)
    racc = re.search(r"\b(float|double) racc = ", kern).group(1)
    assert acc == racc
    return np.float64 if acc == "double" else np.float32


def cfar_model(X, fw, gw, acc):
    """cfar_frames_kernel in NumPy: X read as float32; for a = 0 .. fw-1 the row a of the window is summed over b = 0 .. fw-1
    (the guard hole skipped) into racc, and racc into acc, both of type ``acc``; the cell is X[(i + c - a) mod rows,
    (j + c - b) mod cols] with c = (fw - 1) // 2; CR = X * (1 / mean|X|) / (acc * scale + 1e-10) in ``acc``."""
    X = np.asarray(X, dtype=np.float32)
    rows, cols = X.shape
    hole = np.zeros(fw, dtype=bool)
    e1 = (fw - gw) // 2
    hole[e1:fw - e1 + 1] = True                       # the reference's slice Tfilt[e1:e2, e1:e2]
    c = (fw - 1) // 2
    one = acc(1)
    total = np.zeros(X.shape, dtype=acc)
    for a in range(fw):
        xa = np.roll(X, a - c, axis=0).astype(acc)
        racc = np.zeros_like(xa)
        for b in range(fw):
            if hole[a] and hole[b]:
                continue
            racc = racc + np.roll(xa, b - c, axis=1)
        total = total + racc
    inv_mean = acc(float(rows) * cols / np.abs(X).astype(np.float64).sum())
    scale = acc(one / acc(float(fw) * fw - float(gw) * gw))
    return ((X.astype(acc) * inv_mean) / (total * scale + acc(1e-10))).astype(np.float32)


def test_cfar_frames_kernel_summation_model_matches_float64_oracle():
    acc = _acc_dtype()
    cases = [("rayleigh_256x301", rayleigh(256, 301, 1), 18, 4), ("rayleigh_256x301", rayleigh(256, 301, 1), 64, 10),
             ("ridge_256x301", clutter_ridge(256, 301, 2), 18, 4), ("ridge_256x301", clutter_ridge(256, 301, 2), 64, 3),
             ("rayleigh_9x33", rayleigh(9, 33, 3), 18, 4),            # halo wraps several times
             ("signed_64x101", signed(64, 101, 4), 18, 4)]
    for name, X, fw, gw in cases:
        got = cfar_model(X, fw, gw, acc)
        want = FO.cfar_2d_oracle(X, fw, gw)
        e, cell = cfar_cells(got, want)
        assert e <= TOL and cell <= CELL_TOL, f"{name} fw={fw} gw={gw}: rel-inf {e:.2e}, per cell {cell:.2e} ({acc.__name__})"


# ------------------------------------------------------------------ CFAR_2D on the GPU
def _cfar_gw_grid(fw):
    return sorted({g for g in (0, 1, fw // 2, fw - 2, fw - 1, fw + 1, fw + 2) if g >= 0 and g != fw})


@pytest.mark.gpu
def test_cfar_fw_gw_grid_matches_oracle():
    X = rayleigh(40, 33, 10)
    worst_e = worst_cell = 0.0
    n = 0
    for fw in range(1, 65):
        for gw in _cfar_gw_grid(fw):
            e, cell = cfar_cells(prb.CFAR_2D(X, fw, gw), FO.cfar_2d_oracle(X, fw, gw))
            assert e <= TOL and cell <= CELL_TOL, (fw, gw, e, cell)
            worst_e, worst_cell, n = max(worst_e, e), max(worst_cell, cell), n + 1
        with pytest.raises(_lib.PrcoreError, match="must not be 0"):
            prb.CFAR_2D(X, fw, fw)                     # fw^2 = gw^2: the reference divides by zero
    record_parity("rows/cfar_fw_gw_grid_40x33", cases=n, E_vs_oracle=worst_e, worst_cell=worst_cell)


@pytest.mark.gpu
@pytest.mark.parametrize("fw,gw", [(18, 4), (64, 10)])
def test_cfar_map_sizes_match_oracle(fw, gw):
    worst = {}
    for rows, cols in [(1, 1), (3, 70), (7, 31), (9, 33), (256, 301), (1024, 401), (2048, 301)]:
        X = rayleigh(rows, cols, rows + cols)
        e, cell = cfar_cells(prb.CFAR_2D(X, fw, gw), FO.cfar_2d_oracle(X, fw, gw))
        assert e <= TOL and cell <= CELL_TOL, (rows, cols, e, cell)
        worst[f"E_{rows}x{cols}"], worst[f"cell_{rows}x{cols}"] = e, cell
    record_parity(f"rows/cfar_sizes_fw{fw}_gw{gw}", **worst)


def _cfar_host(x, fw, gw, flags=0, thresh=None):
    """prc_cfar2d_f32 on a host map: CR (float32) or, with ``thresh``, detections."""
    lib = _lib.load()
    rows, cols = x.shape
    out = np.empty((rows, cols), dtype=np.float32 if thresh is None else np.uint8)
    t = None if thresh is None else C.byref(C.c_float(thresh))
    _lib.check(lib.prc_cfar2d_f32(x.ctypes.data, rows, cols, fw, gw, t, out.ctypes.data if thresh is None else None,
                                  None if thresh is None else out.ctypes.data, _lib.MEM_HOST, 0, None, flags))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fw,gw", [(18, 4), (64, 10), (5, 7)])
def test_cfar_map_contents_match_oracle(fw, gw):
    figures = {}
    maps = {"rayleigh": rayleigh(256, 301, 20), "ridge55dB": clutter_ridge(256, 301, 21),
            "zero_plateaus": zero_plateaus(256, 301, 22), "signed": signed(256, 301, 23), "signed_64x101": signed(64, 101, 4)}
    for name, X in maps.items():
        e, cell = cfar_cells(prb.CFAR_2D(X, fw, gw), FO.cfar_2d_oracle(X, fw, gw))
        assert e <= TOL and cell <= CELL_TOL, (name, e, cell)
        figures[f"E_{name}"], figures[f"cell_{name}"] = e, cell
    # float64 maps: the wrapper hands the kernel float32, the oracle keeps float64
    for name in ("rayleigh", "ridge55dB"):
        X64 = maps[name].astype(np.float64) * (1 + 1e-3 * np.random.default_rng(24).random(maps[name].shape))
        e, cell = cfar_cells(prb.CFAR_2D(X64, fw, gw), FO.cfar_2d_oracle(X64, fw, gw))
        assert e <= TOL and cell <= CELL_TOL, (name, "float64", e, cell)
        figures[f"E_{name}_f64"], figures[f"cell_{name}_f64"] = e, cell
    # complex maps: |x| formed on the device (PRC_FLAG_ABS_C64, what cfar_track uses)
    rng = np.random.default_rng(25)
    Z = (rng.standard_normal((256, 301)) + 1j * rng.standard_normal((256, 301))).astype(np.complex64)
    Z[128] *= 300
    e, cell = cfar_cells(_cfar_host(Z, fw, gw, _lib.FLAG_ABS_C64).astype(np.float64), FO.cfar_2d_oracle(np.abs(Z), fw, gw))
    assert e <= TOL and cell <= CELL_TOL, ("complex64", e, cell)
    figures["E_complex64_abs"], figures["cell_complex64_abs"] = e, cell
    record_parity(f"rows/cfar_contents_fw{fw}_gw{gw}", **figures)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ridge55dB", "signed"])
def test_cfar_thresholds_flip_only_at_the_threshold(kind):
    X = clutter_ridge(256, 301, 30) if kind == "ridge55dB" else signed(256, 301, 31)
    fw, gw = 18, 4
    cr = FO.cfar_2d_oracle(X, fw, gw)
    worst = 0
    for q in (0.5, 0.9, 0.99, 0.999, 0.9999):
        th = float(np.quantile(cr, q))
        det = prb.CFAR_2D(X, fw, gw, th)
        assert det.dtype == np.bool_
        flips = det != (cr > th)
        assert np.all(np.abs(cr[flips] - th) <= 1e-5 * abs(th)), (q, th, int(flips.sum()))
        worst = max(worst, int(flips.sum()))
    record_parity(f"rows/cfar_thresholds_{kind}", flips_at_threshold=worst)


@pytest.mark.gpu
def test_cfar_row_limit():
    import torch
    lib = _lib.load()
    # A library without the row check launches a grid it cannot run.  Ask first with fw = 0, which every version
    # rejects before any launch: only a library that checks the rows first names them.
    big = 65535 * 8 + 1
    x = torch.zeros(big, dtype=torch.float32, device="cuda")
    cr = torch.empty_like(x)
    st = lib.prc_cfar2d_f32(x.data_ptr(), big, 1, 0, 0, None, cr.data_ptr(), None, _lib.MEM_DEVICE, 0, None, 0)
    assert st == _lib.PRC_E_INVALID
    msg = lib.prc_last_error().decode()
    if "rows" not in msg:
        pytest.skip("this library has no CFAR row check: " + msg)
    limit = int(re.search(r"maximum of (\d+) rows", msg).group(1))
    assert limit == big - 1
    st = lib.prc_cfar2d_f32(x.data_ptr(), big, 1, 18, 4, None, cr.data_ptr(), None, _lib.MEM_DEVICE, 0, None, 0)
    assert st == _lib.PRC_E_INVALID and str(limit) in lib.prc_last_error().decode()
    X = rayleigh(limit, 2, 32)                 # the tallest map: gridDim.y = 65535
    e, cell = cfar_cells(prb.CFAR_2D(X, 18, 4), FO.cfar_2d_oracle(X, 18, 4))
    assert e <= TOL and cell <= CELL_TOL
    record_parity("rows/cfar_tallest_map", rows=limit, E_vs_oracle=e, worst_cell=cell)


# ------------------------------------------------------------------ resample
RATIO_SET = (1, 2, 3, 5, 7, 13, 119)
RATIOS = [(u, d) for u in RATIO_SET for d in RATIO_SET if u != d]
SAMPLE = np.random.default_rng(40)


def _sampled(n_out, k=200):
    """First and last 40 outputs (the line extension) and a seeded sample of the middle."""
    ends = set(range(min(40, n_out))) | set(range(max(0, n_out - 40), n_out))
    mid = SAMPLE.integers(0, n_out, size=min(k, n_out))
    return np.array(sorted(ends | set(mid.tolist())), dtype=np.int64)


def _resample_check(x, up, dn, ms=None):
    """(GPU-vs-truth, GPU-vs-SciPy, SciPy-vs-truth) of resample(x, up, dn), truth at ``ms`` (default: sampled)."""
    y = prb.resample(x, up, dn)
    want = FO.resample_oracle(x, up, dn)
    assert y.dtype == want.dtype and y.shape == want.shape, (x.dtype, up, dn, y.dtype, want.dtype, y.shape, want.shape)
    ms = _sampled(y.shape[0]) if ms is None else ms
    truth = FO.resample_truth(x, up, dn, ms)
    if not np.iscomplexobj(x):
        truth = truth.real
    den = np.abs(want).max()
    g_t, g_r, r_t = two_sided(y[ms], want[ms], truth, den)
    return g_t, g_r, r_t, rel(y, want, den)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["complex64", "complex128", "float64"])
def test_resample_ratio_grid(dtype):
    ref, _ = synth.make_frame(5000, "P1", 41)
    x = ref.astype(dtype) if dtype != "float64" else ref.real.astype(np.float64)
    worst = {"E_vs_truth": 0.0, "E_vs_scipy": 0.0, "scipy_vs_truth": 0.0}
    refused = []
    for up, dn in RATIOS:
        if _resample_smem(up, dn) > RS_SMEM_LIMIT:     # 1/119; test_resample_shared_memory_limit pins where that starts
            with pytest.raises(_lib.PrcoreError, match="bytes of shared memory"):
                prb.resample(x, up, dn)
            refused.append(f"{up}/{dn}")
            continue
        g_t, g_r, r_t, g_full = _resample_check(x, up, dn)
        assert g_t <= TOL, (up, dn, g_t)
        assert g_r <= TOL + 1.2 * r_t and g_full <= TOL, (up, dn, g_r, r_t, g_full)
        worst = {"E_vs_truth": max(worst["E_vs_truth"], g_t), "E_vs_scipy": max(worst["E_vs_scipy"], g_full),
                 "scipy_vs_truth": max(worst["scipy_vs_truth"], r_t)}
    assert refused == ["1/119"]
    record_parity(f"rows/resample_ratio_grid_{dtype}", ratios=len(RATIOS) - len(refused), **worst)


def _n_for(n_out, up, dn):
    """Shortest input with at least n_out outputs (at 3/2 only every other length is reachable: 255, 257, 512, 513)."""
    n = max(1, (n_out - 1) * dn // up)
    while (n * up + dn - 1) // dn < n_out:
        n += 1
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("up,dn", [(13, 119), (3, 2)])
def test_resample_cta_boundaries(up, dn):
    worst = 0.0
    lengths = set()
    for target in (255, 256, 257, 511, 512, 513):        # RS_THREADS = 256 outputs per CTA
        n = _n_for(target, up, dn)
        n_out = (n * up + dn - 1) // dn
        assert n_out - target <= 1
        lengths.add(n_out)
        ref, _ = synth.make_frame(n, "P1", 42)
        g_t, g_r, r_t, g_full = _resample_check(ref, up, dn, np.arange(n_out))
        assert g_t <= TOL and g_r <= TOL + 1.2 * r_t, (n_out, g_t, g_r, r_t)
        worst = max(worst, g_t)
    assert {255, 257, 512, 513} <= lengths
    record_parity(f"rows/resample_cta_boundaries_{up}_{dn}", n_out=" ".join(map(str, sorted(lengths))), E_vs_truth=worst)


@pytest.mark.gpu
@pytest.mark.parametrize("up,dn", [(13, 119), (3, 2), (119, 13), (1, 7)])
def test_resample_short_inputs(up, dn):
    ref, _ = synth.make_frame(27, "P1", 43)
    worst = 0.0
    for n in (1, 2, 3, 27):
        for x in (ref[:n], ref[:n].astype(np.complex128), ref[:n].real.astype(np.float64)):
            y = prb.resample(x, up, dn)
            with np.errstate(divide="ignore", invalid="ignore"):
                want = FO.resample_oracle(x, up, dn)
            assert y.dtype == want.dtype and y.shape == want.shape
            if n == 1:                                   # the line through one point has slope 0/0
                np.testing.assert_array_equal(np.isnan(y), np.isnan(want))
                assert np.isnan(want).all()
                continue
            ms = np.arange(y.shape[0])
            truth = FO.resample_truth(x, up, dn, ms)
            truth = truth if np.iscomplexobj(x) else truth.real
            den = np.abs(want).max()
            g_t, g_r, r_t = two_sided(y, want, truth, den)
            assert g_t <= TOL and g_r <= TOL + 1.2 * r_t, (n, x.dtype, g_t, g_r, r_t)
            worst = max(worst, g_t)
    record_parity(f"rows/resample_short_{up}_{dn}", E_vs_truth=worst)


RS_SMEM_LIMIT = 200 * 1024          # SMEM_LIMIT of csrc/prcore_host.h


def _resample_smem(up, dn):
    """Shared memory the resampler asks for (csrc/prcore_signal.cu: resample_geo, resample_table), reduced ratio."""
    g = math.gcd(up, dn)
    up, dn = up // g, dn // g
    half_len = 10 * max(up, dn)
    nh = 2 * half_len + 1
    n_pre_pad = dn - half_len % dn
    tpp = -(-(n_pre_pad + nh) // up) | 1
    span = (255 * dn) // up + 2 + tpp
    return ((up * tpp * 4 + 15) & ~15) + span * 8


@pytest.mark.gpu
@pytest.mark.parametrize("up", [1, 2])
def test_resample_shared_memory_limit(up):
    dn = next(d for d in range(up + 1, 1000) if math.gcd(up, d) == 1 and _resample_smem(up, d) > RS_SMEM_LIMIT)
    assert dn == {1: 90, 2: 173}[up]
    last = max(d for d in range(up + 1, dn) if math.gcd(up, d) == 1)
    ref, _ = synth.make_frame(40 * last, "P1", 44)
    g_t, g_r, r_t, g_full = _resample_check(ref, up, last)
    assert g_t <= TOL and g_r <= TOL + 1.2 * r_t, (last, g_t, g_r, r_t)
    with pytest.raises(_lib.PrcoreError, match=f"needs {_resample_smem(up, dn)} bytes of shared memory") as err:
        prb.resample(ref, up, dn)
    assert err.value.code == _lib.PRC_E_INVALID
    record_parity(f"rows/resample_smem_limit_up{up}", last_dn=last, first_rejected_dn=dn, E_vs_truth=g_t)


# ------------------------------------------------------------------ frequency_shift / frontend
N_BIG = 2 ** 25 + 12345


@pytest.mark.gpu
@pytest.mark.parametrize("po", [0.7, np.array([0.7])], ids=["MIX_C64", "MIX_C128"])
def test_frequency_shift_and_frontend_past_2_24_samples(po):
    fc, fs = 300e3, 2.4e6
    assert psu._mix_mode(fc, fs, po)[0] == (_lib.MIX_C64 if isinstance(po, float) else _lib.MIX_C128)
    iq = synth.raw_iq(N_BIG, "int8", 45)
    x = prb.deinterleave_IQ(iq)
    got = prb.frequency_shift(x, fc, fs, po)
    want = frequency_shift_oracle(x, fc, fs, po)
    assert got.dtype == want.dtype
    e_shift = rel(got, want, np.abs(want).max())
    assert e_shift <= TOL
    tail = rel(got[2 ** 24:], want[2 ** 24:], np.abs(want).max())
    del got
    del want
    y = prb.frontend(iq, fc, fs, po, 13, 119)
    ms = _sampled(y.shape[0], 4000)
    ms = np.unique(np.concatenate([ms, np.arange(2 ** 24 * 13 // 119 - 50, 2 ** 24 * 13 // 119 + 50)]))
    want_y = FO.frontend_oracle(iq, fc, fs, po, 13, 119)
    assert y.shape == want_y.shape
    e_front = rel(y[ms], want_y[ms], np.abs(want_y).max())
    assert e_front <= TOL
    record_parity(f"rows/shift_past_2_24_{'c64' if isinstance(po, float) else 'c128'}", n=N_BIG,
                  E_shift=e_shift, E_shift_past_2_24=tail, E_frontend_sampled=e_front)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["int8", "int16", "float32"])
@pytest.mark.parametrize("case", ["MIX_F64", "MIX_FS64", "MIX_C64", "MIX_C128"])
def test_frontend_mix_modes(kind, case):
    # a NumPy float64 fc is multiplied into a Python complex first (it subclasses float), so MIX_F64 needs a strong fc
    fc, fs, po = {"MIX_F64": (np.array(-4321.75), 250e3, 0.25), "MIX_FS64": (4321.75, np.float64(250e3), 0.25),
                  "MIX_C64": (4321.75, 250e3, 0.25), "MIX_C128": (4321.75, 250e3, np.array([0.25]))}[case]
    assert psu._mix_mode(fc, fs, po)[0] == getattr(_lib, case)
    iq = synth.raw_iq(300_001, kind, 46)
    worst = 0.0
    for up, dn in ((13, 119), (3, 2)):
        y = prb.frontend(iq, fc, fs, po, up, dn)
        want = FO.frontend_oracle(iq, fc, fs, po, up, dn)
        assert y.dtype == np.complex64 and y.shape == want.shape
        e = rel(y, want, np.abs(want).max())
        assert e <= TOL, (up, dn, e)
        worst = max(worst, e)
    record_parity(f"rows/frontend_{case}_{kind}", E_vs_oracle=worst)


# ------------------------------------------------------------------ direct_xambg
@pytest.mark.gpu
@pytest.mark.parametrize("n,R,F", [(300, 400, 8), (5000, 33, 1), (4097, 50, 7), (2 ** 16, 60, 32), (2 ** 18, 300, 8)])
def test_direct_xambg_shapes(n, R, F):
    ref, srv = synth.make_frame(n, "P1", 47)
    fs = 1e6
    out = prb.direct_xambg(ref, srv, R, F, fs)
    assert out.dtype == np.complex64 and out.shape == (F, R + 1, 1)
    want = FO.direct_xambg_oracle(ref, srv, R, F, fs)
    truth = FO.direct_xambg_truth(ref, srv, R, F, fs)
    if R >= n:                                     # lags n .. R see only the zero padding
        assert np.all(out[:, :R - n + 1] == 0) and np.all(want[:, :R - n + 1] == 0)
    den = np.abs(truth).max()
    g_t, g_r, r_t = two_sided(out, want, truth, den)
    record_parity(f"rows/direct_xambg_n{n}_R{R}_F{F}", E_vs_truth=g_t, E_vs_reference=g_r, reference_vs_truth=r_t)
    assert g_t <= TOL and g_r <= TOL + 1.2 * r_t, (g_t, g_r, r_t)


@pytest.mark.gpu
def test_direct_xambg_lag_limit():
    ref, srv = synth.make_frame(6000, "P0", 48)
    with pytest.raises(_lib.PrcoreError, match=r"maximum of \d+") as err:
        prb.direct_xambg(ref, srv, 5120, 1, 1e6)
    assert err.value.code == _lib.PRC_E_INVALID
    limit = int(re.search(r"maximum of (\d+)", str(err.value)).group(1))      # lags, R + 1
    assert limit <= 5120
    R = limit - 1
    out = prb.direct_xambg(ref, srv, R, 1, 1e6)
    want = FO.direct_xambg_oracle(ref, srv, R, 1, 1e6)
    truth = FO.direct_xambg_truth(ref, srv, R, 1, 1e6)
    g_t, g_r, r_t = two_sided(out, want, truth, np.abs(truth).max())
    record_parity("rows/direct_xambg_lag_limit", R=R, E_vs_truth=g_t, E_vs_reference=g_r, reference_vs_truth=r_t)
    assert g_t <= TOL and g_r <= TOL + 1.2 * r_t


# ------------------------------------------------------------------ device pointers, threads
@pytest.mark.gpu
def test_device_pointers_on_a_caller_stream_are_bit_identical():
    import torch
    lib = _lib.load()
    st = torch.cuda.Stream()
    sp = C.c_void_p(st.cuda_stream)
    flags = _lib.FLAG_ASYNC
    # frontend: int8 IQ, main.py's ratio and phase-offset array
    iq = synth.raw_iq(200_000, "int8", 49)
    fc, fs, po = 300e3, 2.4e6, np.array([0.7])
    host = prb.frontend(iq, fc, fs, po, 13, 119)
    mode, pov = psu._mix_mode(fc, fs, po)
    h = psu._resample_taps(13, 119, mode == _lib.MIX_C64)     # float32-rounded taps only for a complex64 chain
    d_iq = torch.from_numpy(iq).cuda()
    d_y = torch.empty(host.shape[0], dtype=torch.complex64, device="cuda")
    # CFAR: a real map and a complex map (|x| on the device)
    X = clutter_ridge(256, 301, 50)
    rng = np.random.default_rng(51)
    Z = (rng.standard_normal((64, 101)) + 1j * rng.standard_normal((64, 101))).astype(np.complex64)
    d_X, d_Z = torch.from_numpy(X).cuda(), torch.from_numpy(Z).cuda()
    d_cr, d_crz = torch.empty_like(d_X), torch.empty(Z.shape, dtype=torch.float32, device="cuda")
    d_det = torch.empty(X.shape, dtype=torch.uint8, device="cuda")
    th = C.c_float(3.0)
    # direct_xambg
    ref, srv = synth.make_frame(20_000, "P1", 52)
    d_ref, d_srv = torch.from_numpy(ref).cuda(), torch.from_numpy(srv).cuda()
    d_amb = torch.empty((16, 61), dtype=torch.complex64, device="cuda")
    torch.cuda.synchronize()
    _lib.check(lib.prc_frontend_c64(d_iq.data_ptr(), _lib.IQ_I8, iq.shape[0] // 2, mode, fc, fs, pov, 13, 119, h.ctypes.data,
                                    h.shape[0], d_y.data_ptr(), host.shape[0], _lib.MEM_DEVICE, 0, sp, flags))
    _lib.check(lib.prc_cfar2d_f32(d_X.data_ptr(), 256, 301, 18, 4, C.byref(th), d_cr.data_ptr(), d_det.data_ptr(),
                                  _lib.MEM_DEVICE, 0, sp, flags))
    _lib.check(lib.prc_cfar2d_f32(d_Z.data_ptr(), 64, 101, 9, 2, None, d_crz.data_ptr(), None, _lib.MEM_DEVICE, 0, sp,
                                  flags | _lib.FLAG_ABS_C64))
    _lib.check(lib.prc_direct_xambg_c64(d_ref.data_ptr(), d_srv.data_ptr(), 20_000, 60, 16, 1e6, d_amb.data_ptr(),
                                        _lib.MEM_DEVICE, 0, sp, flags))
    st.synchronize()
    np.testing.assert_array_equal(d_y.cpu().numpy(), host)
    np.testing.assert_array_equal(d_cr.cpu().numpy(), _cfar_host(X, 18, 4))
    np.testing.assert_array_equal(d_det.cpu().numpy(), _cfar_host(X, 18, 4, thresh=3.0))
    np.testing.assert_array_equal(d_crz.cpu().numpy(), _cfar_host(Z, 9, 2, _lib.FLAG_ABS_C64))
    np.testing.assert_array_equal(d_amb.cpu().numpy(), prb.direct_xambg(ref, srv, 60, 16, 1e6)[:, :, 0])


@pytest.mark.gpu
def test_concurrent_threads_are_bit_identical_to_serial_calls():
    """Each thread switches resample ratios, so the per-context polyphase table is re-keyed between its calls."""
    jobs = []
    for t in range(8):
        x, _ = synth.make_frame(30_000 + 997 * t, "P1", 60 + t)
        jobs.append((x, rayleigh(64 + 8 * t, 101, 70 + t) if t % 2 else signed(64, 101 + t, 70 + t)))

    def run(x, X):
        return [prb.resample(x, 13, 119), prb.CFAR_2D(X, 18, 4), prb.resample(x, 3, 2), prb.CFAR_2D(X, 9, 2)]
    serial = [run(*j) for j in jobs]
    results = [[None] * 3 for _ in jobs]

    def worker(i):
        for r in range(3):
            results[i][r] = run(*jobs[i])
    threads = [threading.Thread(target=worker, args=(i,)) for i in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for want, got in zip(serial, results):
        for rounds in got:
            for a, b in zip(want, rounds):
                np.testing.assert_array_equal(a, b)
