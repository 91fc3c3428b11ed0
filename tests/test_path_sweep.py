"""Sweeps of the FFT-domain hot path (csrc/fftcorr.cuh: lscorr_fft_kernel, levinson_kernel, taps_spectrum_kernel,
fir_fft_kernel, caf_fft_kernel<R3, FUSED>) across the edges of the three host planners that choose it (prcore_corr.cu:
ls_fft_plan, caf_fft_plan with and without the fused clutter filter, fir_fft's segment count), against float64 truths.

A Python twin of the planners states, for every case, which transform length and which segments the library uses; the
sweep is generated from it, and a GPU test pins the twin to the library through the batched entry points, which only
the FFT-domain path can serve.  Criteria (SURVEY.md 8d), TOL = 1e-5 rel-inf: cleaned channels over max|srv|, taps over
max|taps|, maps over max|map|.  P1 (strong clutter) maps of the fused frame are held to 1e-5 + 1.2 x the reference's
own complex64 error (DESIGN.md section 6).  Figures go to $PRC_PARITY_DIR/parity.json (conftest.record_parity)."""
import math
from dataclasses import dataclass
from functools import lru_cache

import numpy as np
import pytest
import scipy.signal as signal

import _golden as G
from conftest import record_parity
import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from oracle import clutter_oracle as co
from oracle import xambg_oracle as xo

TOL = 1e-5
FFT_MIN_N = 8192            # the library's default of the "fft_min_n" option


def rel(a, b, den):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / den)


# ------------------------------------------------------------------ planner twin (prcore_corr.cu)
@dataclass(frozen=True)
class LsPlan:
    """ls_fft_plan: on/off, R3, L = 256 R3, the segment bound L - M + 1, segment length Bs, segment count, length of
    the last segment."""
    on: bool
    r3: int = 0
    L: int = 0
    bmax: int = 0
    Bs: int = 0
    nseg: int = 0
    last: int = 0


def ls_plan(n, M, fft_min_n=FFT_MIN_N):
    if n < fft_min_n or not 1 <= M <= 2048:
        return LsPlan(False)
    r3 = 8 if M <= 1024 else 16
    L = 256 * r3
    if n < 2 * L:
        return LsPlan(False, r3, L)
    bmax = L - M + 1                 # lag M - 1 of a segment's last sample reaches L - 1
    nseg = -(-n // bmax)
    Bs = -(-n // nseg)
    nseg = -(-n // Bs)
    return LsPlan(True, r3, L, bmax, Bs, nseg, n - (nseg - 1) * Bs)


def ls_ctas(plan, nf, slots):
    """CTAs per frame of lscorr_fft_kernel: the batch is one wave of ``slots`` CTAs."""
    return max(1, min(plan.nseg, slots // nf))


def fir_nseg(n, M, r3):
    """Segments of fir_fft_kernel (overlap-save, L - M + 1 outputs each)."""
    return -(-n // (256 * r3 - M + 1))


@dataclass(frozen=True)
class CafPlan:
    """caf_fft_plan: on/off, R3, L, Bmax (products of a Doppler block per transform), segments per Doppler block."""
    on: bool
    r3: int = 0
    L: int = 0
    Bmax: int = 0
    nseg: int = 0


def caf_plan(n, R, F, mfuse=0, fft_min_n=FFT_MIN_N):
    """Boxcar decimator (shortFilt, no taps), ``mfuse`` taps of the clutter filter fused into the kernel (0: none)."""
    D = n // F if F >= 1 else 0
    if n < fft_min_n or D < 32 or F < 1:
        return CafPlan(False)
    ntaps = D + 1
    best = None
    for r3 in (4, 8, 16):
        L = 256 * r3
        bmax = L - R - max(mfuse - 1, 0)
        if bmax < L // 4 or n < L:
            continue
        nseg = -(-ntaps // bmax)
        cost = (nseg * (3 if mfuse else 2) + 1) * L * int(math.log2(L))
        if best is None or cost < best[0]:
            best = (cost, CafPlan(True, r3, L, bmax, nseg))
    return CafPlan(False) if best is None else best[1]


def frame_on(n, M, R, F, fft_min_n=FFT_MIN_N):
    """prc_frames_c64 runs the FFT-domain frame (LS plan and fused CAF plan both on); otherwise it runs the direct
    kernels frame by frame."""
    return ls_plan(n, M, fft_min_n).on and caf_plan(n, R, F, M, fft_min_n).on


@lru_cache(maxsize=None)
def one_sample_last(M):
    """Smallest n >= 2L whose last LS segment holds one sample (it needs Bs <= nseg, so n is about bmax^2)."""
    p = ls_plan(1 << 24, M, 0)
    n = np.arange(2 * p.L, (p.bmax + 2) ** 2, dtype=np.int64)
    nseg = -(-n // p.bmax)
    Bs = -(-n // nseg)
    nseg = -(-n // Bs)
    hit = np.flatnonzero(n - (nseg - 1) * Bs == 1)
    return int(n[hit[0]])


LS_M = (1, 2, 1023, 1024, 1025, 1026, 2047, 2048)


def ls_edges(M):
    """(edge, n) of the LS planner at M taps: one below the FFT path's minimum 2L, at it, and a one-sample last
    segment."""
    L = 2048 if M <= 1024 else 4096
    return [("n=2L-1", 2 * L - 1), ("n=2L", 2 * L), ("last_segment_1", one_sample_last(M))]


# (edge, n, R, F): fast_xambg on the planner's edges; D = n // F = 256 keeps one segment per Doppler block, so the
# cheapest eligible transform is the shortest and R = 3L/4 sits on the edge of the L it picks
XAMBG_CASES = [
    ("R=3L/4_L1024", 2 ** 17, 768, 512), ("R=3L/4+1_L1024", 2 ** 17, 769, 512),
    ("R=3L/4_L2048", 2 ** 17, 1536, 512), ("R=3L/4+1_L2048", 2 ** 17, 1537, 512),
    ("R=3L/4_L4096", 2 ** 17, 3072, 512), ("R=3L/4+1_L4096", 2 ** 17, 3073, 512),
    ("D=31", 31 * 1024, 100, 1024), ("D=32", 32 * 1024, 100, 1024),
    ("F=1_n=L-1", 1023, 100, 1), ("F=1_n=L", 1024, 100, 1),
    ("n_not_multiple_of_F", 2 ** 17 + 77, 300, 100),
]

# (edge, n, R, F, filter_len, peek): the fused frame (prc_frames_c64)
FRAME_CASES = [
    ("R+M-1=3072_R3=16", 2 ** 17, 1500, 256, 1563, 10),
    ("R+M-1=3073_direct", 2 ** 17, 1500, 256, 1564, 10),
    ("caf_R3=16_ls_R3=8", 2 ** 18, 1000, 64, 1000, 10),
    ("filterLen=0", 2 ** 17, 200, 128, 0, 10),
    ("peek=0", 2 ** 17, 300, 256, 64, 0),
]
# P1 frames where the reference's own complex64 chain is affordable on the host
FRAME_P1_CASES = [("P1_fused", 2 ** 15, 40, 64, 30, 10), ("P1_filterLen=0", 2 ** 15, 60, 32, 0, 12)]


# ------------------------------------------------------------------ CPU: the twin's invariants
def _all_ls_points():
    pts = [(n, M) for M in LS_M for _, n in ls_edges(M)]
    rng = np.random.default_rng(7)
    pts += [(int(rng.integers(4096, 1 << 23)), int(rng.integers(1, 2049))) for _ in range(400)]
    return pts


def test_ls_twin_segments_cover_the_channel():
    for n, M in _all_ls_points():
        p = ls_plan(n, M, 0)
        if not p.on:
            assert n < 2 * p.L
            continue
        assert p.Bs <= p.L - M + 1, (n, M, p)
        assert (p.nseg - 1) * p.Bs < n <= p.nseg * p.Bs, (n, M, p)
        assert 1 <= p.last <= p.Bs
        assert fir_nseg(n, M, p.r3) * (p.L - M + 1) >= n
        for nf, slots in ((1, 396), (199, 396), (403, 396)):
            assert 1 <= ls_ctas(p, nf, slots) <= p.nseg


def test_ls_twin_sits_on_its_edges():
    for M in LS_M:
        (_, below), (_, at), (_, last1) = ls_edges(M)
        assert not ls_plan(below, M, 0).on and ls_plan(at, M, 0).on
        p = ls_plan(last1, M, 0)
        assert p.on and p.last == 1 and p.r3 == (8 if M <= 1024 else 16)
    assert not ls_plan(10 ** 6, 2049, 0).on
    assert not ls_plan(FFT_MIN_N - 1, 10).on and ls_plan(FFT_MIN_N, 10).on


def test_caf_twin_bounds_and_edges():
    rng = np.random.default_rng(8)
    for _ in range(2000):
        n = int(rng.integers(1000, 1 << 22))
        F = int(rng.integers(1, 2048))
        R = int(rng.integers(0, 3200))
        mfuse = int(rng.choice([0, 1, int(rng.integers(1, 2049))]))
        p = caf_plan(n, R, F, mfuse, 0)
        if p.on:
            assert p.Bmax >= p.L // 4 and n >= p.L and n // F >= 32
            assert p.Bmax + R + max(mfuse - 1, 0) == p.L
            assert (p.nseg - 1) * p.Bmax < n // F + 1 <= p.nseg * p.Bmax
    for edge, n, R, F in XAMBG_CASES[:6]:
        L = int(edge.split("_L")[1])
        p = caf_plan(n, R, F, 0, 0)
        if "+1" in edge:
            assert p.L != L, (edge, p)
        else:
            assert p.on and p.L == L and p.Bmax == L // 4, (edge, p)
    assert not caf_plan(2 ** 17, 3073, 512, 0, 0).on
    assert not caf_plan(31 * 1024, 100, 1024, 0, 0).on and caf_plan(32 * 1024, 100, 1024, 0, 0).on
    assert not caf_plan(1023, 100, 1, 0, 0).on and caf_plan(1024, 100, 1, 0, 0).on
    on = {e: frame_on(n, fl + pk, R, F, 0) for e, n, R, F, fl, pk in FRAME_CASES}
    assert on == {"R+M-1=3072_R3=16": True, "R+M-1=3073_direct": False, "caf_R3=16_ls_R3=8": True,
                  "filterLen=0": True, "peek=0": True}
    assert caf_plan(2 ** 17, 1500, 256, 1573).r3 == 16 and caf_plan(2 ** 18, 1000, 64, 1010).r3 == 16
    assert ls_plan(2 ** 18, 1010).r3 == 8


# ------------------------------------------------------------------ CPU: the truths
@pytest.mark.parametrize("n,R,F,win,short", [
    (1000, 20, 10, False, True), (1003, 7, 9, True, True), (257, 300, 4, False, True),     # R > n
    (64, 5, 64, False, True),                                                               # D = 1
    (500, 10, 1, True, True),                                                               # F = 1
    (400, 6, 8, True, False), (999, 40, 7, False, False),                                   # flat-top decimator
])
def test_block_sums_fft_matches_loop_definition(n, R, F, win, short):
    ref, srv = synth.make_frame(n, "P1", 300 + n)
    w = signal.get_window(("kaiser", 5.0), n) if win else None
    want = xo.block_sums_truth(ref, srv, R, F, w, short)
    got = xo.block_sums_truth_fft(ref, srv, R, F, w, short, max_points=1 << 12)     # several groups of blocks
    assert rel(got, want, np.abs(want).max()) <= 1e-12


@pytest.mark.parametrize("name", G.TOEP_ALL)
def test_toeplitz_truth_is_within_the_reference_arithmetic(name):
    """The golden is the reference's own LS_Filter_Toeplitz (complex64 correlations, complex128 Levinson); the float64
    truth must sit within that arithmetic's error of it, which the reference-pinned oracle's distance measures."""
    g = G.load(name)
    ref, srv = G.inputs(g)
    fl, peek = int(g["filter_len"]), int(g["peek"])
    out, taps = co.ls_filter_toeplitz_truth(ref, srv, fl, peek)
    o_out, o_taps = co.ls_filter_toeplitz_oracle(ref, srv, fl, peek, True)
    den = float(g["srv_absmax"])
    e_taps, e_out = G.rel_inf(taps, g["taps"]), G.rel_inf(out[g["out_idx"]], g["out_sub"], den=den)
    own_taps, own_out = G.rel_inf(o_taps, taps), G.rel_inf(o_out, out, den=den)
    assert e_taps <= 1e-9 + 1.01 * own_taps and e_out <= 1e-9 + 1.01 * own_out, (e_taps, own_taps, e_out, own_out)
    assert own_taps <= 1e-4 and own_out <= 1e-5, (own_taps, own_out)


@pytest.mark.parametrize("name", G.MULTI_ALL)
def test_multiple_truth_is_within_the_reference_arithmetic(name):
    g = G.load(name)
    ref, srv = G.inputs(g)
    fl, fs, bins = int(g["filter_len"]), float(g["sample_rate"]), [float(b) for b in g["bins"]]
    out = co.ls_filter_multiple_truth(ref, srv, fl, fs, bins)
    own = co.ls_filter_multiple_oracle(ref, srv, fl, fs, bins)
    den = float(g["srv_absmax"])
    e_out, own_out = G.rel_inf(out[g["out_idx"]], g["out_sub"], den=den), G.rel_inf(own, out, den=den)
    assert e_out <= 1e-9 + 1.01 * own_out and own_out <= 1e-5, (e_out, own_out)


def test_frame_truth_is_ls_truth_then_map_truth():
    n, fl, peek, R, F = 5000, 20, 5, 30, 50
    ref, srv = synth.make_frame(n, "P1", 310)
    w = signal.get_window(("kaiser", 5.0), n)
    amb, taps, cleaned = xo.frame_truth(ref, srv, fl, 1.0, peek, R, F, w)
    t_clean, t_taps = co.ls_filter_truth(ref, srv, fl, 1.0, peek)
    assert np.array_equal(taps, t_taps) and np.array_equal(cleaned, t_clean)
    want = xo.fast_xambg_truth(ref.astype(np.complex128), t_clean, R, F, None, w)[:, :, 0]
    assert rel(amb, want, np.abs(want).max()) <= 1e-12


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture
def fft_options():
    """Restore the library's "fft" and "fft_min_n" options after a test that sets them."""
    old = (_lib.get_option("fft"), _lib.get_option("fft_min_n"))
    yield
    _lib.set_option("fft", old[0])
    _lib.set_option("fft_min_n", old[1])


def _set_fft(min_n):
    _lib.set_option("fft", 1)
    _lib.set_option("fft_min_n", min_n)


def _ls_multiple(ref, srv, fl, peek, fs, bins):
    """prc_ls_multiple_c64 with any peek (LS_Filter_Multiple passes the reference's 10)."""
    out = np.empty(ref.shape[0], np.complex64)
    taps = np.empty(fl + peek, np.complex64)
    b = np.ascontiguousarray(bins, dtype=np.float64)
    _lib.check(_lib.load().prc_ls_multiple_c64(ref.ctypes.data, srv.ctypes.data, ref.shape[0], fl, peek, fs, b.ctypes.data,
                                               b.shape[0], out.ctypes.data, taps.ctypes.data, _lib.MEM_HOST, 0, None, 0))
    return out, taps


def _noise_pair(n, nf, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((2, nf, n), dtype=np.float32) + 1j * rng.standard_normal((2, nf, n), dtype=np.float32))
    return x.astype(np.complex64)


def _pin_cases():
    """(edge, n, M split as (filter_len, peek), R, F) of every boundary case of the sweep."""
    cases = []
    for M in LS_M:
        for edge, n in ls_edges(M):
            cases.append((f"ls_M{M}_{edge}", n, M - min(M - 1, 10), min(M - 1, 10), 50, 64))
    for edge, n, R, F in XAMBG_CASES:
        cases.append((f"caf_{edge}", n, 1, 0, R, F))
    for edge, n, R, F, fl, peek in FRAME_CASES:
        cases.append((f"frame_{edge}", n, fl, peek, R, F))
    return cases


# ------------------------------------------------------------------ GPU: the twin is the library's planner
@pytest.mark.gpu
def test_planner_twin_matches_the_library(fft_options):
    """With two frames, prc_frames_c64 (host pointers, taps requested) and prc_ls_multiple_frames_c64 are accepted
    exactly when the twin's plans are on and refused with PRC_E_INVALID otherwise; prc_xambg_frames_c64 serves a batch
    in one CAF launch exactly when the twin's CAF plan is on (else it loops over the frames on the direct kernels)."""
    import torch
    lib = _lib.load()
    checked = 0
    pairs = {}
    for min_n in (0, FFT_MIN_N):
        _set_fft(min_n)
        for edge, n, fl, peek, R, F in _pin_cases():
            M = fl + peek
            if n not in pairs:
                pairs[n] = _noise_pair(n, 2, n)
            ref, srv = pairs[n][0], pairs[n][1]
            maps = np.empty((2, F, R + 1), np.complex64)
            taps = np.empty((2, M), np.complex64)
            st = lib.prc_frames_c64(ref.ctypes.data, srv.ctypes.data, n, 2, n, fl, peek, 1.0, R, F, None, maps.ctypes.data,
                                    taps.ctypes.data, None, _lib.MEM_HOST, 0, None, 0)
            want = frame_on(n, M, R, F, min_n)
            assert st == (_lib.PRC_OK if want else _lib.PRC_E_INVALID), (edge, min_n, st, lib.prc_last_error())
            d_ref, d_srv = torch.from_numpy(ref).cuda(), torch.from_numpy(srv).cuda()
            d_out = torch.empty_like(d_srv)
            st = lib.prc_ls_multiple_frames_c64(d_ref.data_ptr(), d_srv.data_ptr(), n, 2, n, fl, peek, 1.0, None, 1,
                                                d_out.data_ptr(), _lib.MEM_DEVICE, 0, None, 0)
            want = ls_plan(n, M, min_n).on
            assert st == (_lib.PRC_OK if want else _lib.PRC_E_INVALID), (edge, min_n, st, lib.prc_last_error())
            _lib.profile_reset()
            _lib.profile(True)
            try:
                _lib.check(lib.prc_xambg_frames_c64(ref.ctypes.data, srv.ctypes.data, n, 2, n, R, F, None, maps.ctypes.data,
                                                    _lib.MEM_HOST, 0, None, 0))
                launches = _lib.profile_read()["lagcorr_caf"][1]
            finally:
                _lib.profile(False)
                _lib.profile_reset()
            assert launches == (1 if caf_plan(n, R, F, 0, min_n).on else 2), (edge, min_n, launches)
            checked += 1
            del d_ref, d_srv, d_out
    record_parity("path/planner_twin", cases=checked)


# ------------------------------------------------------------------ GPU: LS_Filter across the LS planner's edges
def _ls_check(ref, srv, fl, reg, peek, truth):
    out, taps = prb.LS_Filter(ref, srv, fl, reg, peek, True)
    t_out, t_taps = truth
    return rel(taps, t_taps, np.abs(t_taps).max()), rel(out, t_out, np.abs(srv).max())


@pytest.mark.gpu
@pytest.mark.parametrize("M", LS_M)
def test_ls_filter_at_the_planner_edges(M, fft_options):
    worst = {}

    def note(key, e_taps, e_out, what):
        assert e_taps <= TOL and e_out <= TOL, (what, e_taps, e_out)
        worst[key] = max(worst.get(key, 0.0), e_taps, e_out)

    peek0 = min(M - 1, 10)
    for edge, n in ls_edges(M):
        ref, srv = synth.make_frame(n, "P1", 400 + M)
        truth = co.ls_filter_truth(ref, srv, M - peek0, 1.0, peek0)
        for min_n in (0, FFT_MIN_N):                 # FFT-forced and the default switch-over
            _set_fft(min_n)
            e_taps, e_out = _ls_check(ref, srv, M - peek0, 1.0, peek0, truth)
            note(f"E_{edge}", e_taps, e_out, (edge, n, min_n, ls_plan(n, M, min_n)))
    n = 2 * (2048 if M <= 1024 else 4096)
    _set_fft(0)
    ref, srv = synth.make_frame(n, "P1", 500 + M)
    for peek in sorted({0, 1, M - 1, M}):
        truth = co.ls_filter_truth(ref, srv, M - peek, 1.0, peek)
        note("E_peek", *_ls_check(ref, srv, M - peek, 1.0, peek, truth), ("peek", peek))
    p0 = synth.make_frame(n, "P0", 600 + M)
    for (r, s), reg in ((p0, 0.0), ((ref, srv), 1.0), ((ref, srv), 1e3)):
        truth = co.ls_filter_truth(r, s, M - peek0, reg, peek0)
        note("E_reg", *_ls_check(r, s, M - peek0, reg, peek0, truth), ("reg", reg))
    record_parity(f"path/ls_M{M}", n_last_segment_1=ls_edges(M)[2][1], **worst)


@pytest.mark.gpu
def test_ls_taps_above_2048_are_refused_with_the_limit(fft_options):
    ref, srv = synth.make_frame(2 ** 14, "P0", 700)
    for min_n in (0, FFT_MIN_N):
        _set_fft(min_n)
        with pytest.raises(_lib.PrcoreError, match="maximum of 2048") as err:
            prb.LS_Filter(ref, srv, 2039, 1.0, 10)
        assert err.value.code == _lib.PRC_E_INVALID
        with pytest.raises(_lib.PrcoreError, match="maximum of 2048"):
            prb.LS_Filter_Toeplitz(ref, srv, 2039, 10)


# ------------------------------------------------------------------ GPU: LS_Filter_Toeplitz / LS_Filter_Multiple
@pytest.mark.gpu
@pytest.mark.parametrize("M", LS_M)
def test_toeplitz_and_multiple_at_the_planner_edges(M, fft_options):
    fs = synth.P1_SAMPLE_RATE
    bins = (0.0, 2.0)
    peek = min(M - 1, 10)
    worst = {}
    for edge, n in ls_edges(M):
        ref, srv = synth.make_frame(n, "P1", 800 + M)
        t_out, t_taps = co.ls_filter_toeplitz_truth(ref, srv, M - peek, peek)
        m_out = co.ls_filter_multiple_truth(ref, srv, M - peek, fs, bins, peek)
        den = float(np.abs(srv).max())
        for min_n in (0, FFT_MIN_N):
            _set_fft(min_n)
            out, taps = prb.LS_Filter_Toeplitz(ref, srv, M - peek, peek, True)
            e_taps, e_out = rel(taps, t_taps, np.abs(t_taps).max()), rel(out, t_out, den)
            assert e_taps <= TOL and e_out <= TOL, ("toeplitz", edge, n, min_n, e_taps, e_out)
            got, _ = _ls_multiple(ref, srv, M - peek, peek, fs, bins)
            e_multi = rel(got, m_out, den)
            assert e_multi <= TOL, ("multiple", edge, n, min_n, e_multi)
            worst[f"E_toeplitz_{edge}"] = max(worst.get(f"E_toeplitz_{edge}", 0.0), e_taps, e_out)
            worst[f"E_multiple_{edge}"] = max(worst.get(f"E_multiple_{edge}", 0.0), e_multi)
    record_parity(f"path/toeplitz_multiple_M{M}", **worst)


# ------------------------------------------------------------------ GPU: fast_xambg across the CAF planner's edges
def _xambg(ref, srv, R, F, win):
    """(map [F, R+1], the float64 window the map used or None)."""
    n = ref.shape[0]
    if win == "none":
        return prb.fast_xambg(ref, srv, R, F)[:, :, 0], None
    w = signal.get_window(("kaiser", 5.0), n)
    if win == "f64":
        return prb.fast_xambg(ref, srv, R, F, n, w)[:, :, 0], w
    w32 = np.ascontiguousarray(w, dtype=np.float32)
    out = np.empty((F, R + 1), np.complex64)
    _lib.check(_lib.load().prc_xambg_frames_c64(ref.ctypes.data, srv.ctypes.data, n, 1, n, R, F, w32.ctypes.data,
                                                out.ctypes.data, _lib.MEM_HOST, 0, None, _lib.FLAG_WINDOW_F32))
    return out, w32.astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,R,F", XAMBG_CASES, ids=[c[0] for c in XAMBG_CASES])
def test_xambg_at_the_planner_edges(edge, n, R, F, both_paths):
    ref, srv = synth.make_frame(n, "P0", 900 + R + F)
    plan = caf_plan(n, R, F, 0, 0) if both_paths == "fft" else CafPlan(False)
    figures = {}
    for win in ("none", "f64", "f32"):
        got, w = _xambg(ref, srv, R, F, win)
        truth = xo.fast_xambg_truth(ref, srv, R, F, None, w, fast=True)[:, :, 0]
        e = rel(got, truth, np.abs(truth).max())
        assert e <= TOL, (edge, win, plan, e)
        figures[f"E_{win}"] = e
    record_parity(f"path/xambg_{edge}/{both_paths}", fft_r3=plan.r3 if plan.on else 0, **figures)


# ------------------------------------------------------------------ GPU: the fused frame
def _frames_device(refs, srvs, fl, peek, reg, R, F, w32):
    """prc_frames_c64 on device tensors ([nf, n] complex64), taps and cleaned channel requested, the float32 window
    (PRC_FLAG_WINDOW_F32) or a float64 one."""
    import torch
    nf, n = refs.shape
    maps = torch.empty((nf, F, R + 1), dtype=torch.complex64, device=refs.device)
    taps = torch.empty((nf, fl + peek), dtype=torch.complex64, device=refs.device)
    clean = torch.empty((nf, n), dtype=torch.complex64, device=refs.device)
    flags = _lib.FLAG_WINDOW_F32 if w32.dtype == torch.float32 else 0
    _lib.check(_lib.load().prc_frames_c64(refs.data_ptr(), srvs.data_ptr(), n, nf, n, fl, peek, reg, R, F, w32.data_ptr(),
                                          maps.data_ptr(), taps.data_ptr(), clean.data_ptr(), _lib.MEM_DEVICE, 0, None, flags))
    torch.cuda.synchronize()
    return maps, taps, clean


@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,R,F,fl,peek", FRAME_CASES, ids=[c[0] for c in FRAME_CASES])
def test_fused_frame_at_the_planner_edges(edge, n, R, F, fl, peek, fft_options):
    import torch
    _set_fft(FFT_MIN_N)
    M = fl + peek
    assert frame_on(n, M, R, F) == ("direct" not in edge)
    frames = [synth.make_frame(n, "P0", 1000 + i) for i in range(3)]
    w = signal.get_window(("kaiser", 5.0), n).astype(np.float32)
    refs = torch.from_numpy(np.stack([f[0] for f in frames])).cuda()
    srvs = torch.from_numpy(np.stack([f[1] for f in frames])).cuda()
    maps, taps, clean = _frames_device(refs, srvs, fl, peek, 1.0, R, F, torch.from_numpy(w).cuda())
    maps, taps, clean = maps.cpu().numpy(), taps.cpu().numpy(), clean.cpu().numpy()
    worst = {"E_map": 0.0, "E_taps": 0.0, "E_cleaned": 0.0}
    for i, (ref, srv) in enumerate(frames):
        amb, t_taps, t_clean = xo.frame_truth(ref, srv, fl, 1.0, peek, R, F, w.astype(np.float64))
        e = {"E_map": rel(maps[i], amb, np.abs(amb).max()), "E_taps": rel(taps[i], t_taps, np.abs(t_taps).max()),
             "E_cleaned": rel(clean[i], t_clean, np.abs(srv).max())}
        assert max(e.values()) <= TOL, (edge, i, e)
        worst = {k: max(worst[k], e[k]) for k in worst}
    p = caf_plan(n, R, F, M)
    record_parity(f"path/frame_{edge}", caf_r3=p.r3 if p.on else 0, ls_r3=ls_plan(n, M).r3, **worst)


@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,R,F,fl,peek", FRAME_P1_CASES, ids=[c[0] for c in FRAME_P1_CASES])
def test_fused_frame_with_strong_clutter(edge, n, R, F, fl, peek, fft_options):
    """P1: the map is what is left after the cancellation, so it is held to the truth at 1e-5 + 1.2 x the reference's
    own complex64 chain (LS_Filter -> fast_xambg) against the same truth."""
    import torch
    _set_fft(FFT_MIN_N)
    assert frame_on(n, fl + peek, R, F)
    frames = [synth.make_frame(n, "P1", 1100 + i) for i in range(2)]
    w = signal.get_window(("kaiser", 5.0), n)
    refs = torch.from_numpy(np.stack([f[0] for f in frames])).cuda()
    srvs = torch.from_numpy(np.stack([f[1] for f in frames])).cuda()
    maps, taps, clean = _frames_device(refs, srvs, fl, peek, 1.0, R, F, torch.from_numpy(w).cuda())
    maps, taps, clean = maps.cpu().numpy(), taps.cpu().numpy(), clean.cpu().numpy()
    fig = {"E_map": 0.0, "reference_map_vs_truth": 0.0, "E_taps": 0.0, "E_cleaned": 0.0}
    for i, (ref, srv) in enumerate(frames):
        amb, t_taps, t_clean = xo.frame_truth(ref, srv, fl, 1.0, peek, R, F, w)
        ref_map = xo.fast_xambg_oracle(ref, co.ls_filter_oracle(ref, srv, fl, 1.0, peek), R, F, n, w)[:, :, 0]
        den = np.abs(amb).max()
        e_map, r_map = rel(maps[i], amb, den), rel(ref_map, amb, den)
        e_taps, e_clean = rel(taps[i], t_taps, np.abs(t_taps).max()), rel(clean[i], t_clean, np.abs(srv).max())
        assert e_taps <= TOL and e_clean <= TOL and e_map <= TOL + 1.2 * r_map, (edge, i, e_taps, e_clean, e_map, r_map)
        fig = {"E_map": max(fig["E_map"], e_map), "reference_map_vs_truth": max(fig["reference_map_vs_truth"], r_map),
               "E_taps": max(fig["E_taps"], e_taps), "E_cleaned": max(fig["E_cleaned"], e_clean)}
    record_parity(f"path/frame_{edge}", **fig)


# ------------------------------------------------------------------ GPU: batch size
def _slots(M):
    """CTAs of one wave of lscorr_fft_kernel: the library's own figure at R3 = 8, the residency model of
    tests/test_fft_residency.py at R3 = 16 (one CTA per SM when the build's ptxas log is not in this tree)."""
    import os
    import torch
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    if M <= 1024:
        return _lib.get_option("fft_ctas_ls") * nsm
    import test_fft_residency as fr
    from passiveradar_b200 import build as b
    if not os.path.exists(os.path.join(b.PKG, "libprcore.ptxas.log")):
        return nsm
    return fr.expected_ctas(fr.fftc_entries(), "lscorr_fft_kernel", 16) * nsm


# (n, M, R, F, largest batch as a function of slots)
BATCH_CASES = [
    (2 ** 20, 310, 300, 256, lambda s: s + 7),
    (2 ** 21, 1024, 300, 256, lambda s: s // 2 + 1),      # 16 MB per channel: the largest batch stays under 10 GB
    (2 ** 19, 1500, 300, 256, lambda s: s + 7),           # R3 = 16
]
# largest batch-versus-single differences measured on an H100 80GB HBM3: taps 1.4e-6, cleaned 9.7e-7, P0 maps 9.1e-7
# (n = 2^21, M = 1024, one CTA per frame), P1 maps 2.5e-4 (the residual of the cancellation, DESIGN.md section 6)
BATCH_BOUND = {"taps": 3e-6, "cleaned": 3e-6, "map_P0": 3e-6, "map_P1": 5e-4}


@pytest.mark.gpu
@pytest.mark.parametrize("n,M,R,F,top", BATCH_CASES, ids=[f"n{c[0]}_M{c[1]}" for c in BATCH_CASES])
def test_frames_batch_sizes_hold_every_row_to_its_truth(n, M, R, F, top, fft_options):
    """Four distinct frames (two P0, two P1) repeated into batches up to one CTA per frame in lscorr_fft_kernel.  Every
    row's taps and cleaned channel are within TOL of the frame's truth, and so are P0 rows' maps (a P1 map is the
    residual of ~55 dB of cancellation: its batch-versus-single difference is bounded instead).  Rows are not
    bit-identical to single-frame calls: the segments a CTA accumulates depend on the batch size."""
    import torch
    _set_fft(FFT_MIN_N)
    peek = 10
    fl = M - peek
    slots = _slots(M)
    sizes = sorted({1, 2, 25, slots // 2 + 1, top(slots)})
    assert sizes[-1] * 3 * n * 8 < 12 * 2 ** 30
    profiles = ["P0", "P1", "P0", "P1"]
    base = [synth.make_frame(n, profiles[k], 1200 + k) for k in range(4)]
    w = signal.get_window(("kaiser", 5.0), n).astype(np.float32)
    dev = torch.device("cuda", 0)
    d_w = torch.from_numpy(w).to(dev)
    b_ref = torch.from_numpy(np.stack([f[0] for f in base])).to(dev)
    b_srv = torch.from_numpy(np.stack([f[1] for f in base])).to(dev)
    t_maps, t_taps, t_clean = [], [], []
    for k, (ref, srv) in enumerate(base):
        amb, tt, tc = xo.frame_truth(ref, srv, fl, 1.0, peek, R, F, w.astype(np.float64))
        t_maps.append(torch.from_numpy(amb).to(dev))
        t_taps.append(torch.from_numpy(tt).to(dev))
        t_clean.append(torch.from_numpy(tc).to(dev))
    den_srv = [float(np.abs(f[1]).max()) for f in base]
    single = [_frames_device(b_ref[k:k + 1], b_srv[k:k + 1], fl, peek, 1.0, R, F, d_w) for k in range(4)]

    def relt(a, b, den):
        return float((a.to(torch.complex128) - b.to(torch.complex128)).abs().max()) / den

    fig = {"slots": slots, "largest_batch": sizes[-1]}
    worst = {"E_taps": 0.0, "E_cleaned": 0.0, "E_map_P0": 0.0}
    diff = {key: 0.0 for key in BATCH_BOUND}
    for nf in sizes:
        idx = torch.arange(nf, device=dev) % 4
        maps, taps, clean = _frames_device(b_ref[idx], b_srv[idx], fl, peek, 1.0, R, F, d_w)
        for i in range(nf):
            k = i % 4
            e_taps = relt(taps[i], t_taps[k], float(t_taps[k].abs().max()))
            e_clean = relt(clean[i], t_clean[k], den_srv[k])
            assert e_taps <= TOL and e_clean <= TOL, (nf, i, e_taps, e_clean)
            worst["E_taps"], worst["E_cleaned"] = max(worst["E_taps"], e_taps), max(worst["E_cleaned"], e_clean)
            if profiles[k] == "P0":
                e_map = relt(maps[i], t_maps[k], float(t_maps[k].abs().max()))
                assert e_map <= TOL, (nf, i, e_map)
                worst["E_map_P0"] = max(worst["E_map_P0"], e_map)
            s_maps, s_taps, s_clean = single[k]
            diff["taps"] = max(diff["taps"], relt(taps[i], s_taps[0], float(s_taps[0].abs().max())))
            diff["cleaned"] = max(diff["cleaned"], relt(clean[i], s_clean[0], den_srv[k]))
            key = "map_" + profiles[k]
            diff[key] = max(diff[key], relt(maps[i], s_maps[0], float(s_maps[0].abs().max())))
        del maps, taps, clean, idx
        torch.cuda.empty_cache()
    record_parity(f"path/batch_n{n}_M{M}", **fig, **worst, **{f"batch_vs_single_{k}": v for k, v in diff.items()})
    for key, bound in BATCH_BOUND.items():
        assert diff[key] <= bound, (key, diff[key], bound)
