"""GAL_JPE (csrc/gal.cuh, launched from prcore_clutter.cu's gal_device) against the float64 recurrence across its five
kernel variants, its step-size regimes, three input scales and full 2^19-sample runs.

A Python twin of gal_device states which variant a delay line D runs on: one warp per frame with T = 1, 2, 4 or 8
taps per lane (D <= 32, 64, 128, 256), or one CTA of ceil(D / 256) warps per frame (T = 8) up to D = 4096.  CPU tests
pin the twin to the sources, hold oracle/gal_oracle.c's float64 truth to a NumPy statement of the recurrence, and
check that every GPU case sits where its name says (variant and mu1 regime) and that no case's mu1 clamp decision is
close enough to 5e-3 for float32 round-off to take it the other way.  GPU tests hold `out`, `k` and `h` to the truth,
`out` to the reference's complex64 arithmetic (the plain-C oracle), and batches and device pointers to single-frame
calls bit for bit.

mu1 regimes (DESIGN.md section 10): "decay" starts at 1e-3 and decays as 0.999^n; "above" starts at 1e-2, above the
clamp, so the first sample sets it to 5e-3; "held" adds a real offset to srv that keeps e**2 near the positive real
axis with |e|^2 >> 500, so the clamp wins on nearly every sample; and every run past ~1e4 samples ends with mu1 ~
1e-8 sum 0.999^j e_j**2, a complex number whose real part goes negative.  Scaling srv alone by 1e5 (or both channels by
3e4) with no such offset does not hold the clamp: e**2 has a random phase, mu1's real part reaches -1e1 .. -1e2 and
the recurrence diverges to NaN in float64 as in complex64.  The int16-like (x3e4) cases are therefore either
clamp-held or L = 1, where no lattice stage exists and mu1 feeds nothing.

Criteria: out within 1e-5 x max|srv| of the truth and within 1e-5 + 1.2 x (oracle vs truth) of the oracle; k and h
within 5e-5 x max|k_truth|, max|h_truth|.  Figures go to $PRC_PARITY_DIR/parity.json (conftest.record_parity)."""
import ctypes as C
import math
import os
import re
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import passiveradar_b200 as prb
import test_gal_jpe as tg
from conftest import record_parity
from passiveradar_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "passiveradar_b200", "csrc")
TOL = tg.TOL                      # out vs truth, over max|srv|
KH_TOL = 5e-5                     # k and h vs truth, over max|k_truth| and max|h_truth|
MU2 = 1e-2
GAMMA, DELTA, CLAMP = 0.999, 1e-8, 5e-3


# ------------------------------------------------------------------ planner twin (prcore_clutter.cu: gal_device)
def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def gal_constants():
    src = _source("gal.cuh")
    c = {k: int(re.search(rf"constexpr int {k} = (\d+);", src).group(1))
         for k in ("GAL_MAX_D", "GAL_CTA_T", "GAL_WARP_FRAMES")}
    m = re.search(r"constexpr int GAL_WARP_MAX_D = 32 \* (\d+);", src)
    c["GAL_WARP_MAX_D"] = 32 * int(m.group(1))
    return c


GC = gal_constants()
WARP_T = (1, 2, 4, 8)             # gal_device: D <= 32 T runs gal_jpe_kernel<T, false>


def gal_variant(D):
    """(T taps per thread, CTA-per-frame?, warps per frame) of gal_device for a delay line of D taps."""
    if not 1 <= D <= GC["GAL_MAX_D"]:
        raise ValueError(D)
    if D <= GC["GAL_WARP_MAX_D"]:
        return next(t for t in WARP_T if D <= 32 * t), False, 1
    return GC["GAL_CTA_T"], True, -(-D // (32 * GC["GAL_CTA_T"]))


def variant_name(D):
    T, cta, warps = gal_variant(D)
    return f"CTA{warps}" if cta else f"T{T}"


# ------------------------------------------------------------------ cases
# (name, n, L, D, peek, mu1, scale, dc): ref = scale x P1 ref, srv = scale x P1 srv + dc.  The name starts with the
# variant (T<taps per lane> or CTA<warps>); "above", "held", "milli" (x1e-3) and "int16" (x3e4) name the regime and
# scale, everything else is unit power and mu1 = 1e-3.
EDGE_CASES = [
    ("T1_D1_L1", 3000, 1, 1, 10, 1e-3, 1.0, 0.0),
    ("T1_D31_L31_p0", 2500, 31, 31, 0, 1e-3, 1.0, 0.0),
    ("T1_D32_L11_above", 3000, 11, 32, 10, 1e-2, 1.0, 0.0),
    ("T2_D33_L33", 2000, 33, 33, 10, 1e-3, 1.0, 0.0),
    ("T2_D63_L1_p1000", 3000, 1, 63, 1000, 1e-3, 1.0, 0.0),
    ("T2_D64_L19_above", 2000, 19, 64, 10, 1e-2, 1.0, 0.0),
    ("T4_D65_L65_p0", 2000, 65, 65, 0, 1e-3, 1.0, 0.0),
    ("T4_D127_L1", 2000, 1, 127, 10, 1e-3, 1.0, 0.0),
    ("T4_D128_L35_milli", 2000, 35, 128, 10, 1e-3, 1e-3, 0.0),
    ("T8_D129_L129_p1000", 3000, 129, 129, 1000, 1e-3, 1.0, 0.0),
    ("T8_D255_L43_held", 3000, 43, 255, 10, 1e-3, 1.0, 300.0),
    ("T8_D256_L256", 2000, 256, 256, 10, 1e-3, 1.0, 0.0),
    ("CTA2_D257_L257", 2000, 257, 257, 10, 1e-3, 1.0, 0.0),
    ("CTA2_D511_L1_p0", 2000, 1, 511, 0, 1e-3, 1.0, 0.0),
    ("CTA2_D512_L256_above", 2000, 256, 512, 10, 1e-2, 1.0, 0.0),
    ("CTA3_D513_L513", 2000, 513, 513, 10, 1e-3, 1.0, 0.0),
    ("CTA4_D1000_L259_p1000", 3000, 259, 1000, 1000, 1e-3, 1.0, 0.0),
    ("CTA8_D2048_L2048", 1500, 2048, 2048, 10, 1e-3, 1.0, 0.0),
    ("CTA9_D2049_L257_held", 1500, 257, 2049, 10, 1e-3, 1.0, 300.0),
    ("CTA16_D4095_L4095", 1200, 4095, 4095, 10, 1e-3, 1.0, 0.0),
    ("CTA16_D4096_L1_int16", 1500, 1, 4096, 10, 1e-3, 3e4, 0.0),
]
# n - peek - 1 = 1, 31, 32, 33 sample steps: the kernel's 32-sample input chunks and their one-ahead prefetch
CHUNK_CASES = [(f"{v}_D{D}_L{L}_p{peek}_steps{s}", peek + 1 + s, L, D, peek, 1e-3, 1.0, 0.0)
               for v, L, D, peek in (("T1", 32, 32, 0), ("T8", 11, 256, 10), ("CTA16", 256, 4096, 1000))
               for s in (1, 31, 32, 33)]
MID_CASES = [
    ("T2_D64_L64_mid", 2 ** 15, 64, 64, 10, 1e-3, 1.0, 0.0),
    ("T4_D100_L1_int16_mid", 2 ** 15, 1, 100, 10, 1e-3, 3e4, 0.0),
    ("T8_D200_L27_held_mid", 2 ** 15, 27, 200, 10, 1e-3, 1.0, 300.0),
    ("CTA3_D600_L40_int16_held_mid", 2 ** 15, 40, 600, 10, 1e-3, 3e4, 3e5),
    ("CTA4_D1000_L100_above_mid", 2 ** 15, 100, 1000, 10, 1e-2, 1.0, 0.0),
    ("CTA9_D2049_L259_milli_mid", 2 ** 15, 259, 2049, 10, 1e-3, 1e-3, 0.0),
]
LONG_CASES = [
    ("T1_D32_L32_long", 2 ** 19, 32, 32, 10, 1e-3, 1.0, 0.0),
    ("T4_D128_L35_milli_long", 2 ** 19, 35, 128, 10, 1e-3, 1e-3, 0.0),
    ("T8_D256_L256_above_long", 2 ** 19, 256, 256, 10, 1e-2, 1.0, 0.0),
    ("CTA2_D512_L257_long", 2 ** 19, 257, 512, 10, 1e-3, 1.0, 0.0),
    ("CTA16_D4096_L64_long", 2 ** 19, 64, 4096, 10, 1e-3, 1.0, 0.0),
]
CASES = EDGE_CASES + CHUNK_CASES + MID_CASES + LONG_CASES
BY_NAME = {c[0]: c for c in CASES}
EDGE_DS = (1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1000, 2048, 2049, 4095, 4096)


def inputs(case):
    name, n, L, D, peek, mu1, scale, dc = case
    ref, srv = synth.make_frame(n, "P1", frame=zlib.crc32(name.encode()) % 1000)
    if scale != 1.0 or dc:
        ref = (ref * np.float32(scale)).astype(np.complex64)
        srv = (srv * np.float32(scale) + np.float32(dc)).astype(np.complex64)
    return ref, srv


_TRUTH = {}


def truth(case):
    """(out, k, h, stats) of oracle.gal_oracle.gal_jpe_truth_stats, computed once per case."""
    from oracle import gal_oracle as go
    if case[0] not in _TRUTH:
        _, n, L, D, peek, mu1, _, _ = case
        _TRUTH[case[0]] = go.gal_jpe_truth_stats(*inputs(case), L, D, mu1, MU2, peek)
    return _TRUTH[case[0]]


def truths(cases):
    """Truths of all ``cases``, computed side by side (the C recurrence runs without the GIL)."""
    from oracle import gal_oracle as go
    go.build()
    with ThreadPoolExecutor(max_workers=max(1, min(len(cases), os.cpu_count() or 1))) as ex:
        list(ex.map(truth, cases))
    return [_TRUTH[c[0]] for c in cases]


def flip_bound(case):
    """An upper bound on |xr_float32 - xr_float64| / 5e-3 for any clamp decision of the case, where xr = 0.999 Re(mu1)
    + 1e-8 Re(e**2) is what min() compares with 5e-3.  A decision whose margin |xr - 5e-3| / 5e-3 exceeds it is taken
    the same way by every float32 evaluation whose e is within TOL x max|srv| of the truth's.  Per step: the rounding
    of 0.999f x mu1 (2u |xr|max), of e**2 and 1e-8f x e**2 (5u 1e-8 |e|max^2), of the sum (u |xr|max), and the
    error of e (1e-8 (2 |e|max de + de^2)); the error carried in mu1 decays by 0.999 per step, so it adds up over at
    most 1000 steps (fewer in a shorter run).  u = 2^-24."""
    name, n, L, D, peek, mu1, scale, dc = case
    out, _, _, st = truth(case)
    srv = inputs(case)[1]
    u, E, de = 2.0 ** -24, float(np.abs(out).max()), TOL * float(np.abs(srv).max())
    X = max(st["xr_max"], mu1, CLAMP)
    step = 3 * u * X + 5 * u * DELTA * E * E + DELTA * (2 * E * de + de * de)
    return min(max(n - peek - 1, 0), 1000) * step / CLAMP


# ------------------------------------------------------------------ CPU: the twin
def test_twin_is_the_librarys_dispatch():
    """gal_device's thresholds and gal.cuh's constants are what the twin assumes."""
    assert GC == {"GAL_MAX_D": 4096, "GAL_CTA_T": 8, "GAL_WARP_FRAMES": 4, "GAL_WARP_MAX_D": 256}
    src = _source("prcore_clutter.cu")
    body = src[src.index("int gal_device("):]
    body = body[:body.index("\n}\n")]
    assert "if (D <= GAL_WARP_MAX_D) {" in body
    warp = re.findall(r"if \(D <= (\d+)\) gal_jpe_kernel<(\d+), false>", body)
    assert [(int(d), int(t)) for d, t in warp] == [(32 * t, t) for t in WARP_T[:-1]]
    assert re.search(r"else gal_jpe_kernel<(\d+), false>", body).group(1) == str(WARP_T[-1])
    assert 32 * WARP_T[-1] == GC["GAL_WARP_MAX_D"]
    assert "grid = ceil_div(bt.nf, GAL_WARP_FRAMES), threads = 32 * GAL_WARP_FRAMES" in body
    assert "threads = 32 * ceil_div(D, 32 * GAL_CTA_T)" in body
    assert "gal_jpe_kernel<GAL_CTA_T, true><<<bt.nf, threads, gal_smem(threads)" in body
    assert "GAL_MAX_WARPS = GAL_MAX_D / (32 * GAL_CTA_T)" in _source("gal.cuh")
    assert gal_variant(4096) == (8, True, GC["GAL_MAX_D"] // (32 * GC["GAL_CTA_T"]))
    with pytest.raises(ValueError):
        gal_variant(4097)


def test_named_cases_sit_where_their_names_say():
    for name, n, L, D, peek, mu1, scale, dc in CASES:
        assert name.split("_")[0] == variant_name(D), name
        assert f"_D{D}_" in name and f"_L{L}" in name, name
        assert ("above" in name) == (mu1 > CLAMP), name
        assert ("held" in name) == (dc != 0), name
        assert ("milli" in name) == (scale == 1e-3) and ("int16" in name) == (scale == 3e4), name
        assert 1 <= L <= D, name
    assert len(BY_NAME) == len(CASES)
    reached = {variant_name(c[3]) for c in CASES}
    assert {"T1", "T2", "T4", "T8"} <= reached
    assert {int(v[3:]) for v in reached if v.startswith("CTA")} >= {2, 3, 4, 8, 9, 16}
    assert set(EDGE_DS) <= {c[3] for c in CASES}
    # every variant at each of its D edges, and both sides of every edge between variants
    for lo, hi in ((32, 33), (64, 65), (128, 129), (256, 257), (512, 513), (2048, 2049)):
        assert gal_variant(lo) != gal_variant(hi)
    # L against D: L = 1, L = D and L = 8k + 3 in the warp variants; L = 256, 257 and L = 8k + 3 in the CTA variant
    for cta in (False, True):
        Ls = [(c[2], c[3]) for c in CASES if gal_variant(c[3])[1] == cta]
        assert any(L == 1 for L, _ in Ls) and any(L == D for L, D in Ls) and any(L % 8 == 3 for L, _ in Ls)
    assert {256, 257} <= {c[2] for c in CASES if gal_variant(c[3])[1]}
    assert {0, 10, 1000} <= {c[4] for c in CASES}
    assert {c[1] - c[4] - 1 for c in CHUNK_CASES} == {1, 31, 32, 33}
    longs = {variant_name(c[3]) for c in LONG_CASES if c[1] == 2 ** 19}
    assert {"T1", "T4", "T8", "CTA2", "CTA16"} <= longs


# ------------------------------------------------------------------ CPU: the truth against a NumPy statement
def gal_numpy(ref, srv, L, D, mu1, mu2, peek):
    """DESIGN.md section 10's recurrence in plain float64 NumPy, one sample at a time: mu1 is the caller's Python float
    until the first update and a complex number afterwards, min() against 5e-3 compares real parts, then imaginary
    parts, and mu1 is the Python float 5e-3 again whenever the clamp wins.  Returns (out, k, h, clamps, margin)."""
    ref = np.asarray(ref, np.complex128)
    srv = np.asarray(srv, np.complex128)
    n = ref.shape[0]
    b = np.zeros(D, np.complex128)
    k = np.zeros(D, np.complex128)
    h = np.zeros(D, np.complex128)
    P = np.full(D, 1e-8)
    out = np.zeros(n, np.complex128)
    mu = float(mu1)
    clamps, margin = 0, math.inf
    for t in range(n - peek - 1):
        bo = b.copy()
        f = np.empty(L, np.complex128)
        f[0] = ref[t + peek]
        b = np.empty(D, np.complex128)
        b[0] = ref[t + peek]
        for m in range(1, L):
            f[m] = f[m - 1] - np.conj(k[m]) * bo[m - 1]
            b[m] = bo[m - 1] - k[m] * f[m - 1]
        for m in range(1, L):
            Em = abs(f[m - 1]) ** 2 + abs(bo[m - 1]) ** 2
            P[m - 1] = 0.9 * P[m - 1] + (1 - 0.9 ** 2) * Em
            grad = np.conj(f[m - 1]) * b[m] + bo[m - 1] * np.conj(f[m])
            k[m] += mu * grad / (P[m - 1] + 1e-10)
        b[L:] = bo[L - 1:D - 1]
        e = srv[t] - np.vdot(h, b)
        h += mu2 * np.conj(e) * b / (np.vdot(b, b).real + 1e-10)
        out[t] = e
        x = GAMMA * mu + DELTA * e ** 2
        margin = min(margin, abs(x.real - CLAMP) / CLAMP)
        if x.real > CLAMP or (x.real == CLAMP and x.imag > 0):
            mu, clamps = CLAMP, clamps + 1
        else:
            mu = complex(x)
    return out, k, h, clamps, margin


@pytest.mark.parametrize("n,L,D,peek,mu1,dc", [(400, 1, 8, 10, 1e-3, 0.0), (300, 6, 6, 0, 1e-2, 0.0),
                                               (400, 5, 12, 10, 1e-2, 0.0), (350, 3, 20, 0, 1e-3, 0.0),
                                               (300, 4, 10, 10, 1e-3, 300.0), (12, 2, 4, 10, 1e-3, 0.0),
                                               (11, 2, 4, 10, 1e-3, 0.0)])
def test_c_truth_is_the_numpy_recurrence(n, L, D, peek, mu1, dc):
    """gal_jpe_truth_c (and gal_jpe_truth_stats, the same C code) agree with an independent float64 statement to 1e-12
    on L = 1, L = D and L < D, peek 0 and 10, mu1 below and above the clamp, the clamp held, and runs of one and of
    no sample step."""
    from oracle import gal_oracle as go
    ref, srv = synth.make_frame(n, "P1", frame=n + L + D)
    srv = (srv + np.float32(dc)).astype(np.complex64)
    want, wk, wh, clamps, margin = gal_numpy(ref, srv, L, D, mu1, MU2, peek)
    out, k, h = go.gal_jpe_truth_c(ref, srv, L, D, mu1, MU2, peek)
    so, sk, sh, st = go.gal_jpe_truth_stats(ref, srv, L, D, mu1, MU2, peek)
    assert np.array_equal(so, out) and np.array_equal(sk, k) and np.array_equal(sh, h)
    den = float(np.abs(srv).max())
    assert tg._rel(out, want, den) <= 1e-12
    assert tg._rel(k, wk) <= 1e-12 and tg._rel(h, wh) <= 1e-12
    assert st["clamps"] == clamps
    assert st["margin"] == margin if math.isinf(margin) else abs(st["margin"] - margin) <= 1e-9 * max(margin, 1e-3)
    if L == 1:
        assert not k.any()
    if dc:
        assert clamps >= 0.95 * (n - peek - 1)


# ------------------------------------------------------------------ CPU: regimes and clamp margins of the GPU cases
def test_cases_reach_their_regimes():
    """From the truth: "decay" cases never clamp, "above" cases clamp on their first sample, "held" cases on at least
    99% of samples, every run past 1e4 samples without an offset ends in the 1e-8 e**2-dominated regime (mu1 far
    above 0.999^n mu1: 100 times or more), and at least one long run ends with mu1's real part negative."""
    stats = {c[0]: t[3] for c, t in zip(CASES, truths(CASES))}
    negative = 0
    for name, n, L, D, peek, mu1, scale, dc in CASES:
        st, steps = stats[name], max(n - peek - 1, 0)
        if "held" in name:
            assert st["clamps"] >= 0.99 * steps, (name, st)
        elif "above" in name:
            assert st["clamps"] >= 1, (name, st)
        elif "int16" not in name:
            assert st["clamps"] == 0, (name, st)
        if steps > 10_000 and not dc:
            assert abs(st["mu1"]) > 100 * GAMMA ** steps * mu1, (name, st)
            negative += st["mu1"].real < 0
    assert negative >= 1


def test_clamp_decisions_are_not_knife_edge():
    """Every case's smallest clamp margin |xr - 5e-3| / 5e-3 exceeds flip_bound(): no float32 evaluation within the
    out bound of the truth can take a clamp decision the other way.  L = 1 cases are exempt: with no lattice stage,
    mu1 feeds nothing (k stays zero)."""
    for case, (out, k, h, st) in zip(CASES, truths(CASES)):
        name, L = case[0], case[2]
        assert np.isfinite(out).all() and np.isfinite(k).all() and np.isfinite(h).all(), name
        if L == 1:
            assert not k.any(), name
            continue
        bound = flip_bound(case)
        assert st["margin"] > bound, (name, st["margin"], bound)


# ------------------------------------------------------------------ GPU: against the truth and the reference arithmetic
@pytest.mark.gpu
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_gal_matches_truth_and_oracle(name):
    from oracle import gal_oracle as go
    case = BY_NAME[name]
    _, n, L, D, peek, mu1, scale, dc = case
    ref, srv = inputs(case)
    got, gk, gh = prb.GAL_JPE(ref, srv, L, D, mu1, MU2, peek, return_filter=True)
    tout, tk, th, st = truth(case)
    want, wk, wh = go.gal_jpe_oracle_c(ref, srv, L, D, mu1, MU2, peek)
    den = float(np.abs(srv).max())
    e_truth, e_ref, e_rt = tg._rel(got, tout, den), tg._rel(got, want, den), tg._rel(want, tout, den)
    e_k, e_h = tg._rel(gk, tk), tg._rel(gh, th)
    record_parity(f"gal_sweep/{name}", variant=variant_name(D), out_vs_truth=e_truth, out_vs_reference=e_ref,
                  reference_vs_truth=e_rt, k_vs_truth=e_k, h_vs_truth=e_h, k_reference_vs_truth=tg._rel(wk, tk),
                  h_reference_vs_truth=tg._rel(wh, th), clamps=st["clamps"], clamp_margin=st["margin"])
    assert e_truth <= TOL, "out vs float64 truth"
    assert e_ref <= TOL + 1.2 * e_rt, "out vs reference arithmetic"
    assert e_k <= KH_TOL, "k vs float64 truth"
    assert e_h <= KH_TOL, "h vs float64 truth"
    assert not got[max(n - peek - 1, 0):].any()


# ------------------------------------------------------------------ GPU: bitwise invariants of every variant
BATCH_SHAPES = [(8, 20), (19, 50), (35, 100), (43, 200), (259, 700)]      # (L, D): T1, T2, T4, T8, CTA3


def _resident_bound(D):
    """More frames than the GPU can hold at once: past the SM count x the threads an SM holds (2048) per CTA."""
    import torch
    nsm = torch.cuda.get_device_properties(_lib.current_device()).multi_processor_count
    T, cta, warps = gal_variant(D)
    threads, per_cta = (32 * warps, 1) if cta else (32 * GC["GAL_WARP_FRAMES"], GC["GAL_WARP_FRAMES"])
    return nsm * (2048 // threads) * per_cta + per_cta + 1


def _strided_frames(nframes, n, stride, seed):
    """nframes distinct frames (phase-rotated, rescaled P1 frames) laid out `stride` samples apart, the gaps NaN."""
    rng = np.random.default_rng(seed)
    base = [synth.make_frame(n, "P1", frame=i) for i in range(6)]
    ref = np.full((nframes, stride), np.nan, np.complex64)
    srv = np.full((nframes, stride), np.nan, np.complex64)
    ph = np.exp(1j * rng.uniform(0, 2 * np.pi, nframes)).astype(np.complex64)
    sc = rng.uniform(0.5, 1.5, nframes).astype(np.float32)
    for i in range(nframes):
        r, s = base[i % 6]
        ref[i, :n], srv[i, :n] = r * ph[i], s * sc[i]
    return ref, srv


@pytest.mark.gpu
@pytest.mark.parametrize("L,D", BATCH_SHAPES)
def test_gal_batch_is_bit_identical_to_single_frames_in_every_variant(L, D):
    """Batches of 1, 3, 4, 5 frames and one of more frames than the GPU holds at once, frame_stride = n + 13 with NaN
    in the gaps: every row equals its single-frame call bit for bit, and the gaps of `out` are left alone."""
    n, stride, peek, mu1 = 60, 73, 5, 2e-3
    big = _resident_bound(D)
    ref, srv = _strided_frames(big, n, stride, seed=D)
    single = [prb.GAL_JPE(ref[i, :n], srv[i, :n], L, D, mu1, MU2, peek, True) for i in range(big)]
    for nf in (1, 3, 4, 5, big):
        out = np.full((nf, stride), 7 + 7j, np.complex64)
        k = np.empty((nf, D), np.complex64)
        h = np.empty((nf, D), np.complex64)
        _lib.check(tg._frames_call(ref, srv, n, nf, stride, L, D, mu1, MU2, peek, out, k, h, _lib.MEM_HOST))
        assert np.all(out[:, n:] == np.complex64(7 + 7j)), nf
        for i in range(nf):
            o1, k1, h1 = single[i]
            assert np.array_equal(out[i, :n], o1) and np.array_equal(k[i], k1) and np.array_equal(h[i], h1), (nf, i)
    assert variant_name(D) in ("T1", "T2", "T4", "T8", "CTA3")


@pytest.mark.gpu
@pytest.mark.parametrize("L,D", BATCH_SHAPES + [(256, 4096)])
def test_gal_device_pointers_on_a_caller_stream_match_the_host_path(L, D):
    """Five strided frames (NaN gaps) in device memory, on a caller stream, asynchronously: the same bits as the host
    path, and the device `out`'s gaps untouched."""
    import torch
    nframes, n, stride, peek, mu1 = 5, 3000, 3000 + 29, 10, 1e-3
    ref, srv = _strided_frames(nframes, n, stride, seed=D + 1)
    want, wk, wh = prb.gal_jpe_frames(ref[:, :n], srv[:, :n], L, D, mu1, MU2, peek, True)
    dev = torch.device("cuda", _lib.current_device())
    s = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(s):
        dref = torch.from_numpy(ref.view(np.float32)).to(dev)
        dsrv = torch.from_numpy(srv.view(np.float32)).to(dev)
        dout = torch.full((nframes, 2 * stride), 7.0, dtype=torch.float32, device=dev)
        dk = torch.empty((nframes, 2 * D), dtype=torch.float32, device=dev)
        dh = torch.empty_like(dk)
    s.synchronize()
    _lib.check(tg._frames_call(dref, dsrv, n, nframes, stride, L, D, mu1, MU2, peek, dout, dk, dh, _lib.MEM_DEVICE,
                               C.c_void_p(s.cuda_stream), _lib.FLAG_ASYNC))
    s.synchronize()
    got = dout.cpu().numpy().view(np.complex64)
    assert np.all(got[:, n:] == np.complex64(7 + 7j))
    assert np.array_equal(got[:, :n], want)
    assert np.array_equal(dk.cpu().numpy().view(np.complex64), wk)
    assert np.array_equal(dh.cpu().numpy().view(np.complex64), wh)
