"""The channel-offset estimator and xcorr (csrc/chanoff.cuh) across their planner's edges.

A plain-Python twin of prcore_signal.cu's chanoff_device and of prc_channel_offset / prc_xcorr's argument handling gives, for
any call, the lag mapping, the transform size and its passes, the decimator's chunking, the argmax grid and the launches
the call makes.  On the CPU the twin is held to SciPy's 'valid' correlation and to oracle/offset_oracle.py, and a test
names, for every edge of the plan, a sweep case that reaches it.  On the GPU every sweep case runs against a float64 /
complex128 truth, and every call launches exactly what the twin plans."""
import math
import warnings
from dataclasses import dataclass

import numpy as np
import pytest
import scipy.signal as signal

from oracle import offset_oracle as oo

PADLEN = 27                 # sosfiltfilt's default padlen
MAX_ND = 64                 # prcore_signal.cu CHANOFF_MAX_ND
MAX_LOG2 = 26               # prcore_signal.cu CHANOFF_MAX_LOG2
TILE_BITS = 11              # chanoff.cuh FFT_TILE_BITS
TW_LO_BITS = 11
IIR_THREADS = 128
ARG_THREADS = 256
ARG_MAX_BLOCKS = 1024
XCORR_TOL = 1e-12           # xcorr against its complex128 truth, of max|truth| (test_channel_offset.py's bound)
XC_TOL = 1e-9               # |xc| of find_channel_offset against find_channel_offset_truth, of its max


# ------------------------------------------------------------------ the twin
class PlanError(ValueError):
    pass


@dataclass
class Pass:
    lo: int                 # index bits [lo, lo + nb) of the pass
    nb: int
    c: int                  # 2^c consecutive columns per tile
    s0: int                 # global stage of the pass's first stage
    tiles: int              # CTAs of the pass (per buffer)


@dataclass
class Iir:
    next: int               # n + 2 * PADLEN samples through each pass
    chunk: int              # samples per thread
    warm: int               # W
    grid: int               # CTAs of each IIR launch


@dataclass
class Plan:
    n1d: int
    n2d: int
    lenb: int
    nvalid: int
    p0: int                 # valid lag k reads the circular correlation at (k + p0) mod L
    need: int
    m: int
    passes: list
    nhi: int
    argmax_blocks: int
    iir: list               # [s1's, s2's] (find_channel_offset only)
    launches: int

    @property
    def L(self):
        return 1 << self.m

    @property
    def swapped(self):
        return self.n1d < self.lenb


def warmup(sos):
    """chanoff_warmup: W from the largest pole radius of the sections."""
    r = 0.0
    for s in np.asarray(sos, dtype=np.float64):
        a1, a2 = float(s[4]), float(s[5])
        disc = a1 * a1 - 4.0 * a2
        rs = math.sqrt(a2) if disc < 0.0 else max(abs(-a1 + math.sqrt(disc)), abs(-a1 - math.sqrt(disc))) / 2.0
        r = max(r, rs)
    return math.ceil(math.log(1e-18) / math.log(r)) + 256


def iir_plan(n, sos):
    nxt = n + 2 * PADLEN
    chunk = max(256, -(-nxt // 16384))
    return Iir(nxt, chunk, warmup(sos), -(-(-(-nxt // chunk)) // IIR_THREADS))


def fft_passes(m):
    """Top index bits first: 8 bits (x 8 consecutive columns) while more than 11 remain, then the rest."""
    out, top = [], m
    while top > 0:
        nb = top if top <= TILE_BITS else 8
        lo = top - nb
        c = min(3, lo)
        out.append(Pass(lo, nb, c, m - top, 1 << (m - nb - c)))
        top = lo
    return out


def argmax_blocks(nvalid):
    return min(max(-(-nvalid // (ARG_THREADS * 8)), 1), ARG_MAX_BLOCKS)


def device_plan(n1d, n2d, pad_l, pad_r):
    lenb = n2d + pad_l + pad_r
    nvalid = abs(n1d - lenb) + 1
    p0 = (0 if n1d >= lenb else n1d - lenb) + pad_l
    need = max(n1d, n2d, p0 + nvalid - 1 + n2d, n1d - p0, 2)
    m = 1
    while m <= MAX_LOG2 and (1 << m) < need:
        m += 1
    if m > MAX_LOG2:
        raise PlanError(f"the correlation needs a transform of {need} points; the maximum is 2^{MAX_LOG2}")
    return Plan(n1d, n2d, lenb, nvalid, p0, need, m, fft_passes(m), max(1, ((1 << m) // 2) >> TW_LO_BITS),
                argmax_blocks(nvalid), [], 0)


def _sos(nd, dt):
    return oo.decimate_sos(nd, dt)[0]


def offset_plan(n1, n2, nd, nl, dt1="int8", dt2="int8"):
    """prc_channel_offset: 4 IIR launches (forward and backward per channel), the twiddles, P forward passes (X and Y
    in one launch), P inverse passes, the per-block argmax and the final argmax."""
    if nd < 1 or nd > MAX_ND:
        raise PlanError(f"nd={nd} outside [1, {MAX_ND}]")
    if nl < 0:
        raise PlanError(f"nl={nl} invalid")
    if n1 <= PADLEN or n2 <= PADLEN:
        raise PlanError(f"The length of the input vector x must be greater than padlen, which is {PADLEN}.")
    p = device_plan(-(-n1 // nd), -(-n2 // nd), nl, nl)
    p.iir = [iir_plan(n1, _sos(nd, dt1)), iir_plan(n2, _sos(nd, dt2))]
    p.launches = 4 + 1 + 2 * len(p.passes) + 2
    return p


def xcorr_plan(n1, n2, nlead, nlag):
    """prc_xcorr: one load check (two kernels), the twiddles, 2P passes and the argmax kernel writing the lags."""
    if n1 < 1 or n2 < 1 or nlead < 0 or nlag < 0:
        raise PlanError("invalid xcorr arguments")
    p = device_plan(n1, n2, nlag, nlead)
    p.launches = 1 + 1 + 2 * len(p.passes) + 1
    return p


def twiddle_exponents(m, p):
    """Every twiddle exponent chanoff_fft_kernel<false> forms in pass p, and the two rows of each butterfly, as the
    kernel computes them (thread-strided loops flattened)."""
    S = 1 << (p.nb + p.c)
    ucols = 1 << p.c
    tshift = p.lo - p.c
    tile = np.arange(p.tiles, dtype=np.int64)[:, None]
    hi = tile >> tshift
    u0 = (tile & ((1 << tshift) - 1)) << p.c
    b = np.arange(S >> 1, dtype=np.int64)[None, :]
    u, bt = b & (ucols - 1), b >> p.c
    out = []
    for r in range(p.nb):
        half = 1 << (p.nb - 1 - r)
        tt = (bt // half) * 2 * half + bt % half

        def gidx(e):
            return (hi << (p.lo + p.nb)) | ((e >> p.c) << p.lo) | (u0 + (e & (ucols - 1)))
        e1, e2 = (tt << p.c) | u, ((tt + half) << p.c) | u
        ex = (((tt % half) << p.lo) | (u0 + u)) << (p.s0 + r)
        out.append((p.s0 + r, ex, gidx(e1), gidx(e2)))
    return out


def max_twiddle_exponent(p):
    """The largest exponent of pass p: (i mod h) at h - 1 and every column bit set, at the pass's first stage."""
    half = 1 << (p.nb - 1)
    return (((half - 1) << p.lo) | ((1 << p.lo) - 1)) << p.s0


# ------------------------------------------------------------------ the sweep
# xcorr: (name, dtype1, dtype2, n1, n2, nlead, nlag).  need = 2^m exactly at every m; odd m <= 19 with swapped
# operands (len(s1) < len(pad(s2)), need = len(s2) + max(nlag, nlead)); the largest two in int8 to keep host memory
# small; and need = 2^m + 1 at the pass-count changes and elsewhere
XC_DTYPES = [("complex128", "complex128"), ("float64", "float64"), ("complex64", "complex64"), ("int16", "int16"),
             ("complex128", "float32"), ("int8", "complex64"), ("float32", "complex128")]


def _xcorr_cases():
    cases = []
    for m in range(1, MAX_LOG2 + 1):
        L = 1 << m
        dt1, dt2 = ("int8", "int8") if m >= 25 else XC_DTYPES[m % len(XC_DTYPES)]
        if dt1 == "int16" and 12 < m < 24:          # keeps the exact integer truth's direct sum small
            dt1, dt2 = XC_DTYPES[0]
        if m % 2 and m <= 19:
            big = L // 2
            n2, n1 = L - big, max(1, L // 4)
            nlag, nlead = (big, big // 3) if m % 4 == 1 else (big // 5, big)
        else:
            nlead, nlag = (1, 0) if m <= 4 else (m % 3, m % 5)
            n1 = L
            n2 = 48 if dt1.startswith("int") and dt2.startswith("int") and m > 12 else \
                max(1, (L // 3 if m <= 20 else L // 16) - nlead - nlag)
        cases.append((f"xc_m{m}", dt1, dt2, n1, n2, nlead, nlag))
    for m, (dt1, dt2) in ((1, XC_DTYPES[0]), (11, XC_DTYPES[2]), (12, XC_DTYPES[4]), (19, XC_DTYPES[1]),
                          (20, XC_DTYPES[0]), (23, XC_DTYPES[6])):
        cases.append((f"xc_m{m}_plus1", dt1, dt2, (1 << m) + 1, max(1, (1 << m) // 7), 2, 3 if m > 1 else 0))
    cases.append(("xc_nvalid1", "complex128", "complex64", 700, 650, 29, 21))
    cases.append(("xc_single_samples", "float64", "int16", 1, 1, 0, 0))
    return cases


XCORR_CASES = _xcorr_cases()

# find_channel_offset: (name, dtype1, dtype2, n1, n2, nd, nl, delay), s2[j] ~ s1[j + delay]; delay None: no clear
# peak is expected
NDS = (1, 2, 3, 4, 5, 7, 8, 13, 16, 31, 32, 33, 63, 64)
REAL = ("int8", "uint8", "int16", "float32", "float64")
CPLX = ("complex64", "complex128")


def _offset_cases():
    cases = []
    for i, nd in enumerate(NDS):
        base = max(6000, 600 * nd) // nd * nd
        for kind, dt, r in (("real", REAL[i % 5], (0, 1, nd - 1)[i % 3]),
                            ("cplx", CPLX[i % 2], (0, 1, nd - 1)[(i + 1) % 3])):
            n1 = base + r
            cases.append((f"nd{nd}_{kind}", dt, dt, n1, n1 - 3 * nd - i % 2, nd, 40, nd * ((7 * i) % 61 - 30)))
    cases += [
        ("mix_i8_c64", "int8", "complex64", 12000, 11900, 8, 30, 8 * 5),
        ("mix_c64_i8", "complex64", "int8", 9001, 9000, 5, 30, -5 * 11),
        ("mix_f32_f64", "float32", "float64", 10000, 9990, 3, 30, 3 * 17),
        ("mix_f64_f32", "float64", "float32", 8000, 8000, 1, 50, -23),
        ("n28_nd1", "int8", "int8", 28, 28, 1, 3, None),
        ("n29_nd1", "float64", "float64", 29, 28, 1, 5, None),
        ("n28_nd64", "complex64", "complex64", 28, 29, 64, 2, None),
        ("n29_nd63", "int16", "uint8", 29, 29, 63, 4, None),
        ("chunk256_nd1", "int8", "int8", 4194250, 4194250, 1, 100, 37),
        ("chunk257_nd1", "int8", "int8", 4194251, 4194251, 1, 100, -41),
        ("chunk256_nd64", "complex64", "complex64", 4194250, 4194250, 64, 50, -64 * 9),
        ("chunk257_nd64", "int16", "int16", 4194251, 4194251, 64, 50, 64 * 7),
        ("swap_short_s1", "complex128", "complex128", 3000, 9000, 2, 20, 2 * 10),
        ("b1_longer", "uint8", "uint8", 20000, 3000, 4, 30, 4 * 530),
        ("nvalid1_nd1", "float32", "float32", 5040, 5000, 1, 20, 20),
        ("nvalid1_nd4", "uint8", "uint8", 5200, 5160, 4, 5, 4 * 5),
        ("preview", "complex64", "complex64", 2399625, 2399625, 4, 50000, 4 * 1234),
    ]
    return cases


OFFSET_CASES = _offset_cases()

# the two-stage argmax past its 1024-block cap (nvalid > 1024 x 2048 lags): nl = 0 and len(s1) > len(s2), so lag k
# reads s1 from sample k and the planted peak sits at k = delay.  1023 * 256 + 255 + 10 * 262144 is the last lag of
# block 1023's last thread, in its last grid-stride step; 3 145 728 - 4 096 is the last valid lag
ARGMAX_CASES = [
    ("argmax_1024_blocks", "int8", "int8", (1 << 21) + 4095, 4096, 1, 0, (1 << 20) + 17),
    ("argmax_last_step", "int8", "int8", 3145728, 4096, 1, 0, 10 * 262144 + 1023 * 256 + 255),
    ("argmax_last_lag", "int8", "int8", 3145728, 4096, 1, 0, 3145728 - 4096),
]


def _plan(kind, case):
    if kind == "xcorr":
        _, _, _, n1, n2, nlead, nlag = case
        return xcorr_plan(n1, n2, nlead, nlag)
    _, dt1, dt2, n1, n2, nd, nl, _ = case
    return offset_plan(n1, n2, nd, nl, dt1, dt2)


def _all_cases():
    return [("xcorr", c) for c in XCORR_CASES] + [("offset", c) for c in OFFSET_CASES + ARGMAX_CASES]


def _edges():
    """{edge: [names of the cases that reach it]}."""
    reach = {}

    def hit(edge, name):
        reach.setdefault(edge, []).append(name)

    for kind, case in _all_cases():
        name, dt1, dt2 = case[:3]
        p = _plan(kind, case)
        cplx = dt1.startswith("complex") or dt2.startswith("complex")
        hit(f"m{p.m}", name)
        if p.need == p.L:
            hit("need_pow2", name)
        if p.need == p.L // 2 + 1:
            hit("need_pow2_plus_1", name)
        if p.m in (11, 12, 19, 20):
            hit(f"passes{len(p.passes)}_m{p.m}", name)
        if p.swapped:
            hit(f"swapped_{kind}", name)
            if cplx and kind == "xcorr":
                hit("swapped_xcorr_complex", name)
        if p.nvalid == 1:
            hit(f"nvalid1_{kind}", name)
        if kind == "xcorr":
            if not cplx:
                hit("xcorr_real_output", name)
            if case[5] != case[6]:
                hit("xcorr_nlead_ne_nlag", name)
            for dt in (dt1, dt2):
                if dt.startswith("int"):
                    hit("xcorr_integer", name)
            continue
        _, _, _, n1, n2, nd, nl, delay = case
        nb = p.argmax_blocks
        if nb in (1, 2) or (nb == ARG_MAX_BLOCKS and p.nvalid <= ARG_MAX_BLOCKS * 2048):
            hit(f"argmax_blocks_{nb}", name)
        if p.nvalid > ARG_MAX_BLOCKS * 2048:
            hit("argmax_past_cap", name)
            k = delay // nd - p.p0              # the planted peak's lag
            grid = nb * ARG_THREADS
            if k == p.nvalid - 1:
                hit("argmax_peak_at_last_lag", name)
            elif k // grid == (p.nvalid - 1 - k % grid) // grid:
                hit("argmax_peak_in_last_grid_step", name)
        for ip in p.iir:
            if ip.next in (256 * 16384, 256 * 16384 + 1):
                hit(f"iir_chunk{ip.chunk}_nd{nd}", name)
            if ip.chunk > 256:
                hit("iir_chunk_over_256", name)
        hit(f"nd{nd}_{'complex' if cplx else 'real'}", name)
        for dt in (dt1, dt2):
            hit(f"dtype_{dt}", name)
        if dt1 != dt2:
            hit(f"mixed_{dt1}_{dt2}", name)
        for n in (n1, n2):
            if n in (28, 29):
                hit(f"n{n}", name)
        if nd >= 3:
            for r, label in ((0, "0"), (1, "1"), (nd - 1, "nd_minus_1")):
                if n1 % nd == r:
                    hit(f"n_mod_nd_{label}", name)
        if (n1, n2, nd, nl, dt1, dt2) == (2399625, 2399625, 4, 50000, "complex64", "complex64"):
            hit("preview_call", name)
    return reach


# every edge of the plan -> the sweep case named to reach it
EDGE_CASES = {f"m{m}": f"xc_m{m}" for m in range(1, MAX_LOG2 + 1)}
EDGE_CASES.update({
    "need_pow2": "xc_m17", "need_pow2_plus_1": "xc_m11_plus1",
    "passes1_m11": "xc_m11", "passes2_m12": "xc_m11_plus1", "passes2_m19": "xc_m19", "passes3_m20": "xc_m19_plus1",
    "swapped_xcorr": "xc_m15", "swapped_xcorr_complex": "xc_m9", "nvalid1_xcorr": "xc_nvalid1",
    "xcorr_real_output": "xc_m8", "xcorr_nlead_ne_nlag": "xc_m13", "xcorr_integer": "xc_m10",
    "swapped_offset": "preview", "nvalid1_offset": "nvalid1_nd4",
    "iir_chunk256_nd1": "chunk256_nd1", "iir_chunk257_nd1": "chunk257_nd1",
    "iir_chunk256_nd64": "chunk256_nd64", "iir_chunk257_nd64": "chunk257_nd64",
    "argmax_blocks_1": "nd7_real", "argmax_blocks_2": "swap_short_s1", "argmax_blocks_1024": "argmax_1024_blocks",
    "argmax_past_cap": "argmax_last_step", "argmax_peak_in_last_grid_step": "argmax_last_step",
    "argmax_peak_at_last_lag": "argmax_last_lag",
    "n28": "n28_nd1", "n29": "n29_nd63", "n_mod_nd_0": "nd4_real", "n_mod_nd_1": "nd5_real",
    "n_mod_nd_nd_minus_1": "nd3_real", "preview_call": "preview",
    "mixed_int8_complex64": "mix_i8_c64", "mixed_float32_float64": "mix_f32_f64",
})
EDGE_CASES.update({f"nd{nd}_real": f"nd{nd}_real" for nd in NDS})
EDGE_CASES.update({f"nd{nd}_complex": f"nd{nd}_cplx" for nd in NDS})
EDGE_CASES.update({f"dtype_{dt}": c for dt, c in (("int8", "nd1_real"), ("uint8", "nd2_real"), ("int16", "nd3_real"),
                                                  ("float32", "nd4_real"), ("float64", "nd5_real"),
                                                  ("complex64", "nd1_cplx"), ("complex128", "nd2_cplx"))})


# ------------------------------------------------------------------ CPU: the twin
def _circular(a, b, L):
    return np.fft.ifft(np.fft.fft(a, L) * np.conj(np.fft.fft(b, L)))


def test_lag_mapping_is_scipy_valid_correlate_with_a_minimal_transform():
    """xc[k] = cc[(k + p0) mod L] of the twin's L-point circular correlation is correlate(a, pad(b), 'valid') for
    random small shapes, either operand longer, and L is the smallest power of two that holds every valid lag."""
    rng = np.random.default_rng(2024)
    shapes = [tuple(int(v) for v in rng.integers([1, 1, 0, 0], [41, 41, 21, 21])) for _ in range(3000)]
    shapes += [(1, 1, 0, 0), (30, 10, 10, 10), (9, 1, 4, 4), (1, 9, 0, 0), (2, 1, 0, 0)]
    swapped = nvalid1 = 0
    worst = 0.0
    for n1d, n2d, pl, pr in shapes:
        p = device_plan(n1d, n2d, pl, pr)
        assert p.L // 2 < p.need <= p.L or p.need == p.L == 2, (n1d, n2d, pl, pr)
        a = rng.standard_normal(n1d) + 1j * rng.standard_normal(n1d)
        b = rng.standard_normal(n2d) + 1j * rng.standard_normal(n2d)
        want = signal.correlate(a, np.pad(b, (pl, pr)), 'valid', method='direct')
        got = _circular(a, b, p.L)[(np.arange(p.nvalid) + p.p0) % p.L]
        assert got.shape == want.shape == (p.nvalid,)
        worst = max(worst, float(np.abs(got - want).max() / np.abs(want).max()))
        swapped += p.swapped
        nvalid1 += p.nvalid == 1
    assert worst < 1e-13, worst
    assert swapped > 500 and nvalid1 > 10


def test_a_transform_one_point_short_aliases_a_valid_lag():
    """need is tight: a transform of half the twin's L aliases some valid lag, so no smaller L would do."""
    rng = np.random.default_rng(7)
    short = 0
    for _ in range(300):
        n1d, n2d, pl, pr = (int(v) for v in rng.integers([2, 2, 0, 0], [41, 41, 21, 21]))
        p = device_plan(n1d, n2d, pl, pr)
        if p.m == 1:
            continue
        a = rng.standard_normal(n1d) + 1j * rng.standard_normal(n1d)
        b = rng.standard_normal(n2d) + 1j * rng.standard_normal(n2d)
        want = signal.correlate(a, np.pad(b, (pl, pr)), 'valid', method='direct')
        L = p.L // 2
        if L < max(n1d, n2d):
            continue                     # numpy would truncate the operands; the device never does this
        got = _circular(a, b, L)[(np.arange(p.nvalid) + p.p0) % L]
        assert np.abs(got - want).max() > 1e-6 * np.abs(want).max(), (n1d, n2d, pl, pr)
        short += 1
    assert short > 50


@pytest.mark.parametrize("m", range(1, MAX_LOG2 + 1))
def test_passes_cover_every_index_bit_once_within_a_tile(m):
    L = 1 << m
    ps = fft_passes(m)
    assert sorted(b for p in ps for b in range(p.lo, p.lo + p.nb)) == list(range(m))
    nhi = max(1, (L // 2) >> TW_LO_BITS)
    for p in ps:
        assert p.nb <= TILE_BITS and (1 << (p.nb + p.c)) <= 1 << TILE_BITS and p.c <= p.lo
        assert p.s0 == m - p.lo - p.nb
        assert p.tiles * (1 << (p.nb + p.c)) == L
        ex = max_twiddle_exponent(p)
        assert ex < L // 2 and (ex >> TW_LO_BITS) < nhi
    assert len(ps) == (1 if m <= 11 else 2 if m <= 19 else 3)


@pytest.mark.parametrize("m", [1, 2, 5, 11, 12, 13, 14, 19, 20])
def test_pass_index_arithmetic_pairs_every_row_once_per_stage(m):
    """The kernel's tile / column / row arithmetic, flattened: each stage's butterflies pair every index exactly once
    with its partner L >> (s + 1) away, and its twiddle exponents are (i mod h) 2^s, bounded as max_twiddle_exponent
    says."""
    L = 1 << m
    for p in fft_passes(m):
        for s, ex, g1, g2 in twiddle_exponents(m, p):
            h = L >> (s + 1)
            assert np.array_equal(g2 - g1, np.full_like(g1, h))
            both = np.sort(np.concatenate([g1.ravel(), g2.ravel()]))
            assert np.array_equal(both, np.arange(L))
            assert np.array_equal(ex, (g1 % h) << s)
        assert max(int(ex.max()) for _, ex, _, _ in twiddle_exponents(m, p)) == max_twiddle_exponent(p)


def test_twin_agrees_with_the_offset_oracle():
    for m in range(1, MAX_LOG2 + 1):
        assert [(p.lo, p.nb) for p in fft_passes(m)] == oo.pass_plan(m)
    for nd in range(1, MAX_ND + 1):
        for dt in (np.int8, np.complex64):
            sos = oo.decimate_sos(nd, dt)[0]
            assert warmup(sos) == oo.warmup_samples(sos), (nd, dt)
    assert warmup(_sos(1, np.int8)) == 1312 and warmup(_sos(64, np.int8)) == 14731       # DESIGN.md section 12


def test_twin_edges_sit_where_the_library_puts_them():
    """Spot values read off prcore_signal.cu and chanoff.cuh, so that an edit of the twin shows up here."""
    assert [iir_plan(n, _sos(1, np.int8)).chunk for n in (4194250, 4194251)] == [256, 257]
    assert iir_plan(4194250, _sos(1, np.int8)).grid == 128 and iir_plan(100, _sos(1, np.int8)).grid == 1
    assert [argmax_blocks(v) for v in (1, 2048, 2049, 4096, 4097, 2097152, 2097153)] == [1, 1, 2, 2, 3, 1024, 1024]
    assert [len(fft_passes(m)) for m in (11, 12, 19, 20, 26)] == [1, 2, 2, 3, 3]
    # SignalPreview's find_channel_offset(ref, srv, 4, 50000): a 2^20 transform in three passes, swapped operands
    p = offset_plan(2399625, 2399625, 4, 50000, "complex64", "complex64")
    assert (p.m, len(p.passes), p.swapped, p.p0, p.nvalid, p.launches) == (20, 3, True, -50000, 100001, 13)
    assert xcorr_plan(3000, 2000, 40, 33).launches == 1 + 1 + 2 * 2 + 1
    assert offset_plan(100, 100, 1, (1 << 26) - 100).need == 1 << 26
    with pytest.raises(PlanError, match=r"2\^26"):
        offset_plan(100, 100, 1, (1 << 26) - 99)
    with pytest.raises(PlanError, match=r"2\^26"):
        xcorr_plan((1 << 26) + 1, 1, 0, 0)
    with pytest.raises(PlanError, match="padlen"):
        offset_plan(27, 100, 1, 0)


def test_planted_peaks_fall_on_valid_lags():
    """A planted delay d puts the peak at lag d / nd - p0, which must be a valid lag for the offset check to bite."""
    for case in OFFSET_CASES + ARGMAX_CASES:
        name, dt1, dt2, n1, n2, nd, nl, delay = case
        if delay is not None:
            p = offset_plan(n1, n2, nd, nl, dt1, dt2)
            assert delay % nd == 0 and 0 <= delay // nd - p.p0 < p.nvalid, name


def test_sweep_names_a_case_for_every_edge():
    reach = _edges()
    names = [c[0] for _, c in _all_cases()]
    assert len(names) == len(set(names))
    for edge, name in EDGE_CASES.items():
        assert name in names, f"{edge}: no sweep case {name}"
        assert name in reach.get(edge, []), f"{edge}: {name} no longer reaches it (reached by {reach.get(edge)})"
    for m in range(1, MAX_LOG2 + 1):
        if m <= 24 or f"xc_m{m}" in reach["need_pow2"]:
            assert f"xc_m{m}" in reach["need_pow2"], f"xc_m{m} does not sit at need = 2^{m}"


# ------------------------------------------------------------------ GPU helpers
def _lib():
    from passiveradar_b200 import _lib as lib
    return lib


def _counted(call):
    lib = _lib()
    before = lib.launch_count()
    res = call()
    return res, lib.launch_count() - before


def _as(x, dt, small):
    dt = np.dtype(dt)
    if dt.kind == "c":
        return x.astype(dt)
    r = x.real
    if small and dt.kind in "iu":       # xcorr: integer results stay within the dtype, as SciPy's need to
        return np.clip(np.round(10 * r), -30, 30).astype(dt)
    if dt == np.int8:                   # 45 sigma: 2 x[0] - x[k] of the odd extension wraps now and then
        return np.clip(np.round(45 * r), -128, 127).astype(np.int8)
    if dt == np.uint8:
        return (np.clip(np.round(45 * r), -128, 127) + 128).astype(np.uint8)
    if dt == np.int16:
        return np.clip(np.round(12000 * r), -32768, 32767).astype(np.int16)
    return r.astype(dt)


def _signal_pair(dt1, dt2, n1, n2, delay, seed, small=False):
    """s1 and s2 of one complex white source, s2[j] ~ s1[j + delay], with independent noise on each."""
    rng = np.random.default_rng(seed)
    delay = delay or 0
    a = max(0, -delay)
    total = a + max(n1, delay + n2) + 1
    u = rng.standard_normal(total) + 1j * rng.standard_normal(total)
    x1 = u[a:a + n1] + 0.1 * (rng.standard_normal(n1) + 1j * rng.standard_normal(n1))
    x2 = u[a + delay:a + delay + n2] + 0.1 * (rng.standard_normal(n2) + 1j * rng.standard_normal(n2))
    return _as(x1, dt1, small), _as(x2, dt2, small)


def _xcorr_raw(s1, s2, nlead, nlag):
    """prc_xcorr's own float64 / complex128 output (the wrapper rounds integer results)."""
    lib = _lib()
    a1, a2 = np.ascontiguousarray(s1), np.ascontiguousarray(s2)
    cplx = np.iscomplexobj(a1) or np.iscomplexobj(a2)
    out = np.empty(abs(a1.shape[0] - (a2.shape[0] + nlag + nlead)) + 1, np.complex128 if cplx else np.float64)
    code = {np.dtype(k): v for k, v in (("int8", lib.DT_I8), ("uint8", lib.DT_U8), ("int16", lib.DT_I16),
                                        ("float32", lib.DT_F32), ("float64", lib.DT_F64),
                                        ("complex64", lib.DT_C64), ("complex128", lib.DT_C128))}
    lib.check(lib.load().prc_xcorr(a1.ctypes.data, code[a1.dtype], a1.shape[0], a2.ctypes.data, code[a2.dtype],
                                   a2.shape[0], nlead, nlag, out.ctypes.data, lib.MEM_HOST, 0, None, 0))
    return out


def _xcorr_truth(s1, s2, nlead, nlag):
    b = np.pad(s2, (nlag, nlead))
    if s1.dtype.kind in "iu" and s2.dtype.kind in "iu":            # exact integers
        return signal.correlate(s1.astype(np.int64), b.astype(np.int64), 'valid', method='direct').astype(np.float64)
    wide = np.complex128 if np.iscomplexobj(s1) or np.iscomplexobj(s2) else np.float64
    method = 'direct' if s1.shape[0] * b.shape[0] <= 5e7 else 'fft'
    return signal.correlate(s1.astype(wide), b.astype(wide), 'valid', method=method)


def _rel(a, b, den):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / den) if den else float(np.abs(np.asarray(a)).max())


def _offset_and_xc(s1, s2, nd, nl):
    from passiveradar_b200 import signal_utils as psu
    return _counted(lambda: psu._channel_offset(s1, s2, nd, nl, want_xc=True))


def _check_offset(off, xc, nd, nl):
    """The two-stage reduction is np.argmax's first-index rule over the |xc| the device wrote."""
    assert off == (int(np.argmax(xc)) - nl) * nd


def _clear_peak(t_xc):
    """True when the truth's maximum beats every other lag by more than the device's error can close."""
    if t_xc.shape[0] < 2:
        return True
    top2 = np.partition(t_xc, -2)[-2:]
    return top2[1] - top2[0] > 4 * XC_TOL * top2[1]


# ------------------------------------------------------------------ GPU: xcorr at every transform size
@pytest.mark.gpu
@pytest.mark.parametrize("case", XCORR_CASES, ids=[c[0] for c in XCORR_CASES])
def test_xcorr_at_every_transform_size(case):
    import passiveradar_b200 as prb
    name, dt1, dt2, n1, n2, nlead, nlag = case
    plan = xcorr_plan(n1, n2, nlead, nlag)
    s1, s2 = _signal_pair(dt1, dt2, n1, n2, 0, plan.m, small=True)
    got, launches = _counted(lambda: _xcorr_raw(s1, s2, nlead, nlag))
    assert launches == plan.launches, f"{name}: {launches} launches, the plan has {plan.launches}"
    want = _xcorr_truth(s1, s2, nlead, nlag)
    assert got.shape == want.shape == (plan.nvalid,)
    err = _rel(got, want, np.abs(want).max())
    print(f"[sweep] xcorr {name} m={plan.m} {dt1}/{dt2} swapped={plan.swapped} rel_err={err:.3e}")
    assert err <= XCORR_TOL, name
    if plan.m <= 24:                    # the drop-in returns the reference's dtype and values
        pub = prb.xcorr(s1, s2, nlead, nlag)
        ref = oo.xcorr_oracle(s1, s2, nlead, nlag)
        assert pub.dtype == ref.dtype and pub.shape == ref.shape
        if pub.dtype.kind in "iu":
            np.testing.assert_array_equal(pub, ref)
        elif pub.dtype == np.complex128:
            np.testing.assert_array_equal(pub, got)


# ------------------------------------------------------------------ GPU: find_channel_offset across the decimator
@pytest.mark.gpu
@pytest.mark.parametrize("case", OFFSET_CASES + ARGMAX_CASES, ids=[c[0] for c in OFFSET_CASES + ARGMAX_CASES])
def test_channel_offset_across_the_decimator(case):
    name, dt1, dt2, n1, n2, nd, nl, delay = case
    plan = offset_plan(n1, n2, nd, nl, dt1, dt2)
    s1, s2 = _signal_pair(dt1, dt2, n1, n2, delay, 1000 + n1 % 997 + nd)
    (off, xc), launches = _offset_and_xc(s1, s2, nd, nl)
    assert launches == plan.launches, f"{name}: {launches} launches, the plan has {plan.launches}"
    t_off, t_xc = oo.find_channel_offset_truth(s1, s2, nd, nl)
    assert xc.shape == t_xc.shape == (plan.nvalid,)
    err = _rel(xc, t_xc, t_xc.max())
    print(f"[sweep] offset {name} m={plan.m} nd={nd} {dt1}/{dt2} rel_err={err:.3e} offset={off} truth={t_off}")
    assert err <= XC_TOL, name
    _check_offset(off, xc, nd, nl)
    if delay is not None:
        assert _clear_peak(t_xc), f"{name}: the planted delay gives no clear peak"
    if _clear_peak(t_xc):
        assert off == t_off, name
    if name.startswith("argmax_"):
        assert int(np.argmax(xc)) == delay // nd - plan.p0


# ------------------------------------------------------------------ GPU: the argmax's rules
@pytest.mark.gpu
def test_periodic_input_keeps_the_first_of_many_near_equal_peaks():
    """s1 repeats a 97-sample pattern, so |xc| has a peak every 97 lags, equal but for round-off and the filter's
    edges; the device's offset is still the first index of the largest value it wrote."""
    rng = np.random.default_rng(97)
    s1 = np.tile(rng.integers(-60, 60, 97), 420)[:40000].astype(np.int8)
    s2 = s1[300:5300].copy()
    for nd, nl in ((1, 2000), (2, 300)):
        plan = offset_plan(s1.shape[0], s2.shape[0], nd, nl)
        (off, xc), launches = _offset_and_xc(s1, s2, nd, nl)
        assert launches == plan.launches
        _check_offset(off, xc, nd, nl)
        t_xc = oo.find_channel_offset_truth(s1, s2, nd, nl)[1]
        assert _rel(xc, t_xc, t_xc.max()) <= XC_TOL
        k = int(np.argmax(xc))
        assert t_xc[k] >= t_xc.max() * (1 - 4 * XC_TOL)          # one of the truth's peaks
        assert np.sum(t_xc >= t_xc.max() * (1 - 1e-6)) > 1


@pytest.mark.gpu
def test_all_zero_s1_gives_the_first_lag():
    rng = np.random.default_rng(5)
    s1 = np.zeros(5000, np.int8)
    s2 = rng.integers(-50, 50, 4000).astype(np.int8)
    (off, xc), _ = _offset_and_xc(s1, s2, 3, 100)
    assert off == -100 * 3
    assert xc.shape[0] == offset_plan(5000, 4000, 3, 100).nvalid and not xc.any()


def _with(x, i, v):
    y = x.copy()
    y[i] = v
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("bad", ["nan", "inf"])
@pytest.mark.parametrize("nd", [1, 4])
def test_nan_and_inf_inputs_rank_as_numpy_argmax_does(bad, nd):
    """One NaN or inf in s1 reaches every decimated sample and, through the transform, every lag: the reference's |xc|
    is all NaN and np.argmax returns its first index, so the offset is -nl * nd."""
    import passiveradar_b200 as prb
    s1, s2 = _signal_pair("complex128" if bad == "inf" else "float64", "float64", 6000, 2000, 1500, 3 + nd)
    s1 = _with(s1, 2500, float(bad))
    nl = 50
    with np.errstate(invalid="ignore"):
        o_off, o_xc = oo.find_channel_offset_oracle(s1, s2, nd, nl)
    (off, xc), launches = _offset_and_xc(s1, s2, nd, nl)
    assert launches == offset_plan(6000, 2000, nd, nl).launches
    assert o_off == -nl * nd and np.isnan(o_xc).all()
    assert off == o_off
    np.testing.assert_array_equal(np.isnan(xc), np.isnan(o_xc))
    # xcorr of the same input: at this shape SciPy's correlate takes the FFT, which spreads the NaN or inf to every
    # lag, as the device's transform does
    b = np.pad(s2, (33, 40))
    assert signal.choose_conv_method(s1, b, 'valid') == 'fft'
    got = prb.xcorr(s1, s2, 40, 33)
    with np.errstate(invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        want = oo.xcorr_oracle(s1, s2, 40, 33)
    assert np.isnan(want).all()
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))


# ------------------------------------------------------------------ GPU: the transform limit at its edge
@pytest.mark.gpu
def test_one_point_past_the_transform_limit_is_refused_without_a_launch():
    """need = 2^26 runs (xc_m26 above, int8); need = 2^26 + 1 is refused, with the limit in the message, before any
    kernel launches, by both entry points."""
    lib = _lib()
    lb = lib.load()
    assert xcorr_plan(1 << 26, 48, 0, 0).need == 1 << 26
    with pytest.raises(PlanError):
        xcorr_plan((1 << 26) + 1, 48, 0, 0)
    a = np.zeros((1 << 26) + 1, np.int8)
    out = np.empty(a.shape[0] - 48 + 1)
    st, launches = _counted(lambda: lb.prc_xcorr(a.ctypes.data, lib.DT_I8, a.shape[0], a.ctypes.data, lib.DT_I8, 48,
                                                 0, 0, out.ctypes.data, lib.MEM_HOST, 0, None, 0))
    assert st == lib.PRC_E_INVALID and "2^26" in lb.prc_last_error().decode() and launches == 0
    nl = (1 << 26) - 99
    with pytest.raises(PlanError):
        offset_plan(100, 100, 1, nl)
    s = np.ones(100, np.int8)
    sos, zi = (np.ascontiguousarray(np.stack([v, v])) for v in oo.decimate_sos(1, np.int8))
    off = np.zeros(1, np.int64)
    st, launches = _counted(lambda: lb.prc_channel_offset(s.ctypes.data, lib.DT_I8, 100, s.ctypes.data, lib.DT_I8, 100,
                                                          1, nl, sos.ctypes.data, zi.ctypes.data, off.ctypes.data,
                                                          None, lib.MEM_HOST, 0, None, 0))
    assert st == lib.PRC_E_INVALID and "2^26" in lb.prc_last_error().decode() and launches == 0
