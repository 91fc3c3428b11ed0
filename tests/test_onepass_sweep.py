"""The one-pass FFT-domain frame (csrc/framepass.cuh, planned by prcore_corr.cu's onepass_plan) across its planner, its
segment limits, its batch chunks, its CTA walks, the Doppler stages it hands its rows to, and strided frame layouts.

A Python twin of onepass_plan (built on test_path_sweep's ls_plan / caf_plan and the decimator's alignment) states for
every shape whether the one-pass frame runs and how it splits each Doppler block into segments, and for a batch how it
chunks the frames, how many CTAs walk each frame and which Doppler kernel each chunk takes.  CPU tests hold the twin to
its invariants and to scripts/fft/model.py's partition; GPU tests hold the library to the twin (which kernels ran) and
the kernels to float64 truths.  Criteria: taps and P0 maps within 1.5e-6 of the float64 frame truth on shapes the
one-pass frame was measured at (test_frame_onepass.py), 1e-5 (test_path_sweep.py's TOL) where it was not.  Figures go
to $PRC_PARITY_DIR/parity.json (conftest.record_parity)."""
import importlib.util
import math
import os
from dataclasses import dataclass

import numpy as np
import pytest
import scipy.signal as signal

import test_path_sweep as ps
from conftest import record_parity
from passiveradar_b200 import _lib, synth
from oracle import clutter_oracle as co
from oracle import xambg_oracle as xo

HERE = os.path.dirname(os.path.abspath(__file__))
L = 2048                          # the one-pass frame runs at R3 = 8 only
ACC_CAP = 256 << 20               # FP_ACC_CAP: AccP / AccQ spectra of one chunk of frames
TOL1 = 1.5e-6                     # taps and P0 maps of the one-pass frame against the float64 frame truth
TOL = ps.TOL                      # 1e-5: shapes and paths the one-pass bound was never measured on


def rel(a, b, den):
    return float(np.abs(np.asarray(a, np.complex128) - b).max() / den)


def _model():
    spec = importlib.util.spec_from_file_location("fft_model", os.path.join(HERE, "..", "scripts", "fft", "model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ------------------------------------------------------------------ planner twin (prcore_corr.cu: onepass_plan, frame_onepass)
@dataclass(frozen=True)
class OnePlan:
    """on/off and why; bls (LS-only segment limit), Bmax (block segment limit); per Doppler block (lo, hi, ls_end,
    nseg, Bs); the LS-only tail (tail_lo, ntail, Bt)."""
    on: bool
    why: str
    bls: int = 0
    Bmax: int = 0
    blocks: tuple = ()
    tail: tuple = (0, 0, 0)

    @property
    def units(self):
        return len(self.blocks) + self.tail[1]


def onepass_plan(n, F, filter_len, peek, R, fft_min_n=ps.FFT_MIN_N, floor=L // 4):
    """``floor``: the plan's lower bound on Bmax (L / 4); the search for the smallest Bmax lowers it."""
    M = filter_len + peek
    lf, cf = ps.ls_plan(n, M, fft_min_n), ps.caf_plan(n, R, F, M, fft_min_n)
    if not (lf.on and cf.on):
        return OnePlan(False, "no FFT-domain frame")
    if filter_len < 1:
        return OnePlan(False, "filter_len = 0")
    bls = L - 2 * M + 2
    bmax = min(bls, L - M - R - peek + 1)
    if bmax < floor or n < L:
        return OnePlan(False, "Bmax below L/4", bls, bmax)
    D = n // F
    ntaps = D + 1
    c0 = xo.decimator_alignment(ntaps, D)
    if c0 - (ntaps - 1) > 0:
        return OnePlan(False, "samples before the first block", bls, bmax)
    j = np.arange(F, dtype=np.int64)
    base = j * D + c0
    lo = np.maximum(base - (ntaps - 1), 0)
    hi = np.minimum(base + 1, n)
    ls_end = np.where(j + 1 < F, np.minimum(hi, np.maximum(base + D - (ntaps - 1), 0)), hi)
    ln = np.maximum(hi - lo, 0)
    nseg = -(-ln // bmax)
    Bs = np.where(nseg > 0, -(-ln // np.maximum(nseg, 1)), 0)
    tail_lo = min((F - 1) * D + c0 + 1, n)
    ntail = -(-(n - tail_lo) // bls)
    Bt = -(-(n - tail_lo) // ntail) if ntail else 0
    one = (3 * ntail + int((4 * nseg + 1).sum())) * L * 11
    two_caf = int((3 * -(-ln // cf.Bmax) + 1).sum())
    two = 3 * lf.nseg * lf.L * int(math.log2(lf.L)) + two_caf * cf.L * int(math.log2(cf.L))
    blocks = tuple(zip(*(a.tolist() for a in (lo, hi, ls_end, nseg, Bs))))
    on = one < two
    return OnePlan(on, "cheaper than two passes" if on else "two passes cost no more", bls, bmax, blocks,
                   (tail_lo, ntail, Bt))


def doppler_kernel(F, R, nf, nsm):
    """The Doppler stage's kernel for a chunk of nf frames (prcore_corr.cu: doppler_stage)."""
    if F >= 2 and F & (F - 1) == 0 and F <= 8192:
        if F <= 1024 and -(-(R + 1) // 8) * nf >= nsm:
            return "pow2<8>"
        return "pow2<2>" if F <= 4096 else "pow2<1>"
    return "dft"


@dataclass(frozen=True)
class Chunk:
    f0: int
    nf: int
    ncta: int
    runs: tuple                   # units [u0, u1) of each CTA of a frame
    doppler: str


def onepass_batch(plan, F, R, nf, slots, nsm):
    """frame_onepass: chunks of frames whose spectra fit ACC_CAP, one wave of ``slots`` CTAs per chunk."""
    chunk = max(1, min(nf, ACC_CAP // (F * 2 * L * 8)))
    U = plan.units
    out = []
    for f0 in range(0, nf, chunk):
        m = min(chunk, nf - f0)
        ncta = max(1, min(U, slots // m))
        runs = tuple((c * U // ncta, (c + 1) * U // ncta) for c in range(ncta))
        out.append(Chunk(f0, m, ncta, runs, doppler_kernel(F, R, m, nsm)))
    return out


# (edge, n, F, R, filter_len, peek) of the segment limits at equality; test_frame_onepass.EDGE_CASES runs them on the GPU
LIMIT_CASES = {
    "caf_exact": (45712, 16, 300, 300, 10),
    "caf_one_past": (68624, 16, 300, 300, 10),
    "ls_exact": (45744, 16, 100, 300, 10),
    "ls_one_past": (68672, 16, 100, 300, 10),
    "tail_exact": (45745, 16, 100, 300, 10),
    "tail_plus_one": (45746, 16, 100, 300, 10),
    "full_L": (65520, 16, 0, 1, 0),
    "full_L_tail": (65552, 16, 0, 1, 0),
    "smallest_Bmax": (1048708, 1024, 912, 564, 14),
    "Bmax=L/4": (523264, 1024, 768, 769, 0),
}
HEADLINE = (2 ** 20, 256, 300, 300, 10)
# the on/off switches of the cost test at F = 16, filter_len 300, peek 10, R = 300: (D, on) on both sides of each
SWITCHES = [(829, False), (830, True), (1428, True), (1429, False), (1659, False), (1660, True), (2857, True),
            (2858, False), (2877, False), (2878, True)]


def _plan(name):
    n, F, R, fl, peek = LIMIT_CASES[name]
    return onepass_plan(n, F, fl, peek, R)


# ------------------------------------------------------------------ CPU: the twin
def _random_shapes(count, seed, nmax=1 << 22):
    rng = np.random.default_rng(seed)
    for _ in range(count):
        F = int(rng.choice([1, 7, 16, 64, 256, 1000, 1024]))
        yield (int(rng.integers(2048, nmax)), F, int(rng.integers(0, 701)), int(rng.integers(0, 41)),
               int(rng.integers(0, 1501)))


def _check_partition(p, n):
    ls_count = np.zeros(n, np.int64)
    for lo, hi, ls_end, nseg, Bs in p.blocks:
        if hi <= lo:
            assert nseg == 0
            continue
        assert (nseg - 1) * Bs < hi - lo <= nseg * Bs and Bs <= p.Bmax, (lo, hi, nseg, Bs, p.Bmax)
        assert lo <= ls_end <= hi
        ls_count[lo:ls_end] += 1
    tail_lo, ntail, Bt = p.tail
    assert Bt <= p.bls and (ntail == 0) == (tail_lo == n)
    if ntail:
        assert (ntail - 1) * Bt < n - tail_lo <= ntail * Bt
    ls_count[tail_lo:] += 1
    assert (ls_count == 1).all(), np.flatnonzero(ls_count != 1)[:5]


def test_twin_partition_invariants():
    """Every sample is in exactly one X_ls, every segment is within its limit, a block's segments cover [lo, hi)."""
    seen = 0
    for n, F, fl, peek, R in _random_shapes(600, 11):
        p = onepass_plan(n, F, fl, peek, R, 0)
        if p.blocks:
            _check_partition(p, n)
            seen += p.on
    assert seen >= 50, seen
    for name in LIMIT_CASES:
        _check_partition(_plan(name), LIMIT_CASES[name][0])


def test_twin_partition_is_the_models():
    """At model.py's one-pass shapes with L = 2048, the twin's partition is model_onepass's."""
    m = _model()
    shapes = [s for s in m.ONEPASS if s[5] == L]
    assert len(shapes) >= 4
    for n, F, R, M, peek, _, _ in shapes + [(LIMIT_CASES[k][0], LIMIT_CASES[k][1], LIMIT_CASES[k][2],
                                             LIMIT_CASES[k][3] + LIMIT_CASES[k][4], LIMIT_CASES[k][4], L, 0)
                                            for k in LIMIT_CASES]:
        p = onepass_plan(n, F, M - peek, peek, R, 0, floor=1)
        blocks, tail = m.onepass_partition(n, F, M, R, peek, L)
        assert (p.bls, p.Bmax) == m.onepass_limits(L, M, R, peek)
        assert list(p.blocks) == blocks and p.tail == tail, (n, F, R, M, peek)


def test_named_cases_sit_where_their_names_say():
    import test_frame_onepass as tf
    edges = {e: (n, F, R, fl, peek) for e, n, F, R, fl, peek, _ in tf.EDGE_CASES}
    for name in LIMIT_CASES:
        assert _plan(name).on, name
        assert edges[name] == LIMIT_CASES[name], name
    p = _plan("caf_exact")
    assert p.Bmax == 1429 < p.bls and {b[3:] for b in p.blocks[1:]} == {(2, 1429)}
    p = _plan("caf_one_past")
    # blocks of 4290 = 3 x (Bmax + 1): four segments of 1073, three of Bmax + 1 under a CAF limit one too large
    assert p.Bmax == 1429 and {b[3:] for b in p.blocks[1:]} == {(4, 1073)}
    assert {b[1] - b[0] for b in p.blocks[1:]} == {3 * (p.Bmax + 1)}
    p = _plan("ls_exact")
    assert p.Bmax == p.bls == 1430 and {b[3:] for b in p.blocks[1:]} == {(2, 1430)}
    p = _plan("ls_one_past")
    assert p.Bmax == p.bls == 1430 and {b[3:] for b in p.blocks[1:]} == {(4, 1074)}
    assert {b[1] - b[0] for b in p.blocks[1:]} == {3 * (p.bls + 1)}
    p = _plan("tail_exact")
    assert p.tail[1:] == (1, 1430) == (1, p.bls) and 45745 - p.tail[0] == 1430
    p = _plan("tail_plus_one")
    assert p.tail[1:] == (2, 716) and 45746 - p.tail[0] == 1431
    p = _plan("full_L")
    assert p.Bmax == p.bls == L and {b[3:] for b in p.blocks[1:]} == {(2, L)}
    p = _plan("full_L_tail")
    assert p.Bmax == p.bls == L and p.tail[1:] == (1, L)
    assert _plan("smallest_Bmax").Bmax == 545
    assert _plan("Bmax=L/4").Bmax == L // 4
    # the headline: Bmax = 1429, three segments per block, a 2047-sample tail in two segments
    p = onepass_plan(*HEADLINE[:2], HEADLINE[3], HEADLINE[4], HEADLINE[2])
    assert p.on and p.Bmax == 1429 and p.tail[1:] == (2, 1024) and {b[3] for b in p.blocks[1:]} == {3}


def test_switches_of_the_cost_test():
    """The plan switches on and off as D grows: segment counts jump at multiples of Bmax."""
    for D, on in SWITCHES:
        assert onepass_plan(16 * D, 16, 300, 10, 300).on == on, D
    ons = [onepass_plan(16 * D, 16, 300, 10, 300).on for D in range(512, 3200)]
    flips = [512 + i + 1 for i in range(len(ons) - 1) if ons[i] != ons[i + 1]]
    assert flips == [830, 1429, 1660, 2858, 2878], flips


def test_smallest_bmax_is_the_floor():
    """The L/4 floor binds: blocks of one segment (D + 1 = Bmax), peek 0 and the largest R the CAF limit allows are
    the one-pass frame's best case, and there the cost test is passed at Bmax = L/4 and would be below it."""
    best = None
    for bmax in range(L // 4 - 64, L // 4 + 40):
        for M in (769, 770, 800, 1024 - bmax // 2, (L + 2 - bmax) // 2):
            R = L - M - bmax + 1
            if R < 0 or L - 2 * M + 2 < bmax:
                continue
            p = onepass_plan(1024 * (bmax - 1), 1024, M, 0, R, floor=1)
            if p.on and p.Bmax == bmax:
                best = bmax if best is None else min(best, bmax)
    assert best is not None and best < L // 4, best
    assert not onepass_plan(1024 * (best - 1), 1024, (L + 2 - best) // 2, 0, L - (L + 2 - best) // 2 - best + 1).on
    p = _plan("Bmax=L/4")
    assert p.on and p.Bmax == L // 4 and {b[3:] for b in p.blocks[1:]} == {(1, 512)}


def test_batch_twin_walks():
    """CTA runs tile [0, U) in order; chunks tile the batch; the chunk and Doppler columns of the Doppler table."""
    p = onepass_plan(*HEADLINE[:2], HEADLINE[3], HEADLINE[4], HEADLINE[2])
    for nf in (1, 2, 3, 25, 33, 265):
        chunks = onepass_batch(p, HEADLINE[1], HEADLINE[2], nf, 264, 132)
        assert sum(c.nf for c in chunks) == nf and chunks[0].f0 == 0
        for c in chunks:
            assert c.runs[0][0] == 0 and c.runs[-1][1] == p.units
            assert all(a[1] == b[0] for a, b in zip(c.runs, c.runs[1:])) and all(r[1] > r[0] for r in c.runs)
    assert [c.ncta for c in onepass_batch(p, 256, 300, 1, 264, 132)] == [258]
    assert onepass_batch(p, 256, 300, 2, 264, 132)[0].runs[-1] == (256, 258)
    big = onepass_batch(p, 256, 300, 265, 264, 132)
    assert len(big) == 9 and [c.ncta for c in big] == [8] * 8 + [29]
    small = _plan("caf_exact")
    assert [c.ncta for c in onepass_batch(small, 16, 300, 265, 264, 132)] == [1]
    for n, F, nf, want in DOPPLER_CASES:
        q = onepass_plan(n, F, 300, 10, 300)
        assert q.on, (n, F)
        assert [(c.nf, c.doppler) for c in onepass_batch(q, F, 300, nf, 264, 132)] == want, (n, F)


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture
def onepass_options():
    """Restore "frame_onepass", "fft" and "fft_min_n" after a test that sets them."""
    names = ("frame_onepass", "fft", "fft_min_n")
    old = {k: _lib.get_option(k) for k in names}
    yield
    for k in names:
        _lib.set_option(k, old[k])


def _nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _slots():
    return _lib.get_option("fft_ctas_frame") * _nsm()


def _run(refs, srvs, fl, peek, reg, R, F, w, onepass=1, flags=0):
    """prc_frames_c64 on [nf, n] device tensors with taps and the cleaned channel requested; returns (status, maps,
    taps, cleaned, {kernel: launches} from the profiler)."""
    import torch
    nf, n = refs.shape
    maps = torch.empty((nf, F, R + 1), dtype=torch.complex64, device=refs.device)
    taps = torch.empty((nf, fl + peek), dtype=torch.complex64, device=refs.device)
    clean = torch.empty((nf, n), dtype=torch.complex64, device=refs.device)
    wp = None
    if w is not None:
        flags |= _lib.FLAG_WINDOW_F32 if w.dtype == torch.float32 else 0
        wp = w.data_ptr()
    _lib.set_option("frame_onepass", onepass)
    _lib.profile_reset()
    _lib.profile(True)
    try:
        st = _lib.load().prc_frames_c64(refs.data_ptr(), srvs.data_ptr(), n, nf, n, fl, peek, reg, R, F, wp,
                                        maps.data_ptr(), taps.data_ptr(), clean.data_ptr(), _lib.MEM_DEVICE, 0, None,
                                        flags)
        torch.cuda.synchronize()
        prof = {k: v[1] for k, v in _lib.profile_read().items()}
    finally:
        _lib.profile(False)
        _lib.profile_reset()
    return st, maps, taps, clean, prof


def _dev(frames):
    import torch
    refs = torch.from_numpy(np.stack([f[0] for f in frames])).cuda()
    srvs = torch.from_numpy(np.stack([f[1] for f in frames])).cuda()
    return refs, srvs


def _kaiser32(n):
    return signal.get_window(("kaiser", 5.0), n).astype(np.float32)


# ------------------------------------------------------------------ GPU: the twin is the library
def _pin_shapes():
    shapes = [(name, *LIMIT_CASES[name]) for name in LIMIT_CASES]
    shapes += [(f"switch_D{D}", 16 * D, 16, 300, 300, 10) for D, _ in SWITCHES]
    shapes.append(("headline", *HEADLINE))
    rng = np.random.default_rng(23)
    for i in range(150):
        F = int(rng.choice([1, 7, 16, 64, 256]))
        n = int(rng.integers(max(2048, 40 * F), (1 << 18) + 1))
        fl, peek = int(rng.integers(0, 701)), int(rng.integers(0, 41))
        if fl + peek == 0:
            fl = 1
        shapes.append((f"random_{i}", n, F, int(rng.integers(0, 1501)), fl, peek))
    return shapes


@pytest.mark.gpu
def test_twin_is_the_librarys_plan(onepass_options):
    """prc_frames_c64 (profiler on): caf_combine runs and lagcorr_ls does not exactly when the twin's plan is on; with
    "frame_onepass" = 0 caf_combine never runs."""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(5)
    on_count = 0
    for name, n, F, R, fl, peek in _pin_shapes():
        want = onepass_plan(n, F, fl, peek, R)
        x = torch.randn((2, 1, n), dtype=torch.complex64, device="cuda", generator=gen)
        for onepass in (1, 0):
            st, _, _, _, prof = _run(x[0], x[1], fl, peek, 1.0, R, F, None, onepass)
            assert st == _lib.PRC_OK, (name, _lib.load().prc_last_error())
            ran = prof.get("caf_combine", 0) > 0
            assert ran == (want.on and onepass == 1), (name, n, F, R, fl, peek, onepass, want.why, prof)
            assert (prof.get("lagcorr_ls", 0) > 0) == (not ran), (name, onepass, prof)
        on_count += want.on
    assert on_count >= 30, on_count
    record_parity("onepass/twin_is_the_library", shapes=len(_pin_shapes()), on=on_count)


# ------------------------------------------------------------------ GPU: the switch pair and reg at a segment limit
@pytest.mark.gpu
def test_switch_pair_and_reg_at_the_caf_limit(onepass_options):
    """n = 45 712 (D = 2857, one-pass) and n = 45 728 (D = 2858, two passes) against their truths: 1.5e-6 on the
    one-pass side, 1e-5 on the two-pass side; reg = 0 and reg = 1e3 at caf_exact."""
    F, R, fl, peek = 16, 300, 300, 10
    fig = {}
    for n, reg in ((45712, 1.0), (45728, 1.0), (45712, 0.0), (45712, 1e3)):
        plan = onepass_plan(n, F, fl, peek, R)
        assert plan.on == (n == 45712)
        ref, srv = synth.make_frame(n, "P0", 1500 + n % 97)
        w = _kaiser32(n)
        refs, srvs = _dev([(ref, srv)])
        import torch
        st, maps, taps, _, prof = _run(refs, srvs, fl, peek, reg, R, F, torch.from_numpy(w).cuda())
        assert st == _lib.PRC_OK and (prof.get("caf_combine", 0) > 0) == plan.on
        amb, t_taps, _ = xo.frame_truth(ref, srv, fl, reg, peek, R, F, w.astype(np.float64))
        e_map = rel(maps[0].cpu().numpy(), amb, np.abs(amb).max())
        e_taps = rel(taps[0].cpu().numpy(), t_taps, np.abs(t_taps).max())
        bound = TOL1 if plan.on else TOL
        assert e_map <= bound and e_taps <= bound, (n, reg, e_map, e_taps)
        fig[f"n{n}_reg{reg:g}"] = {"E_map": e_map, "E_taps": e_taps}
    for k, v in fig.items():
        record_parity(f"onepass/switch_{k}", **v)


# ------------------------------------------------------------------ GPU: Doppler stages and chunks
# (n, F, nf, [(frames, Doppler kernel) per chunk]) at filter_len 300, peek 10, R = 300 on 132 SMs x 2 CTAs
DOPPLER_CASES = [
    (2 ** 22, 1024, 9, [(8, "pow2<8>"), (1, "pow2<2>")]),
    (2 ** 22, 2048, 5, [(4, "pow2<2>"), (1, "pow2<2>")]),
    (2 ** 23, 8192, 2, [(1, "pow2<1>"), (1, "pow2<1>")]),         # spectra of one frame = the 256 MiB cap
    (2 ** 22, 3000, 3, [(2, "dft"), (1, "dft")]),
    (2 ** 24, 16384, 1, [(1, "dft")]),                            # 512 MiB of spectra: over the cap, chunk of 1
]


@pytest.mark.gpu
@pytest.mark.parametrize("n,F,nf,want", DOPPLER_CASES, ids=[f"F{c[1]}_nf{c[2]}" for c in DOPPLER_CASES])
def test_doppler_stages_and_chunks(n, F, nf, want, onepass_options):
    """P0 frames (two distinct ones alternating), float32 Kaiser window: the chunks and Doppler kernels the twin
    derives from the device's figures are the table's, the profiler counts one frame pass, one combine and one Doppler
    stage per chunk, taps and maps are within 1e-5 of the truth and each map within max(1.5e-6, 2 x the two-pass
    frame's error on the same frame)."""
    import torch
    R, fl, peek = 300, 300, 10
    plan = onepass_plan(n, F, fl, peek, R)
    chunks = onepass_batch(plan, F, R, nf, _slots(), _nsm())
    assert plan.on and [(c.nf, c.doppler) for c in chunks] == want, (plan.why, chunks)
    base = [synth.make_frame(n, "P0", 1600 + k) for k in range(min(nf, 2))]
    w = _kaiser32(n)
    d_w = torch.from_numpy(w).cuda()
    refs, srvs = _dev(base)
    idx = torch.arange(nf, device="cuda") % len(base)
    st, maps1, taps1, _, prof = _run(refs[idx], srvs[idx], fl, peek, 1.0, R, F, d_w, 1)
    assert st == _lib.PRC_OK
    assert prof.get("caf_combine") == prof.get("lagcorr_caf") == prof.get("doppler_fft") == len(chunks), prof
    maps1, taps1 = maps1.cpu().numpy(), taps1.cpu().numpy()
    st, maps0, _, _, prof0 = _run(refs[idx], srvs[idx], fl, peek, 1.0, R, F, d_w, 0)
    assert st == _lib.PRC_OK and prof0.get("caf_combine", 0) == 0, prof0
    maps0 = maps0.cpu().numpy()
    worst = {"E_map": 0.0, "E_taps": 0.0, "E_map_two_pass": 0.0}
    for k, (ref, srv) in enumerate(base):
        cleaned, t_taps = co.ls_filter_truth(ref, srv, fl, 1.0, peek)
        amb = xo.fast_xambg_truth(ref.astype(np.complex128), cleaned, R, F, None, w.astype(np.float64), fast=True)[:, :, 0]
        den = np.abs(amb).max()
        for i in range(k, nf, len(base)):
            e1, e0 = rel(maps1[i], amb, den), rel(maps0[i], amb, den)
            e_taps = rel(taps1[i], t_taps, np.abs(t_taps).max())
            assert e_taps <= TOL and e1 <= TOL and e1 <= max(TOL1, 2 * e0), (i, e_taps, e1, e0)
            worst = {"E_map": max(worst["E_map"], e1), "E_taps": max(worst["E_taps"], e_taps),
                     "E_map_two_pass": max(worst["E_map_two_pass"], e0)}
    record_parity(f"onepass/doppler_F{F}_nf{nf}", chunks=len(chunks), **worst)


# ------------------------------------------------------------------ GPU: CTA walks, isolation and statuses
def _walk_batches(plan, F, R, slots, nsm):
    """nf of the headline batch for each walk: one unit per CTA, a CTA of tail units only, a CTA across the last block
    and the tail, and slots + 1 frames (chunks of the cap, the last one with another ncta)."""
    U = plan.units
    out = {"one_unit_per_cta": 1}
    for nf in range(2, 40):
        runs = onepass_batch(plan, F, R, nf, slots, nsm)[0].runs
        if "tail_only_cta" not in out and any(a >= F for a, _ in runs):
            out["tail_only_cta"] = nf
        if "cta_spans_block_and_tail" not in out and any(a < F < b for a, b in runs):
            out["cta_spans_block_and_tail"] = nf
    out["slots+1"] = slots + 1
    chunks = onepass_batch(plan, F, R, 1, slots, nsm)
    assert chunks[0].ncta == U and all(b - a == 1 for a, b in chunks[0].runs)
    big = onepass_batch(plan, F, R, slots + 1, slots, nsm)
    assert len(big) > 1 and big[-1].ncta != big[0].ncta, big
    assert len(out) == 4, out
    return out


@pytest.mark.gpu
def test_cta_walks_repeat_one_frame_bit_identically(onepass_options):
    """The headline shape with one P0 frame repeated through batches chosen from the twin: rows of the same chunk are
    bit-identical, every row is within 1.5e-6 of the truth.  Rows of different chunks may differ in the last bits (the
    LS lag sums add a different number of CTA partials)."""
    import torch
    n, F, R, fl, peek = HEADLINE
    plan = onepass_plan(n, F, fl, peek, R)
    slots, nsm = _slots(), _nsm()
    batches = _walk_batches(plan, F, R, slots, nsm)
    ref, srv = synth.make_frame(n, "P0", 1700)
    w = _kaiser32(n)
    amb, t_taps, t_clean = xo.frame_truth(ref, srv, fl, 1.0, peek, R, F, w.astype(np.float64))
    d_amb, d_taps = torch.from_numpy(amb).cuda(), torch.from_numpy(t_taps).cuda()
    den, den_t = float(np.abs(amb).max()), float(np.abs(t_taps).max())
    refs, srvs = _dev([(ref, srv)])
    d_w = torch.from_numpy(w).cuda()
    fig = {}
    for what, nf in batches.items():
        idx = torch.zeros(nf, dtype=torch.long, device="cuda")
        st, maps, taps, _, prof = _run(refs[idx], srvs[idx], fl, peek, 1.0, R, F, d_w)
        chunks = onepass_batch(plan, F, R, nf, slots, nsm)
        assert st == _lib.PRC_OK and prof["caf_combine"] == len(chunks), (what, prof)
        e_map = float((maps.to(torch.complex128) - d_amb).abs().amax()) / den
        e_taps = float((taps.to(torch.complex128) - d_taps).abs().amax()) / den_t
        assert e_map <= TOL1 and e_taps <= TOL1, (what, nf, e_map, e_taps)
        for c in chunks:
            rows = slice(c.f0, c.f0 + c.nf)
            assert bool((maps[rows] == maps[c.f0]).all()) and bool((taps[rows] == taps[c.f0]).all()), (what, c.f0)
        fig[what] = {"nf": nf, "chunks": len(chunks), "ncta": chunks[0].ncta, "E_map": e_map, "E_taps": e_taps}
        del maps, taps
    for k, v in fig.items():
        record_parity(f"onepass/walk_{k}", **v)


@pytest.mark.gpu
def test_singular_frame_in_the_second_chunk(onepass_options):
    """The headline shape, reg = 0, a zero reference in a frame of the second chunk: the synchronous call returns
    PRC_E_SINGULAR naming that frame, with PRC_FLAG_ASYNC prc_ls_status flags that index only, and every other row
    still matches its truth."""
    import ctypes as C
    import torch
    n, F, R, fl, peek = HEADLINE
    plan = onepass_plan(n, F, fl, peek, R)
    chunks = onepass_batch(plan, F, R, 40, _slots(), _nsm())
    assert len(chunks) == 2
    bad = chunks[1].f0 + 1
    base = [synth.make_frame(n, "P0", 1800 + k) for k in range(2)]
    w = _kaiser32(n)
    d_w = torch.from_numpy(w).cuda()
    refs, srvs = _dev(base)
    idx = torch.arange(40, device="cuda") % 2
    b_ref, b_srv = refs[idx].contiguous(), srvs[idx].contiguous()
    b_ref[bad] = 0
    lib = _lib.load()
    st, maps, taps, _, _ = _run(b_ref, b_srv, fl, peek, 0.0, R, F, d_w)
    assert st == _lib.PRC_E_SINGULAR and f"frame {bad})" in lib.prc_last_error().decode(), lib.prc_last_error()
    st, maps_a, taps_a, _, _ = _run(b_ref, b_srv, fl, peek, 0.0, R, F, d_w, flags=_lib.FLAG_ASYNC)
    assert st == _lib.PRC_OK
    status = (C.c_int * 40)()
    _lib.check(lib.prc_ls_status(0, None, status, 40))
    assert np.flatnonzero(np.frombuffer(status, np.int32)).tolist() == [bad]
    worst = 0.0
    for k, (ref, srv) in enumerate(base):
        amb, t_taps, _ = xo.frame_truth(ref, srv, fl, 0.0, peek, R, F, w.astype(np.float64))
        d_amb = torch.from_numpy(amb).cuda()
        den = float(np.abs(amb).max())
        for m, t in ((maps, taps), (maps_a, taps_a)):
            for i in range(k, 40, 2):
                if i == bad:
                    continue
                e_map = float((m[i].to(torch.complex128) - d_amb).abs().amax()) / den
                e_taps = rel(t[i].cpu().numpy(), t_taps, np.abs(t_taps).max())
                assert e_map <= TOL1 and e_taps <= TOL1, (i, e_map, e_taps)
                worst = max(worst, e_map, e_taps)
    record_parity("onepass/singular_second_chunk", frame=bad, E_worst=worst)


# ------------------------------------------------------------------ GPU: layouts
@pytest.mark.gpu
def test_strided_frames_window_and_cleaned_gaps(onepass_options):
    """Frames at frame_stride = n + 37 with NaN in the gaps and around the batch, the window in n + 4096 floats whose
    tail is NaN, the cleaned output pre-filled with a sentinel: maps, taps and cleaned samples are finite and
    bit-identical to the packed call, the gaps still hold the sentinel, MEM_HOST with the same strided arrays gives the
    same bits, and FramePipeline.run_device on strided rows equals it on contiguous rows."""
    import torch
    from passiveradar_b200.frames import FramePipeline
    n, F, R, fl, peek = LIMIT_CASES["caf_exact"]
    nf, pad = 3, 37
    stride = n + pad
    assert onepass_plan(n, F, fl, peek, R).on
    frames = [synth.make_frame(n, "P0", 1900 + k) for k in range(nf)]
    nan = np.complex64(complex(np.nan, np.nan))
    sentinel = np.complex64(12345.0 - 6789.0j)
    h_ref = np.full(pad + nf * stride + pad, nan, np.complex64)
    h_srv = h_ref.copy()
    for k, (r, s) in enumerate(frames):
        h_ref[pad + k * stride:pad + k * stride + n] = r
        h_srv[pad + k * stride:pad + k * stride + n] = s
    h_w = np.full(n + 4096, np.nan, np.float32)
    h_w[:n] = _kaiser32(n)
    lib = _lib.load()
    flags = _lib.FLAG_WINDOW_F32
    M = fl + peek

    # packed reference call
    refs, srvs = _dev(frames)
    d_w = torch.from_numpy(h_w).cuda()
    st, p_maps, p_taps, p_clean, prof = _run(refs, srvs, fl, peek, 1.0, R, F, d_w[:n].clone())
    assert st == _lib.PRC_OK and prof["caf_combine"] == 1
    p_maps, p_taps, p_clean = p_maps.cpu().numpy(), p_taps.cpu().numpy(), p_clean.cpu().numpy()
    assert np.isfinite(p_maps).all() and np.isfinite(p_clean).all()

    def gaps(buf):
        keep = np.ones(buf.shape[0], bool)
        for k in range(nf):
            keep[pad + k * stride:pad + k * stride + n] = False
        return buf[keep]

    def rows(buf):
        return np.stack([buf[pad + k * stride:pad + k * stride + n] for k in range(nf)])

    # device pointers, strided
    d_ref, d_srv = torch.from_numpy(h_ref).cuda(), torch.from_numpy(h_srv).cuda()
    d_clean = torch.from_numpy(np.full_like(h_ref, sentinel)).cuda()
    maps = torch.empty((nf, F, R + 1), dtype=torch.complex64, device="cuda")
    taps = torch.empty((nf, M), dtype=torch.complex64, device="cuda")
    _lib.check(lib.prc_frames_c64(d_ref[pad:].data_ptr(), d_srv[pad:].data_ptr(), n, nf, stride, fl, peek, 1.0, R, F,
                                  d_w.data_ptr(), maps.data_ptr(), taps.data_ptr(), d_clean[pad:].data_ptr(),
                                  _lib.MEM_DEVICE, 0, None, flags))
    torch.cuda.synchronize()
    s_clean = d_clean.cpu().numpy()
    assert np.array_equal(maps.cpu().numpy(), p_maps) and np.array_equal(taps.cpu().numpy(), p_taps)
    assert np.array_equal(rows(s_clean), p_clean)
    assert (gaps(s_clean) == sentinel).all()

    # host pointers, the same strided arrays
    h_maps = np.empty((nf, F, R + 1), np.complex64)
    h_taps = np.empty((nf, M), np.complex64)
    h_clean = np.full_like(h_ref, sentinel)
    _lib.check(lib.prc_frames_c64(h_ref[pad:].ctypes.data, h_srv[pad:].ctypes.data, n, nf, stride, fl, peek, 1.0, R, F,
                                  h_w.ctypes.data, h_maps.ctypes.data, h_taps.ctypes.data, h_clean[pad:].ctypes.data,
                                  _lib.MEM_HOST, 0, None, flags))
    assert np.array_equal(h_maps, p_maps) and np.array_equal(h_taps, p_taps)
    assert np.array_equal(rows(h_clean), p_clean) and (gaps(h_clean) == sentinel).all()

    # FramePipeline on strided rows and on contiguous rows
    pipe = FramePipeline(n, R, F, filter_len=fl, peek=peek, nslots=1, batch=nf)
    wide_ref = d_ref[pad:pad + nf * stride].view(nf, stride)[:, :n]
    wide_srv = d_srv[pad:pad + nf * stride].view(nf, stride)[:, :n]
    assert wide_ref.stride(0) == stride
    out_wide = torch.empty((nf, F, R + 1), dtype=torch.complex64, device="cuda")
    out_cont = torch.empty_like(out_wide)
    pipe.run_device(wide_ref, wide_srv, out_wide, check=True)
    pipe.run_device(wide_ref.contiguous(), wide_srv.contiguous(), out_cont, check=True)
    torch.cuda.synchronize()
    assert torch.isfinite(torch.view_as_real(out_wide)).all() and torch.equal(out_wide, out_cont)
    worst = 0.0
    for k, (r, s) in enumerate(frames):
        amb, _, _ = xo.frame_truth(r, s, fl, 1.0, peek, R, F, h_w[:n].astype(np.float64))
        worst = max(worst, rel(p_maps[k], amb, np.abs(amb).max()))
    assert worst <= TOL1, worst
    record_parity("onepass/strided_layouts", stride=stride, E_map=worst)
