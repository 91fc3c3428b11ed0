"""Sweeps of the FP32 direct-form hot path across the edges of the host planners that shape it, against float64 truths.

The kernels: lagstream_kernel and lagcorr_kernel (the CAF's block sums and the LS lag sums), fir_apply_kernel, the
single-CTA levinson_kernel<1> / <4> solve of ls_device, the Doppler stage (doppler_fft_pow2_kernel<8 | 2 | 1>, or
chunk_sum_kernel + doppler_dft_kernel) and nlms_block_kernel<KT, NT>.  They are the library's default for every LS
filter below fft_min_n samples, every tap-weighted (shortFilt=False) or short-block (D < 32) CAF, every CAF of more
than 3072 lags, and all of NLMS.

A Python twin of the planners (prcore_corr.cu: choose_geo, choose_stream, stream_pieces / stream_first_cta, the branches
of xambg_device, doppler_stage, ls_device and nlms_device) states for every case which kernel runs with which
tiling; the sweep is chosen from it so that every edge of the tiling is reached, CPU tests hold the twin's invariants
and name a case per edge, and the GPU tests pin the twin to the library through the per-kernel launch counts of prc_profile_read.
Criteria as in tests/test_path_sweep.py, TOL = 1e-5 rel-inf: maps over max|map|, taps over max|taps|, cleaned
channels over max|srv|; NLMS outputs over max|truth| (taps 5e-5) and within 1e-5 + 1.2 x the reference arithmetic's
own error (tests/test_kernel_variants.py:_nlms_bounds).  Figures go to $PRC_PARITY_DIR/parity.json under direct/."""
from dataclasses import dataclass

import numpy as np
import pytest
import scipy.signal as signal

from conftest import record_parity
from test_kernel_variants import _nlms_bounds
from test_path_sweep import FFT_MIN_N, caf_plan, ls_plan
import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from oracle import clutter_oracle as co
from oracle import xambg_oracle as xo

TOL = 1e-5
TILE_I = TILE_D = 10                  # prcore_corr.cu: register tile of the FP32 sliding-window kernels
SMEM_LIMIT = 200 * 1024
SMEM_SOFT = 100 * 1024                # the tile loops shrink a tile until it fits this, as long as they can
FIR_THREADS = 128
NLMS_TILE, NB_L, NB_PAD, NB_THREADS = 1024, 32, 64, 1024     # nlms_block.cuh
NSM_H100 = (132, 114)                 # SXM and PCIe parts


def cdiv(a, b):
    return -(-a // b)


class PlanError(ValueError):
    """The library refuses the shape (PRC_E_INVALID) with this message."""


# ------------------------------------------------------------------ planner twin (prcore_corr.cu)
@dataclass(frozen=True)
class Geo:
    """choose_geo: lagcorr_kernel, one CTA per (block, chunk).  doublings: how often the nchunk loop halved the chunk
    to bring the tile under 100 KB."""
    H: int
    HT: int
    G: int
    steps: int
    nchunk: int
    chunk_len: int
    smem: int
    threads: int
    doublings: int


def choose_geo(blk_len, outer, nlag, nsm):
    H = cdiv(nlag, TILE_D)
    HT = H * TILE_D
    if H > 512:
        raise PlanError(f"{nlag} lags exceed the supported maximum of {512 * TILE_D}")
    gmax = max(1, min(32, 256 // H))
    nchunk = max(1, cdiv(nsm * 8, outer))
    nchunk = min(nchunk, max(1, blk_len // (TILE_I * gmax * 2)))
    doublings = 0
    while True:
        chunk_len = cdiv(blk_len, nchunk)
        nch = cdiv(blk_len, chunk_len)
        G = max(1, min(gmax, cdiv(chunk_len, TILE_I * 4)))
        steps = cdiv(cdiv(chunk_len, G), TILE_I)
        Lpad = G * steps * TILE_I
        smem = max(3 * Lpad + HT, G * HT) * 8
        if smem <= SMEM_SOFT or chunk_len <= TILE_I:
            break
        nchunk *= 2
        doublings += 1
    if smem > SMEM_LIMIT:
        raise PlanError(f"lag-correlation tile needs {smem} B of shared memory")
    return Geo(H, HT, G, steps, nch, chunk_len, smem, cdiv(H * G, 32) * 32, doublings)


@dataclass(frozen=True)
class StreamGeo:
    """choose_stream: lagstream_kernel, the blocks laid end to end and cut into ncta ranges of per_cta samples."""
    H: int
    HT: int
    G: int
    steps: int
    ncta: int
    per_cta: int
    total: int
    maxpieces: int
    smem: int
    threads: int


def choose_stream(blk_len, nblk, nprob, nlag, nsm):
    H = cdiv(nlag, TILE_D)
    HT = H * TILE_D
    if H > 512:
        raise PlanError(f"{nlag} lags exceed the supported maximum of {512 * TILE_D}")
    G0 = max(1, min(32, 256 // H))
    total = nblk * blk_len
    want = max(1, 2 * nsm // nprob)
    want = min(want, max(1, total // (G0 * TILE_I * 2)))
    per_cta = cdiv(total, want)
    ncta = cdiv(total, per_cta)
    G = max(1, min(G0, cdiv(per_cta, TILE_I)))
    steps = max(2, 100 // TILE_I)
    while steps > 1 and G * steps * TILE_I > per_cta + G * TILE_I:
        steps -= 1
    while True:
        Lmax = G * steps * TILE_I
        smem = (2 * (2 * Lmax + HT) + 2 * G * HT) * 8
        if smem <= SMEM_SOFT or steps == 1:
            break
        steps -= 1
    if smem > SMEM_LIMIT:
        raise PlanError(f"lag-correlation tile needs {smem} B of shared memory")
    maxpieces = min(ncta, (blk_len + per_cta - 2) // per_cta + 1)
    return StreamGeo(H, HT, G, steps, ncta, per_cta, total, maxpieces, smem, cdiv(H * G, 32) * 32)


def stream_first_cta(blk, blk_len, per_cta):
    return (blk * blk_len) // per_cta


def stream_pieces(blk, blk_len, per_cta):
    return ((blk + 1) * blk_len - 1) // per_cta - (blk * blk_len) // per_cta + 1


def blocks_per_cta(sg, blk_len):
    """Most Doppler blocks one CTA's range of the stream touches."""
    c = np.arange(sg.ncta, dtype=np.int64)
    last = np.minimum((c + 1) * sg.per_cta, sg.total) - 1
    return int((last // blk_len - (c * sg.per_cta) // blk_len + 1).max())


def doppler_branch(F, R, nf, nsm):
    """doppler_stage: "ct8" / "ct2" / "ct1" (doppler_fft_pow2_kernel<CT>) or "dft" (chunk sums
    and the direct DFT, frame by frame)."""
    pow2 = F >= 2 and F & (F - 1) == 0
    if pow2 and F <= 8192:
        if F <= 1024 and cdiv(R + 1, 8) * nf >= nsm:
            return "ct8"
        return "ct2" if F <= 4096 else "ct1"
    return "dft"


@dataclass(frozen=True)
class CafDirect:
    """What one fast_xambg call runs: the block-sum kernel ("fft" when the FFT-domain CAF takes it), its tiling, the
    Doppler branch and the launches prc_profile_read and prc_launch_count see on a call whose twiddles are cached."""
    kernel: str
    ntaps: int
    geo: object
    doppler: str
    profile: tuple            # (lagcorr_caf, misc, doppler_fft)
    launches: int


def caf_direct(n, R, F, window, short_filt, nsm, fft_min_n=None):
    """fft_min_n None: the FFT-domain path off ("fft" = 0); else on with that minimum length."""
    D = n // F
    taps = not short_filt and D > 1
    ntaps = 1 if D == 1 else (10 * D + 1 if taps else D + 1)
    if fft_min_n is not None and not taps and caf_plan(n, R, F, 0, fft_min_n).on:
        return CafDirect("fft", ntaps, None, doppler_branch(F, R, 1, nsm), (), 0)
    if not taps and ntaps >= 64:
        kernel, geo = "lagstream", choose_stream(ntaps, F, 1, R + 1, nsm)
    else:
        kernel, geo = "lagcorr", choose_geo(ntaps, F, R + 1, nsm)
    dop = doppler_branch(F, R, 1, nsm)
    misc = int(kernel == "lagstream" and window)
    staged = int(bool(window)) + int(taps)                   # f64_to_f32_kernel of the window / the decimator taps
    return CafDirect(kernel, ntaps, geo, dop, (1, misc, 1), staged + misc + 1 + (2 if dop == "dft" else 1))


@dataclass(frozen=True)
class LsDirect:
    """ls_device's direct branch: the two lag sums (lagstream_kernel, 2 problems), the single-CTA Levinson solve
    (levinson_kernel<E>) and fir_apply_kernel with Mpad reversed taps."""
    stream: StreamGeo
    levinson: int
    lev_smem: int
    Mpad: int
    fir_smem: int


def levinson_smem(M, threads):
    nparts = min(3, threads // (2 * M))
    return (2 * M + max(nparts * 2 * M, 4 + 2 * 32 * 2)) * 16


def ls_direct(n, M, nsm):
    if M > 2048:
        raise PlanError(f"{M} taps exceed the Toeplitz solver's maximum of 2048")
    sg = choose_stream(n, 1, 2, M, nsm)
    E = 1 if M <= 1024 else 4
    Mpad = cdiv(M, TILE_I) * TILE_I
    if Mpad & 1:
        Mpad += TILE_I
    fir_smem = (2 * Mpad + FIR_THREADS * TILE_D) * 8
    if fir_smem > SMEM_LIMIT:
        raise PlanError(f"{M} taps exceed the FIR kernel's shared memory")
    return LsDirect(sg, E, levinson_smem(M, 1024 if E == 1 else 512), Mpad, fir_smem)


def nlms_kernel(M, nf, nsm):
    """(KT, NT) of nlms_block_kernel: 512-thread CTAs for more frames than SMs up to 2048 taps."""
    if M > 4096:
        raise PlanError(f"{M} taps exceed the NLMS kernel's maximum of 4096")
    if nf > nsm and M <= 2048:
        return (1 if M <= 512 else 2 if M <= 1024 else 4), 512
    return (1 if M <= 1024 else 2 if M <= 2048 else 4), NB_THREADS


def nlms_smem(M):
    Mpad = (M + 1) & ~1
    return (NLMS_TILE + Mpad + NB_PAD + NLMS_TILE + Mpad + 32 * NB_L + NB_L * (NB_L + 1) + NB_L) * 8 + NB_L * 4


def nlms_subblocks(n, M, block_len):
    """The (tile, first sample in the tile, length, user block) of every exact block nlms_block_kernel evaluates:
    1024-sample tiles of the n - M recurrence steps, 32-sample exact blocks inside a tile, cut short where a user
    block (block_len > 1) ends."""
    nsteps = n - M
    out, in_block, ub = [], 0, 0
    for ts in range(0, max(nsteps, 0), NLMS_TILE):
        tl = min(NLMS_TILE, nsteps - ts)
        kk0 = 0
        while kk0 < tl:
            Lb = min(NB_L, tl - kk0)
            if block_len > 1:
                Lb = min(Lb, block_len - in_block)
            out.append((ts, kk0, Lb, ub))
            kk0 += Lb
            if block_len > 1:
                in_block += Lb
                if in_block == block_len:
                    in_block, ub = 0, ub + 1
    return out


# ------------------------------------------------------------------ the sweep
# (edge, n, R, F, shortFilt, window, fft_min_n): fast_xambg on the direct form; fft_min_n None runs with the FFT
# path off, a number with it on (the direct form is then the library's own choice)
CAF_CASES = [
    ("D1_F_nonpow2", 1500, 12, 1500, True, False, None),
    ("F1_one_block_over_all_ctas", 100003, 77, 1, True, True, None),
    ("F2_blocks_over_many_ctas", 2 ** 16 + 1, 40, 2, True, False, None),
    ("D31_lagcorr", 31 * 256 + 17, 99, 256, True, True, None),
    ("D32_flattop", 32 * 128 + 5, 45, 128, False, False, None),
    ("D62_ntaps63", 62 * 200 + 9, 20, 200, True, True, None),
    ("D63_ntaps64_cta_over_blocks", 63 * 128, 20, 128, True, True, None),
    ("D64_lagstream", 64 * 512 + 100, 300, 512, True, False, None),
    ("D64_flattop", 64 * 64 + 3, 130, 64, False, True, None),
    ("flattop_G32", 1024 * 250 + 7, 60, 1024, False, True, None),
    ("R1100_ct8", 2 ** 15, 1100, 64, True, True, None),
    ("R2600_G1_dft", 50000, 2600, 100, True, False, None),
    ("H512_ct8", 2 ** 16, 5119, 32, True, True, None),
    ("flattop_H512", 2 ** 14, 5119, 16, False, False, None),
    ("ct2_F4096", 4096 * 3 + 1, 50, 4096, True, False, None),
    ("ct1_F8192", 8192 * 4 + 3, 30, 8192, True, True, None),
    ("dft_F16384", 16384 * 2 + 5, 20, 16384, True, False, None),
    ("fft_on_R3073", 2 ** 17, 3073, 512, True, True, FFT_MIN_N),
    ("fft_on_R5119", 2 ** 17 + 77, 5119, 64, True, True, FFT_MIN_N),
    ("fft_on_R4000_nowin", 2 ** 17, 4000, 128, True, False, FFT_MIN_N),
    ("fft_on_flattop_nchunk_loop", 2 ** 19, 5119, 2048, False, False, FFT_MIN_N),
]

# (edge, n, filter_len, peek): LS_Filter and LS_Filter_Toeplitz below fft_min_n (the library's default switch-over)
LS_CASES = [
    ("M1_peek0", 300, 1, 0), ("M9", 1000, 9, 0), ("M10", 777, 5, 5), ("M11", 4096, 1, 10),
    ("M1024_levinson1", 8191, 1014, 10), ("M1025_levinson4", 5000, 1025, 0), ("M2048", 8191, 2038, 10),
    ("M2048_peek0", 6000, 2048, 0),
]
# LS_Filter_Toeplitz with peek >= n / 2 (the rolled reference wraps at n - peek)
TOEP_WRAP_CASES = [("peek_half", 600, 5, 300), ("peek_most", 1000, 3, 900)]

# (edge, n, filter_len, peek, block_len, initial taps)
NLMS_CASES = [
    ("M1_last1", 1 + 1025, 1, 0, 1, False),
    ("M2_fl0_last31", 2 + 2048 + 31, 0, 2, 2, False),
    ("M31_last32", 31 + 2048 + 32, 21, 10, 31, False),
    ("M32_last33", 32 + 1024 + 33, 32, 0, 33, False),
    ("M33_last1024", 33 + 3072, 23, 10, 1000, False),
    ("M64_last1", 64 + 2049, 54, 10, 1025, False),
    ("M65_block_over_frame", 65 + 5000, 65, 0, 10000, False),
    ("M511_last33", 511 + 4096 + 33, 501, 10, 1, False),
    ("M512_init", 512 + 3000, 502, 10, 31, True),
    ("M513_last31", 513 + 2048 + 31, 513, 0, 1, False),
    ("M1024_last1024", 1024 + 2048, 1014, 10, 33, False),
    ("M1025_init_last1", 1025 + 1025, 1015, 10, 1, True),
    ("M2048_init", 2048 + 2081, 2038, 10, 1000, True),
    ("M2049_last32", 2049 + 1056, 2039, 10, 1, False),
    ("M4096_init", 4096 + 1055, 4086, 10, 1025, True),
]
NLMS_FRAME_M = (512, 513, 1025, 2048, 2049)       # prc_nlms_frames_c64 with more frames than SMs
NLMS_MU = 0.05


# ------------------------------------------------------------------ CPU: the twin's invariants
def _random_caf_shapes(rng, count):
    shapes = []
    for _ in range(count):
        F = int(rng.choice([1, 2, 3, 64, 100, 256, 1000, 1024, 4096, 8192, 16384]))
        D = int(rng.choice([1, 2, 31, 32, 62, 63, 64, 100, 500, 2048, int(rng.integers(1, 70000))]))
        n = F * D + int(rng.integers(0, F))
        if n >= 2 ** 31 - 4096 or n < 1:
            continue
        R = int(rng.choice([0, 9, 10, 79, 80, 2559, 2560, 5110, 5119, int(rng.integers(0, 5120))]))
        shapes.append((n, R, F, bool(rng.integers(0, 2)), bool(rng.integers(0, 2))))
    return shapes


def _case_shapes():
    return [(n, R, F, short, win) for _, n, R, F, short, win, _ in CAF_CASES]


def test_twin_plans_fit_shared_memory_and_the_block_size():
    rng = np.random.default_rng(11)
    for nsm in NSM_H100:
        for n, R, F, short, win in _case_shapes() + _random_caf_shapes(rng, 1500):
            p = caf_direct(n, R, F, win, short, nsm)
            g = p.geo
            assert g.smem <= SMEM_LIMIT and 32 <= g.threads <= 512 and g.H * g.G <= g.threads, (n, R, F, p)
            assert g.HT >= R + 1 and g.HT % TILE_D == 0 and g.G >= 1 and g.steps >= 1
            if p.kernel == "lagcorr":
                assert g.nchunk * g.chunk_len >= p.ntaps > (g.nchunk - 1) * g.chunk_len
                assert g.G * g.steps * TILE_I >= g.chunk_len
            else:
                assert g.G * g.steps * TILE_I <= g.per_cta + g.G * TILE_I or g.steps == 1
        for M in list(range(1, 40)) + [511, 512, 513, 1023, 1024, 1025, 2047, 2048]:
            for n in (M + 1, 300, 1000, 4096, 8191):
                if n <= M:
                    continue
                p = ls_direct(n, M, nsm)
                assert max(p.stream.smem, p.lev_smem, p.fir_smem) <= SMEM_LIMIT, (n, M, p)
                assert p.Mpad >= M and p.Mpad % TILE_I == 0 and p.Mpad % 2 == 0
                assert p.stream.maxpieces == p.stream.ncta          # levinson sums every CTA's row
        for M in range(1, 4097):
            for nf in (1, nsm + 1):
                KT, NT = nlms_kernel(M, nf, nsm)
                assert KT * NT >= M and nlms_smem(M) <= SMEM_LIMIT


def _stream_shapes(rng):
    shapes = [(ntaps, F, R) for n, R, F, short, _ in _case_shapes() for ntaps in [n // F + 1] if short and ntaps >= 64]
    for _ in range(400):
        shapes.append((int(rng.integers(64, 300000)), int(rng.integers(1, 3000)), int(rng.integers(0, 5120))))
    return shapes


def test_stream_pieces_tile_every_block_exactly_once():
    """Every sample of the stream belongs to exactly one (CTA, piece) and the pieces of block j are the CTAs
    stream_first_cta(j) .. + stream_pieces(j) - 1, each a row below maxpieces."""
    rng = np.random.default_rng(12)
    for nsm in NSM_H100:
        for blk_len, F, R in _stream_shapes(rng):
            if F * blk_len > 4_000_000:
                F = max(1, 4_000_000 // blk_len)
            sg = choose_stream(blk_len, F, 1, R + 1, nsm)
            j = np.arange(F, dtype=np.int64)
            first = (j * blk_len) // sg.per_cta
            pieces = ((j + 1) * blk_len - 1) // sg.per_cta - first + 1
            assert (pieces >= 1).all() and int(pieces.max()) <= sg.maxpieces, (blk_len, F, R, sg)
            assert sg.maxpieces <= sg.ncta
            # the CTAs a block's pieces name cover its samples: piece k of block j is CTA first + k
            lo = np.maximum(j * blk_len, (first + pieces - 1) * sg.per_cta)
            hi = np.minimum((j + 1) * blk_len, (first + pieces) * sg.per_cta)
            assert (lo < hi).all()                                        # the last piece is not empty
            assert ((first * sg.per_cta) <= j * blk_len).all() and ((first + 1) * sg.per_cta > j * blk_len).all()
            # the CTAs' ranges cut the stream into consecutive pieces: summed over blocks, every CTA is counted once
            # per block it touches, and the total is what the CTAs' own walks flush
            flushes = sum(min((c + 1) * sg.per_cta, sg.total) // blk_len - (c * sg.per_cta) // blk_len
                          + (1 if min((c + 1) * sg.per_cta, sg.total) % blk_len else 0)
                          for c in range(sg.ncta))
            assert flushes == int(pieces.sum()), (blk_len, F, R, sg)
            assert (sg.ncta - 1) * sg.per_cta < sg.total <= sg.ncta * sg.per_cta


def test_maxpieces_is_the_largest_count_a_block_can_need():
    """maxpieces = (blk_len + per_cta - 2) // per_cta + 1 (capped at ncta) is reached by some block start offset:
    without the + 1 a block that starts late in a CTA's range would write a row past its slots."""
    for blk_len in (64, 65, 100, 2049, 10000):
        for per_cta in (1, 7, 63, 64, 65, 640, 10001):
            bound = (blk_len + per_cta - 2) // per_cta + 1
            worst = max(((o + blk_len - 1) // per_cta) - (o // per_cta) + 1 for o in range(per_cta))
            assert worst == bound, (blk_len, per_cta, worst, bound)


def _edges(nsm):
    """{edge: [cases that reach it]} over the sweep at nsm SMs."""
    reach = {}

    def hit(edge, case):
        reach.setdefault(edge, []).append(case)

    for edge, n, R, F, short, win, fmin in CAF_CASES:
        p = caf_direct(n, R, F, win, short, nsm, fmin)
        if p.kernel == "fft":
            continue
        g = p.geo
        if p.kernel == "lagstream":
            if blocks_per_cta(g, p.ntaps) >= 3:
                hit("cta_range_covers_3_blocks", edge)
            if max(stream_pieces(j, p.ntaps, g.per_cta) for j in range(F)) >= 3:
                hit("block_split_over_3_ctas", edge)
            if g.steps == 1:
                hit("stream_steps_1", edge)
            if p.ntaps == 64:
                hit("ntaps64_lagstream", edge)
        else:
            if g.doublings:
                hit("lagcorr_nchunk_loop", edge)
            if p.ntaps == 63:
                hit("ntaps63_lagcorr", edge)
            if p.ntaps == 1:
                hit("D1_one_tap", edge)
            if not short and n // F > 1:
                hit("tap_weighted_decimator", edge)
        if g.G == 1 and g.H > 256:
            hit(f"G1_H_over_256_{p.kernel}", edge)
        if g.G == 32:
            hit(f"G32_cap_{p.kernel}", edge)
        if g.H == 512:
            hit(f"H512_{p.kernel}", edge)
        if (R + 1) % TILE_D:
            hit("lags_not_multiple_of_TD", edge)
        hit(f"doppler_{p.doppler}", edge)
        if p.doppler == "ct2" and F <= 1024:
            hit("doppler_ct2_small_grid", edge)
        if F == 1:
            hit("F1", edge)
        if n % F:
            hit("n_not_multiple_of_F", edge)
        hit("window" if win else "no_window", edge)
        if fmin is not None and R > 3072:
            hit("R_over_3072_fft_on", edge)
    for edge, n, fl, peek in LS_CASES:
        M = fl + peek
        p = ls_direct(n, M, nsm)
        hit(f"levinson{p.levinson}_M{M}" if M in (1024, 1025, 2048) else f"ls_M{M}", edge)
        if peek == 0:
            hit("ls_peek0", edge)
    for edge, n, fl, peek, B, init in NLMS_CASES:
        M = fl + peek
        KT, NT = nlms_kernel(M, 1, nsm)
        hit(f"nlms_KT{KT}_NT{NT}", edge)
        hit(f"nlms_M{M}", edge)
        if M < NB_L:
            hit("nlms_M_below_32", edge)
        if fl == 0:
            hit("nlms_filter_len_0", edge)
        if peek == 0:
            hit("nlms_peek_0", edge)
        if init and KT == 4:
            hit("nlms_init_KT4", edge)
        sub = nlms_subblocks(n, M, B)
        last_tile = (n - M) - sub[-1][0]
        if last_tile in (1, 31, 32, 33, 1024):
            hit(f"nlms_last_tile_{last_tile}", edge)
        if B > 1:
            hit(f"nlms_block_len_{B}" if B <= 1025 else "nlms_block_longer_than_frame", edge)
            ends = {}
            for ts, kk0, Lb, ub in sub:
                ends.setdefault(ub, set()).add(ts)
            if any(len(t) > 1 for t in ends.values()):
                hit("nlms_user_block_straddles_tile", edge)
            if any(Lb < NB_L and kk0 + Lb < min(NLMS_TILE, n - M - ts) for ts, kk0, Lb, _ in sub):
                hit("nlms_user_block_ends_inside_exact_block", edge)
    for M in NLMS_FRAME_M:
        KT, NT = nlms_kernel(M, nsm + 1, nsm)
        hit(f"nlms_frames_KT{KT}_NT{NT}", f"frames_M{M}")
    return reach


EXPECTED_EDGES = [
    "cta_range_covers_3_blocks", "block_split_over_3_ctas", "stream_steps_1", "lagcorr_nchunk_loop",
    "G1_H_over_256_lagstream", "G1_H_over_256_lagcorr", "G32_cap_lagstream", "G32_cap_lagcorr", "H512_lagstream",
    "H512_lagcorr", "lags_not_multiple_of_TD", "ntaps63_lagcorr", "ntaps64_lagstream", "D1_one_tap",
    "tap_weighted_decimator", "doppler_ct8", "doppler_ct2", "doppler_ct2_small_grid", "doppler_ct1", "doppler_dft",
    "F1", "n_not_multiple_of_F", "window", "no_window", "R_over_3072_fft_on",
    "levinson1_M1024", "levinson4_M1025", "levinson4_M2048", "ls_M1", "ls_M9", "ls_M10", "ls_M11", "ls_peek0",
    "nlms_M_below_32", "nlms_filter_len_0", "nlms_peek_0", "nlms_init_KT4",
    "nlms_last_tile_1", "nlms_last_tile_31", "nlms_last_tile_32", "nlms_last_tile_33", "nlms_last_tile_1024",
    "nlms_block_len_2", "nlms_block_len_31", "nlms_block_len_33", "nlms_block_len_1000", "nlms_block_len_1025",
    "nlms_block_longer_than_frame", "nlms_user_block_straddles_tile", "nlms_user_block_ends_inside_exact_block",
    "nlms_KT1_NT1024", "nlms_KT2_NT1024", "nlms_KT4_NT1024",
    "nlms_frames_KT1_NT512", "nlms_frames_KT2_NT512", "nlms_frames_KT4_NT512", "nlms_frames_KT4_NT1024",
] + [f"nlms_M{M}" for M in (1, 2, 31, 32, 33, 64, 65, 511, 512, 513, 1024, 1025, 2048, 2049, 4096)]


@pytest.mark.parametrize("nsm", NSM_H100)
def test_sweep_reaches_every_edge(nsm):
    reach = _edges(nsm)
    missing = [e for e in EXPECTED_EDGES if e not in reach]
    assert not missing, f"edges no case reaches at {nsm} SMs: {missing}"
    for edge in EXPECTED_EDGES:
        print(f"{edge}: {reach[edge][0]}")


def test_twin_edges_sit_where_the_library_puts_them():
    """Spot values of the branches, read off prcore_corr.cu, so that an edit of the twin shows up here."""
    assert caf_direct(62 * 200 + 9, 20, 200, False, True, 132).kernel == "lagcorr"
    assert caf_direct(63 * 128, 20, 128, False, True, 132).kernel == "lagstream"
    assert caf_direct(63 * 128, 20, 128, False, False, 132).kernel == "lagcorr"      # taps: always lagcorr
    assert caf_direct(2 ** 17, 3072, 512, True, True, 132, FFT_MIN_N).kernel == "fft"
    assert caf_direct(2 ** 17, 3073, 512, True, True, 132, FFT_MIN_N).kernel == "lagstream"
    assert caf_direct(31 * 1024, 100, 1024, False, True, 132, FFT_MIN_N).kernel == "lagcorr"   # D < 32
    with pytest.raises(PlanError, match="maximum of 5120"):
        caf_direct(2 ** 17, 5120, 64, False, True, 132)
    with pytest.raises(PlanError, match="maximum of 5120"):
        caf_direct(2 ** 14, 5120, 16, False, False, 132)
    assert caf_direct(2 ** 17, 5119, 64, False, True, 132).geo.H == 512
    # CT = 8 needs a grid of at least one CTA per SM; below it the 2-column kernel fills more SMs
    assert doppler_branch(1024, 8 * 132 - 1, 1, 132) == "ct8" and doppler_branch(1024, 8 * 131 - 1, 1, 132) == "ct2"
    assert doppler_branch(1024, 8 * 131 - 1, 1, 114) == "ct8"
    assert doppler_branch(2048, 5000, 1, 132) == "ct2" and doppler_branch(8192, 5, 1, 132) == "ct1"
    assert [doppler_branch(F, 5, 1, 132) for F in (1, 3, 16384)] == ["dft"] * 3
    assert ls_direct(1000, 1024, 132).levinson == 1 and ls_direct(2000, 1025, 132).levinson == 4
    assert ls_direct(1000, 11, 132).Mpad == 20 and ls_direct(1000, 1, 132).Mpad == 10 and ls_direct(1000, 2048, 132).Mpad == 2050
    assert nlms_kernel(2048, 133, 132) == (4, 512) and nlms_kernel(2049, 133, 132) == (4, 1024)
    assert nlms_kernel(2048, 132, 132) == (2, 1024)
    assert [len(nlms_subblocks(M + s, M, 1)) for M, s in ((1, 1025), (10, 1024), (10, 1056))] == [33, 32, 33]
    assert [b[2] for b in nlms_subblocks(10 + 70, 10, 33)] == [32, 1, 32, 1, 4]


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture
def fft_options():
    """Restore the library's "fft" and "fft_min_n" options after a test that sets them."""
    old = (_lib.get_option("fft"), _lib.get_option("fft_min_n"))
    yield
    _lib.set_option("fft", old[0])
    _lib.set_option("fft_min_n", old[1])


def _set_path(fft_min_n):
    if fft_min_n is None:
        _lib.set_option("fft", 0)
    else:
        _lib.set_option("fft", 1)
        _lib.set_option("fft_min_n", fft_min_n)


def _nsm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _counted(call):
    """(result, {kernel: launches} of prc_profile_read, prc_launch_count delta) of one call."""
    _lib.profile_reset()
    _lib.profile(True)
    try:
        before = _lib.launch_count()
        res = call()
        launches = _lib.launch_count() - before
        prof = {k: v[1] for k, v in _lib.profile_read().items() if v[1]}
    finally:
        _lib.profile(False)
        _lib.profile_reset()
    return res, prof, launches


def rel(a, b, den):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / den)


# ------------------------------------------------------------------ GPU: the CAF on the direct form
@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,R,F,short,win,fmin", CAF_CASES, ids=[c[0] for c in CAF_CASES])
def test_caf_direct_form_at_the_planner_edges(edge, n, R, F, short, win, fmin, fft_options):
    nsm = _nsm()
    _set_path(fmin)
    plan = caf_direct(n, R, F, win, short, nsm, fmin)
    assert plan.kernel != "fft", (edge, plan)
    ref, srv = synth.make_frame(n, "P0", 1300 + F)
    w = signal.get_window(("kaiser", 5.0), n) if win else None
    got = prb.fast_xambg(ref, srv, R, F, n, w, short)[:, :, 0]
    truth = xo.fast_xambg_truth(ref, srv, R, F, None, w, short, fast=True)[:, :, 0]
    e = rel(got, truth, np.abs(truth).max())
    assert e <= TOL, (edge, plan, e)
    # the same call again, its twiddles cached: the launches are the twin's
    again, prof, launches = _counted(lambda: prb.fast_xambg(ref, srv, R, F, n, w, short)[:, :, 0])
    assert np.array_equal(again, got), edge
    want = dict(zip(("lagcorr_caf", "misc", "doppler_fft"), plan.profile))
    assert prof == {k: v for k, v in want.items() if v}, (edge, plan, prof)
    assert launches == plan.launches, (edge, plan, launches)
    g = plan.geo
    record_parity(f"direct/caf_{edge}", E=e, nsm=nsm, kernel=plan.kernel, doppler=plan.doppler, H=g.H, G=g.G,
                  steps=g.steps, ctas=g.ncta if plan.kernel == "lagstream" else F * g.nchunk)


@pytest.mark.gpu
def test_caf_direct_form_with_strong_clutter(fft_options):
    """P1: the map is dominated by the direct-path clutter the channels share; held to 1e-5 + 1.2 x the reference's
    own complex64 error against the same truth (lagstream with a window, and the tap-weighted decimator)."""
    nsm = _nsm()
    _set_path(None)
    n, R, F = 63 * 256 + 11, 70, 256
    ref, srv = synth.make_frame(n, "P1", 1400)
    w = signal.get_window(("kaiser", 5.0), n)
    fig = {}
    for short in (True, False):
        got = prb.fast_xambg(ref, srv, R, F, n, w, short)[:, :, 0]
        truth = xo.fast_xambg_truth(ref, srv, R, F, None, w, short, fast=True)[:, :, 0]
        own = xo.fast_xambg_oracle(ref, srv, R, F, n, w, short)[:, :, 0]
        den = np.abs(truth).max()
        e, r = rel(got, truth, den), rel(own, truth, den)
        assert e <= TOL + 1.2 * r, (short, caf_direct(n, R, F, True, short, nsm), e, r)
        fig[f"E_short{short}"], fig[f"reference_vs_truth_short{short}"] = e, r
    record_parity("direct/caf_P1", **fig)


@pytest.mark.gpu
def test_caf_lag_limit_of_the_direct_form(fft_options):
    """R + 1 = 5120 lags run (H = 512 lag groups); 5121 are refused before any launch, with the limit in the message,
    on the boxcar (lagstream) and the tap-weighted (lagcorr) decimator, with the FFT path on and off."""
    import torch
    lib = _lib.load()
    n, F = 2 ** 17, 64
    ref, srv = synth.make_frame(n, "P0", 1500)
    for fmin in (None, FFT_MIN_N):
        _set_path(fmin)
        for short in (True, False):
            dt = None if short else np.ascontiguousarray(signal.firwin(10 * (n // F) + 1, 1. / (n // F), window="flattop"))
            for R, ok in ((5119, True), (5120, False)):
                out = np.empty((F, R + 1), np.complex64)
                before = _lib.launch_count()
                st = lib.prc_xambg_c64(ref.ctypes.data, srv.ctypes.data, n, R, F, None,
                                       None if dt is None else dt.ctypes.data, 0 if dt is None else dt.shape[0],
                                       out.ctypes.data, _lib.MEM_HOST, 0, None, 0)
                if ok:
                    assert st == _lib.PRC_OK, (fmin, short, lib.prc_last_error())
                else:
                    assert st == _lib.PRC_E_INVALID, (fmin, short, st)
                    assert b"5121 lags exceed the supported maximum of 5120" in lib.prc_last_error()
                    assert _lib.launch_count() - before == (0 if short else 1)       # only the taps' conversion
    torch.cuda.synchronize()
    record_parity("direct/caf_lag_limit", largest_range_bins=5119)


# ------------------------------------------------------------------ GPU: LS_Filter / LS_Filter_Toeplitz
@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,fl,peek", LS_CASES, ids=[c[0] for c in LS_CASES])
def test_ls_direct_form_at_the_planner_edges(edge, n, fl, peek, fft_options):
    """The library's default options: every case is below fft_min_n, so ls_device takes its direct branch."""
    nsm = _nsm()
    _set_path(FFT_MIN_N)
    M = fl + peek
    assert not ls_plan(n, M).on
    plan = ls_direct(n, M, nsm)
    ref, srv = synth.make_frame(n, "P1", 1600 + M)
    den = float(np.abs(srv).max())
    fig = {}
    t_out, t_taps = co.ls_filter_truth(ref, srv, fl, 1.0, peek)
    (out, taps), prof, launches = _counted(lambda: prb.LS_Filter(ref, srv, fl, 1.0, peek, True))
    fig["E_taps"], fig["E_cleaned"] = rel(taps, t_taps, np.abs(t_taps).max()), rel(out, t_out, den)
    assert max(fig.values()) <= TOL, (edge, plan, fig)
    assert prof == {"lagcorr_ls": 1, "levinson": 1, "fir_apply": 1} and launches == 3, (edge, prof, launches)
    t_out, t_taps = co.ls_filter_toeplitz_truth(ref, srv, fl, peek)
    (out, taps), prof, launches = _counted(lambda: prb.LS_Filter_Toeplitz(ref, srv, fl, peek, True))
    fig["E_toeplitz_taps"], fig["E_toeplitz_cleaned"] = rel(taps, t_taps, np.abs(t_taps).max()), rel(out, t_out, den)
    assert max(fig.values()) <= TOL, (edge, plan, fig)
    assert prof == {"lagcorr_ls": 1, "levinson": 1, "fir_apply": 1, "misc": 1} and launches == 4, (edge, prof, launches)
    s = plan.stream
    record_parity(f"direct/ls_{edge}", nsm=nsm, levinson=plan.levinson, ctas=s.ncta, G=s.G, steps=s.steps, **fig)


@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,fl,peek", TOEP_WRAP_CASES, ids=[c[0] for c in TOEP_WRAP_CASES])
def test_toeplitz_direct_form_with_peek_past_half_the_frame(edge, n, fl, peek, fft_options):
    _set_path(FFT_MIN_N)
    ref, srv = synth.make_frame(n, "P0", 1700 + peek)
    t_out, t_taps = co.ls_filter_toeplitz_truth(ref, srv, fl, peek)
    out, taps = prb.LS_Filter_Toeplitz(ref, srv, fl, peek, True)
    e_taps, e_out = rel(taps, t_taps, np.abs(t_taps).max()), rel(out, t_out, np.abs(srv).max())
    assert e_taps <= TOL and e_out <= TOL, (edge, e_taps, e_out)
    record_parity(f"direct/toeplitz_{edge}", E_taps=e_taps, E_cleaned=e_out)


# ------------------------------------------------------------------ GPU: NLMS / block_NLMS
def _init_taps(M, seed):
    rng = np.random.default_rng(seed)
    return (0.02 * (rng.standard_normal(M) + 1j * rng.standard_normal(M))).astype(np.complex64)


@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,fl,peek,B,init", NLMS_CASES, ids=[c[0] for c in NLMS_CASES])
def test_nlms_at_the_tiling_edges(edge, n, fl, peek, B, init):
    M = fl + peek
    ref, srv = synth.make_frame(n, "P1", 1800 + M)
    w0 = _init_taps(M, M) if init else None
    (got, gw), prof, launches = _counted(lambda: prb.block_NLMS(ref, srv, fl, NLMS_MU, peek, B, w0, True))
    assert prof == {"nlms": 1} and launches == 1, (edge, prof, launches)
    want = co.block_nlms_oracle_c(ref, srv, fl, NLMS_MU, peek, B, w0)
    truth = co.block_nlms_truth_c(ref, srv, fl, NLMS_MU, peek, B, w0)
    fig = _nlms_bounds(got, gw, *want, *truth, edge)
    assert not got[:fl].any() and not got[n - peek:].any(), edge
    assert np.abs(got[fl:n - peek]).min() > 0, edge
    KT, NT = nlms_kernel(M, 1, _nsm())
    record_parity(f"direct/nlms_{edge}", KT=KT, NT=NT, last_tile=(n - M - 1) % NLMS_TILE + 1, **fig)


@pytest.mark.gpu
@pytest.mark.parametrize("fl,peek", [(1, 0), (0, 1), (2, 0), (3, 2)])
def test_nlms_with_fewer_taps_than_an_exact_block_keeps_small_powers(fl, peek):
    """Regression: with M < 32 the Gram windows g(m, k) of an exact block were formed by telescoping sliding-window
    increments, so the power p_m of a one- or two-sample regressor near zero came out as the rounding of its
    neighbours' products, and mu / p_m put that into the taps (M = 1: 6.4e-4 of max|truth| on an H100).  Each window
    is now summed directly."""
    M = fl + peek
    n = 4096 + M
    ref, srv = synth.make_frame(n, "P1", 2000 + M)
    got, gw = prb.NLMS_filter(ref, srv, fl, NLMS_MU, peek, None, True)
    want = co.block_nlms_oracle_c(ref, srv, fl, NLMS_MU, peek, 1)
    truth = co.block_nlms_truth_c(ref, srv, fl, NLMS_MU, peek, 1)
    fig = _nlms_bounds(got, gw, *want, *truth, (fl, peek))
    assert fig["out_vs_truth"] <= 1e-6, fig
    record_parity(f"direct/nlms_short_window_M{M}_peek{peek}", **fig)


@pytest.mark.gpu
@pytest.mark.parametrize("M", NLMS_FRAME_M)
def test_nlms_frames_past_the_sm_count_at_the_kt_edges(M):
    """prc_nlms_frames_c64 with more frames than SMs: 512-thread CTAs up to M = 2048 (KT = 1 / 2 / 4 either side of
    512 and 1024 taps), 1024-thread CTAs at 2049.  Four distinct frames repeated; every distinct row is held to the
    float64 recurrence and the reference arithmetic, its repeats are bit-identical, and its zero head and tail hold."""
    import torch
    nsm = _nsm()
    nf = nsm + 5
    n, peek = M + 1024 + 33, 10
    fl = M - peek
    base = [synth.make_frame(n, "P1", 1900 + i) for i in range(4)]
    dev = torch.device("cuda", 0)
    ref_d = torch.from_numpy(np.stack([base[i % 4][0] for i in range(nf)])).to(dev)
    srv_d = torch.from_numpy(np.stack([base[i % 4][1] for i in range(nf)])).to(dev)
    out = torch.empty((nf, n), dtype=torch.complex64, device=dev)
    taps = torch.empty((nf, M), dtype=torch.complex64, device=dev)
    lib = _lib.load()
    _, prof, launches = _counted(lambda: _lib.check(lib.prc_nlms_frames_c64(
        ref_d.data_ptr(), srv_d.data_ptr(), n, nf, n, fl, peek, NLMS_MU, 1, None, out.data_ptr(), taps.data_ptr(),
        _lib.MEM_DEVICE, 0, None, 0)))
    assert prof == {"nlms": 1} and launches == 1, (prof, launches)
    got, gt = out.cpu().numpy(), taps.cpu().numpy()
    fig = {}
    for k, (ref, srv) in enumerate(base):
        want = co.block_nlms_oracle_c(ref, srv, fl, NLMS_MU, peek, 1)
        truth = co.block_nlms_truth_c(ref, srv, fl, NLMS_MU, peek, 1)
        for key, v in _nlms_bounds(got[k], gt[k], *want, *truth, (M, k)).items():
            fig[key] = max(fig.get(key, 0.0), v)
        assert not got[k, :fl].any() and not got[k, n - peek:].any(), k
        for i in range(k + 4, nf, 4):
            assert np.array_equal(got[i], got[k]) and np.array_equal(gt[i], gt[k]), (k, i)
    KT, NT = nlms_kernel(M, nf, nsm)
    record_parity(f"direct/nlms_frames_M{M}", frames=nf, KT=KT, NT=NT, **fig)
