"""Residency of the FFT-domain correlation kernels (csrc/fftcorr.cuh) and the grids sized from it.

lscorr_fft_kernel and fir_fft_kernel launch one wave of CTAs for the whole batch, so their grids are only as good as
the number of CTAs an SM really holds.  On the CPU that number is worked out from the build's ptxas log and the
shared-memory layout of fftcorr.cuh against the H100's limits, and caf_fft_kernel's (one CTA per Doppler block) is
held to three per SM; on the GPU the library reports what it sized its grids from (prc_get_option "fft_ctas_*"), and
the fused frame path is checked at Doppler block counts that leave a partial last group of blocks.
"""
import os
import re

import numpy as np
import pytest
import scipy.signal as signal

from passiveradar_b200 import _lib, synth

# H100 (sm_90): per SM
REGS_PER_SM = 65536
SMEM_PER_SM = 233472            # 228 KB
SMEM_RESERVED_PER_CTA = 1024
MAX_WARPS_PER_SM = 64
MAX_CTAS_PER_SM = 32
REG_UNIT = 8                    # registers are allocated per thread in multiples of 8 (256 per warp)


def smem_bytes(kernel, r3):
    """Dynamic shared memory the kernel is launched with: fft::Geo<R3>::SMEM_FLOAT2 (two padded exchange buffers and
    the twiddle tables) plus the staging of fftcorr.cuh (lscorr/fir: L float2, caf: L float2 + L float)."""
    L = 256 * r3
    geo = 2 * 16 * 17 * r3 + L + 16 * r3
    extra = {"lscorr_fft_kernel": L, "fir_fft_kernel": L, "caf_fft_kernel": L + L // 2}[kernel]
    return (geo + extra) * 8


def ctas_per_sm(regs, threads, smem):
    warps = threads // 32
    per_warp = -(-regs // REG_UNIT) * REG_UNIT * 32
    by_regs = (REGS_PER_SM // per_warp) // warps
    by_smem = SMEM_PER_SM // (smem + SMEM_RESERVED_PER_CTA)
    return min(by_regs, by_smem, MAX_WARPS_PER_SM // warps, MAX_CTAS_PER_SM)


def fftc_entries():
    """{(kernel, r3, fused or None): (registers, spill text)} of every fftc:: entry in the build's ptxas log."""
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    out = {}
    for blk in open(log).read().split("Compiling entry function")[1:]:
        head = blk.split("\n")[0]
        m = re.search(r"_ZN3prc4fftc\d+(\w+?_kernel)ILi(\d+)(?:ELb([01]))?E", head)
        if not m:
            continue
        assert "'sm_90a'" in head
        regs = int(re.search(r"Used (\d+) registers", blk).group(1))
        spills = re.search(r"\d+ bytes spill stores, \d+ bytes spill loads", blk).group(0)
        fused = None if m.group(3) is None else m.group(3) == "1"
        out[(m.group(1), int(m.group(2)), fused)] = (regs, spills)
    return out


def expected_ctas(entries, kernel, r3):
    regs, _ = entries[(kernel, r3, None)]
    return ctas_per_sm(regs, 16 * r3, smem_bytes(kernel, r3))


# ------------------------------------------------------------------ CPU
def test_fftc_kernels_have_no_spills():
    entries = fftc_entries()
    names = {k[0] for k in entries}
    assert {"lscorr_fft_kernel", "fir_fft_kernel", "caf_fft_kernel", "taps_spectrum_kernel"} <= names, names
    for key, (_, spills) in entries.items():
        assert spills == "0 bytes spill stores, 0 bytes spill loads", (key, spills)


def test_lscorr_fft_r3_8_fits_three_ctas_per_sm():
    entries = fftc_entries()
    regs, _ = entries[("lscorr_fft_kernel", 8, None)]
    assert smem_bytes("lscorr_fft_kernel", 8) == 68608
    n = expected_ctas(entries, "lscorr_fft_kernel", 8)
    assert n >= 3, f"lscorr_fft_kernel<8>: {regs} registers x 128 threads -> {n} CTAs per SM"


def test_residency_model_matches_the_known_h100_limits():
    # 175 registers (rounded to 176) x 128 threads = 22 528: two CTAs in 65 536; 168 x 128 = 21 504: three
    assert ctas_per_sm(175, 128, 68608) == 2
    assert ctas_per_sm(168, 128, 68608) == 3
    # caf_fft_kernel<8, *>: 76 800 B + 1 KB three times is the whole 233 472 B
    assert smem_bytes("caf_fft_kernel", 8) == 76800
    assert ctas_per_sm(128, 128, 76800) == 3
    # R3 = 16: 137 KB of shared memory, one CTA per SM whatever the registers
    assert ctas_per_sm(64, 256, smem_bytes("lscorr_fft_kernel", 16)) == 1


# ------------------------------------------------------------------ GPU
OPTIONS = {"fft_ctas_ls": "lscorr_fft_kernel", "fft_ctas_fir": "fir_fft_kernel"}


@pytest.mark.gpu
def test_residency_options_report_what_the_build_fits():
    from passiveradar_b200 import build as b
    have_log = os.path.exists(os.path.join(b.PKG, "libprcore.ptxas.log"))
    entries = fftc_entries() if have_log else None
    for name, kernel in OPTIONS.items():
        got = _lib.get_option(name)
        want = expected_ctas(entries, kernel, 8) if entries else 3
        assert got == want, (name, got, want)
        with pytest.raises(_lib.PrcoreError):
            _lib.set_option(name, got)
    assert _lib.get_option("fft_ctas_ls") >= 3


def _fused_maps(n, F, R, fl, frames, batch):
    from passiveradar_b200.frames import FramePipeline
    pipe = FramePipeline(n, R, F, filter_len=fl, batch=batch, nslots=1)
    return pipe.run_host(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))


@pytest.mark.gpu
@pytest.mark.parametrize("n,F,R,fl,nf", [
    (2 ** 17, 6, 50, 50, 3),            # F not a multiple of 4 (Doppler blocks per CTA group)
    (2 ** 17, 13, 100, 40, 2),          # odd F, one frame per call and a batch of two
    (2 ** 16, 3, 40, 30, 1),            # one frame, F < 4
])
def test_fused_frames_at_small_and_odd_doppler_counts(n, F, R, fl, nf):
    """prc_frames_c64 on the FFT path (clutter filter fused into caf_fft_kernel) against the float64 LS filter
    followed by the CAF oracle, one frame per call and the whole batch in one call."""
    from oracle import clutter_oracle as co
    from oracle import xambg_oracle as xo
    frames = [synth.make_frame(n, "P0", frame=250 + i) for i in range(nf)]
    old = (_lib.get_option("fft"), _lib.get_option("fft_min_n"))
    try:
        _lib.set_option("fft", 1)
        _lib.set_option("fft_min_n", 8192)
        res = [_fused_maps(n, F, R, fl, frames, batch) for batch in sorted({1, nf})]
    finally:
        _lib.set_option("fft", old[0])
        _lib.set_option("fft_min_n", old[1])
    w = signal.get_window(("kaiser", 5.0), n)
    worst = 0.0
    for maps in res:
        assert maps.shape[0] == nf
        for i, (ref, srv) in enumerate(frames):
            t_clean, _ = co.ls_filter_truth(ref, srv, fl, 1.0, 10)
            want = xo.fast_xambg_oracle(ref, t_clean.astype(np.complex64), R, F, n, w)
            worst = max(worst, float(np.abs(maps[i].reshape(want.shape) - want).max() / np.abs(want).max()))
    assert worst <= 1e-5, worst
