"""The one-pass FFT-domain frame (csrc/framepass.cuh): LS lag sums and the CAF's per-block spectra from one set of
window transforms, then the Toeplitz solve, W' and AccP - AccQ conj(W') per Doppler block.

CPU: every launch of framepass.cuh has a covering GPU test, and the build's ptxas log holds frame_pass_kernel<8> to two
CTAs per SM without spills.  GPU: prc_frames_c64 with the option "frame_onepass" at 1 (default) against the float64
frame truth and against the two-pass frame ("frame_onepass" = 0) on the same frames, at the headline shape, at the
edges of the one-pass plan, and for a batch larger than the spectra workspace's cap.
"""
import os
import re

import numpy as np
import pytest
import scipy.signal as signal

from conftest import record_parity
from passiveradar_b200 import _lib, synth
from oracle import clutter_oracle as co
from oracle import xambg_oracle as xo

HERE = os.path.dirname(os.path.abspath(__file__))
FRAMEPASS = os.path.join(HERE, "..", "passiveradar_b200", "csrc", "framepass.cuh")
TOL = 1.5e-6                 # P0 maps and taps against the float64 frame truth
L = 2048


def rel(a, b, den):
    return float(np.abs(np.asarray(a, np.complex128) - b).max() / den)


# ------------------------------------------------------------------ CPU
# every launch in framepass.cuh -> the GPU tests that reach it
COVERAGE = {
    "frame_pass_kernel<FP_R3>": ["test_headline_batches_match_truth_and_two_pass", "test_onepass_at_the_plan_edges"],
    "caf_combine_kernel<FP_R3>": ["test_headline_batches_match_truth_and_two_pass", "test_onepass_at_the_plan_edges"],
}


def test_every_framepass_launch_has_a_covering_gpu_test():
    src = open(FRAMEPASS).read()
    sites = {m.group(1) + (m.group(2) or "") for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", src)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    this = open(os.path.abspath(__file__)).read()
    for tests in COVERAGE.values():
        for t in tests:
            i = this.index(f"\ndef {t}(")
            decorators = this[this.rindex("\n\n", 0, i):i]
            assert "@pytest.mark.gpu" in decorators, f"{t} is not a GPU test"


def framepass_smem_bytes(r3=8):
    """fft::Geo<R3>::SMEM_FLOAT2 + staging L float2 + accC, accX 2 L float2 + window L float"""
    Lr = 256 * r3
    return (2 * 16 * 17 * r3 + Lr + 16 * r3 + 3 * Lr + Lr // 2) * 8


def expected_frame_ctas():
    import test_fft_residency as fr
    entries = fr.fftc_entries()
    regs, spills = entries[("frame_pass_kernel", 8, None)]
    return fr.ctas_per_sm(regs, 128, framepass_smem_bytes()), regs, spills


def test_frame_pass_fits_two_ctas_per_sm_without_spills():
    import test_fft_residency as fr
    assert framepass_smem_bytes() == 109568
    n, regs, spills = expected_frame_ctas()
    assert spills == "0 bytes spill stores, 0 bytes spill loads"
    assert n == 2, f"frame_pass_kernel<8>: {regs} registers x 128 threads, {framepass_smem_bytes()} B -> {n} CTAs per SM"
    regs_c, spills_c = fr.fftc_entries()[("caf_combine_kernel", 8, None)]
    assert spills_c == "0 bytes spill stores, 0 bytes spill loads", regs_c


# ------------------------------------------------------------------ GPU
def _frames(refs, srvs, fl, peek, R, F, w, onepass, profile=False):
    """prc_frames_c64 on device tensors with taps and the cleaned channel requested; returns numpy maps, taps, cleaned
    and whether the one-pass kernels ran"""
    import torch
    nf, n = refs.shape
    maps = torch.empty((nf, F, R + 1), dtype=torch.complex64, device=refs.device)
    taps = torch.empty((nf, fl + peek), dtype=torch.complex64, device=refs.device)
    clean = torch.empty((nf, n), dtype=torch.complex64, device=refs.device)
    flags, wp = 0, None
    if w is not None:
        flags = _lib.FLAG_WINDOW_F32 if w.dtype == torch.float32 else 0
        wp = w.data_ptr()
    old = _lib.get_option("frame_onepass")
    _lib.set_option("frame_onepass", onepass)
    try:
        if profile:
            _lib.profile_reset()
            _lib.profile(True)
        _lib.check(_lib.load().prc_frames_c64(refs.data_ptr(), srvs.data_ptr(), n, nf, n, fl, peek, 1.0, R, F, wp,
                                              maps.data_ptr(), taps.data_ptr(), clean.data_ptr(), _lib.MEM_DEVICE, 0,
                                              None, flags))
        torch.cuda.synchronize()
        ran = None
        if profile:
            prof = _lib.profile_read()
            ran = prof["caf_combine"][1] > 0
    finally:
        if profile:
            _lib.profile(False)
        _lib.set_option("frame_onepass", old)
    return maps.cpu().numpy(), taps.cpu().numpy(), clean.cpu().numpy(), ran


@pytest.mark.gpu
def test_frame_ctas_option_reports_what_the_build_fits():
    from passiveradar_b200 import build as b
    got = _lib.get_option("fft_ctas_frame")
    want = expected_frame_ctas()[0] if os.path.exists(os.path.join(b.PKG, "libprcore.ptxas.log")) else 2
    assert got == want == 2, (got, want)
    with pytest.raises(_lib.PrcoreError):
        _lib.set_option("fft_ctas_frame", got)


@pytest.mark.gpu
def test_headline_batches_match_truth_and_two_pass():
    """The headline shape (2^20 samples, 256 x 300, filterLen 300, peek 10, float32 Kaiser window): four distinct frames
    (P0, P1, P0, P1) repeated into batches of 25 and of 33 frames (over the 32 frames the 256 MiB spectra workspace holds
    at this shape, so the batch runs in two chunks).  Every row's taps and every P0 row's map are within 1.5e-6 of the
    float64 frame truth; every P1 map is no further from the truth than twice the two-pass frame's error on the same
    frame, and within 5e-4 of the two-pass map (the fused-versus-separate bound of the residual)."""
    import torch
    n, F, R, fl, peek = 2 ** 20, 256, 300, 300, 10
    profiles = ["P0", "P1", "P0", "P1"]
    base = [synth.make_frame(n, profiles[k], 1300 + k) for k in range(4)]
    w = signal.get_window(("kaiser", 5.0), n).astype(np.float32)
    truths = [xo.frame_truth(ref, srv, fl, 1.0, peek, R, F, w.astype(np.float64)) for ref, srv in base]
    dev = torch.device("cuda", 0)
    b_ref = torch.from_numpy(np.stack([f[0] for f in base])).to(dev)
    b_srv = torch.from_numpy(np.stack([f[1] for f in base])).to(dev)
    d_w = torch.from_numpy(w).to(dev)
    for nf in (25, 33):
        idx = torch.arange(nf, device=dev) % 4
        maps1, taps1, clean1, ran = _frames(b_ref[idx], b_srv[idx], fl, peek, R, F, d_w, 1, profile=True)
        assert ran
        maps0, taps0, _, ran0 = _frames(b_ref[idx], b_srv[idx], fl, peek, R, F, d_w, 0, profile=True)
        assert not ran0
        for i in range(nf):
            k = i % 4
            amb, t_taps, t_clean = truths[k]
            den = np.abs(amb).max()
            assert rel(taps1[i], t_taps, np.abs(t_taps).max()) <= TOL, (nf, i)
            assert rel(clean1[i], t_clean, np.abs(base[k][1]).max()) <= 1e-5, (nf, i)
            e1 = rel(maps1[i], amb, den)
            if profiles[k] == "P0":
                assert e1 <= TOL, (nf, i, e1)
            else:
                e0 = rel(maps0[i], amb, den)
                assert e1 <= 2 * e0, (nf, i, e1, e0)
                assert rel(maps1[i], maps0[i], np.abs(maps0[i]).max()) <= 5e-4, (nf, i)


# (edge, n, F, R, filter_len, peek, profile): shapes where the one-pass plan is on, at its edges (D = 32 and R + M near
# L are off: there the two passes cost fewer transforms; scripts/fft/model.py covers their algebra)
EDGE_CASES = [
    ("M=1", 2 ** 17, 16, 100, 1, 0, "P0"),
    ("M=2_peek=0", 2 ** 17, 16, 100, 2, 0, "P0"),
    ("M=2_peek=1", 2 ** 17, 16, 100, 1, 1, "P0"),
    ("peek=M-1", 2 ** 17, 16, 100, 1, 39, "P0"),
    ("F=1", 2 ** 14, 1, 100, 60, 10, "P0"),
    ("n_not_multiple_of_F", 2 ** 17 + 3, 7, 60, 30, 9, "P0"),
    ("Bmax=1429", 2 ** 17, 16, 300, 300, 10, "P0"),
    ("P1", 2 ** 17, 16, 100, 50, 10, "P1"),
    # segments at their limits (test_onepass_sweep.py's planner twin states each partition): blocks of 2 x Bmax under
    # the CAF limit, of 3 x (Bmax + 1) (what a CAF limit one too large would make), the same for the LS limit bls, a
    # tail of exactly bls and of bls + 1, segments and a tail of the whole transform, and the smallest Bmax the plan
    # takes (545 from a sample of shapes, and L / 4 = 512, the plan's floor)
    ("caf_exact", 45712, 16, 300, 300, 10, "P0"),
    ("caf_one_past", 68624, 16, 300, 300, 10, "P0"),
    ("ls_exact", 45744, 16, 100, 300, 10, "P0"),
    ("ls_one_past", 68672, 16, 100, 300, 10, "P0"),
    ("tail_exact", 45745, 16, 100, 300, 10, "P0"),
    ("tail_plus_one", 45746, 16, 100, 300, 10, "P0"),
    ("full_L", 65520, 16, 0, 1, 0, "P0"),
    ("full_L_tail", 65552, 16, 0, 1, 0, "P0"),
    ("smallest_Bmax", 1048708, 1024, 912, 564, 14, "P0"),
    ("Bmax=L/4", 523264, 1024, 768, 769, 0, "P0"),
    ("caf_exact_P1", 45712, 16, 300, 300, 10, "P1"),
    ("ls_exact_P1", 45744, 16, 100, 300, 10, "P1"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,F,R,fl,peek,prof", EDGE_CASES, ids=[c[0] for c in EDGE_CASES])
def test_onepass_at_the_plan_edges(edge, n, F, R, fl, peek, prof):
    """At the edges of the one-pass plan, with no window, a float64 window and PRC_FLAG_WINDOW_F32: the one-pass
    kernels run, taps and P0 maps are within 1.5e-6 of the float64 frame truth, and a P1 map is within 1e-5 + 1.2 x the
    reference chain's own error (LS_Filter -> fast_xambg in complex64) and no worse than twice the two-pass frame's."""
    import torch
    ref, srv = synth.make_frame(n, prof, 1400 + F)
    w64 = signal.get_window(("kaiser", 5.0), n)
    dev = torch.device("cuda", 0)
    refs = torch.from_numpy(ref[None]).to(dev)
    srvs = torch.from_numpy(srv[None]).to(dev)
    ref_err = None
    fig = {}
    for win in ("none", "f64", "f32"):
        w = None if win == "none" else (w64 if win == "f64" else w64.astype(np.float32))
        d_w = None if w is None else torch.from_numpy(w).to(dev)
        amb, t_taps, _ = xo.frame_truth(ref, srv, fl, 1.0, peek, R, F, None if w is None else w.astype(np.float64))
        maps1, taps1, _, ran = _frames(refs, srvs, fl, peek, R, F, d_w, 1, profile=True)
        assert ran, edge
        den = np.abs(amb).max()
        e_taps = rel(taps1[0], t_taps, np.abs(t_taps).max())
        assert e_taps <= TOL, (edge, win)
        e1 = rel(maps1[0], amb, den)
        fig[f"E_taps_{win}"], fig[f"E_map_{win}"] = e_taps, e1
        if prof == "P0":
            assert e1 <= TOL, (edge, win, e1)
            continue
        maps0, _, _, _ = _frames(refs, srvs, fl, peek, R, F, d_w, 0)
        e0 = rel(maps0[0], amb, den)
        if ref_err is None or win != "none":
            chain = xo.fast_xambg_oracle(ref, co.ls_filter_oracle(ref, srv, fl, 1.0, peek), R, F, n, w)[:, :, 0]
            ref_err = rel(chain, amb, den)
        fig[f"E_map_two_pass_{win}"], fig[f"reference_map_vs_truth_{win}"] = e0, ref_err
        assert e1 <= 1e-5 + 1.2 * ref_err and e1 <= 2 * e0, (edge, win, e1, e0, ref_err)
    record_parity(f"onepass/edge_{edge}", **fig)
