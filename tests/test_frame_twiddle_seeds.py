"""frame_pass_kernel's pass-1 / pass-3 twiddles from per-thread seeds (csrc/fftcore.cuh: Tw1Seeds, SmemSeeded).

The one-pass frame kernel forms each twiddle W_2048^{t k1} from five float64-built table values held in registers, at
most one product of two of them, instead of reading the tw1 table from shared memory.  CPU: ``scripts/fft/emul.cu
seeds`` runs the seeded pass functions thread by thread (host rounding of the same expressions) against float64; every
twiddle is within 2 ulp of 1.0 and each transform's error (test_fft_emulation.py's definitions: largest error over
largest magnitude) within 1.5x the table transform's.  The shared-memory layout without tw1 and the build's ptxas log
hold the kernel to two CTAs per SM without spills.  GPU: the one-pass frame at the headline shape and at two plan edges
against the float64 frame truth at the bounds of test_frame_onepass.py.
"""
import os
import subprocess

import numpy as np
import pytest
import scipy.signal as signal

from conftest import record_parity
from test_fft_emulation import ROOT, _nvcc

L, R3, T = 2048, 8, 128
ULP = 2.0 ** -23                     # 1 ulp of 1.0 in float32


@pytest.fixture(scope="module")
def seeds_report(tmp_path_factory):
    if _nvcc() is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("emul") / "fft_emul")
    res = subprocess.run([_nvcc(), "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-I",
                          os.path.join(ROOT, "passiveradar_b200", "csrc"), "-o", exe,
                          os.path.join(ROOT, "scripts", "fft", "emul.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    run = subprocess.run([exe, "seeds"], capture_output=True, text=True)
    assert run.returncode == 0, run.stdout + run.stderr
    return {k: float(v) for k, v in (kv.split("=") for kv in run.stdout.split())}


def framepass_seeded_smem_bytes():
    """SmemSeeded<8> (two padded exchange buffers + tw2) + staging L float2 + accC, accX 2 L float2 + window L float"""
    return (2 * 16 * 17 * R3 + 16 * R3 + 3 * L + L // 2) * 8


# ------------------------------------------------------------------ CPU
def test_every_seeded_twiddle_is_within_two_ulp_of_float64(seeds_report):
    assert seeds_report["twiddle_ulp"] <= 2.0, seeds_report


@pytest.mark.parametrize("direction", ["n2p", "p2n"])
def test_seeded_transform_error_within_one_and_a_half_times_the_table(seeds_report, direction):
    table, seeded = seeds_report[f"table_{direction}"], seeds_report[f"seeded_{direction}"]
    assert seeded <= 1.5 * table, (direction, seeded, table)
    assert seeded < 2e-6 if direction == "n2p" else seeded < 4e-6       # emul.cu's own bounds on the table transform


def test_seeded_layout_drops_tw1_and_keeps_two_ctas_per_sm_without_spills(seeds_report):
    import test_fft_residency as fr
    assert seeds_report["smem_seeded_float2"] == seeds_report["smem_table_float2"] - L == 2 * 16 * 17 * R3 + 16 * R3
    smem = framepass_seeded_smem_bytes()
    assert smem == 93184 == 109568 - L * 8
    regs, spills = fr.fftc_entries()[("frame_pass_kernel", R3, None)]
    assert spills == "0 bytes spill stores, 0 bytes spill loads"
    assert fr.ctas_per_sm(regs, T, smem) == 2, f"frame_pass_kernel<8>: {regs} registers x {T} threads, {smem} B"


# ------------------------------------------------------------------ GPU
EDGES = ("n_not_multiple_of_F", "caf_exact_P1")


@pytest.mark.gpu
@pytest.mark.parametrize("prof", ["P0", "P1"])
def test_headline_frame_with_seeded_twiddles(prof):
    """One frame at the headline shape (2^20 samples, 256 x 300, filterLen 300, peek 10, float32 Kaiser window): taps
    and a P0 map within 1.5e-6 of the float64 frame truth; a P1 map no further from it than twice the two-pass frame
    (whose transforms read the table) and within 5e-4 of the two-pass map."""
    import torch
    from passiveradar_b200 import synth
    from test_frame_onepass import TOL, _frames, rel
    from oracle import xambg_oracle as xo
    n, F, R, fl, peek = 2 ** 20, 256, 300, 300, 10
    ref, srv = synth.make_frame(n, prof, 1500)
    w = signal.get_window(("kaiser", 5.0), n).astype(np.float32)
    amb, t_taps, _ = xo.frame_truth(ref, srv, fl, 1.0, peek, R, F, w.astype(np.float64))
    dev = torch.device("cuda", 0)
    refs, srvs = torch.from_numpy(ref[None]).to(dev), torch.from_numpy(srv[None]).to(dev)
    d_w = torch.from_numpy(w).to(dev)
    maps1, taps1, _, ran = _frames(refs, srvs, fl, peek, R, F, d_w, 1, profile=True)
    assert ran
    den = np.abs(amb).max()
    e_taps, e1 = rel(taps1[0], t_taps, np.abs(t_taps).max()), rel(maps1[0], amb, den)
    fig = {"E_taps": e_taps, "E_map": e1}
    assert e_taps <= TOL, e_taps
    if prof == "P0":
        assert e1 <= TOL, e1
    else:
        maps0, _, _, _ = _frames(refs, srvs, fl, peek, R, F, d_w, 0)
        e0 = rel(maps0[0], amb, den)
        fig["E_map_two_pass"] = e0
        assert e1 <= 2 * e0, (e1, e0)
        assert rel(maps1[0], maps0[0], np.abs(maps0[0]).max()) <= 5e-4
    record_parity(f"twiddle_seeds/headline_{prof}", **fig)


@pytest.mark.gpu
@pytest.mark.parametrize("edge", EDGES)
def test_plan_edges_with_seeded_twiddles(edge):
    """Two of test_frame_onepass.py's EDGE_CASES with no window, a float64 and a float32 window, at its bounds."""
    import test_frame_onepass as fo
    case = next(c for c in fo.EDGE_CASES if c[0] == edge)
    fo.test_onepass_at_the_plan_edges(*case)
