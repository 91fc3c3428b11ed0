"""Several surveillance channels against one shared reference: prc_frames_multi_c64 (csrc/framemulti.cuh, planned in
prcore_corr.cu: frames_multi_device) and FramePipeline(channels=K).

CPU: the refusals (before any CUDA call and any launch), the build's ptxas log (no spills, shared memory and residency
by the formula of DESIGN.md section 20), every launch of framemulti.cuh covered by a GPU test, and a Python twin of the
planner that states which path each (shape, K) takes and how many transforms it runs.  GPU: every channel bit for bit
prc_frames_c64(ref, srv_k) with the same frames per call, within 1.5e-6 of the float64 frame truth, across chunks, on
the fallback paths, with permuted, aliased, zero and singular channels, and through FramePipeline.
"""
import os
import re
import sys

import numpy as np
import pytest
import scipy.signal as signal

import test_onepass_sweep as ops
from passiveradar_b200 import _lib, synth
from oracle import xambg_oracle as xo

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "passiveradar_b200", "csrc")
FRAMEMULTI = os.path.join(CSRC, "framemulti.cuh")
TOL = 1.5e-6
L = 2048
C2 = (2 ** 20, 256, 300, 300, 10)            # n, F, R, filter_len, peek
_BUF = np.zeros(1 << 16, np.complex128)
P = _BUF.ctypes.data


def min_shared_k():
    src = open(os.path.join(CSRC, "prcore_corr.cu")).read()
    return int(re.search(r"constexpr int FM_MIN_SHARED_K = (\d+);", src).group(1))


# ------------------------------------------------------------------ CPU: refusals
def _call(**kw):
    a = dict(ref=P, srv=P, n=1 << 14, nframes=2, frame_stride=1 << 14, nchan=2, chan_stride=1 << 15, filter_len=10,
             peek=2, reg=1.0, range_bins=20, freq_bins=8, window=None, maps=P, taps=None, device=0, stream=None, flags=0)
    a.update(kw)
    return _lib.load().prc_frames_multi_c64(*a.values())


REFUSALS = [dict(nchan=0), dict(nchan=5), dict(nchan=-1), dict(ref=None), dict(srv=None), dict(maps=None), dict(n=0),
            dict(nframes=0), dict(frame_stride=100), dict(freq_bins=0), dict(range_bins=-1), dict(filter_len=-1),
            dict(peek=-1), dict(filter_len=0, peek=0)]


@pytest.mark.parametrize("kw", REFUSALS, ids=[",".join(f"{k}={v}" for k, v in r.items()) for r in REFUSALS])
def test_refusals_come_before_any_cuda_call(kw):
    before = _lib.launch_count()
    assert _call(**kw) == _lib.PRC_E_INVALID
    assert _lib.launch_count() == before
    assert _lib.load().prc_last_error()


@pytest.mark.parametrize("chan_stride", [0, -(1 << 15), 1, 1 << 40])
def test_any_channel_stride_passes_the_checks(chan_stride):
    """The inputs are only read, so channels may alias or lie in any order: a call with any chan_stride gets past the
    argument checks (here it then needs a device: PRC_E_CUDA without one, and it runs with one)."""
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("with a device the call would read the dummy operands")
    except ImportError:
        pass
    assert _call(chan_stride=chan_stride) == _lib.PRC_E_CUDA


# ------------------------------------------------------------------ CPU: build
def multi_entries():
    """{(kernel, K or None): (registers, spill text)} of framemulti.cuh's kernels in the build's ptxas log"""
    import test_fft_residency as fr
    fr.fftc_entries()                        # builds the library, skips without a log
    from passiveradar_b200 import build as b
    out = {}
    for blk in open(os.path.join(b.PKG, "libprcore.ptxas.log")).read().split("Compiling entry function")[1:]:
        head = blk.split("\n")[0]
        m = re.search(r"_ZN3prc4fftc\d+(frame_multi_pass_kernel|caf_combine_multi_kernel)ILi8E(?:Li(\d)E)?E", head)
        if m:
            assert "'sm_90a'" in head
            regs = int(re.search(r"Used (\d+) registers", blk).group(1))
            spills = re.search(r"\d+ bytes spill stores, \d+ bytes spill loads", blk).group(0)
            out[(m.group(1), None if m.group(2) is None else int(m.group(2)))] = (regs, spills)
    return out


def framemulti_smem_bytes(K):
    """DESIGN.md section 20: frame_pass_kernel's layout without its AccP / AccQ slots (FpSmem, staging L float2,
    window L float) plus AccQ, K AccP_k and K - 1 accX_k slots of L float2"""
    fp_smem = 2 * 16 * 17 * 8 + 8 * 18                # two exchange buffers + tw2 rows (fft::SmemSeeded<8, Tw2Rows<8>>)
    return (fp_smem + L + L // 2 + 2 * K * L) * 8


def test_kernels_have_no_spills_and_one_cta_per_sm():
    import test_fft_residency as fr
    entries = multi_entries()
    assert set(entries) == {("frame_multi_pass_kernel", 2), ("frame_multi_pass_kernel", 3),
                            ("frame_multi_pass_kernel", 4), ("caf_combine_multi_kernel", None)}, entries
    for key, (_, spills) in entries.items():
        assert spills == "0 bytes spill stores, 0 bytes spill loads", (key, spills)
    assert [framemulti_smem_bytes(K) for K in (2, 3, 4)] == [126080, 158848, 191616]
    assert framemulti_smem_bytes(0) == 60544            # frame_pass_kernel's 93 312 B less its two L-float2 slots
    for K in (2, 3, 4):
        regs, _ = entries[("frame_multi_pass_kernel", K)]
        assert fr.ctas_per_sm(regs, 128, framemulti_smem_bytes(K)) == 1, (K, regs)
        assert framemulti_smem_bytes(K) <= 200 * 1024      # SMEM_LIMIT, the opt-in the library sets


# every launch in framemulti.cuh -> the GPU tests that reach it
COVERAGE = {
    "frame_multi_pass_kernel<FP_R3, K>": ["test_channels_are_single_channel_frames_bit_for_bit",
                                          "test_edge_shapes_bit_for_bit_and_against_truth"],
    "caf_combine_multi_kernel<FP_R3>": ["test_channels_are_single_channel_frames_bit_for_bit",
                                        "test_edge_shapes_bit_for_bit_and_against_truth"],
}


def test_every_framemulti_launch_has_a_covering_gpu_test():
    src = open(FRAMEMULTI).read()
    code = "\n".join(line.split("//", 1)[0] for line in src.splitlines())
    sites = {m.group(1) + (m.group(2) or "") for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", code)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    this = open(os.path.abspath(__file__)).read()
    for tests in COVERAGE.values():
        for t in tests:
            i = this.index(f"\ndef {t}(")
            decorators = this[this.rindex("\n\n", 0, i):i]
            assert "@pytest.mark.gpu" in decorators, f"{t} is not a GPU test"


# ------------------------------------------------------------------ CPU: planner twin
def multi_path(n, F, R, filter_len, peek, K):
    """prcore_corr.cu: frames_multi_device -- 'shared' (frame_multi_pass_kernel) or the path prc_frames_c64 takes for
    each channel: 'onepass', 'two-pass' (the FFT-domain LS and fused CAF kernels) or 'direct'"""
    plan = ops.onepass_plan(n, F, filter_len, peek, R)
    if plan.on and K >= min_shared_k():
        return "shared", plan
    if plan.on:
        return "onepass", plan
    M = filter_len + peek
    fft = ops.ps.ls_plan(n, M, ops.ps.FFT_MIN_N).on and ops.ps.caf_plan(n, R, F, M, ops.ps.FFT_MIN_N).on
    return ("two-pass" if fft else "direct"), plan


def twin_transforms(plan, F, K, ncta):
    """length-L transforms per frame: K one-pass frames, and the shared pass"""
    seg = sum(b[3] for b in plan.blocks)
    ntail = plan.tail[1]
    return K * (4 * seg + 3 * ntail + 2 * ncta + F), (3 + K) * seg + (2 + K) * ntail + (1 + K) * ncta + K * F


PATH_CASES = [
    ("config2", C2, {1: "onepass", 2: "shared", 3: "shared", 4: "shared"}),
    ("onepass_off", (2 ** 20, 256, 1300, 310, 10), {k: "two-pass" for k in (1, 2, 3, 4)}),
    ("direct", (4096, 8, 20, 10, 0), {k: "direct" for k in (1, 2, 3, 4)}),
    ("M=1024", (2 ** 17, 16, 100, 1014, 10), {k: "two-pass" for k in (1, 2, 3, 4)}),
]


@pytest.mark.parametrize("name,shape,want", PATH_CASES, ids=[c[0] for c in PATH_CASES])
def test_twin_states_each_path(name, shape, want):
    n, F, R, fl, peek = shape
    for K, path in want.items():
        if path == "shared" and K < min_shared_k():
            path = "onepass"
        assert multi_path(n, F, R, fl, peek, K)[0] == path, (name, K)


def test_twin_transform_counts_match_the_issue_table_at_config_2():
    n, F, R, fl, peek = C2
    _, plan = multi_path(n, F, R, fl, peek, 2)
    assert plan.on and sum(b[3] for b in plan.blocks) == 767 and plan.tail[1] == 2
    table = {2: (6700, 4385), 3: (10050, 5420), 4: (13400, 6455)}
    sys.path.insert(0, os.path.join(HERE, "..", "scripts"))
    import multichannel_bench as mb
    for K, want in table.items():
        assert twin_transforms(plan, F, K, 10) == want, K
        assert mb.transforms(n, F, R, fl, peek, K, 26, 264) == (26 * want[0], 26 * want[1])   # 264 // 26 = 10 CTAs


# ------------------------------------------------------------------ GPU helpers
def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", 0))


def _multi(refs, srvs, fl, peek, R, F, w, reg=1.0, chan_stride=None, K=None, profile=False):
    """prc_frames_multi_c64 (asynchronous, status read with prc_ls_status) -> maps (K, nf, F, R+1), taps (K, nf, M),
    status (K, nf), and whether frame_multi ran (None unless profiled)"""
    import ctypes as C
    import torch
    nf, n = refs.shape
    K = srvs.shape[0] if K is None else K
    cs = srvs.stride(0) if chan_stride is None else chan_stride
    maps = torch.empty((K, nf, F, R + 1), dtype=torch.complex64, device=refs.device)
    taps = torch.empty((K, nf, fl + peek), dtype=torch.complex64, device=refs.device)
    flags = _lib.FLAG_ASYNC
    wp = None
    if w is not None:
        flags |= _lib.FLAG_WINDOW_F32 if w.dtype == torch.float32 else 0
        wp = w.data_ptr()
    lib = _lib.load()
    if profile:
        _lib.profile_reset()
        _lib.profile(True)
    try:
        _lib.check(lib.prc_frames_multi_c64(refs.data_ptr(), srvs.data_ptr(), n, nf, refs.stride(0) if nf > 1 else n, K,
                                            cs, fl, peek, reg, R, F, wp, maps.data_ptr(), taps.data_ptr(), 0, None,
                                            flags))
        st = (C.c_int * (K * nf))()
        _lib.check(lib.prc_ls_status(0, None, st, K * nf))
        ran = None
        if profile:
            ran = _lib.profile_read()["frame_multi"][1] > 0
    finally:
        if profile:
            _lib.profile(False)
    return (maps.cpu().numpy(), taps.cpu().numpy(), np.frombuffer(st, np.int32).reshape(K, nf).copy(), ran)


def _single(refs, srv, fl, peek, R, F, w, reg=1.0):
    """prc_frames_c64 on one channel's frames -> maps (nf, F, R+1), taps (nf, M)"""
    import torch
    nf, n = refs.shape
    maps = torch.empty((nf, F, R + 1), dtype=torch.complex64, device=refs.device)
    taps = torch.empty((nf, fl + peek), dtype=torch.complex64, device=refs.device)
    flags, wp = 0, None
    if w is not None:
        flags = _lib.FLAG_WINDOW_F32 if w.dtype == torch.float32 else 0
        wp = w.data_ptr()
    _lib.check(_lib.load().prc_frames_c64(refs.data_ptr(), srv.data_ptr(), n, nf, refs.stride(0) if nf > 1 else n, fl,
                                          peek, reg, R, F, wp, maps.data_ptr(), taps.data_ptr(), None, _lib.MEM_DEVICE,
                                          0, None, flags))
    torch.cuda.synchronize()
    return maps.cpu().numpy(), taps.cpu().numpy()


def _channels(n, nf, K, seed):
    """P0 frames: nf white references, K x nf white surveillance channels"""
    refs = np.stack([synth.make_frame(n, "P0", seed + f)[0] for f in range(nf)])
    srvs = np.stack([np.stack([synth.make_frame(n, "P0", seed + 100 + 10 * k + f)[1] for f in range(nf)])
                     for k in range(K)])
    return refs, srvs


def rel(a, b):
    b = np.asarray(b, np.complex128)
    return float(np.abs(np.asarray(a, np.complex128) - b).max() / np.abs(b).max())


def _check_against_single_and_truth(refs, srvs, fl, peek, R, F, w, K, truth_frames=(0,)):
    d_refs, d_srvs = _dev(refs), _dev(srvs)
    d_w = None if w is None else _dev(w)
    maps, taps, st, ran = _multi(d_refs, d_srvs[:K], fl, peek, R, F, d_w, profile=True)
    assert not st.any()
    n = refs.shape[1]
    shared = multi_path(n, F, R, fl, peek, K)[0] == "shared"
    assert ran == shared, (K, ran)
    worst = 0.0
    for k in range(K):
        m1, t1 = _single(d_refs, d_srvs[k], fl, peek, R, F, d_w)
        assert np.array_equal(maps[k].view(np.uint64), m1.view(np.uint64)), k
        assert np.array_equal(taps[k].view(np.uint64), t1.view(np.uint64)), k
        for f in truth_frames:
            amb, t_taps, _ = xo.frame_truth(refs[f], srvs[k, f], fl, 1.0, peek, R, F,
                                            None if w is None else w.astype(np.float64))
            e = max(rel(taps[k, f], t_taps), rel(maps[k, f], amb))
            worst = max(worst, e)
            assert e <= TOL, (k, f, e)
    return worst


# ------------------------------------------------------------------ GPU: bit for bit, truth
@pytest.mark.gpu
@pytest.mark.parametrize("window", ["none", "kaiser_f32"])
def test_channels_are_single_channel_frames_bit_for_bit(window):
    """Config 2, four frames per call (one chunk of both paths): K = 1 .. 4, every channel's taps and map are the bytes
    of prc_frames_c64(ref, srv_k) on the same frames, and within 1.5e-6 of the float64 frame truth."""
    n, F, R, fl, peek = C2
    refs, srvs = _channels(n, 4, 4, 700)
    w = None if window == "none" else signal.get_window(("kaiser", 5.0), n).astype(np.float32)
    for K in (1, 2, 3, 4):
        _check_against_single_and_truth(refs, srvs, fl, peek, R, F, w, K, truth_frames=(0, 3) if K == 4 else (0,))


EDGE_SHAPES = [
    ("M=1", 2 ** 17, 16, 100, 1, 0),
    ("M=2_peek=0", 2 ** 17, 16, 100, 2, 0),
    ("M=2_peek=1", 2 ** 17, 16, 100, 1, 1),
    ("peek=M-1", 2 ** 17, 16, 100, 1, 39),
    ("F=1", 2 ** 14, 1, 100, 60, 10),
    ("n_not_multiple_of_F", 2 ** 17 + 3, 7, 60, 30, 9),
    ("M=1023", 2 ** 17, 16, 100, 1013, 10),
    ("M=1024_peek=M-1", 2 ** 17, 16, 100, 1, 1023),
    ("smallest_Bmax", 1048708, 1024, 912, 564, 14),
]


@pytest.mark.gpu
@pytest.mark.parametrize("edge,n,F,R,fl,peek", EDGE_SHAPES, ids=[c[0] for c in EDGE_SHAPES])
def test_edge_shapes_bit_for_bit_and_against_truth(edge, n, F, R, fl, peek):
    """The one-pass plan's edge shapes (and two beyond it, M = 1023 and 1024, where it is off), two frames per call,
    Kaiser window: K = 2, 3, 4 channels bit for bit per-channel prc_frames_c64, and within 1.5e-6 of the truth."""
    refs, srvs = _channels(n, 2, 4, 900 + F)
    w = signal.get_window(("kaiser", 5.0), n)
    for K in (2, 3, 4):
        _check_against_single_and_truth(refs, srvs, fl, peek, R, F, w, K, truth_frames=(1,))


@pytest.mark.gpu
def test_batch_spanning_two_chunks():
    """Config 2, K = 4 and 14 frames: chunks of 12 and 2 frames (the (1 + K) F L complex64 spectra of a frame against
    the 256 MiB cap).  Every channel of every frame is within 1.5e-6 of the truth, and with reg = 0 and frame 13's
    reference all zero exactly the four status words [k][13] are set."""
    n, F, R, fl, peek = C2
    nf, K = 14, 4
    base_refs, base_srvs = _channels(n, 2, K, 1100)
    idx = np.arange(nf) % 2
    refs = base_refs[idx].copy()
    refs[13] = 0
    srvs = base_srvs[:, idx]
    w = signal.get_window(("kaiser", 5.0), n).astype(np.float32)
    maps, taps, st, ran = _multi(_dev(refs), _dev(srvs), fl, peek, R, F, _dev(w), reg=0.0, profile=True)
    assert ran
    want = np.zeros((K, nf), np.int32)
    want[:, 13] = 1
    assert np.array_equal(st, want), st
    truths = {}
    for k in range(K):
        for f in range(13):
            key = (k, idx[f])
            if key not in truths:
                truths[key] = xo.frame_truth(base_refs[idx[f]], base_srvs[k, idx[f]], fl, 0.0, peek, R, F,
                                             w.astype(np.float64))
            amb, t_taps, _ = truths[key]
            assert rel(taps[k, f], t_taps) <= TOL, (k, f)
            assert rel(maps[k, f], amb) <= TOL, (k, f)


@pytest.mark.gpu
@pytest.mark.parametrize("name,n,F,R,fl,peek", [("two-pass", 2 ** 17, 16, 1300, 310, 10), ("direct", 4096, 8, 20, 10, 0)])
def test_fallback_paths_are_per_channel_frames(name, n, F, R, fl, peek):
    """Where the one-pass plan is off (the two-pass FFT path; the direct form below 8192 samples) every channel is the
    bytes of prc_frames_c64 on it, and frame_multi does not run."""
    refs, srvs = _channels(n, 3, 3, 1200)
    d_refs, d_srvs = _dev(refs), _dev(srvs)
    assert multi_path(n, F, R, fl, peek, 3)[0] == name
    maps, taps, st, ran = _multi(d_refs, d_srvs, fl, peek, R, F, None, profile=True)
    assert ran is False and not st.any()
    for k in range(3):
        m1, t1 = _single(d_refs, d_srvs[k], fl, peek, R, F, None)
        assert np.array_equal(maps[k].view(np.uint64), m1.view(np.uint64)), k
        assert np.array_equal(taps[k].view(np.uint64), t1.view(np.uint64)), k


# ------------------------------------------------------------------ GPU: channels are independent
SMALL = (2 ** 17, 16, 100, 50, 10)           # one-pass plan on


@pytest.mark.gpu
def test_permuted_aliased_and_zero_channels():
    """Permuting the channels permutes the outputs bit for bit; chan_stride = 0 gives every channel channel 0's
    output; an all-zero channel gets zero taps and a zero map and leaves the others' bytes unchanged."""
    n, F, R, fl, peek = SMALL
    refs, srvs = _channels(n, 3, 4, 1300)
    w = _dev(signal.get_window(("kaiser", 5.0), n).astype(np.float32))
    d_refs = _dev(refs)
    maps, taps, _, _ = _multi(d_refs, _dev(srvs), fl, peek, R, F, w)
    perm = [2, 0, 3, 1]
    pm, pt, _, _ = _multi(d_refs, _dev(srvs[perm]), fl, peek, R, F, w)
    assert np.array_equal(pm.view(np.uint64), maps[perm].view(np.uint64))
    assert np.array_equal(pt.view(np.uint64), taps[perm].view(np.uint64))
    am, at, _, _ = _multi(d_refs, _dev(srvs), fl, peek, R, F, w, chan_stride=0)
    for k in range(4):
        assert np.array_equal(am[k].view(np.uint64), maps[0].view(np.uint64)), k
        assert np.array_equal(at[k].view(np.uint64), taps[0].view(np.uint64)), k
    z = srvs.copy()
    z[1] = 0
    zm, zt, st, _ = _multi(d_refs, _dev(z), fl, peek, R, F, w)
    assert not st.any()
    assert not zm[1].any() and not zt[1].any()
    for k in (0, 2, 3):
        assert np.array_equal(zm[k].view(np.uint64), maps[k].view(np.uint64)), k


@pytest.mark.gpu
def test_singular_reference_flags_every_channel_of_its_frame_only():
    n, F, R, fl, peek = SMALL
    refs, srvs = _channels(n, 3, 3, 1400)
    refs[1] = 0
    _, _, st, ran = _multi(_dev(refs), _dev(srvs), fl, peek, R, F, None, reg=0.0, profile=True)
    assert ran == (3 >= min_shared_k())
    assert np.array_equal(st, np.array([[0, 1, 0]] * 3, np.int32)), st


# ------------------------------------------------------------------ GPU: FramePipeline(channels=K)
@pytest.mark.gpu
def test_frame_pipeline_channels():
    """run_host equals run_device, and any batch and slot count gives the bytes of one call"""
    from passiveradar_b200.frames import FramePipeline
    import torch
    n, F, R, fl, peek = SMALL
    K, nf = 3, 5
    refs, srvs = _channels(n, nf, K, 1500)
    one = FramePipeline(n, R, F, filter_len=fl, peek=peek, batch=nf, nslots=1, channels=K)
    d_maps = torch.empty((K, nf, F, R + 1), dtype=torch.complex64, device="cuda")
    one.run_device(_dev(refs), _dev(srvs), d_maps, check=True)
    torch.cuda.synchronize()
    want = d_maps.cpu().numpy()
    wm, _, _, _ = _multi(_dev(refs), _dev(srvs), fl, peek, R, F, one.window)
    assert np.array_equal(want.view(np.uint64), wm.view(np.uint64))
    assert one.ls_status(0, nf).shape == (K, nf)
    for batch, nslots in ((nf, 1), (2, 1), (2, 3), (1, 2)):
        pipe = FramePipeline(n, R, F, filter_len=fl, peek=peek, batch=batch, nslots=nslots, channels=K)
        got = pipe.run_host(refs, srvs)
        assert got.shape == (K, nf, F, R + 1, 1)
        assert np.array_equal(got[..., 0].view(np.uint64), want.view(np.uint64)), (batch, nslots)
        d_maps.zero_()
        pipe.run_device(_dev(refs), _dev(srvs), d_maps)
        torch.cuda.synchronize()
        assert np.array_equal(d_maps.cpu().numpy().view(np.uint64), want.view(np.uint64)), (batch, nslots)
