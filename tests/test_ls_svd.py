"""SVD least-squares clutter filter (reference passiveRadar/clutter_removal.py:58-107): the goldens' provenance, the
oracle and the two float64 truths against them, the wrappers' contract and the build (no GPU needed); the sm_90a
kernels against the truth and the reference across shapes, on rank-deficient inputs and in batches (GPU)."""
import ctypes as C
import hashlib
import inspect
import json
import os
import re
import threading

import numpy as np
import pytest

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth

import _golden as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LSSVD = os.path.join(ROOT, "passiveradar_b200", "csrc", "lssvd.cuh")
GOLDENS = ["ls_svd_p0", "ls_svd_p1", "ls_svd_peek0", "ls_svd_short", "ls_svd_zero", "ls_svd_periodic", "ls_svd_c128",
           "ls_svd_f32", "ls_svd_c4"]


def golden(name):
    g = G.load(name)
    ref, srv = G.inputs(g)
    return g, ref, srv, int(g["filter_len"]), int(g["peek"])


def periodic_pair(n, period, seed):
    rng = np.random.default_rng(seed)
    base = (rng.standard_normal(period) + 1j * rng.standard_normal(period)).astype(np.complex64)
    ref = np.tile(base, n // period)
    srv = (0.8 * np.roll(ref, 5) + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    return ref, srv


def _truth(ref, srv, fl, peek):
    from oracle import svd_oracle as so
    r, s = np.asarray(ref).astype(np.complex64), np.asarray(srv).astype(np.complex64)
    return so.ls_filter_svd_truth_gram(r, s, fl, peek)


# ------------------------------------------------------------------ CPU: goldens, oracle, truths, wrapper contract
@pytest.mark.parametrize("name", GOLDENS)
def test_svd_golden_is_what_the_reference_produces(name):
    with open(os.path.join(G.GOLDEN_DIR, "svd_reference_digests.json")) as f:
        want = json.load(f)[name]
    committed = G.load(name)
    assert set(want) == set(committed) - {"seconds"}
    for key, digest in want.items():
        a = np.ascontiguousarray(committed[key])
        hsh = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
        hsh.update(a.tobytes())
        assert hsh.hexdigest() == digest, f"{name}[{key}] differs from the reference's output"
    assert os.path.getsize(os.path.join(G.GOLDEN_DIR, name + ".npz")) < 300_000


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_reproduces_the_golden(name):
    from oracle import svd_oracle as so
    g, ref, srv, fl, peek = golden(name)
    out, taps = so.ls_filter_svd_oracle(ref, srv, fl, peek, True)
    assert out.dtype == g["out"].dtype and taps.dtype == g["taps"].dtype
    den = float(g["srv_absmax"])
    assert G.rel_inf(out, g["out"], den) <= 1e-6
    assert G.rel_inf(taps, g["taps"], max(float(np.abs(g["taps"]).max()), 1e-30)) <= 1e-6


@pytest.mark.parametrize("name", GOLDENS)
def test_truths_agree_and_the_reference_is_near_them(name):
    """The explicit complex128 SVD and the float64 Gram eigendecomposition give the same solution, rank-deficient
    cases (short, zero, periodic) included; the reference's complex64 SVD is within 1e-5 max|srv| of it."""
    from oracle import svd_oracle as so
    g, ref, srv, fl, peek = golden(name)
    r, s = ref.astype(np.complex64), srv.astype(np.complex64)
    o1, t1, k1 = so.ls_filter_svd_truth(r, s, fl, peek)
    o2, t2, k2 = so.ls_filter_svd_truth_gram(r, s, fl, peek)
    den = float(g["srv_absmax"])
    assert k1 == k2
    assert G.rel_inf(o1, o2, den) <= 1e-9
    assert G.rel_inf(t1, t2, max(float(np.abs(t1).max()), 1e-30)) <= 1e-9
    assert G.rel_inf(g["out"], o1, den) <= 1e-5
    expect_rank = {"ls_svd_short": 24, "ls_svd_zero": 0, "ls_svd_periodic": 13}
    assert k1 == expect_rank.get(name, fl + peek)


def test_truncation_rule_separates_a_periodic_null_space():
    """DESIGN.md section 13: the float64 Gram of an exactly 13-periodic reference has its null eigenvalues near
    1e-16 lambda_max, far below the 1e-10 lambda_max floor, and its smallest kept one far above it."""
    ref, _ = periodic_pair(65533 // 13 * 13, 13, 1)
    fr = np.fft.fft(ref.astype(np.complex128))
    c = np.fft.ifft(np.conj(fr) * fr)
    m = 60
    lam = np.linalg.eigvalsh(c[(np.arange(m)[:, None] - np.arange(m)[None, :]) % ref.shape[0]])
    lam = np.sort(lam)[::-1] / lam.max()
    assert lam[12] > 1e-4 and np.abs(lam[13:]).max() < 1e-13


def test_signature_defaults_exports_and_install():
    def names(f):
        return [p for p in inspect.signature(f).parameters if p != "device"]
    assert names(prb.LS_Filter_SVD) == ["refChannel", "srvChannel", "filterLen", "peek", "return_filter"]
    sig = inspect.signature(prb.LS_Filter_SVD)
    assert sig.parameters["peek"].default == 10 and sig.parameters["return_filter"].default is False
    assert sig.parameters["device"].kind is inspect.Parameter.KEYWORD_ONLY
    sig = inspect.signature(prb.ls_filter_svd_frames)
    assert list(sig.parameters)[:5] == ["ref_frames", "srv_frames", "filterLen", "peek", "return_filter"]
    assert sig.parameters["return_rank"].kind is inspect.Parameter.KEYWORD_ONLY
    assert "LS_Filter_SVD" in prb.__all__ and "ls_filter_svd_frames" in prb.__all__
    assert "LS_Filter_SVD" not in inspect.getsource(prb.install)


def test_argument_errors_and_empty_filters_never_load_the_library(monkeypatch):
    def no_library(*a, **k):
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "load", no_library)
    a = np.ones(16, np.complex64)
    with pytest.raises(ValueError, match="Input vectors must have the same length"):
        prb.LS_Filter_SVD(a, a[:15], 4)
    with pytest.raises(ValueError, match="filterLen"):
        prb.LS_Filter_SVD(a, a, -1, 2)
    with pytest.raises(ValueError, match="peek"):
        prb.LS_Filter_SVD(a, a, 4, -1)
    with pytest.raises(ValueError, match="two-dimensional"):
        prb.ls_filter_svd_frames(a, a, 4)
    with pytest.raises(ValueError, match="peek"):
        prb.ls_filter_svd_frames(a[None], a[None], 4, -3)
    for srv in (a * 2, (a * 2).astype(np.complex128), np.arange(16, dtype=np.float32), np.arange(16.0)):
        out, taps = prb.LS_Filter_SVD(a, srv, 0, 0, True)
        rt = np.result_type(np.complex64, srv.dtype)
        assert out.dtype == rt and taps.dtype == rt and taps.shape == (0,)
        np.testing.assert_array_equal(out, srv)
    out, taps = prb.ls_filter_svd_frames(np.ones((2, 8)), np.full((2, 8), 3.0), 0, 0, True)
    assert out.dtype == np.complex128 and taps.shape == (2, 0)
    np.testing.assert_array_equal(out, 3.0)


def test_no_cpu_fallback_without_a_device():
    if _lib.device_count() > 0:
        pytest.skip("a CUDA device is present")
    a = np.ones(64, np.complex64)
    with pytest.raises(_lib.PrcoreError):
        prb.LS_Filter_SVD(a, a, 4)


def test_lssvd_kernels_build_for_sm90a_without_spills():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    blocks = [blk for blk in open(log).read().split("Compiling entry function")[1:]
              if "5lssvd" in blk.split("\n")[0]]
    assert len(blocks) == 4, "corr, reduce, eig, fir"
    for blk in blocks:
        assert "'sm_90a'" in blk.split("\n")[0]
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in blk


# every launch in lssvd.cuh -> the GPU tests that reach it
COVERAGE = {
    "svd_corr_kernel": ["test_goldens_match_truth_and_reference", "test_parameter_grid_matches_truth"],
    "svd_reduce_kernel": ["test_goldens_match_truth_and_reference", "test_parameter_grid_matches_truth"],
    "svd_eig_kernel": ["test_goldens_match_truth_and_reference", "test_parameter_grid_matches_truth"],
    "svd_fir_kernel": ["test_goldens_match_truth_and_reference", "test_parameter_grid_matches_truth"],
}


def test_every_lssvd_launch_has_a_covering_gpu_test():
    src = open(LSSVD).read()
    sites = {m.group(1) + (m.group(2) or "") for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", src)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    this = open(os.path.abspath(__file__)).read()
    for tests in COVERAGE.values():
        for t in tests:
            i = this.index(f"\ndef {t}(")
            decorators = this[this.rindex("\n\n", 0, i):i]
            assert "@pytest.mark.gpu" in decorators, f"{t} is not a GPU test"


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", GOLDENS)
def test_goldens_match_truth_and_reference(name):
    g, ref, srv, fl, peek = golden(name)
    out, taps = prb.LS_Filter_SVD(ref, srv, fl, peek, True)
    assert out.dtype == g["out"].dtype and taps.dtype == g["taps"].dtype
    t_out, t_taps, _ = _truth(ref, srv, fl, peek)
    den = float(g["srv_absmax"])
    tden = max(float(np.abs(t_taps).max()), 1e-30)
    assert G.rel_inf(out, t_out, den) <= 1e-6
    assert G.rel_inf(taps, t_taps, tden) <= 1e-6
    assert G.rel_inf(out, g["out"], den) <= 1e-5 + 1.2 * G.rel_inf(t_out, g["out"], den)
    assert G.rel_inf(taps, g["taps"], tden) <= 1e-5 + 1.2 * G.rel_inf(t_taps, g["taps"], tden)


GRID = [(24, 1, 0, "P0"), (24, 40, 10, "P1"), (1000, 11, 0, "P1"), (1000, 175, 10, "P0"), (8192, 40, 10, "P1"),
        (8192, 300, 10, "P0"), (8192, 1014, 10, "P1"), (65543, 1, 0, "P1"), (65543, 50, 0, "P0"),
        (65543, 175, 10, "P1"), (65543, 300, 10, "P1"), (1000, 1024, 0, "P0")]


@pytest.mark.gpu
@pytest.mark.parametrize("n,fl,peek,profile", GRID)
def test_parameter_grid_matches_truth(n, fl, peek, profile):
    """M = 1, 11, 50, 185, 310 and 1024; n from below M to past 2^16; peek 0 and 10.  M <= 86 keeps A and Z in shared
    memory, M <= 105 A alone, larger M both in the per-frame global workspace."""
    ref, srv = synth.make_frame(n, profile, frame=n % 7)
    out, taps = prb.LS_Filter_SVD(ref, srv, fl, peek, True)
    t_out, t_taps, _ = _truth(ref, srv, fl, peek)
    assert G.rel_inf(out, t_out, float(np.abs(srv).max())) <= 1e-6
    assert G.rel_inf(taps, t_taps) <= 1e-6


@pytest.mark.gpu
def test_periodic_reference_rank_and_minimum_norm_taps():
    ref, srv = periodic_pair(8190, 13, 3)
    out, taps, rank = prb.ls_filter_svd_frames(ref[None], srv[None], 30, 10, True, return_rank=True)
    assert rank[0] == 13
    t_out, t_taps, t_rank = _truth(ref, srv, 30, 10)
    assert t_rank == 13
    assert G.rel_inf(out[0], t_out, float(np.abs(srv).max())) <= 1e-6
    assert G.rel_inf(taps[0], t_taps) <= 1e-6
    with pytest.raises(np.linalg.LinAlgError):
        prb.LS_Filter(ref, srv, 30, 0.0, 10)


@pytest.mark.gpu
def test_zero_reference_returns_srv_bit_for_bit():
    _, srv = synth.make_frame(5000, "P1", 2)
    ref = np.zeros_like(srv)
    out, taps, rank = prb.ls_filter_svd_frames(ref[None], srv[None], 20, 10, True, return_rank=True)
    assert rank[0] == 0 and not taps.any()
    np.testing.assert_array_equal(out[0].view(np.uint32), srv.view(np.uint32))


@pytest.mark.gpu
def test_non_finite_input_raises_linalgerror():
    ref, srv = synth.make_frame(2000, "P0", 1)
    bad = ref.copy()
    bad[100] = np.nan
    with pytest.raises(np.linalg.LinAlgError, match="^SVD did not converge$"):
        prb.LS_Filter_SVD(bad, srv, 10)
    bad_srv = srv.copy()
    bad_srv[5] = np.inf
    with pytest.raises(np.linalg.LinAlgError, match="^SVD did not converge$"):
        prb.LS_Filter_SVD(ref, bad_srv, 10)
    out, rank = prb.ls_filter_svd_frames(np.stack([ref, bad]), np.stack([srv, srv]), 10, return_rank=True)
    assert list(rank) == [20, -1] and np.isnan(out[1]).all() and np.isfinite(out[0]).all()


@pytest.mark.gpu
def test_mixed_batch_is_correct_frame_by_frame_and_rows_equal_single_calls():
    frames = [synth.make_frame(6000, "P1", k) for k in range(3)]
    frames.insert(2, periodic_pair(6000, 12, 4))
    frames.insert(4, (np.zeros(6000, np.complex64), frames[0][1]))
    ref = np.stack([f[0] for f in frames])
    srv = np.stack([f[1] for f in frames])
    out, taps, rank = prb.ls_filter_svd_frames(ref, srv, 40, 10, True, return_rank=True)
    assert list(rank) == [50, 50, 12, 50, 0]
    for i in range(ref.shape[0]):
        o1, t1 = prb.LS_Filter_SVD(ref[i], srv[i], 40, 10, True)
        np.testing.assert_array_equal(out[i], o1)
        np.testing.assert_array_equal(taps[i], t1)
        t_out, t_taps, _ = _truth(ref[i], srv[i], 40, 10)
        assert G.rel_inf(out[i], t_out, float(np.abs(srv[i]).max())) <= 1e-6
        if rank[i]:
            assert G.rel_inf(taps[i], t_taps) <= 1e-6


@pytest.mark.gpu
def test_device_pointers_frame_stride_and_caller_stream():
    import torch
    n, nf, stride, fl, peek = 7000, 3, 7300, 60, 10
    frames = [synth.make_frame(n, "P1", k) for k in range(nf)]
    ref_h = np.zeros((nf, stride), np.complex64)
    srv_h = np.zeros((nf, stride), np.complex64)
    for i, (r, s) in enumerate(frames):
        ref_h[i, :n], srv_h[i, :n] = r, s
    want, want_t, want_r = prb.ls_filter_svd_frames(ref_h[:, :n], srv_h[:, :n], fl, peek, True, return_rank=True)
    ref_d = torch.from_numpy(ref_h.view(np.float32)).cuda()
    srv_d = torch.from_numpy(srv_h.view(np.float32)).cuda()
    out_d = torch.zeros((nf, 2 * stride), dtype=torch.float32, device="cuda")
    taps_d = torch.zeros((nf, 2 * (fl + peek)), dtype=torch.float32, device="cuda")
    rank_d = torch.zeros(nf, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    lib = _lib.load()
    _lib.check(lib.prc_ls_svd_frames_c64(ref_d.data_ptr(), srv_d.data_ptr(), n, nf, stride, fl, peek, out_d.data_ptr(),
                                         taps_d.data_ptr(), rank_d.data_ptr(), _lib.MEM_DEVICE, 0,
                                         C.c_void_p(st.cuda_stream), _lib.FLAG_ASYNC))
    st.synchronize()
    out = out_d.cpu().numpy().view(np.complex64)
    np.testing.assert_array_equal(out[:, :n], want)
    assert not out[:, n:].any()                     # nothing written past n in a frame
    np.testing.assert_array_equal(taps_d.cpu().numpy().view(np.complex64), want_t)
    np.testing.assert_array_equal(rank_d.cpu().numpy(), want_r)


@pytest.mark.gpu
def test_concurrent_threads_are_bit_identical():
    cases = [synth.make_frame(5000 + 500 * k, "P1", k) for k in range(4)]
    serial = [prb.LS_Filter_SVD(r, s, 50, 10, True) for r, s in cases]
    results = [None] * 4

    def run(i):
        results[i] = prb.LS_Filter_SVD(cases[i][0], cases[i][1], 50, 10, True)
    threads = [threading.Thread(target=run, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for (o1, t1), (o2, t2) in zip(serial, results):
        np.testing.assert_array_equal(o1, o2)
        np.testing.assert_array_equal(t1, t2)


@pytest.mark.gpu
def test_limit_and_returned_dtypes():
    ref, srv = synth.make_frame(3000, "P0", 6)
    with pytest.raises(_lib.PrcoreError, match="1024"):
        prb.LS_Filter_SVD(ref, srv, 1015, 10)
    lib = _lib.load()
    out = np.empty_like(srv)
    st = lib.prc_ls_svd_frames_c64(ref.ctypes.data, srv.ctypes.data, 3000, 1, 3000, 1020, 5, out.ctypes.data, None, None,
                                   _lib.MEM_HOST, 0, None, 0)
    assert st == _lib.PRC_E_INVALID and "1024" in lib.prc_last_error().decode()
    for dt in (np.complex64, np.complex128, np.float32, np.float64):
        s = srv.astype(dt) if np.dtype(dt).kind == "c" else srv.real.astype(dt)
        from oracle import svd_oracle as so
        w_out, w_taps = so.ls_filter_svd_oracle(ref, s, 12, 3, True)
        out, taps = prb.LS_Filter_SVD(ref, s, 12, 3, True)
        assert out.dtype == w_out.dtype and taps.dtype == w_taps.dtype
        assert G.rel_inf(out, w_out, float(np.abs(s).max())) <= 1e-5
