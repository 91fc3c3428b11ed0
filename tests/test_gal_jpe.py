"""GAL_JPE (reference passiveRadar/clutter_removal.py:251-364): the plain-C oracle against the reference's own outputs,
the drop-in's signature and argument checks (no GPU needed), and the sm_90a kernel against the goldens, the oracle and
the float64 truth (GPU)."""
import ctypes as C
import hashlib
import inspect
import json
import os
import threading

import numpy as np
import pytest

import _golden as G
import passiveradar_b200 as prb
from conftest import record_parity
from passiveradar_b200 import _lib, synth

GAL_ALL = ["gal_full", "gal_partial", "gal_clamp", "gal_peek0", "gal_lattice1", "gal_mid"]
TOL = 1e-5


def _args(g):
    return (int(g["lattice_len"]), int(g["delay_line_len"]), float(g["mu1"]), float(g["mu2"]), int(g["peek"]))


def _rel(a, b, den=None):
    """max|a - b| / den (default max|b|); exact equality is required when b is all zero."""
    d = float(np.abs(b).max()) if den is None else den
    if d == 0.0:
        return 0.0 if not np.asarray(a).any() else float("inf")
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / d)


# ------------------------------------------------------------------ CPU: oracle, goldens, wrapper contract
@pytest.mark.parametrize("name", GAL_ALL)
def test_c_oracle_matches_reference_golden(name):
    from oracle import gal_oracle as co
    g = G.load(name)
    out, k, h = co.gal_jpe_oracle_c(g["ref"], g["srv"], *_args(g))
    assert _rel(out, g["out"], den=float(np.abs(g["srv"]).max())) < 1e-6
    assert _rel(k, g["k"]) < 1e-6
    assert _rel(h, g["h"]) < 1e-6
    assert not out[-(int(g["peek"]) + 1):].any()


@pytest.mark.parametrize("name", GAL_ALL)
def test_gal_golden_is_what_the_reference_produces(name):
    with open(os.path.join(G.GOLDEN_DIR, "gal_reference_digests.json")) as f:
        want = json.load(f)[name]
    committed = G.load(name)
    assert set(want) == set(committed) - {"seconds"}
    for key, digest in want.items():
        a = np.ascontiguousarray(committed[key])
        hsh = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
        hsh.update(a.tobytes())
        assert hsh.hexdigest() == digest, f"{name}[{key}] differs from the reference's output"


def test_truth_is_close_to_reference():
    from oracle import gal_oracle as co
    g = G.load("gal_mid")
    out, k, h = co.gal_jpe_truth_c(g["ref"], g["srv"], *_args(g))
    assert _rel(g["out"], out, den=float(np.abs(g["srv"]).max())) < 1e-5
    assert _rel(g["h"], h) < 1e-5


def test_signature_matches_reference():
    params = inspect.signature(prb.GAL_JPE).parameters
    assert [p for p in params if p != "device"] == ["refChannel", "srvChannel", "latticeLen", "delayLineLen", "mu1",
                                                   "mu2", "peek", "return_filter"]
    assert params["peek"].default == 10 and params["return_filter"].default is False
    assert params["device"].kind is inspect.Parameter.KEYWORD_ONLY
    assert prb.gal_jpe_frames in (getattr(prb, n) for n in prb.__all__)


def test_argument_errors_raise_before_touching_the_gpu(monkeypatch):
    def no_library(*a, **k):
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "load", no_library)
    a = np.zeros(100, np.complex64)
    with pytest.raises(ValueError, match="Input vectors must have the same length"):
        prb.GAL_JPE(a, a[:99], 4, 8, 1e-3, 1e-2)
    with pytest.raises(ValueError, match="^Delay line order must be greater than"):
        prb.GAL_JPE(a, a, 9, 8, 1e-3, 1e-2)
    with pytest.raises(ValueError):
        prb.GAL_JPE(a, a, 0, 8, 1e-3, 1e-2)
    with pytest.raises(ValueError):
        prb.gal_jpe_frames(a.reshape(4, 25), a.reshape(4, 25), 9, 8, 1e-3, 1e-2)
    with pytest.raises(ValueError):
        prb.gal_jpe_frames(a, a, 4, 8, 1e-3, 1e-2)


def test_c_abi_rejects_delay_lines_above_4096():
    lib = _lib.load()
    a = np.zeros(64, np.complex64)
    st = lib.prc_gal_jpe_frames_c64(a.ctypes.data, a.ctypes.data, 64, 1, 64, 8, 4097, 1e-3, 1e-2, 10, a.ctypes.data,
                                    None, None, _lib.MEM_HOST, 0, None, 0)
    assert st == _lib.PRC_E_INVALID
    assert "4096" in lib.prc_last_error().decode()


def test_no_cpu_fallback_without_a_device():
    if _lib.device_count() > 0:
        pytest.skip("a CUDA device is present")
    a = np.ones(256, np.complex64)
    with pytest.raises(_lib.PrcoreError):
        prb.GAL_JPE(a, a, 4, 8, 1e-3, 1e-2)
    with pytest.raises(_lib.PrcoreError):
        prb.gal_jpe_frames(np.ones((2, 64), np.complex64), np.ones((2, 64), np.complex64), 4, 8, 1e-3, 1e-2)


def test_gal_kernels_build_for_sm90a_without_spills():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    text = open(log).read()
    blocks = [blk for blk in text.split("Compiling entry function")[1:] if "gal_jpe_kernel" in blk.split("\n")[0]]
    assert len(blocks) == 5, "four warp-per-frame and one CTA-per-frame instantiation"
    for blk in blocks:
        assert "'sm_90a'" in blk.split("\n")[0]
        assert "0 bytes spill stores, 0 bytes spill loads" in blk


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", GAL_ALL)
def test_gal_matches_reference_golden(name):
    g = G.load(name)
    out, k, h = prb.GAL_JPE(g["ref"], g["srv"], *_args(g), return_filter=True)
    assert out.dtype == k.dtype == h.dtype == np.complex64
    assert out.shape == g["out"].shape and k.shape == h.shape == (int(g["delay_line_len"]),)
    e_out = _rel(out, g["out"], den=float(np.abs(g["srv"]).max()))
    record_parity(f"gal/{name}", out_vs_reference=e_out, k_vs_reference=_rel(k, g["k"]), h_vs_reference=_rel(h, g["h"]))
    assert e_out <= TOL
    assert _rel(k, g["k"]) <= 5e-5
    assert _rel(h, g["h"]) <= 5e-5
    assert not out[-(int(g["peek"]) + 1):].any()


@pytest.mark.gpu
def test_gal_long_run_matches_c_oracle_and_truth():
    """One 2**19-sample CPI (the PRconfig.yaml chunk) with 32 lattice stages and a 185-tap delay line: within 1e-5 of
    the float64 recurrence, and within 1e-5 + 1.2 x (reference-vs-truth) of the reference's complex64 arithmetic."""
    from oracle import gal_oracle as co
    n, L, D = 2 ** 19, 32, 185
    ref, srv = synth.make_frame(n, "P1", frame=5)
    want, wk, wh = co.gal_jpe_oracle_c(ref, srv, L, D, 1e-3, 1e-2, 10)
    truth, tk, th = co.gal_jpe_truth_c(ref, srv, L, D, 1e-3, 1e-2, 10)
    got, gk, gh = prb.GAL_JPE(ref, srv, L, D, 1e-3, 1e-2, 10, True)
    den = float(np.abs(srv).max())
    e_truth, e_ref, e_rt = _rel(got, truth, den), _rel(got, want, den), _rel(want, truth, den)
    record_parity("gal/long_2p19_L32_D185", out_vs_truth=e_truth, out_vs_reference=e_ref, reference_vs_truth=e_rt,
                  k_vs_truth=_rel(gk, tk), h_vs_truth=_rel(gh, th), k_vs_reference=_rel(gk, wk),
                  h_vs_reference=_rel(gh, wh))
    assert e_truth <= TOL, "GAL_JPE vs float64 truth"
    assert e_ref <= TOL + 1.2 * e_rt, "GAL_JPE vs reference arithmetic"
    assert not got[-11:].any()


@pytest.mark.gpu
@pytest.mark.parametrize("L,D,n", [(4096, 4096, 700), (100, 4096, 700), (13, 77, 3000), (200, 300, 2000),
                                   (1, 500, 1500)])
def test_gal_shapes_match_c_oracle(L, D, n):
    """The largest delay line, delay lines that are not a multiple of 32, and both kernel variants (one warp per frame
    up to 256 taps, one CTA above)."""
    from oracle import gal_oracle as co
    ref, srv = synth.make_frame(n, "P1", frame=6)
    want, wk, wh = co.gal_jpe_oracle_c(ref, srv, L, D, 1e-3, 1e-2, 7)
    got, gk, gh = prb.GAL_JPE(ref, srv, L, D, 1e-3, 1e-2, 7, True)
    e = _rel(got, want, den=float(np.abs(srv).max()))
    record_parity(f"gal/shape_L{L}_D{D}_n{n}", out_vs_reference=e, k_vs_reference=_rel(gk, wk), h_vs_reference=_rel(gh, wh))
    assert e <= TOL
    assert _rel(gk, wk) <= 5e-5 and _rel(gh, wh) <= 5e-5


@pytest.mark.gpu
def test_gal_edge_cases():
    ref, srv = synth.make_frame(12, "P0", frame=1)
    for n in (1, 5, 11):                                    # n <= peek + 1: nothing to filter
        out, k, h = prb.GAL_JPE(ref[:n], srv[:n], 3, 5, 1e-3, 1e-2, 10, True)
        assert out.shape == (n,) and not out.any() and not k.any() and not h.any()
    from oracle import gal_oracle as co
    ref, srv = synth.make_frame(2000, "P1", frame=2)
    for L, D in [(1, 1), (1, 40), (40, 40), (256, 256), (257, 257)]:
        want, wk, wh = co.gal_jpe_oracle_c(ref, srv, L, D, 1e-3, 1e-2, 10)
        got, gk, gh = prb.GAL_JPE(ref, srv, L, D, 1e-3, 1e-2, 10, True)
        assert _rel(got, want, den=float(np.abs(srv).max())) <= TOL, (L, D)
        assert _rel(gk, wk) <= 5e-5 and _rel(gh, wh) <= 5e-5, (L, D)


def _frames_call(ref, srv, n, nframes, stride, L, D, mu1, mu2, peek, out, k, h, mem, stream=None, flags=0):
    lib = _lib.load()
    return lib.prc_gal_jpe_frames_c64(_lib.ptr(ref), _lib.ptr(srv), n, nframes, stride, L, D, mu1, mu2, peek,
                                      _lib.ptr(out), _lib.ptr(k), _lib.ptr(h), mem, 0, stream, flags)


@pytest.mark.gpu
@pytest.mark.parametrize("L,D", [(16, 64), (64, 4000)])
def test_gal_batch_is_bit_identical_to_single_frames(L, D):
    """300 frames, laid out frame_stride = n + 37 apart, in one call (more frames than the GPU runs at once for the
    CTA variant) give exactly the 300 single-frame results."""
    nframes, n, stride, peek = 300, 900, 937, 5
    rng = np.random.default_rng(3)
    base = [synth.make_frame(n, "P1", frame=i) for i in range(6)]
    ref = np.zeros((nframes, stride), np.complex64)
    srv = np.zeros((nframes, stride), np.complex64)
    for i in range(nframes):
        r, s = base[i % 6]
        ph = np.complex64(np.exp(1j * rng.uniform(0, 2 * np.pi)))
        ref[i, :n], srv[i, :n] = r * ph, s * np.complex64(rng.uniform(0.5, 1.5))
        ref[i, n:] = srv[i, n:] = np.nan                   # never read
    out = np.full((nframes, stride), 7 + 7j, np.complex64)
    k = np.empty((nframes, D), np.complex64)
    h = np.empty((nframes, D), np.complex64)
    _lib.check(_frames_call(ref, srv, n, nframes, stride, L, D, 1e-3, 1e-2, peek, out, k, h, _lib.MEM_HOST))
    assert np.all(out[:, n:] == np.complex64(7 + 7j))      # the gap between frames is left alone
    for i in range(nframes):
        o1, k1, h1 = prb.GAL_JPE(ref[i, :n], srv[i, :n], L, D, 1e-3, 1e-2, peek, True)
        assert np.array_equal(out[i, :n], o1) and np.array_equal(k[i], k1) and np.array_equal(h[i], h1), i
    o2, k2, h2 = prb.gal_jpe_frames(ref[:7, :n], srv[:7, :n], L, D, 1e-3, 1e-2, peek, True)
    assert np.array_equal(o2, out[:7, :n]) and np.array_equal(k2, k[:7]) and np.array_equal(h2, h[:7])


@pytest.mark.gpu
def test_gal_device_pointers_async_on_caller_stream():
    import torch
    nframes, n, L, D = 5, 5000, 24, 300
    frames = [synth.make_frame(n, "P1", frame=20 + i) for i in range(nframes)]
    ref = np.stack([f[0] for f in frames])
    srv = np.stack([f[1] for f in frames])
    want, wk, wh = prb.gal_jpe_frames(ref, srv, L, D, 2e-3, 1e-2, 10, True)
    dev = torch.device("cuda", _lib.current_device())
    s = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(s):
        dref = torch.from_numpy(ref.view(np.float32)).to(dev)
        dsrv = torch.from_numpy(srv.view(np.float32)).to(dev)
        dout = torch.empty_like(dref)
        dk = torch.empty((nframes, 2 * D), dtype=torch.float32, device=dev)
        dh = torch.empty_like(dk)
    s.synchronize()
    _lib.check(_frames_call(dref, dsrv, n, nframes, n, L, D, 2e-3, 1e-2, 10, dout, dk, dh, _lib.MEM_DEVICE,
                            C.c_void_p(s.cuda_stream), _lib.FLAG_ASYNC))
    s.synchronize()
    got = dout.cpu().numpy().view(np.complex64)
    assert np.array_equal(got, want)
    assert np.array_equal(dk.cpu().numpy().view(np.complex64), wk)
    assert np.array_equal(dh.cpu().numpy().view(np.complex64), wh)


@pytest.mark.gpu
def test_gal_concurrent_threads_give_serial_results():
    jobs = [(synth.make_frame(20000, "P1", frame=40 + i), 8 + 4 * i, 24 + 30 * i) for i in range(8)]
    serial = [prb.GAL_JPE(r, s, L, D, 1e-3, 1e-2, 10, True) for (r, s), L, D in jobs]
    results = [None] * len(jobs)
    errors = []

    def run(i):
        try:
            (r, s), L, D = jobs[i]
            results[i] = prb.GAL_JPE(r, s, L, D, 1e-3, 1e-2, 10, True)
        except Exception as exc:           # pragma: no cover - reported below
            errors.append(exc)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for a, b in zip(results, serial):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
