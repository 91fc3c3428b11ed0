"""Channel-offset estimator (reference passiveRadar/signal_utils.py:29-78): the oracle against the reference's goldens,
NumPy models of the device decimator and transform, the drop-ins' signatures and argument checks, the install table and
the build (no GPU needed); the sm_90a kernels against the goldens, the oracle and the float64 truth (GPU)."""
import ctypes as C
import hashlib
import inspect
import os
import re
import threading

import numpy as np
import pytest
import scipy.signal as signal

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200 import signal_utils as psu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHANOFF = os.path.join(ROOT, "passiveradar_b200", "csrc", "chanoff.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden", "offset_goldens.npz")
SMALL = ["i8_pos", "i8_neg_nd2", "i8_edge_neg", "u8_zero_nd3", "c64_edge_nd8", "c64_outside", "c64_b1_longer",
         "i8_unequal_nd64"]


def golden(name):
    with np.load(GOLDEN, allow_pickle=False) as z:
        g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}
    n1, n2, nd, nl, delay, seed = (int(v) for v in g["args"])
    s1, s2 = synth.offset_pair(n1, n2, str(g["kind"]), delay, seed)
    for a, want in zip((s1, s2), g["digest"]):
        h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
        h.update(a.tobytes())
        assert h.hexdigest() == str(want), f"{name}: synth.offset_pair no longer makes the golden's inputs"
    return g, s1, s2, nd, nl, delay


def _rel(a, b, den):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / den)


# ------------------------------------------------------------------ CPU: oracle, models, wrapper contract
@pytest.mark.parametrize("name", SMALL)
def test_oracle_matches_reference_golden(name):
    from oracle import offset_oracle as oo
    g, s1, s2, nd, nl, _ = golden(name)
    off, xc = oo.find_channel_offset_oracle(s1, s2, nd, nl)
    assert off == int(g["offset"]) and xc.shape[0] == int(g["nvalid"])
    # SciPy's FFT rounds differently from host to host, so the same calls agree with the golden to round-off only
    assert _rel(xc[g["lags"]], g["xc"], g["xc"].max()) < 1e-12
    t_off, t_xc = oo.find_channel_offset_truth(s1, s2, nd, nl)
    assert t_off == off
    assert _rel(t_xc[g["lags"]], g["xc"], g["xc"].max()) < (1e-12 if s1.dtype.kind in "iu" else 1e-5)


@pytest.mark.parametrize("nd", [1, 2, 3, 8, 16, 32, 64])
@pytest.mark.parametrize("kind", ["int8", "complex64"])
def test_chunked_warmup_decimator_model_matches_sosfiltfilt(nd, kind):
    """The device decimator's chunking (every chunk but a pass's first starts from zero W samples early) against
    scipy.signal.sosfiltfilt.  Raising W further does not lower the nd = 64 figure (1.7e-13): what remains there is the
    float64 round-off of the recursion itself, whose poles lie at radius 0.9971."""
    from oracle import offset_oracle as oo
    s1, _ = synth.offset_pair(60000, 10, kind, 0, 100 + nd)
    sos, zi = oo.decimate_sos(nd, s1.dtype)
    w = oo.warmup_samples(sos)
    got = oo.decimate_chunked(s1, nd, 256, w)
    want = oo.decimate_truth(s1, nd)
    if s1.dtype.kind in "iu":
        np.testing.assert_array_equal(want, signal.decimate(s1, nd))     # the truth is the reference for integers
    assert _rel(got, want, np.abs(want).max()) <= (1e-13 if nd <= 32 else 3e-13)


@pytest.mark.parametrize("m", [1, 2, 5, 11, 12, 15, 20])
def test_fft_pass_model_matches_numpy(m):
    from oracle import offset_oracle as oo
    rng = np.random.default_rng(m)
    L = 1 << m
    x = rng.standard_normal(max(1, L // 2)) + 1j * rng.standard_normal(max(1, L // 2))
    y = rng.standard_normal(max(1, L // 3)) + 1j * rng.standard_normal(max(1, L // 3))
    want = np.fft.ifft(np.fft.fft(x, L) * np.conj(np.fft.fft(y, L)))
    assert _rel(oo.fft_passes_correlate(x, y, m), want, np.abs(want).max()) < 1e-14
    assert all(nb + min(3, lo) <= 11 for lo, nb in oo.pass_plan(m))


def test_signatures_match_reference():
    def names(f):
        return [p for p in inspect.signature(f).parameters if p != "device"]
    assert names(prb.find_channel_offset) == ["s1", "s2", "nd", "nl"]
    assert names(prb.offset_compensation) == ["x1", "x2", "ns", "ndec", "nlag"]
    assert inspect.signature(prb.offset_compensation).parameters["nlag"].default == 2000
    assert names(prb.xcorr) == ["s1", "s2", "nlead", "nlag"]
    assert names(prb.shift) == ["x", "n"]
    for f in (prb.find_channel_offset, prb.offset_compensation, prb.xcorr):
        assert inspect.signature(f).parameters["device"].kind is inspect.Parameter.KEYWORD_ONLY


def test_argument_errors_raise_before_the_library_loads(monkeypatch):
    def no_library(*a, **k):
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "load", no_library)
    a = np.zeros(100, np.int8)
    with pytest.raises(ValueError, match=r"^The length of the input vector x must be greater than padlen, which is 27\.$"):
        prb.find_channel_offset(a[:27], a, 1, 5)
    with pytest.raises(ValueError, match="padlen"):
        prb.find_channel_offset(a, a[:10], 1, 5)
    with pytest.raises(ZeroDivisionError):
        prb.find_channel_offset(a, a, 0, 5)
    with pytest.raises(ValueError):
        prb.find_channel_offset(a, a, -2, 5)
    with pytest.raises(TypeError):
        prb.find_channel_offset(a, a, 1.5, 5)
    with pytest.raises(ValueError, match="negative"):
        prb.find_channel_offset(a, a, 1, -1)
    with pytest.raises(ValueError, match="negative"):
        prb.xcorr(a, a, -1, 0)
    with pytest.raises(TypeError):
        prb.xcorr(a, a, 1.0, 0)


@pytest.mark.parametrize("n", [0, 1, 3, -1, -3, 7, 8, 20, -8, -20])
def test_shift_is_the_reference_shift(n):
    x = np.arange(1, 9, dtype=np.complex64)
    e = np.zeros_like(x)
    if n >= 0:
        e[n:] = x[:max(0, 8 - n)]
    else:
        e[:max(0, 8 + n)] = x[-n:]
    got = prb.shift(x, n)
    np.testing.assert_array_equal(got, e)
    assert (got is x) == (n == 0)


def test_no_cpu_fallback_without_a_device():
    if _lib.device_count() > 0:
        pytest.skip("a CUDA device is present")
    a = np.ones(256, np.int8)
    with pytest.raises(_lib.PrcoreError):
        prb.find_channel_offset(a, a, 1, 10)
    with pytest.raises(_lib.PrcoreError):
        prb.xcorr(a, a, 3, 3)


def test_install_swaps_the_offset_finder_and_leaves_xcorr(tmp_path, monkeypatch):
    import sys
    pkg = tmp_path / "offRadar"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    (pkg / "range_doppler_processing.py").write_text("def fast_xambg(*a, **k):\n    return 'cpu'\n")
    (pkg / "clutter_removal.py").write_text("def LS_Filter(*a, **k):\n    return 'cpu'\n")
    (pkg / "signal_utils.py").write_text("def find_channel_offset(*a, **k):\n    return 'cpu'\n"
                                         "def offset_compensation(*a, **k):\n    return 'cpu'\n"
                                         "def xcorr(*a, **k):\n    return 'untouched'\n")
    (pkg / "target_detection.py").write_text("raise AttributeError('np.float')\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    replaced = prb.install("offRadar")
    from offRadar import signal_utils as su
    assert su.find_channel_offset is prb.find_channel_offset and su.offset_compensation is prb.offset_compensation
    assert su.xcorr() == "untouched"
    assert "offRadar.signal_utils.find_channel_offset" in replaced and "offRadar.signal_utils.xcorr" not in replaced
    for m in [k for k in sys.modules if k.startswith("offRadar")]:
        del sys.modules[m]


def test_chanoff_kernels_build_for_sm90a_without_spills():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    blocks = [blk for blk in open(log).read().split("Compiling entry function")[1:]
              if "7chanoff" in blk.split("\n")[0]]
    assert len(blocks) == 10, "4 IIR, 2 FFT, load, twiddle, argmax, argmax_final"
    for blk in blocks:
        assert "'sm_90a'" in blk.split("\n")[0]
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in blk


# every launch in chanoff.cuh -> the GPU tests that reach it
COVERAGE = {
    "chanoff_iir_kernel<CPLX, BACKWARD>": ["test_offsets_and_lags_match_goldens", "test_main_py_shapes"],
    "chanoff_load_kernel": ["test_xcorr_dtypes_and_values"],
    "chanoff_twiddle_kernel": ["test_offsets_and_lags_match_goldens", "test_xcorr_dtypes_and_values"],
    "chanoff_fft_kernel<true>": ["test_offsets_and_lags_match_goldens", "test_xcorr_dtypes_and_values"],
    "chanoff_fft_kernel<false>": ["test_offsets_and_lags_match_goldens", "test_xcorr_dtypes_and_values"],
    "chanoff_argmax_kernel": ["test_offsets_and_lags_match_goldens", "test_xcorr_dtypes_and_values"],
    "chanoff_argmax_final_kernel": ["test_offsets_and_lags_match_goldens"],
}


def test_every_chanoff_launch_has_a_covering_gpu_test():
    src = open(CHANOFF).read()
    sites = {m.group(1) + (m.group(2) or "") for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", src)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    this = open(os.path.abspath(__file__)).read()
    for tests in COVERAGE.values():
        for t in tests:
            i = this.index(f"\ndef {t}(")
            decorators = this[this.rindex("\n\n", 0, i):i]
            assert "@pytest.mark.gpu" in decorators, f"{t} is not a GPU test"


# ------------------------------------------------------------------ GPU
def _check_xc(name, s1, xc, g, t_xc):
    den = float(g["xc"].max())
    e_ref = _rel(xc[g["lags"]], g["xc"], den)
    if s1.dtype.kind in "iuf" and s1.dtype != np.float32:
        assert e_ref <= 1e-10, name
    else:
        e_truth = _rel(xc, t_xc, float(t_xc.max()))
        r_ref = _rel(t_xc[g["lags"]], g["xc"], den)
        assert e_truth <= 1e-9, name
        assert e_ref <= 1e-5 + 1.2 * r_ref, name


@pytest.mark.gpu
@pytest.mark.parametrize("name", SMALL)
def test_offsets_and_lags_match_goldens(name):
    from oracle import offset_oracle as oo
    g, s1, s2, nd, nl, delay = golden(name)
    off, xc = psu._channel_offset(s1, s2, nd, nl, want_xc=True)
    assert isinstance(off, np.integer) and off == int(g["offset"])
    assert prb.find_channel_offset(s1, s2, nd, nl) == off
    if abs(delay) <= nl * nd and name not in ("c64_b1_longer", "i8_unequal_nd64"):
        assert off == delay
    assert xc.shape[0] == int(g["nvalid"])
    _check_xc(name, s1, xc, g, oo.find_channel_offset_truth(s1, s2, nd, nl)[1])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["int8", "complex64"])
def test_main_py_shapes(kind):
    """main.py:78-83 (10 CPIs of raw int8 per channel) and :49-54 (deinterleaved complex64), nl = 5 000 000."""
    from oracle import offset_oracle as oo
    if kind == "int8":
        g, s1, s2, nd, nl, delay = golden("i8_main")
    else:
        s1, s2 = synth.offset_pair(2621440, 2621440, "complex64", -4321, 12)
        nd, nl, delay = 1, 5000000, -4321
        o_off, o_xc = oo.find_channel_offset_oracle(s1, s2, nd, nl)
        k = int(np.argmax(o_xc))
        lags = np.unique(np.concatenate([np.arange(k - 64, k + 65), np.random.default_rng(3).integers(0, o_xc.shape[0], 256)]))
        g = {"offset": o_off, "nvalid": o_xc.shape[0], "lags": lags, "xc": o_xc[lags]}
    off, xc = psu._channel_offset(s1, s2, nd, nl, want_xc=True)
    assert off == int(g["offset"]) == delay
    assert xc.shape[0] == int(g["nvalid"])
    t_xc = oo.find_channel_offset_truth(s1, s2, nd, nl)[1] if kind != "int8" else None
    _check_xc(kind, s1, xc, g, t_xc)


@pytest.mark.gpu
@pytest.mark.parametrize("dt1,dt2", [("complex64", "complex64"), ("float64", "float64"), ("int16", "int16"),
                                     ("complex128", "float32"), ("int8", "complex64")])
@pytest.mark.parametrize("nlead,nlag", [(0, 0), (5, 0), (0, 7), (40, 33)])
def test_xcorr_dtypes_and_values(dt1, dt2, nlead, nlag):
    from oracle import offset_oracle as oo
    rng = np.random.default_rng(nlead + 3 * nlag)

    def sig(dt, n):
        if dt.startswith("int"):
            return rng.integers(-30, 30, n).astype(dt)
        x = rng.standard_normal(n) + (1j * rng.standard_normal(n) if dt.startswith("complex") else 0)
        return x.astype(dt)
    s1, s2 = sig(dt1, 3000), sig(dt2, 2000)
    got = prb.xcorr(s1, s2, nlead, nlag)
    want = oo.xcorr_oracle(s1, s2, nlead, nlag)
    assert got.dtype == want.dtype and got.shape == want.shape
    truth = oo.xcorr_oracle(s1.astype(np.complex128), s2.astype(np.complex128), nlead, nlag)
    if got.dtype.kind in "iu":
        np.testing.assert_array_equal(got, want)
    else:
        wide = prb.xcorr(s1.astype(np.complex128), s2.astype(np.complex128), nlead, nlag)
        assert _rel(wide, truth, np.abs(truth).max()) <= 1e-12
        assert _rel(got, want, np.abs(want).max()) <= (1e-12 if got.dtype.itemsize >= 8 and got.dtype != np.complex64 else 1e-5)
    short = prb.xcorr(s2, s1, nlead, nlag)          # len(s1) < len(padded s2): SciPy's swapped operands
    assert short.shape == oo.xcorr_oracle(s2, s1, nlead, nlag).shape


@pytest.mark.gpu
@pytest.mark.parametrize("delay", [37, -53, 0])
def test_offset_compensation_and_shift(delay):
    s1, s2 = synth.offset_pair(20000, 20000, "complex64", delay, 21)
    got = prb.offset_compensation(s1, s2, 8000, 1, 100)
    if delay == 0:
        assert got is s2
    else:
        np.testing.assert_array_equal(got, prb.shift(s2, delay))


def _sos(nd, single):
    s, z = psu._decimate_sos(nd, single)
    return np.ascontiguousarray(np.stack([s, s])), np.ascontiguousarray(np.stack([z, z]))


@pytest.mark.gpu
def test_device_pointers_and_caller_stream_are_bit_identical_to_the_host_path():
    import torch
    g, s1, s2, nd, nl, _ = golden("i8_neg_nd2")
    off_h, xc_h = psu._channel_offset(s1, s2, nd, nl, want_xc=True)
    lib = _lib.load()
    sos, zi = _sos(nd, False)
    t1 = torch.from_numpy(s1).cuda()
    t2 = torch.from_numpy(s2).cuda()
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    xc = torch.empty(xc_h.shape[0], dtype=torch.float64, device="cuda")
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    _lib.check(lib.prc_channel_offset(t1.data_ptr(), _lib.DT_I8, s1.shape[0], t2.data_ptr(), _lib.DT_I8, s2.shape[0], nd,
                                      nl, sos.ctypes.data, zi.ctypes.data, off.data_ptr(), xc.data_ptr(),
                                      _lib.MEM_DEVICE, 0, C.c_void_p(st.cuda_stream), _lib.FLAG_ASYNC))
    st.synchronize()
    assert int(off.item()) == off_h
    np.testing.assert_array_equal(xc.cpu().numpy(), xc_h)


@pytest.mark.gpu
def test_concurrent_threads_are_bit_identical_to_serial_calls():
    names = ["i8_pos", "u8_zero_nd3", "c64_edge_nd8", "i8_neg_nd2"] * 2
    data = [golden(n) for n in names]
    serial = [psu._channel_offset(s1, s2, nd, nl, want_xc=True) for _, s1, s2, nd, nl, _ in data]
    results = [None] * len(data)

    def run(i):
        _, s1, s2, nd, nl, _ = data[i]
        results[i] = psu._channel_offset(s1, s2, nd, nl, want_xc=True)
    threads = [threading.Thread(target=run, args=(i,)) for i in range(len(data))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for (o1, x1), (o2, x2) in zip(serial, results):
        assert o1 == o2
        np.testing.assert_array_equal(x1, x2)


@pytest.mark.gpu
def test_limits_return_invalid_with_the_limit_in_the_message():
    lib = _lib.load()
    a = np.zeros(4096, np.int8)
    sos, zi = _sos(64, False)
    off = np.zeros(1, np.int64)
    st = lib.prc_channel_offset(a.ctypes.data, _lib.DT_I8, 4096, a.ctypes.data, _lib.DT_I8, 4096, 65, 10,
                                sos.ctypes.data, zi.ctypes.data, off.ctypes.data, None, _lib.MEM_HOST, 0, None, 0)
    assert st == _lib.PRC_E_INVALID and "64" in lib.prc_last_error().decode()
    sos, zi = _sos(1, False)
    st = lib.prc_channel_offset(a.ctypes.data, _lib.DT_I8, 4096, a.ctypes.data, _lib.DT_I8, 4096, 1, 1 << 26,
                                sos.ctypes.data, zi.ctypes.data, off.ctypes.data, None, _lib.MEM_HOST, 0, None, 0)
    assert st == _lib.PRC_E_INVALID and "2^26" in lib.prc_last_error().decode()
    with pytest.raises(_lib.PrcoreError, match="64"):
        prb.find_channel_offset(a, a, 65, 3)
