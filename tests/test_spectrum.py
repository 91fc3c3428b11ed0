"""Welch PSD (mlab.psd's definition) and signal_preview.py's chain: the oracle against scipy.signal.welch, a direct
DFT and (when it imports) matplotlib itself, the goldens' provenance, prc_psd_frames' refusals, the wrapper's errors and
the preview's geometry (no GPU needed); the sm_90a kernels against the float64 oracle, batching, streams, threads and
the reference's preview goldens (GPU).

Which GPU test reaches which kernel instantiation of csrc/spectrum.cuh is listed in COVERAGE below; launch_segments
picks spec_segments_kernel<ACC> with ACC = max(1, pad_to / 256)."""
import json
import os
import re
import shutil
import subprocess
import threading

import numpy as np
import pytest
import scipy.signal as signal

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200 import spectrum as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPECTRUM = os.path.join(ROOT, "passiveradar_b200", "csrc", "spectrum.cuh")
GOLDEN = os.path.join(ROOT, "tests", "golden")
PREVIEW_CASES = ["i8_split", "i16_split", "i8_inter", "i16_inter"]

# every launch in spectrum.cuh -> the GPU tests that reach it
COVERAGE = {
    "spec_twiddle_kernel": ["test_psd_matches_float64_oracle", "test_psd_frames_rows_are_bit_identical_to_psd"],
    "spec_segments_kernel<1>": ["test_psd_matches_float64_oracle"],          # pad_to 16 .. 256
    "spec_segments_kernel<2>": ["test_psd_matches_float64_oracle"],          # 512
    "spec_segments_kernel<4>": ["test_psd_matches_float64_oracle", "test_psd_frames_rows_are_bit_identical_to_psd"],
    "spec_segments_kernel<8>": ["test_psd_matches_float64_oracle", "test_preview_goldens_host_and_device"],   # 2048
    "spec_segments_kernel<16>": ["test_psd_matches_float64_oracle"],         # 4096
    "spec_segments_kernel<32>": ["test_psd_matches_float64_oracle", "test_preview_goldens_host_and_device"],  # 8192
    "spec_finish_kernel": ["test_psd_matches_float64_oracle", "test_psd_frames_rows_are_bit_identical_to_psd"],
}


def _golden(name):
    with np.load(os.path.join(GOLDEN, f"preview_{name}.npz"), allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


def _preview_inputs(name):
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_preview_golden", os.path.join(GOLDEN, "make_preview_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.config(name), mod.sources(name), mod


def _deinterleave(raw):
    x = np.asarray(raw)
    return (x[0:-1:2] + 1j * x[1::2]).astype(np.complex64)


def _channels(config, a, b):
    icl = config["input_chunk_length"]
    if config["interleaved_input_channels"]:
        iq = _deinterleave(a[:icl])
        return iq[0::2], iq[1::2]
    return _deinterleave(a[:icl]), _deinterleave(b[:icl])


# ------------------------------------------------------------------ CPU: the oracle
WELCH_CASES = [  # (n, NFFT, noverlap, pad_to, complex)
    (5000, 256, 0, None, True), (5000, 256, 128, None, True), (5000, 256, 255, None, False),
    (4097, 16, 8, None, True), (3001, 100, 50, 128, False), (3001, 100, 99, 128, True),
    (20000, 2048, 1024, None, True), (40000, 8192, 0, None, False), (8192, 8192, 4096, None, True),
]


@pytest.mark.parametrize("n,NFFT,noverlap,pad_to,cplx", WELCH_CASES)
@pytest.mark.parametrize("scale_by_freq", [True, False])
def test_oracle_psd_matches_scipy_welch(n, NFFT, noverlap, pad_to, cplx, scale_by_freq):
    from oracle import spectrum_oracle as so
    rng = np.random.default_rng(n + NFFT)
    x = rng.standard_normal(n) + (1j * rng.standard_normal(n) if cplx else 0)
    Fs = 1e3
    P, f = so.psd_oracle(x, NFFT=NFFT, Fs=Fs, Fc=5.0, noverlap=noverlap, pad_to=pad_to, scale_by_freq=scale_by_freq)
    fw, W = signal.welch(x, fs=Fs, window=np.hanning(NFFT), nperseg=NFFT, noverlap=noverlap, nfft=pad_to or NFFT,
                         detrend=False, return_onesided=not cplx, scaling="density" if scale_by_freq else "spectrum")
    if cplx:
        W, fw = np.fft.fftshift(W), np.fft.fftshift(fw)
    assert np.abs(P - W).max() <= 1e-13 * W.max()
    np.testing.assert_allclose(f, fw + 5.0, rtol=1e-15, atol=1e-12)


@pytest.mark.parametrize("n,NFFT,pad_to,cplx", [(10, 16, None, True), (100, 256, None, False), (1, 16, 32, True),
                                                (70, 100, 128, False)])
def test_oracle_psd_of_short_signals_matches_a_direct_dft(n, NFFT, pad_to, cplx):
    """n < NFFT: mlab zero-pads to one segment (welch shortens nperseg instead, so it is no yardstick here)."""
    from oracle import spectrum_oracle as so
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n) + (1j * rng.standard_normal(n) if cplx else 0)
    P, _ = so.psd_oracle(x, NFFT=NFFT, pad_to=pad_to)
    D, _ = so.psd_dft(x, NFFT=NFFT, pad_to=pad_to)
    assert np.abs(P - D).max() <= 1e-12 * D.max()


def test_oracle_psd_matches_matplotlib_mlab():
    mlab = pytest.importorskip("matplotlib.mlab")
    from oracle import spectrum_oracle as so
    rng = np.random.default_rng(7)
    for n, NFFT, nov, pad_to, cplx, sides, sbf in [(5000, 256, 128, None, True, None, None),
                                                   (3001, 100, 50, 128, False, None, False),
                                                   (3001, 15, 5, 16, False, "onesided", True),
                                                   (10, 16, 0, None, True, "twosided", True)]:
        x = rng.standard_normal(n) + (1j * rng.standard_normal(n) if cplx else 0)
        P, f = so.psd_oracle(x, NFFT=NFFT, Fs=3.0, noverlap=nov, pad_to=pad_to, sides=sides, scale_by_freq=sbf)
        M, fm = mlab.psd(x, NFFT=NFFT, Fs=3.0, noverlap=nov, pad_to=pad_to, sides=sides, scale_by_freq=sbf)
        assert np.abs(P - M).max() <= 1e-13 * M.max()
        np.testing.assert_allclose(f, fm, rtol=1e-15, atol=1e-12)


def test_onesided_nyquist_bin_follows_mlab_rule():
    """mlab doubles the pad_to/2 bin only when NFFT is odd (its slice is chosen on NFFT, not on pad_to)."""
    from oracle import spectrum_oracle as so
    x = np.random.default_rng(3).standard_normal(400)
    for NFFT in (15, 16):
        P, _ = so.psd_oracle(x, NFFT=NFFT, pad_to=16)
        D, _ = so.psd_dft(x, NFFT=NFFT, pad_to=16, sides="twosided")        # rotated: bin 0 is -Fs/2
        assert P[-1] == pytest.approx(D[0] * (2 if NFFT % 2 else 1), rel=1e-12)
        assert P[1] == pytest.approx(2 * D[9], rel=1e-12)


# ------------------------------------------------------------------ CPU: goldens
def test_preview_goldens_keep_their_recorded_digests():
    with open(os.path.join(GOLDEN, "preview_reference_digests.json")) as f:
        table = json.load(f)
    assert sorted(table["cases"]) == sorted(PREVIEW_CASES)
    for name in PREVIEW_CASES:
        g = _golden(name)
        config, (a, b), mod = _preview_inputs(name)
        assert table["cases"][name] == {k: mod.digest(v) for k, v in g.items()}, name
        assert [mod.digest(s) for s in (a, b) if s is not None] == list(g["source_digest"]), \
            f"{name}: synth no longer makes the golden's inputs"
    total = sum(os.path.getsize(os.path.join(GOLDEN, f"preview_{n}.npz")) for n in PREVIEW_CASES)
    assert total < 200 * 1024


# ------------------------------------------------------------------ CPU: the C entry point's refusals
PSD_PARAMS = "x dtype n nframes frame_stride nfft noverlap pad_to window scale onesided out out_stride device stream flags"
_BUF = np.zeros(1 << 12, np.float64)
_P = _BUF.ctypes.data
PSD_VALID = dict(x=_P, dtype=_lib.DT_C64, n=1000, nframes=2, frame_stride=1000, nfft=256, noverlap=128, pad_to=256,
                 window=_P, scale=1.0, onesided=0, out=_P, out_stride=256, device=0, stream=None, flags=0)
PSD_ROWS = [
    ({"x": None}, "x/window/out must not be NULL"),
    ({"window": None}, "x/window/out must not be NULL"),
    ({"out": None}, "x/window/out must not be NULL"),
    ({"dtype": _lib.DT_I8}, "dtype=0 invalid: PRC_DT_F32, PRC_DT_F64, PRC_DT_C64 or PRC_DT_C128"),
    ({"dtype": _lib.DT_I16}, "dtype=2 invalid"),
    ({"dtype": 7}, "dtype=7 invalid"),
    ({"pad_to": 8, "nfft": 8, "noverlap": 0}, "pad_to=8 must be a power of two in [16, 8192]"),
    ({"pad_to": 16384, "nfft": 256}, "pad_to=16384 must be a power of two in [16, 8192]"),
    ({"pad_to": 384}, "pad_to=384 must be a power of two in [16, 8192]"),
    ({"nfft": 0, "noverlap": 0}, "nfft=0 outside [1, pad_to=256]"),
    ({"nfft": 512}, "nfft=512 outside [1, pad_to=256]"),
    ({"noverlap": -1}, "noverlap=-1 outside [0, nfft=256)"),
    ({"noverlap": 256}, "noverlap=256 outside [0, nfft=256)"),
    ({"n": 0}, "n=0 invalid"),
    ({"nframes": 0}, "nframes=0 invalid"),
    ({"frame_stride": 999}, "frame_stride=999 smaller than n=1000"),
    ({"onesided": 2}, "onesided=2 must be 0 or 1"),
    ({"out_stride": 255}, "out_stride=255 smaller than the 256 output bins"),
    ({"onesided": 1, "out_stride": 128}, "out_stride=128 smaller than the 129 output bins"),
]


def test_psd_frames_declaration_matches_the_ctypes_table():
    with open(os.path.join(ROOT, "include", "prcore.h")) as f:
        decls = dict(re.findall(r"^int (prc_\w+)\(([^;]*)\);", f.read(), re.M | re.S))
    assert "mem_kind" not in decls["prc_psd_frames"]       # device pointers only
    assert len(PSD_PARAMS.split()) == len(decls["prc_psd_frames"].split(",")) == \
        len(_lib.SIGNATURES["prc_psd_frames"][1])


@pytest.mark.parametrize("kw,msg", PSD_ROWS, ids=[m.split(" ")[0] + "-" + str(i) for i, (_, m) in enumerate(PSD_ROWS)])
def test_psd_frames_refuses_malformed_calls_before_any_launch(kw, msg):
    lib = _lib.load()
    before = _lib.launch_count()
    args = dict(PSD_VALID, **kw)
    st = lib.prc_psd_frames(*[args[p] for p in PSD_PARAMS.split()])
    err = lib.prc_last_error().decode()
    assert st == _lib.PRC_E_INVALID, (kw, st, err)
    assert msg in err, (kw, msg, err)
    assert _lib.launch_count() == before


# ------------------------------------------------------------------ CPU: the Python wrapper
def test_wrapper_errors_are_raised_before_the_library_loads(monkeypatch):
    def no_library(*a, **k):
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "load", no_library)
    x = np.zeros(1000, np.complex64)
    with pytest.raises(ValueError, match="^noverlap must be less than NFFT$"):
        prb.psd(x, NFFT=256, noverlap=256)
    with pytest.raises(ValueError, match="pad_to=128 must not be smaller than NFFT=256"):
        prb.psd(x, NFFT=256, pad_to=128)
    with pytest.raises(ValueError, match="^The window length must match the data's first dimension$"):
        prb.psd(x, NFFT=256, window=np.ones(255))
    with pytest.raises(ValueError, match="powers of two"):
        prb.psd(x, NFFT=100)
    with pytest.raises(ValueError, match="powers of two"):
        prb.psd(x, NFFT=8, pad_to=8)
    with pytest.raises(ValueError, match="powers of two"):
        prb.psd(x, NFFT=8192, pad_to=16384)
    with pytest.raises(ValueError, match="not a valid value for sides"):
        prb.psd(x, sides="both")
    with pytest.raises(ValueError, match="window must be real"):
        prb.psd(x, NFFT=16, window=np.ones(16) * 1j)
    with pytest.raises(NotImplementedError, match="detrend='mean'"):
        prb.psd(x, detrend="mean")
    with pytest.raises(NotImplementedError, match="detrend"):
        prb.psd(x, detrend=lambda s: s - s.mean())
    with pytest.raises(ValueError, match="one-dimensional"):
        prb.psd(np.zeros((2, 300)))
    with pytest.raises(ValueError, match="two-dimensional"):
        prb.psd_frames(np.zeros(300), 256)
    with pytest.raises(ValueError, match="must not be empty"):
        prb.psd(np.zeros(0))
    with pytest.raises(TypeError):
        prb.psd(x, NFFT=256.0)


def test_wrapper_plan_follows_mlab_defaults():
    def detrend_none(s):
        return s
    for dt, onesided in ((np.complex64, False), (np.complex128, False), (np.float32, True), (np.int16, True)):
        nfft, nov, pad_to, w, scale, one, f = sp._plan(np.dtype(dt), None, None, None, detrend_none, None, None, None,
                                                       None, None)
        assert (nfft, nov, pad_to, one) == (256, 0, 256, onesided)
        np.testing.assert_array_equal(w, np.hanning(256))
        assert scale == 1.0 / (2 * (np.hanning(256) ** 2).sum())
        assert f.shape[0] == (129 if onesided else 256)
        assert f[0] == (0.0 if onesided else -1.0) and f[-1] == (1.0 if onesided else 1.0 - 2 / 256)
    *_, scale, _, _ = sp._plan(np.dtype(np.complex64), 64, 10.0, 0, "none", lambda s: np.blackman(len(s)) * s, None, None,
                                None, False)
    assert scale == 1.0 / np.abs(np.blackman(64)).sum() ** 2
    assert sp._host_dtype(np.int8) == np.float64 and sp._host_dtype(np.complex64) == np.complex64
    assert sp._host_dtype(np.float16) == np.float64 and sp._host_dtype(np.clongdouble) == np.complex128


@pytest.mark.parametrize("name", PREVIEW_CASES)
def test_preview_geometry(name):
    config, (a, b), _ = _preview_inputs(name)
    g = _golden(name)
    pre = prb.SignalPreview.from_config(config)
    geo = pre.geometry(a.shape[0])
    ref, srv = _channels(config, a, b)
    assert (geo["n_ref"], geo["n_srv"]) == (ref.shape[0], srv.shape[0])
    assert (geo["n_ref_resampled"], geo["n_srv_resampled"]) == (g["ref_resampled"].shape[0], g["srv_resampled"].shape[0])
    assert geo["xcorr_lags"].shape[0] == int(g["xcorr_len"])
    assert geo["xcorr_lags"][0] == -2000
    if ref.shape[0] == srv.shape[0]:
        np.testing.assert_array_equal(geo["xcorr_lags"], np.arange(-2000, 2001))     # the script's xx
    else:
        assert config["interleaved_input_channels"] and ref.shape[0] == srv.shape[0] + 1
    np.testing.assert_allclose(geo["input_freqs"], np.fft.fftshift(np.fft.fftfreq(8192, 1 / 2400000)) + 102000000)
    np.testing.assert_allclose(geo["channel_freqs"], np.fft.fftshift(np.fft.fftfreq(2048, 1 / 200000)) + 101900000)
    with pytest.raises(ValueError):
        pre._chain(a, None if b is not None else a)


def test_shipped_preview_geometry():
    config = dict(synth.RECORDING_CONFIGS["shipped"], input_center_freq=102000000, channel_freq=101900000,
                  channel_bandwidth=200000)
    geo = prb.SignalPreview.from_config(config).geometry(10 ** 8)
    assert (geo["n_ref"], geo["n_ref_resampled"]) == (2399625, 262144)
    assert (geo["n_ref"] - 0) // 8192 == 292 and geo["n_ref_resampled"] // 2048 == 128
    inter = prb.SignalPreview.from_config(dict(config, interleaved_input_channels=True)).geometry(10 ** 8)
    assert (inter["n_ref"], inter["n_srv"]) == (1199813, 1199812)
    assert inter["xcorr_lags"].shape[0] == 4000


def test_spectrum_kernels_compile_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    tu = tmp_path / "t.cu"
    tu.write_text('#include "spectrum.cuh"\n'
                  "void f(const prc::spec::SegParams& p, const prc::spec::FinParams& q, cudaStream_t st) {\n"
                  "  prc::spec::launch_segments(p, 1, st); prc::spec::launch_finish(q, 1, st);\n"
                  "  prc::spec::launch_twiddle(nullptr, 4, st); }\n")
    res = subprocess.run([nvcc, "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                          "-I", os.path.dirname(SPECTRUM), "-c", str(tu), "-o", str(tmp_path / "t.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    log = res.stdout + res.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)'", log)
    assert len([k for k in kernels if "spec_segments_kernel" in k]) == 6 and len(kernels) == 8
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 8 and all(s == ("0", "0") for s in spills), log


def test_every_spectrum_launch_has_a_covering_gpu_test():
    src = open(SPECTRUM).read()
    sites = {m.group(1) + (m.group(2) or "") for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", src)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    this = open(os.path.abspath(__file__)).read()
    for tests in COVERAGE.values():
        for t in tests:
            i = this.index(f"\ndef {t}(")
            assert "@pytest.mark.gpu" in this[this.rindex("\n\n", 0, i):i], f"{t} is not a GPU test"


# ------------------------------------------------------------------ GPU
def _check_tight(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == np.float64, what
    peak = want.max()
    assert np.abs(got - want).max() <= 1e-12 * peak, what
    big = want > 1e-10 * peak
    assert (np.abs(got - want)[big] / want[big]).max() <= 1e-10, what


def _signal(rng, n, dt):
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    x = x if np.dtype(dt).kind == "c" else x.real
    x = x + 0.3 * np.exp(2j * np.pi * 0.123 * np.arange(n)) if np.dtype(dt).kind == "c" else \
        x + 0.3 * np.cos(2 * np.pi * 0.123 * np.arange(n))
    return x.astype(dt)


GPU_CASES = [  # (NFFT, pad_to, noverlap, n)
    (16, None, 0, 1000), (16, None, 8, 1000), (16, None, 15, 333), (16, None, 0, 10), (16, None, 0, 16),
    (100, 128, 0, 1234), (100, 128, 50, 1234), (100, 128, 99, 777), (100, 128, 0, 64),
    (256, None, 0, 5000), (256, None, 128, 5000), (256, None, 255, 3000), (256, None, 0, 256), (256, None, 0, 100),
    (20, 32, 10, 500), (40, 64, 0, 500), (512, None, 256, 9000), (1000, 1024, 500, 20000),
    (2048, None, 0, 300000), (2048, None, 1024, 20000), (2048, None, 2047, 6000), (2048, None, 0, 2048),
    (4096, None, 2048, 50000), (8192, None, 0, 100000), (8192, None, 4096, 60000), (8192, None, 8191, 9000),
    (8192, None, 0, 5000), (15, 16, 5, 400),
]


@pytest.mark.gpu
def test_psd_matches_float64_oracle():
    from oracle import spectrum_oracle as so
    rng = np.random.default_rng(2026)
    for dt in (np.complex64, np.complex128, np.float32, np.float64):
        for NFFT, pad_to, nov, n in GPU_CASES:
            x = _signal(rng, n, dt)
            what = (np.dtype(dt).name, NFFT, pad_to, nov, n)
            P, f = prb.psd(x, NFFT=NFFT, Fs=1e5, Fc=7.0, noverlap=nov, pad_to=pad_to)
            W, fw = so.psd_oracle(x, NFFT=NFFT, Fs=1e5, Fc=7.0, noverlap=nov, pad_to=pad_to)
            _check_tight(P, W, what)
            np.testing.assert_array_equal(f, fw)
        x = _signal(rng, 7000, dt)
        other = "onesided" if np.dtype(dt).kind == "c" else "twosided"
        custom = rng.uniform(0.1, 1.0, 256)
        for kw in ({"sides": other}, {"scale_by_freq": False}, {"window": custom},
                   {"window": lambda s: np.blackman(len(s)) * s}, {"window": custom, "scale_by_freq": False,
                                                                   "sides": other, "noverlap": 100}):
            P, _ = prb.psd(x, NFFT=256, Fs=3.0, **kw)
            W, _ = so.psd_oracle(x, NFFT=256, Fs=3.0, **kw)
            _check_tight(P, W, (np.dtype(dt).name, kw))
    # integers are widened to float64 on the host, as NumPy widens them for mlab
    xi = rng.integers(-128, 128, 5000).astype(np.int8)
    P, _ = prb.psd(xi, NFFT=512)
    _check_tight(P, so.psd_oracle(xi.astype(np.float64), NFFT=512)[0], "int8")


def _torch_frames(B, n, stride, seed, dt=np.complex64):
    import torch
    rng = np.random.default_rng(seed)
    host = np.zeros((B, stride), dt)
    host[:, :n] = rng.standard_normal((B, n)) + (1j * rng.standard_normal((B, n)) if np.dtype(dt).kind == "c" else 0)
    return torch.from_numpy(host).cuda()[:, :n], host[:, :n]


@pytest.mark.gpu
def test_psd_frames_rows_are_bit_identical_to_psd():
    n = 100000                                   # 195 segments at NFFT 1024: 4 segments per CTA, a ragged last chunk
    t1200, h1200 = _torch_frames(1200, n, n + 37, 5)
    for B in (1, 2, 133):
        P, f = prb.psd_frames(h1200[:B], 1024, Fs=10.0, noverlap=512)
        Pt, ft = prb.psd_frames(t1200[:B], 1024, Fs=10.0, noverlap=512)      # padded row stride on the device
        np.testing.assert_array_equal(Pt.cpu().numpy(), P)
        for b in range(B):
            np.testing.assert_array_equal(P[b], prb.psd(h1200[b], NFFT=1024, Fs=10.0, noverlap=512)[0])
    P1200, _ = prb.psd_frames(t1200, 1024, Fs=10.0, noverlap=512)
    P1200 = P1200.cpu().numpy()
    np.testing.assert_array_equal(P1200[:133], P)
    for b in np.random.default_rng(1).integers(0, 1200, 24):
        np.testing.assert_array_equal(P1200[b], prb.psd(h1200[b], NFFT=1024, Fs=10.0, noverlap=512)[0])


@pytest.mark.gpu
def test_psd_frames_on_a_caller_stream_async_matches_host_path():
    import torch
    t, h = _torch_frames(7, 30000, 30011, 9)
    want = np.stack([prb.psd(h[b], NFFT=2048, noverlap=1000, Fs=4.0)[0] for b in range(7)])
    nfft, nov, pad_to, w, scale, onesided, _ = sp._plan(np.dtype(np.complex64), 2048, 4.0, 0, None, None, 1000, None,
                                                        None, None)
    lib = _lib.load()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        wd = torch.from_numpy(w).cuda()
        out = torch.full((7, 2048 + 5), -1.0, dtype=torch.float64, device="cuda")
        _lib.check(lib.prc_psd_frames(t.data_ptr(), _lib.DT_C64, 30000, 7, t.stride(0), nfft, nov, pad_to,
                                      wd.data_ptr(), scale, int(onesided), out.data_ptr(), out.stride(0), 0,
                                      s.cuda_stream, _lib.FLAG_ASYNC))
    s.synchronize()
    got = out.cpu().numpy()
    np.testing.assert_array_equal(got[:, :2048], want)
    assert (got[:, 2048:] == -1.0).all()


@pytest.mark.gpu
def test_psd_threads_are_bit_identical_to_serial_calls():
    rng = np.random.default_rng(11)
    xs = [_signal(rng, 50000 + 999 * k, np.complex64) for k in range(8)]
    serial = [prb.psd(x, NFFT=4096, noverlap=1024)[0] for x in xs]
    got = [None] * 8
    errors = []

    def work(k):
        try:
            for _ in range(3):
                got[k] = prb.psd(xs[k], NFFT=4096, noverlap=1024)[0]
        except Exception as exc:          # reported below
            errors.append(exc)
    threads = [threading.Thread(target=work, args=(k,)) for k in range(8)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for k in range(8):
        np.testing.assert_array_equal(got[k], serial[k])


@pytest.mark.gpu
@pytest.mark.parametrize("name", PREVIEW_CASES)
def test_preview_goldens_host_and_device(name):
    import torch
    from oracle import spectrum_oracle as so
    g = _golden(name)
    config, (a, b), _ = _preview_inputs(name)
    pre = prb.SignalPreview.from_config(config)
    r = pre.run(a, b)
    rd = pre.run_device(torch.from_numpy(a).cuda(), None if b is None else torch.from_numpy(b).cuda())
    assert r["offset"] == rd["offset"] == int(g["offset"])
    for k in ("input_psd", "channel_psd", "xcorr_abs", "input_freqs", "channel_freqs", "xcorr_lags"):
        np.testing.assert_array_equal(rd[k].cpu().numpy(), r[k], err_msg=k)
    ref, srv = _channels(config, a, b)
    t = so.xcorr_truth(ref, srv, 2000, 2000)
    assert r["xcorr_abs"].shape == t.shape == (int(g["xcorr_len"]),)
    assert np.abs(r["xcorr_abs"] - t).max() <= 1e-9 * t.max()
    np.testing.assert_array_equal(r["xcorr_lags"], np.arange(t.shape[0]) - 2000)
    lo = int(g["xcorr_peak_lo"])
    assert np.abs(r["xcorr_abs"][lo:lo + g["xcorr_peak"].shape[0]] - g["xcorr_peak"]).max() <= 1e-5 * t.max()
    for q, s in enumerate((ref, srv)):
        W, f = so.psd_oracle(s, NFFT=8192, Fs=config["input_sample_rate"], Fc=config["input_center_freq"])
        _check_tight(r["input_psd"][q], W, (name, "input", q))
        np.testing.assert_array_equal(r["input_freqs"], f)
        rs = g["ref_resampled" if q == 0 else "srv_resampled"]
        W, f = so.psd_oracle(rs, NFFT=2048, Fs=config["channel_bandwidth"], Fc=config["channel_freq"])
        assert np.abs(r["channel_psd"][q] - W).max() <= 1e-5 * W.max(), (name, q)
        np.testing.assert_array_equal(r["channel_freqs"], f)
        P, _ = prb.psd(rs, NFFT=2048, Fs=config["channel_bandwidth"], Fc=config["channel_freq"])
        _check_tight(P, W, (name, "resampled", q))


@pytest.mark.gpu
def test_preview_at_the_shipped_shape_finds_the_planted_offset():
    config = dict(synth.RECORDING_CONFIGS["shipped"], input_center_freq=102000000, channel_freq=101900000,
                  channel_bandwidth=200000)
    ref, srv, _, _ = synth.recording_for(config, 1, channel_delay=12, seed=4)
    _lib.profile_reset()
    _lib.profile(True)
    try:
        r = prb.SignalPreview.from_config(config).run(ref, srv)
        prof = _lib.profile_read()
    finally:
        _lib.profile(False)
    assert r["offset"] == -12
    assert r["input_psd"].shape == (2, 8192) and r["channel_psd"].shape == (2, 2048)
    assert r["xcorr_abs"].shape == (4001,) and r["xcorr_abs"].dtype == np.float64
    assert int(np.argmax(r["xcorr_abs"])) - 2000 == -12
    assert prof["psd_segments"][1] >= 4 and prof["psd_finish"][1] == 2          # one call per pair of spectra
