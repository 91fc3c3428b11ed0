"""decimate, channel_preprocessing and normalize (reference passiveRadar/signal_utils.py:7-13, :80-85) on the device.

CPU tests: the host tap design, SciPy's shapes and dtypes, the argument errors (raised before the library loads),
install() and the goldens' provenance.  GPU tests: the decimator against the float64 closed form

    y[m] = sum_{j=0}^{20q} b[j] x[m q + 10 q - j],   x = 0 outside [0, n)

and against the reference's goldens, across q (beyond resample's limit of 89 at up = 1), n, dtypes and batches; the fused
raw-I/Q front end against the composition of the drop-ins; normalize against NumPy.
"""
import importlib.util
import json
import math
import os

import numpy as np
import pytest
import scipy.signal as signal

import passiveradar_b200 as prb
from passiveradar_b200 import _lib
from passiveradar_b200 import signal_utils as su

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_decimate_golden", os.path.join(GOLDEN, "make_decimate_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GEN = _generator()
DTYPES = ["int8", "uint8", "int16", "float32", "float64", "complex64", "complex128"]


def _goldens():
    with np.load(os.path.join(GOLDEN, "decimate_goldens.npz"), allow_pickle=False) as z:
        out = {}
        for key in z.files:
            case, field = key.split("/")
            out.setdefault(case, {})[field] = z[key]
        return out


def truth(x, q):
    """The closed form in float64 / complex128 with decimate's taps in the result dtype, along axis 0."""
    x = np.asarray(x)
    rd = su._decimate_dtype(x.dtype)
    b = su._decimate_taps(q, rd in (np.float32, np.complex64))
    n = x.shape[0]
    xs = x.reshape(n, -1).astype(np.complex128 if x.dtype.kind == "c" else np.float64)
    full = signal.oaconvolve(xs, b[:, None], axes=0) if n * b.size > 1 << 22 else \
        np.stack([np.convolve(xs[:, c], b) for c in range(xs.shape[1])], axis=1)
    y = full[10 * q::q][:-(-n // q)]
    return y.reshape((-(-n // q),) + x.shape[1:])


def rel(a, b, den=None):
    a, b = np.asarray(a), np.asarray(b)
    d = np.abs(b).max() if den is None else den
    return float(np.abs(a.astype(np.complex128) - b).max() / d) if a.size else 0.0


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("q", [2, 3, 7, 12, 90])
@pytest.mark.parametrize("dtype", ["float32", "complex64", "float64", "complex128", "int16"])
def test_host_taps_are_decimates_own(q, dtype):
    """SciPy's decimate of impulses at 10q - r in column r returns b[m q + r]: every tap, in the result dtype."""
    x = np.zeros((21 * q, q), dtype=dtype)
    x[10 * q - np.arange(q), np.arange(q)] = 1
    y = signal.decimate(x, q, 20 * q, ftype="fir", axis=0)
    rd = su._decimate_dtype(np.dtype(dtype))
    b = su._decimate_taps(q, rd in (np.float32, np.complex64))
    got = np.zeros(21 * q)
    for r in range(q):
        got[r::q][:y.shape[0]] = np.real(y[:, r])
    np.testing.assert_array_equal(got[:20 * q + 1], b)
    assert np.array_equal(b, b.astype(rd).real.astype(np.float64))


SHAPES = [((50,), 3), ((1,), 2), ((0,), 5), ((4,), 7), ((7,), 7), ((8,), 7), ((40, 3), 2), ((0, 4), 3), ((13, 2, 2), 4),
          ((6, 0), 3)]


@pytest.mark.parametrize("shape,q", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES + ["float16", "bool", "int32", "uint16"])
def test_shape_and_dtype_match_scipy(shape, q, dtype):
    x = np.ones(shape, dtype=dtype)
    y = signal.decimate(x, q, 20 * q, ftype="fir", axis=0)
    assert su._decimate_dtype(x.dtype) == y.dtype
    assert (-(-shape[0] // q),) + shape[1:] == y.shape
    if 0 in shape:                                      # answered on the host
        r = prb.decimate(x, q)
        assert r.shape == y.shape and r.dtype == y.dtype


def test_argument_errors_are_raised_before_the_library_loads(monkeypatch):
    def no_load(*a, **k):
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(_lib, "load", no_load)
    x = np.ones(100, np.complex64)
    raw = np.ones(200, np.int8)
    for fn, args, exc in [(prb.decimate, (x, 1), ValueError), (prb.decimate, (x, 0), ZeroDivisionError),
                          (prb.decimate, (x, -3), ValueError), (prb.decimate, (x, 2.0), TypeError),
                          (prb.decimate, (x, "4"), TypeError), (prb.decimate, (np.array(1.0), 2), IndexError),
                          (prb.decimate, (np.ones(4, object), 2), TypeError),
                          (prb.channel_preprocessing, (raw, 1, 0.0, 1.0), ValueError),
                          (prb.channel_preprocessing, (raw, 2.5, 0.0, 1.0), TypeError),
                          (prb.channel_preprocessing, (raw.reshape(2, 100), 4, 0.0, 1.0), ValueError),
                          (prb.normalize, (np.ones(4, np.int32),), TypeError),
                          (prb.normalize, (np.ones(4, np.float16),), TypeError),
                          (prb.normalize, (np.ones(4, bool),), TypeError)]:
        with pytest.raises(exc):
            fn(*args)
        ref_exc = None
        try:
            if fn is prb.decimate:
                signal.decimate(args[0], args[1], 20 * args[1] if not isinstance(args[1], str) else 1, ftype="fir",
                                axis=0)
        except Exception as e:                          # noqa: BLE001  SciPy's own exception for the same call
            ref_exc = e
        if fn is prb.decimate and exc is not TypeError:
            assert isinstance(ref_exc, exc), (args, ref_exc)
    assert prb.decimate(np.ones(0, np.int8), 4).dtype == np.float64
    assert prb.channel_preprocessing(np.ones(1, np.int8), 4, 0.0, 1.0).dtype == np.complex64
    assert prb.normalize(np.ones((0, 3), np.int16)).shape == (0, 3)


def test_install_swaps_the_three_names(tmp_path, monkeypatch):
    import sys
    pkg = tmp_path / "fakeRadarDec"
    pkg.mkdir()
    (pkg / "__init__.py").write_text("")
    (pkg / "range_doppler_processing.py").write_text("def fast_xambg(*a, **k):\n    return 'cpu'\n")
    (pkg / "clutter_removal.py").write_text("def LS_Filter(*a, **k):\n    return 'cpu'\n")
    (pkg / "signal_utils.py").write_text("def decimate(x, q):\n    return 'cpu'\ndef normalize(x):\n    return 'cpu'\n"
                                         "def channel_preprocessing(sig, dec, fc, Fs):\n    return 'cpu'\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    replaced = prb.install("fakeRadarDec")
    from fakeRadarDec import signal_utils as mod
    assert mod.decimate is prb.decimate and mod.normalize is prb.normalize
    assert mod.channel_preprocessing is prb.channel_preprocessing
    for name in ("decimate", "normalize", "channel_preprocessing"):
        assert f"fakeRadarDec.signal_utils.{name}" in replaced
        assert name in prb.__all__
    for m in [k for k in sys.modules if k.startswith("fakeRadarDec")]:
        del sys.modules[m]


def test_goldens_keep_their_recorded_digests():
    with open(os.path.join(GOLDEN, "decimate_reference_digests.json")) as f:
        table = json.load(f)
    gold = _goldens()
    assert sorted(table["cases"]) == sorted(list(GEN.DECIMATE) + list(GEN.CHANNEL) + list(GEN.NORMALIZE))
    for case, fields in gold.items():
        assert table["cases"][case] == {k: GEN.digest(v) for k, v in fields.items()}, case
    for name, (dtype, n, k, q, seed) in GEN.DECIMATE.items():
        assert GEN.digest(GEN.decimate_input(dtype, n, k, seed)) == str(gold[name]["input"]), name
    for name, args in GEN.CHANNEL.items():
        assert GEN.digest(GEN.channel_args(*args)[0]) == str(gold[name]["input"]), name
    for name, args in GEN.NORMALIZE.items():
        assert GEN.digest(GEN.normalize_input(*args)) == str(gold[name]["input"]), name
    assert os.path.getsize(os.path.join(GOLDEN, "decimate_goldens.npz")) < 200 * 1024


# ------------------------------------------------------------------ GPU
QS = [2, 3, 7, 12, 89, 90, 96, 173, 1000, 4096]


def _tol(dtype):
    return 1e-5 if np.dtype(dtype) in (np.float32, np.complex64) else 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("q", QS)
def test_decimate_against_the_float64_truth(q):
    """n in {1, q-1, q, q+1, 20q, 20q+1} for every dtype; float32 / complex64 within 1e-5, the rest within 1e-12."""
    for dtype in DTYPES:
        for n in sorted({1, q - 1, q, q + 1, 20 * q, 20 * q + 1}):
            x = GEN.signal(dtype, n, seed=n + q)
            y = prb.decimate(x, q)
            t = truth(x, q)
            assert y.dtype == su._decimate_dtype(x.dtype) and y.shape == t.shape
            assert rel(y, t) <= _tol(dtype), (dtype, n, q, rel(y, t))


@pytest.mark.gpu
@pytest.mark.parametrize("q", [12, 96, 4096])
def test_decimate_at_a_large_n(q):
    n = (1 << 23) + 5
    x = GEN.signal("complex64", n, seed=q)
    assert rel(prb.decimate(x, q), truth(x, q)) <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("q", [2, 12, 96, 1000])
@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("dtype", ["float32", "complex64", "int16", "complex128"])
def test_columns_of_a_2d_call_are_bit_identical_to_1d_calls(q, k, dtype):
    n = 20 * q + 37
    x = GEN.signal(dtype, n * k, seed=k * q).reshape(n, k)
    y = prb.decimate(x, q)
    assert y.shape == (-(-n // q), k)
    assert rel(y, truth(x, q)) <= _tol(dtype)
    for c in range(k):
        np.testing.assert_array_equal(y[:, c], prb.decimate(np.ascontiguousarray(x[:, c]), q))


@pytest.mark.gpu
def test_decimate_matches_the_reference_goldens():
    gold = _goldens()
    for name, (dtype, n, k, q, seed) in GEN.DECIMATE.items():
        g = gold[name]
        x = GEN.decimate_input(dtype, n, k, seed)
        y = prb.decimate(x, q)
        assert y.shape == tuple(g["shape"]) and y.dtype == g["y"].dtype, name
        got, ref, tru = y.reshape(-1)[g["idx"]], g["y"], truth(x, q).reshape(-1)[g["idx"]]
        den = np.abs(tru).max()
        r_ref = rel(ref, tru, den)
        assert rel(got, tru, den) <= 1e-5, name
        assert rel(got, ref, den) <= 1e-5 + 1.2 * r_ref, name


CHAN_MODES = [(-3.0e4, 2.4e5, ""), (1.0e4, 2.4e5, "fc16"), (5.0e3, 1.0e5, "Fs")]


def _chan_args(fc, Fs, strong):
    return (np.float16(fc) if strong == "fc16" else fc), (np.float64(Fs) if strong == "Fs" else Fs)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["int8", "int16", "float32"])
@pytest.mark.parametrize("mode", range(len(CHAN_MODES)))
@pytest.mark.parametrize("dec", [12, 96, 173])
def test_channel_preprocessing_equals_the_composition_of_the_drop_ins(kind, mode, dec):
    fc, Fs = _chan_args(*CHAN_MODES[mode])
    sig = GEN.channel_args(kind, 20 * dec + 1001, dec, 0, 1, "", dec + mode)[0]
    y = prb.channel_preprocessing(sig, dec, fc, Fs)
    comp = prb.decimate(prb.frequency_shift(prb.deinterleave_IQ(sig), fc, Fs), dec)
    assert y.dtype == comp.dtype == (np.complex64 if mode == 0 else np.complex128)
    np.testing.assert_array_equal(y, comp)
    # the reference's arithmetic, stated in float64 on the GPU drop-ins' tuned signal
    tuned = prb.frequency_shift(prb.deinterleave_IQ(sig), fc, Fs)
    assert rel(y, truth(tuned, dec)) <= _tol(y.dtype)


@pytest.mark.gpu
def test_channel_preprocessing_matches_the_reference_goldens():
    gold = _goldens()
    for name, args in GEN.CHANNEL.items():
        g = gold[name]
        sig, dec, fc, Fs = GEN.channel_args(*args)
        y = prb.channel_preprocessing(sig, dec, fc, Fs)
        assert y.shape == tuple(g["shape"]) and y.dtype == g["y"].dtype, name
        tuned = prb.frequency_shift(prb.deinterleave_IQ(sig), fc, Fs)
        tru = truth(tuned, dec).reshape(-1)[g["idx"]]
        den = np.abs(tru).max()
        got, ref = y[g["idx"]], g["y"]
        assert rel(got, tru, den) <= 1e-5, name
        assert rel(got, ref, den) <= 1e-5 + 1.2 * rel(ref, tru, den), name


@pytest.mark.gpu
def test_decimate_limits():
    x = GEN.signal("complex64", 3 * 65536 + 5, seed=1)
    assert rel(prb.decimate(x, 65536), truth(x, 65536)) <= 1e-5
    with pytest.raises(_lib.PrcoreError, match=r"q=65537 outside \[2, 65536\]"):
        prb.decimate(x[:10], 65537)


@pytest.mark.gpu
def test_every_decimator_instantiation_runs():
    """dec_kernel<float> (float32), <float2> (complex64, raw I/Q with a float32 mix), <double> (integers, float64),
    <double2> (complex128, raw I/Q with a float64 mix), norm_sum and norm_scale: each counted by the profiler."""
    cases = [lambda: prb.decimate(GEN.signal("float32", 999, 1), 5),
             lambda: prb.decimate(GEN.signal("complex64", 999, 2), 40),
             lambda: prb.channel_preprocessing(GEN.channel_args("int8", 999, 5, 0, 1, "", 3)[0], 5, 1e3, 1e4),
             lambda: prb.decimate(GEN.signal("int8", 999, 4), 17),
             lambda: prb.decimate(GEN.signal("float64", 999, 5), 3),
             lambda: prb.decimate(GEN.signal("complex128", 999, 6), 300),
             lambda: prb.channel_preprocessing(GEN.channel_args("int16", 999, 5, 0, 1, "", 7)[0], 5, 1e3,
                                               np.float64(1e4)),
             lambda: prb.normalize(GEN.signal("complex64", 999, 8))]
    _lib.profile(True)
    try:
        for fn in cases:
            _lib.profile_reset()
            fn()
            prof = _lib.profile_read()
            assert prof["decimate"][1] + prof["norm_sum"][1] >= 1
    finally:
        _lib.profile(False)
    assert prof["norm_sum"][1] == 1 and prof["norm_scale"][1] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_normalize_matches_numpy(dtype):
    for shape in [(1,), (1000,), (123, 7), (5000, 41)]:
        x = GEN.normalize_input(dtype, shape, seed=int(np.prod(shape)))
        want = x / np.mean(np.abs(x).flatten())
        got = prb.normalize(x)
        assert got.dtype == want.dtype and got.shape == want.shape
        assert rel(got, want) <= 1e-6, (dtype, shape)
    z = np.zeros(10, dtype)
    with np.errstate(invalid="ignore", divide="ignore"):
        want = z / np.mean(np.abs(z).flatten())
    got = prb.normalize(z)
    assert got.dtype == want.dtype and np.isnan(got).all() and np.isnan(want).all()


@pytest.mark.gpu
def test_normalize_matches_the_reference_goldens_and_wraps_int8():
    gold = _goldens()
    for name, (dtype, shape, seed) in GEN.NORMALIZE.items():
        x = GEN.normalize_input(dtype, shape, seed)
        got = prb.normalize(x)
        assert got.dtype == gold[name]["y"].dtype and got.shape == gold[name]["y"].shape
        assert rel(got, gold[name]["y"]) <= 1e-6, name
    x = np.array([-128, 1, 2], np.int8)             # numpy: |-128| = -128, mean -125 / 3
    np.testing.assert_allclose(prb.normalize(x), x / np.mean(np.abs(x)), rtol=1e-15)


@pytest.mark.gpu
def test_tensors_in_give_the_same_bytes_as_numpy():
    import torch
    dev = torch.device("cuda", _lib.current_device())
    for dtype in DTYPES:
        x = GEN.signal(dtype, 4000 * 3, seed=9).reshape(4000, 3)
        t = torch.from_numpy(x).to(dev)
        for q in (3, 96):
            yt = prb.decimate(t, q)
            assert yt.is_cuda
            np.testing.assert_array_equal(yt.cpu().numpy(), prb.decimate(x, q))
        nt = prb.normalize(t)
        assert nt.is_cuda
        np.testing.assert_array_equal(nt.cpu().numpy(), prb.normalize(x))
    sig = GEN.channel_args("int8", 5000, 12, 0, 1, "", 4)[0]
    ct = prb.channel_preprocessing(torch.from_numpy(sig).to(dev), 12, 2e3, 1e5)
    np.testing.assert_array_equal(ct.cpu().numpy(), prb.channel_preprocessing(sig, 12, 2e3, 1e5))
