"""Every kernel instantiation prcore's host code can launch, run against the suite's oracles and float64 truths.

Three parts:

* Direct-form cases (GPU).  LS, Toeplitz, CAF and whole-frame inputs at config 2 and below run on the FP32 direct form
  ("fft" set to 0 for the test), and NLMS at 410 .. 3010 taps on its one path.  Outputs are held to the float64 truth
  (1e-5) and to the reference-pinned oracle or golden (1e-5 + 1.2 x reference-vs-truth), as in
  tests/test_gpu_parity.py.  Each oracle is computed once per module.
* GPU cases for dispatches of the default configuration no other test reaches: NLMS with more than 1024 taps, the
  Doppler stage at F = 4096 .. 16384, the tap-weighted decimator at full size, and 5-frame CAF batches.
* A CPU guard: every kernel launch site of the library's sources must appear in COVERAGE with the GPU tests that reach it.

Per-case figures go to $PRC_PARITY_DIR/parity.json (tests/conftest.py:record_parity).
"""
import os
import re

import numpy as np
import pytest
import scipy.signal as signal

import _golden as G
from conftest import record_parity
from passiveradar_b200 import _lib, build, synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TOL = 1e-5

DIRECT = ["ls_big", "ls_small", "ls_wide", "toep", "caf_big", "caf_small", "frame"]


# ------------------------------------------------------------------ case inputs
# Output keys are "<case>.<item>.<profile>.<field>"; the profile is the channel model (P0: independent channels, P1:
# strong clutter).
KAISER = ("kaiser", 5.0)


def ls_items(case):
    """LS_Filter inputs: (item, profile, golden name or None, ref, srv, filter_len, reg, peek)."""
    if case == "ls_big":          # n = 2**20, 310 taps: lagstream_kernel, levinson_kernel<1>, fir_apply_kernel
        for name in ("ls_c2_p1", "frame_c2_p0"):
            g = G.load(name)
            ref, srv = G.inputs(g)
            yield name, str(g["profile"]), name, ref, srv, 300, 1.0, 10
    elif case == "ls_small":      # lagstream_kernel, fir_apply_kernel, levinson_kernel<1>
        ref, srv = synth.make_frame(5000, "P0", frame=9)
        yield "n5000", "P0", None, ref, srv, 20, 1.0, 10
        for name in ("ls_small", "ls_small_peek0", "ls_small_reg0"):
            g = G.load(name)
            ref, srv = G.inputs(g)
            yield name, str(g["profile"]), name, ref, srv, int(g["filter_len"]), float(g["reg"]), int(g["peek"])
    elif case == "ls_wide":       # 1110 taps: levinson_kernel<4>
        for profile in ("P1", "P0"):
            ref, srv = synth.make_frame(2 ** 18, profile, frame=2)
            yield f"n262144_{profile}", profile, None, ref, srv, 1100, 1.0, 10


def toep_items():
    for name in ("toep_small", "toep_mid"):
        g = G.load(name)
        ref, srv = G.inputs(g)
        yield name, str(g["profile"]), g, ref, srv


def caf_items(case):
    """fast_xambg inputs: (item, profile, golden or None, ref, srv, R, F, input_len, window, short_filt)."""
    if case == "caf_big":         # D = 4096: weight_kernel, lagstream_kernel (CAF)
        n = 2 ** 20
        ref, srv = synth.make_frame(n, "P0", frame=21)
        yield "n1048576", "P0", None, ref, srv, 300, 256, n, signal.get_window(KAISER, n), True
    elif case == "caf_small":     # Doppler blocks of < 64 taps and the tap-weighted decimator: lagcorr_kernel
        ref, srv = synth.make_frame(1000, "P0", frame=3)
        yield "n1000", "P0", None, ref, srv, 9, 16, None, None, True
        g = G.load("xambg_longfilt")
        ref, srv = G.inputs(g)
        R, F, input_len, window, short = G.xambg_args(g)
        yield "xambg_longfilt", str(g["profile"]), g, ref, srv, R, F, input_len, window, short


FRAME = dict(name="frame_c2_p0", filter_len=300, reg=1.0, peek=10)


def frame_inputs():
    g = G.load(FRAME["name"])
    ref, srv = G.inputs(g)
    return g, ref, srv, int(g["n"]), int(g["R"]), int(g["F"])


NLMS = dict(n=2 ** 15, profile="P1", frame=4, mu=0.05, peek=10)
NLMS_FILTER_LENS = (400, 1100, 3000)       # M = 410, 1110, 3010: nlms_block_kernel<1>, <2>, <4>
NLMS_BLOCK = dict(filter_len=1100, block_len=64)


def nlms_inputs():
    return synth.make_frame(NLMS["n"], NLMS["profile"], frame=NLMS["frame"])


# ------------------------------------------------------------------ runners: each fills `res` with its case's outputs
def run_ls(case, res):
    import passiveradar_b200 as prb
    for item, profile, _, ref, srv, fl, reg, peek in ls_items(case):
        out, taps = prb.LS_Filter(ref, srv, fl, reg, peek, True)
        res[f"{case}.{item}.{profile}.out"] = out
        res[f"{case}.{item}.{profile}.taps"] = taps


def run_toep(res):
    import passiveradar_b200 as prb
    for item, profile, g, ref, srv in toep_items():
        out, taps = prb.LS_Filter_Toeplitz(ref, srv, int(g["filter_len"]), int(g["peek"]), True)
        res[f"toep.{item}.{profile}.out"] = out
        res[f"toep.{item}.{profile}.taps"] = taps


def run_caf(case, res):
    import passiveradar_b200 as prb
    for item, profile, _, ref, srv, R, F, input_len, window, short in caf_items(case):
        res[f"{case}.{item}.{profile}.map"] = prb.fast_xambg(ref, srv, R, F, input_len, window, short)


def run_frame(res):
    """One frame through prc_frame_c64 (the entry point of FramePipeline) on the direct form: the LS stage's kernels, then
    the CAF of the cleaned channel against the reference weighted by weight_kernel."""
    g, ref, srv, n, R, F = frame_inputs()
    M = FRAME["filter_len"] + FRAME["peek"]
    w = np.ascontiguousarray(signal.get_window(KAISER, n), dtype=np.float64)
    maps = np.empty((F, R + 1), np.complex64)
    taps = np.empty(M, np.complex64)
    clean = np.empty(n, np.complex64)
    lib = _lib.load()
    _lib.check(lib.prc_frame_c64(ref.ctypes.data, srv.ctypes.data, n, FRAME["filter_len"], FRAME["peek"], FRAME["reg"], R, F,
                                 w.ctypes.data, maps.ctypes.data, taps.ctypes.data, clean.ctypes.data, _lib.MEM_HOST,
                                 _lib.current_device(), None, 0))
    prof = str(g["profile"])
    res[f"frame.{FRAME['name']}.{prof}.map"] = maps[:, :, None]
    res[f"frame.{FRAME['name']}.{prof}.taps"] = taps
    res[f"frame.{FRAME['name']}.{prof}.out"] = clean


def run_nlms(res):
    import passiveradar_b200 as prb
    ref, srv = nlms_inputs()
    p = NLMS["profile"]
    for fl in NLMS_FILTER_LENS:
        out, taps = prb.NLMS_filter(ref, srv, fl, NLMS["mu"], NLMS["peek"], None, True)
        res[f"nlms.M{fl + NLMS['peek']}.{p}.out"] = out
        res[f"nlms.M{fl + NLMS['peek']}.{p}.taps"] = taps
    fl, B = NLMS_BLOCK["filter_len"], NLMS_BLOCK["block_len"]
    out, taps = prb.block_NLMS(ref, srv, fl, NLMS["mu"], NLMS["peek"], B, None, True)
    res[f"nlms.M{fl + NLMS['peek']}_B{B}.{p}.out"] = out
    res[f"nlms.M{fl + NLMS['peek']}_B{B}.{p}.taps"] = taps


RUNNERS = {
    "ls_big": lambda res: run_ls("ls_big", res),
    "ls_small": lambda res: run_ls("ls_small", res),
    "ls_wide": lambda res: run_ls("ls_wide", res),
    "toep": run_toep,
    "caf_big": lambda res: run_caf("caf_big", res),
    "caf_small": lambda res: run_caf("caf_small", res),
    "frame": run_frame,
}


def _rel_columns(got, want_cols, lags, R, peak):
    """max over the sampled lags d of |got[:, R - d] - want column| / peak."""
    return max(float(np.abs(got[:, R - d, 0] - want_cols[d]).max()) / peak for d in lags)


# ------------------------------------------------------------------ oracles and truths, computed once per session
class Oracles:
    """Lazily computed CPU oracles / float64 truths of the cases, cached for the whole module."""

    def __init__(self):
        self._cache = {}

    def get(self, key, fn):
        if key not in self._cache:
            self._cache[key] = fn()
        return self._cache[key]

    def ls(self, case):
        """item -> dict(truth=(out, taps), oracle=(out at idx or None, taps) or None, idx, den = max|srv|, profile).
        The oracle is the item's golden (made by the reference) or, for small synthetic items, the live complex64 oracle."""
        def make():
            from oracle import clutter_oracle as co
            d = {}
            for item, profile, golden, ref, srv, fl, reg, peek in ls_items(case):
                t_out, t_taps = co.ls_filter_truth(ref, srv, fl, reg, peek)
                den = float(np.abs(srv).max())
                e = dict(truth=(t_out, t_taps), den=den, profile=profile, oracle=None)
                if golden is not None:
                    g = G.load(golden)
                    idx = g["out_idx"] if "out_idx" in g else None
                    e["oracle"] = (None if idx is None else g["out_sub"], g["taps"])
                    e["idx"] = idx
                elif fl + peek <= 64:          # the complex64 oracle forms the n x M data matrix: small problems only
                    o_out, o_taps = co.ls_filter_oracle(ref, srv, fl, reg, peek, True)
                    e["oracle"] = (o_out, o_taps)
                    e["idx"] = np.arange(ref.shape[0])
                d[item] = e
            return d
        return self.get(("ls", case), make)

    def toep(self):
        def make():
            from oracle import clutter_oracle as co
            d = {}
            for item, profile, g, ref, srv in toep_items():
                t_out, t_taps = co.ls_filter_toeplitz_oracle(ref, srv, int(g["filter_len"]), int(g["peek"]), True)
                d[item] = dict(truth=(t_out, t_taps), golden=g, den=float(g["srv_absmax"]))
            return d
        return self.get("toep", make)

    def caf(self, case):
        """item -> dict(lags, oracle columns, truth columns) for caf_big; whole maps for caf_small."""
        def make():
            from oracle import xambg_oracle as xo
            d = {}
            for item, profile, golden, ref, srv, R, F, input_len, window, short in caf_items(case):
                if case == "caf_big":
                    n = ref.shape[0]
                    lags = sorted({0, 1, R // 3, R // 2, R - 1, R})
                    oc = {k: xo.fast_xambg_oracle(ref, np.roll(srv, -k), 0, F, n, window)[:, 0, 0] for k in lags}
                    tc = {k: xo.fast_xambg_truth(ref, np.roll(srv, -k), 0, F, n, window)[:, 0, 0] for k in lags}
                    d[item] = dict(lags=lags, oracle=oc, truth=tc, R=R, profile=profile)
                else:
                    truth = xo.fast_xambg_truth(ref, srv, R, F, input_len, window, short)
                    oracle = golden["out"] if golden is not None else xo.fast_xambg_oracle(ref, srv, R, F, input_len, window, short)
                    d[item] = dict(truth=truth, oracle=oracle, profile=profile)
            return d
        return self.get(("caf", case), make)

    def frame(self):
        def make():
            from oracle import clutter_oracle as co
            from oracle import xambg_oracle as xo
            g, ref, srv, n, R, F = frame_inputs()
            t_clean, t_taps = co.ls_filter_truth(ref, srv, FRAME["filter_len"], FRAME["reg"], FRAME["peek"])
            t_map = xo.fast_xambg_truth(ref, t_clean, R, F, n, signal.get_window(KAISER, n))
            return dict(golden=g, t_clean=t_clean, t_taps=t_taps, t_map=t_map, den=float(np.abs(srv).max()))
        return self.get("frame", make)

    def nlms(self):
        """key (as run_nlms names it) ->(oracle out, oracle taps, truth out, truth taps) of the C oracle."""
        def make():
            from oracle import clutter_oracle as co
            ref, srv = nlms_inputs()
            mu, peek = NLMS["mu"], NLMS["peek"]
            d = {}
            for fl in NLMS_FILTER_LENS:
                d[f"M{fl + peek}"] = co.block_nlms_oracle_c(ref, srv, fl, mu, peek, 1) + co.block_nlms_truth_c(ref, srv, fl, mu, peek, 1)
            fl, B = NLMS_BLOCK["filter_len"], NLMS_BLOCK["block_len"]
            d[f"M{fl + peek}_B{B}"] = co.block_nlms_oracle_c(ref, srv, fl, mu, peek, B) + co.block_nlms_truth_c(ref, srv, fl, mu, peek, B)
            return d
        return self.get("nlms", make)


@pytest.fixture(scope="module")
def oracles():
    return Oracles()


@pytest.fixture
def direct_form():
    """Run a test on the FP32 direct-form kernels ("fft" = 0) and restore the library's "fft" option afterwards."""
    old = _lib.get_option("fft")
    _lib.set_option("fft", 0)
    yield
    _lib.set_option("fft", old)


# ------------------------------------------------------------------ per-case checks against truth and oracle
def _check_ls(case, res, orc, fig):
    for item, e in orc.ls(case).items():
        p = f"{case}.{item}.{e['profile']}"
        out, taps = res[p + ".out"], res[p + ".taps"]
        t_out, t_taps = e["truth"]
        fig[f"{item}/taps_vs_truth"] = et = G.rel_inf(taps, t_taps)
        fig[f"{item}/out_vs_truth"] = eo = G.rel_inf(out, t_out, den=e["den"])
        assert et <= TOL and eo <= TOL, (case, item, et, eo)
        if e["oracle"] is not None:
            o_out, o_taps = e["oracle"]
            er = G.rel_inf(o_taps, t_taps)
            fig[f"{item}/taps_vs_reference"] = ed = G.rel_inf(taps, o_taps)
            assert ed <= TOL + 1.2 * er, (case, item, ed, er)
            if o_out is not None:
                idx = e["idx"]
                er_o = G.rel_inf(o_out, t_out[idx], den=e["den"])
                fig[f"{item}/out_vs_reference"] = ed = G.rel_inf(out[idx], o_out, den=e["den"])
                assert ed <= TOL + 1.2 * er_o, (case, item, ed, er_o)


def _check_toep(res, orc, fig):
    for item, e in orc.toep().items():
        g = e["golden"]
        p = f"toep.{item}.{g['profile']}"
        out, taps = res[p + ".out"], res[p + ".taps"]
        t_out, t_taps = e["truth"]               # the complex128 Levinson solve of the reference's formulation
        fig[f"{item}/taps_vs_truth"] = et = G.rel_inf(taps, t_taps)
        fig[f"{item}/out_vs_truth"] = eo = G.rel_inf(out, t_out, den=e["den"])
        assert et <= TOL and eo <= TOL, (item, et, eo)
        er = G.rel_inf(g["taps"], t_taps)
        er_o = G.rel_inf(g["out_sub"], t_out[g["out_idx"]], den=e["den"])
        assert G.rel_inf(taps, g["taps"]) <= TOL + 1.2 * er, item
        assert G.rel_inf(out[g["out_idx"]], g["out_sub"], den=e["den"]) <= TOL + 1.2 * er_o, item


def _check_caf(case, res, orc, fig):
    for item, e in orc.caf(case).items():
        got = res[f"{case}.{item}.{e['profile']}.map"]
        if case == "caf_big":
            peak = float(np.abs(got).max())
            et = _rel_columns(got, e["truth"], e["lags"], e["R"], peak)
            eo = _rel_columns(got, e["oracle"], e["lags"], e["R"], peak)
            er = max(float(np.abs(e["oracle"][d] - e["truth"][d]).max()) / peak for d in e["lags"])
        else:
            et, eo, er = G.rel_inf(got, e["truth"]), G.rel_inf(got, e["oracle"]), G.rel_inf(e["oracle"], e["truth"])
        fig[f"{item}/map_vs_truth"], fig[f"{item}/map_vs_reference"] = et, eo
        assert et <= TOL, (case, item, et)
        assert eo <= TOL + 1.2 * er, (case, item, eo, er)


def _check_frame(res, orc, fig):
    e = orc.frame()
    g = e["golden"]
    p = f"frame.{FRAME['name']}.{g['profile']}"
    fig["map_vs_truth"] = em = G.rel_inf(res[p + ".map"], e["t_map"])
    fig["taps_vs_truth"] = et = G.rel_inf(res[p + ".taps"], e["t_taps"])
    fig["out_vs_truth"] = eo = G.rel_inf(res[p + ".out"], e["t_clean"], den=e["den"])
    assert em <= TOL and et <= TOL and eo <= TOL, (em, et, eo)
    er_map, er_taps = G.rel_inf(g["out"], e["t_map"]), G.rel_inf(g["taps"], e["t_taps"])
    fig["map_vs_reference"] = ed = G.rel_inf(res[p + ".map"], g["out"])
    assert ed <= TOL + 1.2 * er_map, (ed, er_map)
    assert G.rel_inf(res[p + ".taps"], g["taps"]) <= TOL + 1.2 * er_taps


def _nlms_bounds(out, taps, want, ww, truth, tw, what):
    """NLMS output against the float64 recurrence (1e-5 of max|truth|) and the reference-pinned C oracle
    (1e-5 + 1.2 x oracle-vs-truth); taps within 5e-5 of both, as tests/test_gpu_parity.py holds config 4."""
    den = float(np.abs(truth).max())
    et, eo, er = G.rel_inf(out, truth, den=den), G.rel_inf(out, want, den=den), G.rel_inf(want, truth, den=den)
    assert et <= TOL, (what, et)
    assert eo <= TOL + 1.2 * er, (what, eo, er)
    assert G.rel_inf(taps, tw) <= 5e-5 and G.rel_inf(taps, ww) <= 5e-5, what
    return dict(out_vs_truth=et, out_vs_reference=eo, reference_vs_truth=er)


def _check_nlms(res, orc, fig):
    prof = NLMS["profile"]
    for key, (want, ww, truth, tw) in orc.nlms().items():
        out, taps = res[f"nlms.{key}.{prof}.out"], res[f"nlms.{key}.{prof}.taps"]
        for k, v in _nlms_bounds(out, taps, want, ww, truth, tw, key).items():
            fig[f"{key}/{k}"] = v
        fl = int(key[1:].split("_")[0]) - NLMS["peek"]
        assert not out[:fl].any() and not out[-NLMS["peek"]:].any(), key


def _check(case, res, orc, fig):
    if case in ("ls_big", "ls_small", "ls_wide"):
        _check_ls(case, res, orc, fig)
    elif case == "toep":
        _check_toep(res, orc, fig)
    elif case in ("caf_big", "caf_small"):
        _check_caf(case, res, orc, fig)
    elif case == "frame":
        _check_frame(res, orc, fig)
    else:
        _check_nlms(res, orc, fig)


@pytest.mark.gpu
@pytest.mark.parametrize("case", DIRECT)
def test_direct_form_matches_truth_and_reference(case, direct_form, oracles):
    res, fig = {}, {}
    RUNNERS[case](res)
    _check(case, res, oracles, fig)
    record_parity(f"variants/default/{case}", **fig)


@pytest.mark.gpu
def test_nlms_matches_truth_and_reference(oracles):
    res, fig = {}, {}
    run_nlms(res)
    _check("nlms", res, oracles, fig)
    record_parity("variants/default/nlms", **fig)


@pytest.mark.parametrize("name", ["stream", "packed", "tile", "nlms_block", "tma", "tma_l2", "tc", "tc_caf", "tc_fir",
                                  "tune_nchunk", "tune_g", "tma_active", "caf_wave", "fft_ctas_caf"])
def test_retired_switches_are_unknown_options(name):
    """The switches INTEGRATION.md section 6 lists as no longer read ("tune_nchunk" and "tune_g" reported PRC_TUNE_NCHUNK
    and PRC_TUNE_G) and the options it lists as removed ("tma_active" reported the loader the "tma" switch selected,
    "fft_ctas_caf" the residency the "caf_wave" grid was sized from): their option names are unknown, not read-only,
    so a library that still kept one of them fails here."""
    lib = _lib.load()
    with pytest.raises(_lib.PrcoreError):
        _lib.get_option(name)
    assert b"unknown option" in lib.prc_last_error()
    assert lib.prc_set_option(name.encode(), 1) == _lib.PRC_E_INVALID
    assert b"unknown option" in lib.prc_last_error()


# ------------------------------------------------------------------ default-configuration dispatches (in process)
@pytest.mark.gpu
@pytest.mark.parametrize("fl", [1100, 3000])
def test_nlms_with_more_than_1024_taps_matches_c_oracle(fl, oracles):
    """M = 1110 and 3010: nlms_block_kernel<2> and <4> (two and four taps per thread)."""
    import passiveradar_b200 as prb
    ref, srv = nlms_inputs()
    mu, peek = NLMS["mu"], NLMS["peek"]
    got, gw = prb.NLMS_filter(ref, srv, fl, mu, peek, None, True)
    fig = _nlms_bounds(got, gw, *oracles.nlms()[f"M{fl + peek}"], fl)
    record_parity(f"nlms/n32768_M{fl + peek}", **fig)
    assert not got[:fl].any() and not got[-peek:].any()


@pytest.mark.gpu
def test_nlms_accepts_4096_taps_and_names_the_limit_above():
    import passiveradar_b200 as prb
    from oracle import clutter_oracle as co
    ref, srv = synth.make_frame(6000, "P1", frame=12)
    got, gw = prb.NLMS_filter(ref, srv, 4086, 0.05, 10, None, True)
    want = co.block_nlms_oracle_c(ref, srv, 4086, 0.05, 10, 1) + co.block_nlms_truth_c(ref, srv, 4086, 0.05, 10, 1)
    record_parity("nlms/n6000_M4096", **_nlms_bounds(got, gw, *want, 4086))
    with pytest.raises(_lib.PrcoreError, match="4096"):
        prb.NLMS_filter(ref, srv, 4087, 0.05, 10)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1000, 2000])
def test_nlms_frames_past_the_sm_count_with_many_taps(M):
    """More frames than SMs at M = 1000 and 2000: nlms_block_kernel<2, 512> and <4, 512> against single-frame calls and
    the C oracle (bounds of test_nlms_large_batch_uses_the_half_size_ctas_and_matches)."""
    import torch
    import passiveradar_b200 as prb
    from oracle import clutter_oracle as co
    nf = torch.cuda.get_device_properties(0).multi_processor_count + 12
    n, peek, mu = 2 ** 13, 10, 0.05
    fl = M - peek
    base = [synth.make_frame(n, "P1", frame=180 + i) for i in range(4)]
    dev = torch.device("cuda", 0)
    ref_d = torch.from_numpy(np.stack([base[i % 4][0] for i in range(nf)])).to(dev)
    srv_d = torch.from_numpy(np.stack([base[i % 4][1] for i in range(nf)])).to(dev)
    out = torch.empty((nf, n), dtype=torch.complex64, device=dev)
    taps = torch.empty((nf, M), dtype=torch.complex64, device=dev)
    lib = _lib.load()
    st = torch.cuda.Stream(device=dev)
    _lib.check(lib.prc_nlms_frames_c64(ref_d.data_ptr(), srv_d.data_ptr(), n, nf, n, fl, peek, mu, 1, None, out.data_ptr(),
                                       taps.data_ptr(), _lib.MEM_DEVICE, 0, st.cuda_stream, 0))
    got, gt = out.cpu().numpy(), taps.cpu().numpy()
    for i in (0, 1, 2, 3, nf - 1):
        ref, srv = base[i % 4]
        want, _ = co.block_nlms_oracle_c(ref, srv, fl, mu, peek, 1)
        single, st1 = prb.NLMS_filter(ref, srv, fl, mu, peek, None, True)
        den = float(np.abs(want).max())
        assert G.rel_inf(got[i], want, den=den) <= TOL, i
        assert G.rel_inf(got[i], single, den=den) <= 2e-6, i
        assert G.rel_inf(gt[i], st1) <= 5e-5, i
    assert np.array_equal(got[0], got[4])


_DOPPLER_SHAPES = [(2 ** 20, 4096), (2 ** 20, 8192), (2 ** 20, 16384), (2 ** 22, 8192), (2 ** 22, 16384)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,F", _DOPPLER_SHAPES)
def test_doppler_stage_at_large_F(n, F, both_paths, oracles):
    """F = 4096: doppler_fft_pow2_kernel<2>; 8192: <1>; 16384: chunk sums + direct DFT.  Sampled range columns against
    the oracle (columns are independent: lag d of srv is lag 0 of srv rolled by -d)."""
    import passiveradar_b200 as prb
    from oracle import xambg_oracle as xo
    R = 40
    ref, srv = synth.make_frame(n, "P1", frame=25)
    w = signal.get_window(KAISER, n)
    lags = [0, 1, R // 2, R - 1, R]
    cols = oracles.get(("doppler", n, F), lambda: {d: xo.fast_xambg_oracle(ref, np.roll(srv, -d), 0, F, n, w)[:, 0, 0] for d in lags})
    got = prb.fast_xambg(ref, srv, R, F, n, w)
    e = _rel_columns(got, cols, lags, R, float(np.abs(got).max()))
    record_parity(f"xambg/doppler_n{n}_F{F}/{both_paths}", E_vs_oracle_sampled_columns=e)
    assert e <= TOL, e


@pytest.mark.gpu
def test_tap_weighted_decimator_at_full_size(both_paths, oracles):
    """fast_xambg(..., shortFilt=False) at config 2: 40 961 flat-top taps per Doppler block, lagcorr_kernel with taps
    on either path (the FFT-domain CAF takes the boxcar decimator only)."""
    import passiveradar_b200 as prb
    from oracle import xambg_oracle as xo
    n, F, R = 2 ** 20, 256, 300
    ref, srv = synth.make_frame(n, "P1", frame=26)
    lags = sorted({0, 1, R // 3, R // 2, R - 1, R})

    def make():
        oc = {d: xo.fast_xambg_oracle(ref, np.roll(srv, -d), 0, F, n, None, False)[:, 0, 0] for d in lags}
        tc = {d: xo.fast_xambg_truth(ref, np.roll(srv, -d), 0, F, n, None, False)[:, 0, 0] for d in lags}
        return oc, tc
    oc, tc = oracles.get("longfilt_c2", make)
    got = prb.fast_xambg(ref, srv, R, F, shortFilt=False)
    peak = float(np.abs(got).max())
    eo, et = _rel_columns(got, oc, lags, R, peak), _rel_columns(got, tc, lags, R, peak)
    record_parity(f"xambg/longfilt_n{n}/{both_paths}", E_vs_oracle_sampled_columns=eo, E_vs_truth_sampled_columns=et)
    assert eo <= TOL, eo


@pytest.mark.gpu
@pytest.mark.parametrize("n,F,R", [(2 ** 20, 256, 300), (2 ** 18, 1024, 100)])
def test_xambg_frames_batch_matches_oracle(n, F, R):
    """A 5-frame prc_xambg_frames_c64 batch on the FFT-domain CAF (one CTA per Doppler block and frame), sampled range
    columns of the first and last frame against the oracle.  At (2**20, 256, 300) the batch also takes
    doppler_fft_pow2_kernel<8>."""
    from oracle import xambg_oracle as xo
    nf = 5
    frames = [synth.make_frame(n, "P0", frame=190 + i) for i in range(nf)]
    ref = np.ascontiguousarray(np.stack([f[0] for f in frames]))
    srv = np.ascontiguousarray(np.stack([f[1] for f in frames]))
    w = np.ascontiguousarray(signal.get_window(KAISER, n), dtype=np.float64)
    lib = _lib.load()
    old = (_lib.get_option("fft"), _lib.get_option("fft_min_n"))
    try:
        _lib.set_option("fft", 1)
        _lib.set_option("fft_min_n", 8192)
        xb = np.empty((nf, F, R + 1), np.complex64)
        _lib.check(lib.prc_xambg_frames_c64(ref.ctypes.data, srv.ctypes.data, n, nf, n, R, F, w.ctypes.data, xb.ctypes.data,
                                            _lib.MEM_HOST, 0, None, 0))
    finally:
        _lib.set_option("fft", old[0])
        _lib.set_option("fft_min_n", old[1])
    lags = sorted({0, 1, R // 2, R - 1, R})
    worst = 0.0
    for i in (0, nf - 1):
        cols = {d: xo.fast_xambg_oracle(ref[i], np.roll(srv[i], -d), 0, F, n, w)[:, 0, 0] for d in lags}
        worst = max(worst, _rel_columns(xb[i][:, :, None], cols, lags, R, float(np.abs(xb[i]).max())))
    record_parity(f"xambg/frames_n{n}_F{F}_R{R}", E_vs_oracle_sampled_columns=worst)
    assert worst <= TOL, worst


# ------------------------------------------------------------------ CPU guard: every launch site is covered
# (host function, kernel<template arguments>) of every launch in build.SOURCES -> [(test id, variant, what it reaches)].
# The launches in the headers' own launchers are covered where those headers are tested: the front end's in
# tests/test_recording.py, CFAR_2D's and the frame chain's in tests/test_render.py.
# Variant: "default" (shipped configuration), or "fft" / "direct" (the both_paths fixture; "direct" also marks the
# direct_form fixture).
# A row is checked against the source, not the other way round: read the dispatch code before adding one.
PAR, FFT, KV = "tests/test_gpu_parity.py::", "tests/test_gpu_fft.py::", "tests/test_kernel_variants.py::"
FE, GAL, TRK = "tests/test_gpu_frontend.py::", "tests/test_gal_jpe.py::", "tests/test_tracking.py::"
RS = "tests/test_rows_sweep.py::"
PS = "tests/test_path_sweep.py::"
DS = "tests/test_direct_sweep.py::"
DIRECT_TEST = KV + "test_direct_form_matches_truth_and_reference"
NLMS_TEST = KV + "test_nlms_matches_truth_and_reference"
COVERAGE = {
    "launch_lagstream: lagstream_kernel<TILE_I, TILE_D>": [(PAR + "test_ls_matches_live_oracle", "direct", "LS, n <= 20000"),
                                                           (DIRECT_TEST, "direct", "ls_big, caf_big, frame: LS and CAF at config 2"),
        (DS + "test_caf_direct_form_at_the_planner_edges", "default", "CAF: G = 1 at H = 512, G = 32, blocks over >= 3 CTAs, CTAs over >= 3 blocks"), (DS + "test_ls_direct_form_at_the_planner_edges", "default", "LS lag sums, M = 1 .. 2048")],
    "fft_twiddles: fft::fft_twiddle_kernel<R3>": [
        (FFT + "test_frame_fused_equals_separate_operators_at_awkward_sizes", "fft", "R3 = 4 (n = 200000) and 8 (n = 10**6)"),
        (PAR + "test_ls_many_taps_uses_the_wide_solver", "fft", "R3 = 16")],
    "ls_fft_corr: fftc::lscorr_fft_kernel<R3>": [
        (PAR + "test_ls_matches_live_oracle", "fft", "R3 = 8 (M <= 1024)"),
        (PAR + "test_ls_many_taps_uses_the_wide_solver", "fft", "R3 = 16; ls_fft_plan never picks R3 = 4"),
        (PS + "test_ls_filter_at_the_planner_edges", "default", "M = 1 .. 2048 at n = 2L and a one-sample last segment"),
        (PS + "test_frames_batch_sizes_hold_every_row_to_its_truth", "default", "one CTA per frame (nf > slots / 2)")],
    "levinson_launch: levinson_kernel<1>": [(PAR + "test_ls_matches_live_oracle", "fft", "M <= 1024, batched solve"),
                                            (PS + "test_ls_filter_at_the_planner_edges", "default", "M = 1, 2, 1023, 1024"),
                                            (DIRECT_TEST, "direct", "single-CTA solve: ls_big, ls_small"),
                                            (PAR + "test_ls_matches_live_oracle", "direct", "single-CTA solve"),
        (DS + "test_ls_direct_form_at_the_planner_edges", "default", "single-CTA solve, M = 1 .. 1024")],
    "levinson_launch: levinson_kernel<4>": [(PAR + "test_ls_many_taps_uses_the_wide_solver", "fft", "M = 1110"),
                                            (PS + "test_ls_filter_at_the_planner_edges", "default", "M = 1025 .. 2048 against the truth"),
                                            (DIRECT_TEST, "direct", "single-CTA solve: ls_wide"),
                                            (PAR + "test_ls_many_taps_uses_the_wide_solver", "direct", "single-CTA solve"),
        (DS + "test_ls_direct_form_at_the_planner_edges", "default", "single-CTA solve, M = 1025, 2048")],
    "taps_spectrum: fftc::taps_spectrum_kernel<R3>": [
        (FFT + "test_frame_fused_equals_separate_operators_at_awkward_sizes", "fft", "R3 = 4 and 8 (CAF transform)"),
        (PAR + "test_ls_matches_live_oracle", "fft", "R3 = 8 (FIR transform)"),
        (PAR + "test_ls_many_taps_uses_the_wide_solver", "fft", "R3 = 16")],
    "fir_fft: fftc::fir_fft_kernel<R3>": [
        (PAR + "test_ls_matches_live_oracle", "fft", "R3 = 8"),
        (PAR + "test_ls_many_taps_uses_the_wide_solver", "fft", "R3 = 16; the LS transform is never R3 = 4"),
        (PS + "test_toeplitz_and_multiple_at_the_planner_edges", "default", "linear mode, M = 1 .. 2048")],
    "caf_fft: fftc::caf_fft_kernel<R3, true>": [
        (FFT + "test_frame_fused_equals_separate_operators_at_awkward_sizes", "fft", "R3 = 4 and 8"),
        (FFT + "test_long_range_and_long_filter_take_the_larger_transforms", "fft", "R3 = 16"),
        (PS + "test_fused_frame_at_the_planner_edges", "default",
         "R3 = 16 against the frame truth (R + M - 1 = 3072); filterLen = 0: the staging without reuse; peek = 0")],
    "caf_fft: fftc::caf_fft_kernel<R3, false>": [
        (PS + "test_xambg_at_the_planner_edges", "fft", "R = 3L/4 at L = 1024, 2048, 4096; D = 32; F = 1; f32 window"),
        (PAR + "test_xambg_matches_live_oracle", "fft", "R3 = 4"),
        (FFT + "test_xambg_large_shapes_sampled_columns", "fft", "R3 = 8 (F = 64, D >= 16384)"),
        (FFT + "test_long_range_and_long_filter_take_the_larger_transforms", "fft", "R3 = 16 (R = 1200)"),
        (KV + "test_xambg_frames_batch_matches_oracle", "default", "5-frame batches, one CTA per Doppler block and frame")],
    "xambg_device: weight_kernel": [(DIRECT_TEST, "direct", "caf_big, frame"),
                                    (PAR + "test_xambg_matches_live_oracle", "direct", "lagstream CAF with a window"),
        (DS + "test_caf_direct_form_at_the_planner_edges", "default", "windowed lagstream cases")],
    "xambg_device: lagcorr_kernel<TILE_I, TILE_D>": [
        (DIRECT_TEST, "direct", "caf_small: blocks of < 64 taps and the tap-weighted decimator"),
        (KV + "test_tap_weighted_decimator_at_full_size", "direct", "40 961 taps"),
        (DS + "test_caf_direct_form_at_the_planner_edges", "default", "D = 1, ntaps 32 / 63, tap-weighted at G = 32, H = 512 and the nchunk loop")],
    "doppler_stage: twiddle_kernel": [(PAR + "test_xambg_matches_live_oracle", "fft", "every fast_xambg")],
    "doppler_stage: doppler_fft_pow2_kernel<8>": [
        (KV + "test_xambg_frames_batch_matches_oracle", "default", "5 frames x 38 column groups >= SM count"),
        (FFT + "test_long_range_and_long_filter_take_the_larger_transforms", "direct", "R = 1200, F = 64"),
        (DS + "test_caf_direct_form_at_the_planner_edges", "default", "R = 1100, 3073, 5119")],
    "doppler_stage: doppler_fft_pow2_kernel<2>": [(PAR + "test_xambg_matches_live_oracle", "direct", "F <= 4096"),
                                                 (KV + "test_doppler_stage_at_large_F", "fft", "F = 4096"),
        (DS + "test_caf_direct_form_at_the_planner_edges", "direct", "F = 2 .. 4096")],
    "doppler_stage: doppler_fft_pow2_kernel<1>": [(KV + "test_doppler_stage_at_large_F", "fft", "F = 8192"),
        (DS + "test_caf_direct_form_at_the_planner_edges", "direct", "F = 8192")],
    "doppler_stage: chunk_sum_kernel": [(PAR + "test_xambg_matches_reference_golden", "direct", "xambg_nonpow2_F"),
                                       (KV + "test_doppler_stage_at_large_F", "fft", "F = 16384"),
        (DS + "test_caf_direct_form_at_the_planner_edges", "direct", "F = 1, 100, 200, 1500, 16384")],
    "doppler_stage: doppler_dft_kernel": [(PAR + "test_xambg_matches_reference_golden", "direct", "xambg_nonpow2_F"),
                                         (KV + "test_doppler_stage_at_large_F", "fft", "F = 16384"),
        (DS + "test_caf_direct_form_at_the_planner_edges", "direct", "F = 1, 100, 200, 1500, 16384")],
    "ls_device: fir_apply_kernel<TILE_I, TILE_D>": [(DIRECT_TEST, "direct", "ls_small, ls_wide, toep"),
                                                    (DIRECT_TEST, "direct", "ls_big, frame at config 2"),
        (DS + "test_ls_direct_form_at_the_planner_edges", "default", "Mpad = 10 .. 2050, circular and linear")],
    "ls_toeplitz_device: shift_roll_kernel": [(DIRECT_TEST, "direct", "toep"),
                                              (PAR + "test_ls_multiple_matches_reference_golden", "direct", "shifted bins"),
        (DS + "test_toeplitz_direct_form_with_peek_past_half_the_frame", "default", "peek >= n / 2")],
    "direct_xambg_device: piece_sum_kernel": [
        (FE + "test_direct_xambg_matches_reference_golden", "default", ""),
        (RS + "test_direct_xambg_shapes", "default", "R >= n, F = 1, odd F, n = 2^18"),
        (RS + "test_direct_xambg_lag_limit", "default", "R + 1 = the lag limit")],
    "nlms_device: nlms_block_kernel<1, 512>": [(FFT + "test_nlms_large_batch_uses_the_half_size_ctas_and_matches", "default", "M = 410"),
        (DS + "test_nlms_frames_past_the_sm_count_at_the_kt_edges", "default", "M = 512")],
    "nlms_device: nlms_block_kernel<2, 512>": [(KV + "test_nlms_frames_past_the_sm_count_with_many_taps", "default", "M = 1000"),
        (DS + "test_nlms_frames_past_the_sm_count_at_the_kt_edges", "default", "M = 513")],
    "nlms_device: nlms_block_kernel<4, 512>": [(KV + "test_nlms_frames_past_the_sm_count_with_many_taps", "default", "M = 2000"),
        (DS + "test_nlms_frames_past_the_sm_count_at_the_kt_edges", "default", "M = 1025, 2048")],
    "nlms_device: nlms_block_kernel<1>": [(PAR + "test_nlms_matches_reference_golden", "default", ""),
                                          (NLMS_TEST, "default", "M = 410"),
        (DS + "test_nlms_at_the_tiling_edges", "default", "M = 1 .. 1024, every last-tile length")],
    "nlms_device: nlms_block_kernel<2>": [(KV + "test_nlms_with_more_than_1024_taps_matches_c_oracle", "default", "M = 1110"),
        (DS + "test_nlms_at_the_tiling_edges", "default", "M = 1025, 2048")],
    "nlms_device: nlms_block_kernel<4>": [(KV + "test_nlms_with_more_than_1024_taps_matches_c_oracle", "default", "M = 3010"),
                                          (KV + "test_nlms_accepts_4096_taps_and_names_the_limit_above", "default", "M = 4096"),
        (DS + "test_nlms_at_the_tiling_edges", "default", "M = 2049, 4096 with initial taps"),
        (DS + "test_nlms_frames_past_the_sm_count_at_the_kt_edges", "default", "M = 2049: more frames than SMs, 1024-thread CTAs")],
    "gal_device: gal_jpe_kernel<1, false>": [(GAL + "test_gal_edge_cases", "default", "D = 1")],
    "gal_device: gal_jpe_kernel<2, false>": [(GAL + "test_gal_edge_cases", "default", "D = 40")],
    "gal_device: gal_jpe_kernel<4, false>": [(GAL + "test_gal_shapes_match_c_oracle", "default", "D = 77")],
    "gal_device: gal_jpe_kernel<8, false>": [(GAL + "test_gal_long_run_matches_c_oracle_and_truth", "default", "D = 185")],
    "gal_device: gal_jpe_kernel<GAL_CTA_T, true>": [(GAL + "test_gal_shapes_match_c_oracle", "default", "D = 300, 4096")],
    "stage_window: f64_to_f32_kernel": [(PAR + "test_xambg_matches_live_oracle", "fft", "float64 window")],
    "prc_xambg_c64: f64_to_f32_kernel": [(PAR + "test_xambg_matches_reference_golden", "direct", "xambg_longfilt taps")],
    "trk_meas_launch: track_meas_kernel<T, TRK_MODE_MEAN>": [
        (TRK + "test_float32_equals_float64_and_frame_layouts_agree", "default", "T = float, double (simple tracker)")],
    "trk_meas_launch: track_meas_kernel<T, TRK_MODE_SLOTS>": [
        (TRK + "test_float32_equals_float64_and_frame_layouts_agree", "default", "T = float, double (multi-target tracker)")],
    "trk_meas_launch: track_meas_kernel<T, TRK_MODE_MEAS>": [
        (TRK + "test_float32_equals_float64_and_frame_layouts_agree", "default", "T = float, double (get_measurements)")],
    "prc_multitarget_track_frames: track_multi_kernel": [(TRK + "test_multitarget_tracker_matches_golden", "default", "")],
    "prc_simple_track_frames: track_simple_kernel<double>": [(TRK + "test_simple_target_tracker_matches_golden", "default", "")],
    "prc_simple_track_frames: track_simple_kernel<float>": [(TRK + "test_float32_equals_float64_and_frame_layouts_agree", "default", "")],
}

_FUNC_DEF = re.compile(r"^(?!(?:return|typedef|using|namespace|struct|enum|extern|template|#))[A-Za-z_][\w:<>*&\s]*?\b([A-Za-z_]\w*)\s*\(")
_LAUNCH = re.compile(r"([A-Za-z_][\w:]*)\s*(<[^<>;()]*>)?\s*<<<")


def launch_sites(paths=build.SOURCES):
    """{'host function: kernel<template arguments>': [(file, line number)]} of every kernel launch in the files,
    including the ones inside macros (PRC_R3_SWITCH, PRC_TRK_MEAS)."""
    sites = {}
    for path in paths:
        func = None
        with open(path) as f:
            for no, line in enumerate(f, 1):
                m = _FUNC_DEF.match(line)
                if m:
                    func = m.group(1)
                code = line.split("//", 1)[0]
                for k in _LAUNCH.finditer(code):
                    targs = ""
                    if k.group(2):
                        targs = "<" + ", ".join(a.strip() for a in k.group(2)[1:-1].split(",")) + ">"
                    sites.setdefault(f"{func}: {k.group(1)}{targs}", []).append((os.path.basename(path), no))
    return sites


def _is_gpu_test(test_id):
    path, name = test_id.split("::")
    with open(os.path.join(ROOT, path)) as f:
        src = f.read()
    m = re.search(rf"^def {re.escape(name)}\(", src, re.M)
    assert m, f"{test_id} does not exist"
    decorators = src[:m.start()].rstrip("\n").rsplit("\n\n", 1)[-1]       # the block right above the def
    return re.search(r"^pytestmark = pytest\.mark\.gpu$", src, re.M) is not None or "@pytest.mark.gpu" in decorators


def test_every_launch_site_of_the_library_sources_has_a_covering_gpu_test():
    sites = launch_sites()
    assert len(sites) == 39
    missing = sorted(set(sites) - set(COVERAGE))
    stale = sorted(set(COVERAGE) - set(sites))
    assert not missing, "launch sites without a covering test in COVERAGE: " + \
        "; ".join(f"{s} ({sites[s][0][0]}, line {sites[s][0][1]})" for s in missing)
    assert not stale, f"COVERAGE rows that are no launch site of the library's sources: {stale}"
    for site, reached in COVERAGE.items():
        assert reached, f"{site}: no test"
        for test_id, variant, _ in reached:
            assert _is_gpu_test(test_id), f"{site}: {test_id} is not a GPU test"
            assert variant in ("default", "fft", "direct"), f"{site}: unknown variant {variant}"


def test_coverage_guard_sees_a_new_launch(tmp_path):
    """The guard fails for a launch it has not been told about."""
    paths = []
    for path in build.SOURCES:
        scratch = tmp_path / os.path.basename(path)
        scratch.write_text(open(path).read())
        paths.append(str(scratch))
    with open(paths[-1], "a") as f:
        f.write("\nint new_entry(Ctx* c) {\n    new_kernel<3><<<1, 32, 0, c->stream>>>();\n    return 0;\n}\n")
    extra = set(launch_sites(paths)) - set(COVERAGE)
    assert extra == {"new_entry: new_kernel<3>"}
