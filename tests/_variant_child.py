"""Child process of tests/test_kernel_variants.py: runs the GPU cases under the PRC_* switches of its environment and
saves every output to an .npz.  The parent computes the oracles and float64 truths and makes every comparison.

    python tests/_variant_child.py OUT.npz CASE [CASE ...]
    python tests/_variant_child.py --switches          # print the switches in force as JSON (no GPU needed)

libprcore latches its environment switches once per process (prcore.cu, read_env), so each variant needs a process of
its own.  The child sets no switch itself.  Before it runs any case it checks that the library reports the switches its
environment asks for (prc_get_option): a misspelt variable would otherwise test the default configuration twice.

The case inputs are defined here and nowhere else; the parent imports this module to rebuild the same inputs.
"""
import json
import os
import sys

import numpy as np
import scipy.signal as signal

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (HERE, os.path.dirname(HERE)):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import _golden as G                      # noqa: E402
from passiveradar_b200 import synth     # noqa: E402

# prc_get_option name -> (environment variable, value when the variable is unset: prcore.cu's defaults)
SWITCHES = {"tune_nchunk": ("PRC_TUNE_NCHUNK", -1), "tune_g": ("PRC_TUNE_G", -1)}


def expected_switches(env):
    """What the library must report for environment `env`."""
    return {k: int(env[var]) if var in env else default for k, (var, default) in SWITCHES.items()}


def library_switches():
    from passiveradar_b200 import _lib
    return {k: _lib.get_option(k) for k in SWITCHES}


# ------------------------------------------------------------------ case inputs
# Output keys are "<case>.<item>.<profile>.<field>"; the profile tells the parent whether a cross-variant comparison
# applies (P0: independent channels) or only the comparison with the truth (P1: strong clutter).
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


# ------------------------------------------------------------------ what the child runs
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
    from passiveradar_b200 import _lib
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
    "nlms": run_nlms,
}


def main(argv):
    if argv[1:] == ["--switches"]:
        print(json.dumps(library_switches()))
        return 0
    out_path, cases = argv[1], argv[2:]
    unknown = [c for c in cases if c not in RUNNERS]
    if unknown:
        raise SystemExit(f"unknown cases {unknown}")
    got, want = library_switches(), expected_switches(os.environ)
    if got != want:
        raise SystemExit(f"the library reports switches {got}, the environment asks for {want}")
    from passiveradar_b200 import _lib
    _lib.set_option("fft", 0)            # every case but NLMS is a direct-form (FP32) case
    res = {}
    for case in cases:
        RUNNERS[case](res)
    res["switches"] = np.array([got[k] for k in SWITCHES], dtype=np.int64)
    res["cases"] = np.array(cases)
    np.savez(out_path, **res)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
