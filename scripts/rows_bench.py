#!/usr/bin/env python
"""Device-resident timings of the rows either side of the hot path (SURVEY.md 8f), CUDA events on the
launching stream, inputs already in HBM.  Prints one JSON object.

    python scripts/rows_bench.py [--reps 20]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from passiveradar_b200 import _lib, synth                      # noqa: E402
from passiveradar_b200.signal_utils import _resample_taps      # noqa: E402


STREAM = None


def timeit(fn, reps):
    """fn enqueues on STREAM (a non-default stream handed to the library: a NULL stream would make the
    library use its private one and the events would bracket nothing)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(STREAM)
    for _ in range(reps):
        fn()
    e1.record(STREAM)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3      # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    global STREAM
    STREAM = torch.cuda.Stream(dev)
    st = STREAM.cuda_stream
    hbm = 6571.6
    try:
        hbm = float(json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    res = {"hbm_peak_GBps": hbm}

    # ---- front end: one main.py chunk, IQ -> mix -> 13/119 resample, and the mix alone; int8 is what main.py reads,
    # int16 and float32 load I and Q as wider scalars
    n = 9_600_000
    h = _resample_taps(13, 119, False)
    n_out = (n * 13 + 118) // 119
    out = torch.empty(n_out, dtype=torch.complex64, device=dev)
    x64 = torch.empty(n, dtype=torch.complex64, device=dev)
    for name, kind, ib in (("int8", _lib.IQ_I8, 2), ("int16", _lib.IQ_I16, 4), ("float32", _lib.IQ_C64, 8)):
        iq = torch.from_numpy(synth.raw_iq(n, name, 1)).to(dev)

        def fe():
            _lib.check(lib.prc_frontend_c64(iq.data_ptr(), kind, n, _lib.MIX_C128, 300e3, 2.4e6, 0.7, 13, 119,
                                            h.ctypes.data, h.shape[0], out.data_ptr(), n_out, _lib.MEM_DEVICE, 0, st,
                                            _lib.FLAG_ASYNC))
        us = timeit(fe, args.reps)
        alg = ib * n + 8 * n_out
        res[f"frontend_{name}_9.6M"] = {"us": round(us, 1), "alg_bytes": alg, "alg_GBps": round(alg / us / 1e3, 1),
                                        "frac_hbm": round(alg / us / 1e3 / hbm, 4),
                                        "Msamples_in_per_s": round(n / us, 1)}

        def mix():
            _lib.check(lib.prc_iq_mix_c64(iq.data_ptr(), kind, n, _lib.MIX_C128, 300e3, 2.4e6, 0.7, x64.data_ptr(),
                                          _lib.MEM_DEVICE, 0, st, _lib.FLAG_ASYNC))
        us = timeit(mix, args.reps)
        alg = ib * n + 8 * n
        res[f"iq_mix_{name}_9.6M"] = {"us": round(us, 1), "alg_bytes": alg, "alg_GBps": round(alg / us / 1e3, 1),
                                      "frac_hbm": round(alg / us / 1e3 / hbm, 4)}
        del iq

    # ---- CFAR on a config-2 map
    rows, cols = 256, 301
    amb = torch.randn(rows, cols, dtype=torch.complex64, device=dev)
    cr = torch.empty(rows, cols, dtype=torch.float32, device=dev)

    def cfar():
        _lib.check(lib.prc_cfar2d_f32(amb.data_ptr(), rows, cols, 18, 4, None, cr.data_ptr(), None, _lib.MEM_DEVICE, 0, st,
                                      _lib.FLAG_ASYNC | _lib.FLAG_ABS_C64))
    us = timeit(cfar, args.reps)
    alg = rows * cols * (8 + 4)
    res["cfar_256x301"] = {"us": round(us, 1), "alg_bytes": alg, "alg_GBps": round(alg / us / 1e3, 2)}

    # ---- direct_xambg at config 2 (256 Doppler bins x 301 lags x 2^20 samples, time domain)
    nn, R, F = 2 ** 20, 300, 256
    r, s = synth.make_frame(nn, "P1", 0)
    rd, sd = torch.from_numpy(r).to(dev), torch.from_numpy(s).to(dev)
    od = torch.empty(F, R + 1, dtype=torch.complex64, device=dev)

    def direct():
        _lib.check(lib.prc_direct_xambg_c64(rd.data_ptr(), sd.data_ptr(), nn, R, F, float(nn), od.data_ptr(), _lib.MEM_DEVICE, 0, st,
                                            _lib.FLAG_ASYNC))
    us = timeit(direct, max(2, args.reps // 10))
    flops = 8.0 * nn * (R + 1) * F
    res["direct_xambg_c2"] = {"us": round(us, 1), "alg_flops": flops, "alg_TFLOPs": round(flops / us / 1e6, 2),
                              "fp32_pipe_peak_TFLOPs": 74.4}

    # ---- LS_Filter_Multiple, 5 Doppler bins (what main.py runs), config-2 block
    bins = np.array([0.0, 1.0, -1.0, 2.0, -2.0])
    cl = torch.empty(nn, dtype=torch.complex64, device=dev)

    def multi():
        _lib.check(lib.prc_ls_multiple_c64(rd.data_ptr(), sd.data_ptr(), nn, 300, 10, 2.4e6 * 13 / 119, bins.ctypes.data, 5,
                                           cl.data_ptr(), None, _lib.MEM_DEVICE, 0, st, _lib.FLAG_ASYNC))
    us = timeit(multi, max(2, args.reps // 4))
    res["ls_multiple_5bins_c2"] = {"us": round(us, 1)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
