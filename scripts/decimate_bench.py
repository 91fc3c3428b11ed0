#!/usr/bin/env python
"""Time decimate, channel_preprocessing and normalize on the GPU; print one JSON line.

    python scripts/decimate_bench.py [--reps 20] [--no-host-reference]

Shapes: channel_preprocessing of 2^24 raw int8 I/Q pairs at dec = 12 and 96; decimate of 2^24 complex64 samples at
q = 2, 12, 96 and 1000; decimate (q = 12) and normalize of a (2^22, 8) float32 array.  Each is timed with its data
resident on the device (CUDA events around `reps` calls) and from host arrays (wall clock, copies included).  Beside
them: per-kernel times from the library's profiler, the algorithmic bytes (inputs read once, outputs written once) and
flops (4 (20q+1) per complex output, 2 (20q+1) per real output: the taps are real), the share of the larger of the two
bounds (3.35 TB/s HBM3, 67 TFLOP/s FP32: the H100 SXM data sheet), and scipy.signal.decimate plus the reference's
functions (oracle/_ref, when build() installed them) on the host.  Fails without a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import passiveradar_b200 as prb                                         # noqa: E402
from passiveradar_b200 import _lib, synth                               # noqa: E402

HBM, FP32 = 3.35e12, 67e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def reference():
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "passiveRadar")):
        return None
    sys.path.insert(0, ref)
    from passiveRadar import signal_utils
    return signal_utils


def dev_time(torch, fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def host_time(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps


def kernels(torch, fn, reps):
    _lib.profile(True)
    _lib.profile_reset()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    prof = _lib.profile_read()
    _lib.profile(False)
    return {k: round(v[0] / reps * 1e3, 2) for k, v in prof.items() if v[1] and k in ("decimate", "norm_sum", "norm_scale")}


def bounds(in_bytes, out_bytes, flops, sec):
    tb, tf = (in_bytes + out_bytes) / HBM, flops / FP32
    return {"bytes": int(in_bytes + out_bytes), "flops": int(flops), "bound": "hbm" if tb >= tf else "fp32",
            "share_of_bound": round(max(tb, tf) / sec, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-host-reference", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available() or _lib.device_count() < 1:
        raise SystemExit("decimate_bench needs a CUDA device (there is no CPU fallback)")
    import scipy.signal as signal
    dev = torch.device("cuda", _lib.current_device())
    ref = None if args.no_host_reference else reference()
    res = {"card": card(), "reps": args.reps, "cases": []}
    n = 1 << 24

    def case(name, fn_dev, fn_host, in_b, out_b, flops, host_ref=None):
        r = {"case": name}
        sec = dev_time(torch, fn_dev, args.reps)
        r["device_us"] = round(sec * 1e6, 1)
        r.update(bounds(in_b, out_b, flops, sec))
        r["kernels_us"] = kernels(torch, fn_dev, args.reps)
        r["host_arrays_ms"] = round(host_time(fn_host, max(3, args.reps // 4)) * 1e3, 2)
        if host_ref is not None:
            r["host_reference"] = {k: round(host_time(f, 1), 3) for k, f in host_ref.items()}
        res["cases"].append(r)
        print(json.dumps(r), file=sys.stderr)

    raw = synth.raw_iq(n, "int8", seed=1)
    raw_t = torch.from_numpy(raw).to(dev)
    for d in (12, 96):
        nout = -(-n // d)
        hr = None
        if not args.no_host_reference:
            hr = {"scipy_s": lambda d=d: signal.decimate(
                (raw[0:-1:2] + 1j * raw[1::2]).astype(np.complex64) * np.exp(
                    1j * 2 * np.pi * 1e4 * np.arange(n, dtype=np.complex64) / 2.4e6), d, 20 * d, ftype="fir", axis=0)}
            if ref is not None:
                hr["reference_s"] = lambda d=d: ref.channel_preprocessing(raw, d, 1e4, 2.4e6)
        case(f"channel_preprocessing_int8_dec{d}", lambda d=d: prb.channel_preprocessing(raw_t, d, 1e4, 2.4e6),
             lambda d=d: prb.channel_preprocessing(raw, d, 1e4, 2.4e6), 2 * n, 8 * nout, 4 * (20 * d + 1) * nout, hr)
    x = synth.raw_iq(n, "float32", seed=2).view(np.complex64)
    x_t = torch.from_numpy(x).to(dev)
    for q in (2, 12, 96, 1000):
        nout = -(-n // q)
        hr = None
        if not args.no_host_reference:
            hr = {"scipy_s": lambda q=q: signal.decimate(x, q, 20 * q, ftype="fir", axis=0)}
            if ref is not None:
                hr["reference_s"] = lambda q=q: ref.decimate(x, q)
        case(f"decimate_c64_q{q}", lambda q=q: prb.decimate(x_t, q), lambda q=q: prb.decimate(x, q), 8 * n, 8 * nout,
             4 * (20 * q + 1) * nout, hr)
    m = 1 << 22
    f = synth.raw_iq(4 * m, "float32", seed=3).reshape(m, 8)
    f_t = torch.from_numpy(f).to(dev)
    nout = -(-m // 12)
    hr = None if args.no_host_reference else {"scipy_s": lambda: signal.decimate(f, 12, 240, ftype="fir", axis=0)}
    if hr is not None and ref is not None:
        hr["reference_s"] = lambda: ref.decimate(f, 12)
    case("decimate_f32_4Mx8_q12", lambda: prb.decimate(f_t, 12), lambda: prb.decimate(f, 12), 4 * 8 * m, 4 * 8 * nout,
         2 * 241 * nout * 8, hr)
    hr = None if args.no_host_reference else {"numpy_s": lambda: f / np.mean(np.abs(f).flatten())}
    if hr is not None and ref is not None:
        hr["reference_s"] = lambda: ref.normalize(f)
    case("normalize_f32_4Mx8", lambda: prb.normalize(f_t), lambda: prb.normalize(f), 2 * 4 * 8 * m, 4 * 8 * m,
         3 * 8 * m, hr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
