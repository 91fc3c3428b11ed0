#!/usr/bin/env python
"""Time the channel-offset estimator (find_channel_offset) at main.py's shapes and print one JSON line.

    python scripts/offset_bench.py [--reps 5] [--no-reference]

Shapes: main.py:78-83 (10 CPIs of raw int8 per channel at the shipped PRconfig.yaml, 5 242 880 samples), :49-54
(the interleaved-file path: 2 621 440 complex64 samples per channel) and 10 CPIs of a 2^20-sample CPI (10 485 760
int8), all with main.py's nl = 5 000 000 and nd = 1.  For each: the host-array call (numpy in, offset out), the
device-resident call (inputs already in HBM, prc_channel_offset on device pointers), the per-kernel times of one
device-resident call from the library's event profiler, the bytes each kernel must move at least and the rate that
gives, and the reference's find_channel_offset on the host (from oracle/_ref when build() installed it).  The card's
name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import passiveradar_b200 as prb                                    # noqa: E402
from passiveradar_b200 import _lib, synth                          # noqa: E402
from passiveradar_b200 import signal_utils as psu                  # noqa: E402

NL = 5000000
SHAPES = [("main_int8", "int8", 5242880), ("main_interleaved_c64", "complex64", 2621440),
          ("cpi2e20_int8", "int8", 10485760)]


def plan(n, nl):
    """Transform length and pass count of the device path (csrc/prcore.cu chanoff_device, nd = 1)."""
    nvalid = 2 * nl + 1
    p0 = -nl
    need = max(n, n, p0 + nvalid - 1 + n, n - p0, 2)
    m = max(1, int(np.ceil(np.log2(need))))
    npass, top = 0, m
    while top > 0:
        top -= top if top <= 11 else 8
        npass += 1
    return m, npass, nvalid


def algorithmic_bytes(n, itemsize, cplx, nl):
    m, npass, nvalid = plan(n, nl)
    L = 1 << m
    w = 16 if cplx else 8
    iir = 2 * (n * itemsize + (n + 54) * w          # forward: raw in, full-rate out
               + (n + 54) * w + n * 16)              # backward: full-rate in, complex128 into the transform buffer
    fft = npass * 2 * 2 * L * 16 + npass * 2 * L * 16 + L * 16    # forward X and Y, inverse, Y read by the product
    arg = nvalid * 16                                              # the valid lags read once
    return {"chanoff_iir": iir, "chanoff_fft": fft, "chanoff_argmax": arg}, L


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:                  # the numbers still stand; say the card was not read
        return {"name": f"not read ({exc})"}


def reference_finder():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    try:
        from passiveRadar.signal_utils import find_channel_offset
        return find_channel_offset
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    import torch
    assert _lib.device_count() >= 1, "offset_bench.py needs a CUDA device"
    ref_fn = None if args.no_reference else reference_finder()
    lib = _lib.load()
    out = {"bench": "find_channel_offset", "card": card(), "nd": 1, "nl": NL, "shapes": {}}
    for name, kind, n in SHAPES:
        s1, s2 = synth.offset_pair(n, n, kind, 1234, 40)
        a1, d1, single = psu._offset_input(s1)
        a2, d2, _ = psu._offset_input(s2)
        row = {"samples": n, "dtype": kind}
        # host arrays in, offset out
        got = prb.find_channel_offset(s1, s2, 1, NL)
        ts = []
        for _ in range(args.reps):
            t = time.perf_counter()
            prb.find_channel_offset(s1, s2, 1, NL)
            ts.append(time.perf_counter() - t)
        row["offset"] = int(got)
        row["host_call_ms"] = {"median": 1e3 * statistics.median(ts), "min": 1e3 * min(ts), "max": 1e3 * max(ts)}
        # device-resident inputs, device offset
        s, z = psu._decimate_sos(1, single)
        sos = np.ascontiguousarray(np.stack([s, s]))
        zi = np.ascontiguousarray(np.stack([z, z]))
        t1 = torch.from_numpy(a1.view(np.uint8)).cuda()
        t2 = torch.from_numpy(a2.view(np.uint8)).cuda()
        off = torch.zeros(1, dtype=torch.int64, device="cuda")

        def dev_call():
            _lib.check(lib.prc_channel_offset(t1.data_ptr(), d1, n, t2.data_ptr(), d2, n, 1, NL, sos.ctypes.data,
                                              zi.ctypes.data, off.data_ptr(), None, _lib.MEM_DEVICE, 0, None, 0))
        dev_call()
        assert int(off.item()) == int(got)
        ts = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            dev_call()
            ts.append(time.perf_counter() - t)
        row["device_call_ms"] = {"median": 1e3 * statistics.median(ts), "min": 1e3 * min(ts), "max": 1e3 * max(ts)}
        _lib.profile_reset()
        _lib.profile(True)
        dev_call()
        prof = _lib.profile_read()
        _lib.profile(False)
        nbytes, L = algorithmic_bytes(n, a1.dtype.itemsize, np.iscomplexobj(a1), NL)
        row["transform_points"] = L
        row["kernels"] = {}
        for k, b in nbytes.items():
            ms, cnt = prof.get(k, (0.0, 0))
            row["kernels"][k] = {"ms": ms, "launches": cnt, "bytes": b, "GB_per_s": (b / (ms * 1e-3) / 1e9) if ms else None}
        ms, cnt = prof.get("chanoff_load", (0.0, 0))
        if cnt:
            row["kernels"]["chanoff_load"] = {"ms": ms, "launches": cnt}
        if ref_fn is not None:
            t = time.perf_counter()
            r = ref_fn(s1, s2, 1, NL)
            row["reference_host_s"] = time.perf_counter() - t
            row["reference_offset"] = int(r)
        else:
            row["reference_host_s"] = "not measured (no oracle/_ref)"
        out["shapes"][name] = row
        del t1, t2
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
