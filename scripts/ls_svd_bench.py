#!/usr/bin/env python
"""LS_Filter_SVD throughput on the GPU against the reference's own LS_Filter_SVD on the host.  Prints one JSON line.

    python scripts/ls_svd_bench.py [--workloads 1048576x310,524288x185,2097152x410,1048576x1024] [--reps 3]

Per (n, M) workload (M = filterLen + peek, peek = 10): a device-resident batch of frames goes through
prc_ls_svd_frames_c64 in one call on a caller stream, timed with CUDA events: frames/s and the per-stage time from the
library's profile table (svd_corr: lag sums, svd_eig: eigendecomposition and pseudo-inverse, svd_fir: residual), taken
in a separate profiled pass.  LS_Filter (Tikhonov-regularised solve, reg = 1) on the same frame is timed for scale.
Frames 0 and -1 of the timed batch are checked bit for bit against single-frame LS_Filter_SVD calls.  The reference
column times the reference's LS_Filter_SVD (oracle/_ref, placed there by build()) on a short slice of the frame on the
host and scales it linearly in n to the whole frame, which is labelled as extrapolated.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import passiveradar_b200 as prb                                 # noqa: E402
from passiveradar_b200 import _lib, synth                      # noqa: E402

PEEK = 10


def card():
    """Name and power limit of GPU 0, read now (nvidia-smi query only)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": q[0].strip(), "power_limit": q[1].strip()}
    except Exception as exc:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({exc.__class__.__name__})"}


def reference_seconds(n_slice, M):
    """The reference's LS_Filter_SVD on an n_slice-sample frame, one call on the host: seconds, or None."""
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref_dir, "passiveRadar")):
        return None
    sys.path.insert(0, ref_dir)
    try:
        from passiveRadar.clutter_removal import LS_Filter_SVD as ref_svd
    finally:
        sys.path.remove(ref_dir)
    ref, srv = synth.make_frame(n_slice, "P1", frame=0)
    t0 = time.perf_counter()
    ref_svd(ref, srv, M - PEEK, PEEK)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="1048576x310,524288x185,2097152x410,1048576x1024",
                    help="n x M, comma-separated")
    ap.add_argument("--frames", type=int, default=0, help="frames per batch (0: one per SM, capped by --mem-gb)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--mem-gb", type=float, default=16.0, help="device memory for the batch's inputs and outputs")
    ap.add_argument("--ref-samples", type=int, default=16384, help="samples of the reference's frame timed on the host")
    args = ap.parse_args()

    lib = _lib.load()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    stream = torch.cuda.Stream(dev)
    res = {"what": "LS_Filter_SVD (clutter_removal.py:58-107), device-resident batch, one call per batch",
           "peek": PEEK, **card(), "sms": nsm, "workloads": []}
    for wl in args.workloads.split(","):
        n, M = (int(v) for v in wl.lower().split("x"))
        fl = M - PEEK
        base = [synth.make_frame(n, "P1", frame=200 + i) for i in range(2)]
        cap = int(args.mem_gb * 1e9 // (3 * 8 * n))
        nframes = max(1, min(args.frames or nsm, cap))
        with torch.cuda.stream(stream):
            dref = torch.empty((nframes, 2 * n), dtype=torch.float32, device=dev)
            dsrv = torch.empty_like(dref)
            for i in range(nframes):
                dref[i].copy_(torch.from_numpy(base[i % 2][0].view(np.float32)))
                dsrv[i].copy_(torch.from_numpy(base[i % 2][1].view(np.float32)))
            dout = torch.empty_like(dref)
            dtaps = torch.empty((nframes, 2 * M), dtype=torch.float32, device=dev)
            drank = torch.empty(nframes, dtype=torch.int32, device=dev)
        stream.synchronize()

        def launch():
            _lib.check(lib.prc_ls_svd_frames_c64(dref.data_ptr(), dsrv.data_ptr(), n, nframes, n, fl, PEEK,
                                                 dout.data_ptr(), dtaps.data_ptr(), drank.data_ptr(), _lib.MEM_DEVICE,
                                                 0, C.c_void_p(stream.cuda_stream), _lib.FLAG_ASYNC))

        launch()                                      # warm-up
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.reps):
            launch()
        e1.record(stream)
        stream.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        _lib.profile_reset()                          # per-stage times: a separate, profiled pass
        _lib.profile(True)
        launch()
        prof = _lib.profile_read()
        _lib.profile(False)
        stages = {k: round(prof[k][0], 3) for k in ("svd_corr", "svd_eig", "svd_fir")}
        checked = True
        for i in (0, nframes - 1):
            o1, t1 = prb.LS_Filter_SVD(base[i % 2][0], base[i % 2][1], fl, PEEK, True)
            checked &= bool(np.array_equal(dout[i].cpu().numpy().view(np.complex64), o1)
                            and np.array_equal(dtaps[i].cpu().numpy().view(np.complex64), t1))
        ranks = drank.cpu().numpy()
        # LS_Filter on one frame of the same shape, for scale (host arrays in and out, as a user calls it)
        prb.LS_Filter(base[0][0], base[0][1], fl, 1.0, PEEK)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.reps):
            prb.LS_Filter(base[0][0], base[0][1], fl, 1.0, PEEK)
        ls_ms = (time.perf_counter() - t0) / args.reps * 1e3
        t0 = time.perf_counter()
        prb.LS_Filter_SVD(base[0][0], base[0][1], fl, PEEK)
        svd1_ms = (time.perf_counter() - t0) * 1e3
        row = {"n": n, "M": M, "frames": nframes, "batch_ms": round(ms, 2),
               "frames_per_s": round(nframes / (ms * 1e-3), 2), "stage_ms_per_batch": stages,
               "ranks": sorted(set(int(r) for r in ranks)),
               "single_frame_host_call_ms": round(svd1_ms, 2),
               "ls_filter_single_frame_host_call_ms": round(ls_ms, 2),
               "batch_matches_single_frame_calls": checked}
        s_ref = reference_seconds(args.ref_samples, M)
        if s_ref is not None:
            row["reference_cpu"] = {"slice_samples": args.ref_samples, "slice_s": round(s_ref, 3),
                                    "frame_s": round(s_ref * n / args.ref_samples, 1),
                                    "frame_s_is": "extrapolated linearly in n from the slice (thin SVD of n x M)"}
        res["workloads"].append(row)
        del dref, dsrv, dout, dtaps, drank
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if not all(w["batch_matches_single_frame_calls"] for w in res["workloads"]):
        sys.exit(1)


if __name__ == "__main__":
    main()
