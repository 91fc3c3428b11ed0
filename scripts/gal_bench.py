#!/usr/bin/env python
"""GAL_JPE throughput on the GPU against the reference's own GAL_JPE on the host.  Prints one JSON line.

    python scripts/gal_bench.py [--n 524288] [--workloads 16x64,32x185,512x512] [--reps 2]

Per (latticeLen, delayLineLen) workload: a device-resident batch of frames (enough to fill every SM, capped by
--mem-gb) goes through prc_gal_jpe_frames_c64 in one launch on a caller stream, timed with CUDA events; frames/s,
ns per sample step (launch time / n: every frame is a serial recurrence of n steps, all frames run side by side)
and the kernel's own time from the library's profile table ("gal_jpe").  Frames 0 and -1 of the timed batch are
checked bit for bit against single-frame GAL_JPE calls.  The reference column times a short slice of the
reference's GAL_JPE (oracle/_ref, placed there by build()) on one host core and extrapolates to a whole frame.
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

MU1, MU2, PEEK = 1e-3, 1e-2, 10


def card():
    """Name and power limit of GPU 0, read now (nvidia-smi query only)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": q[0].strip(), "power_limit": q[1].strip()}
    except Exception as exc:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({exc.__class__.__name__})"}


def reference_us_per_sample(L, D, samples):
    """The reference's GAL_JPE on `samples` samples, one host core: microseconds per sample, or None."""
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref_dir, "passiveRadar")):
        return None
    sys.path.insert(0, ref_dir)
    try:
        from passiveRadar.clutter_removal import GAL_JPE as ref_gal
    finally:
        sys.path.remove(ref_dir)
    ref, srv = synth.make_frame(samples + PEEK + 1, "P1", frame=0)
    t0 = time.perf_counter()
    ref_gal(ref, srv, L, D, MU1, MU2, PEEK)
    return (time.perf_counter() - t0) / samples * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=524288, help="samples per frame (PRconfig.yaml chunk)")
    ap.add_argument("--workloads", default="16x64,32x185,512x512", help="latticeLen x delayLineLen, comma-separated")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--mem-gb", type=float, default=24.0, help="device memory for the batch's inputs and outputs")
    ap.add_argument("--ref-samples", type=int, default=1500, help="samples of the reference timed on the host")
    args = ap.parse_args()

    lib = _lib.load()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    stream = torch.cuda.Stream(dev)
    n = args.n
    base = [synth.make_frame(n, "P1", frame=100 + i) for i in range(4)]
    res = {"what": "GAL_JPE (clutter_removal.py:251-364), device-resident batch, one launch per batch", "n": n,
           "mu1": MU1, "mu2": MU2, "peek": PEEK, **card(), "sms": nsm, "workloads": []}
    for wl in args.workloads.split(","):
        L, D = (int(v) for v in wl.lower().split("x"))
        variant = "warp_per_frame" if D <= 256 else "cta_per_frame"
        per_sm = 16 if variant == "warp_per_frame" else 8
        cap = int(args.mem_gb * 1e9 // (3 * 8 * n))
        nframes = max(1, min(nsm * per_sm, cap))
        with torch.cuda.stream(stream):
            dref = torch.empty((nframes, 2 * n), dtype=torch.float32, device=dev)
            dsrv = torch.empty_like(dref)
            for i in range(nframes):
                dref[i].copy_(torch.from_numpy(base[i % 4][0].view(np.float32)))
                dsrv[i].copy_(torch.from_numpy(base[i % 4][1].view(np.float32)))
            dout = torch.empty_like(dref)
            dk = torch.empty((nframes, 2 * D), dtype=torch.float32, device=dev)
            dh = torch.empty_like(dk)
        stream.synchronize()

        def launch():
            _lib.check(lib.prc_gal_jpe_frames_c64(dref.data_ptr(), dsrv.data_ptr(), n, nframes, n, L, D, MU1, MU2, PEEK,
                                                  dout.data_ptr(), dk.data_ptr(), dh.data_ptr(), _lib.MEM_DEVICE, 0,
                                                  C.c_void_p(stream.cuda_stream), _lib.FLAG_ASYNC))

        launch()                                      # warm-up
        stream.synchronize()
        _lib.profile_reset()
        _lib.profile(True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.reps):
            launch()
        e1.record(stream)
        stream.synchronize()
        prof = _lib.profile_read()
        _lib.profile(False)
        ms = e0.elapsed_time(e1) / args.reps
        kms, kcnt = prof.get("gal_jpe", (0.0, 0))
        # the timed batch against single-frame calls of the public operator
        checked = True
        for i in (0, nframes - 1):
            o1, k1, h1 = prb.GAL_JPE(base[i % 4][0], base[i % 4][1], L, D, MU1, MU2, PEEK, True)
            checked &= bool(np.array_equal(dout[i].cpu().numpy().view(np.complex64), o1)
                            and np.array_equal(dk[i].cpu().numpy().view(np.complex64), k1)
                            and np.array_equal(dh[i].cpu().numpy().view(np.complex64), h1))
        us_ref = reference_us_per_sample(L, D, args.ref_samples)
        row = {"latticeLen": L, "delayLineLen": D, "variant": variant, "frames": nframes,
               "batch_ms": round(ms, 2), "frames_per_s": round(nframes / (ms * 1e-3), 2),
               "ns_per_sample_step": round(ms * 1e6 / n, 2),
               "sample_steps_per_s": round(nframes * n / (ms * 1e-3), 1),
               "kernel_ms_per_launch": round(kms / kcnt, 2) if kcnt else None,
               "batch_matches_single_frame_calls": checked}
        if us_ref is not None:
            cores = os.cpu_count()
            frame_s = us_ref * 1e-6 * n
            row["reference_cpu"] = {"us_per_sample": round(us_ref, 2), "frame_s": round(frame_s, 1),
                                    "frame_s_is": "extrapolated from %d samples" % args.ref_samples,
                                    "host_cores": cores,
                                    "frames_per_s_all_cores": round(cores / frame_s, 5),
                                    "frames_per_s_all_cores_is": "extrapolated: one frame per core, no contention"}
            row["speedup_vs_all_host_cores"] = round(row["frames_per_s"] / (cores / frame_s), 1)
        res["workloads"].append(row)
        del dref, dsrv, dout, dk, dh
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if not all(w["batch_matches_single_frame_calls"] for w in res["workloads"]):
        sys.exit(1)


if __name__ == "__main__":
    main()
