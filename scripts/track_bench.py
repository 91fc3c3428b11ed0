#!/usr/bin/env python
"""Kalman trackers on the GPU against the reference's own trackers on the host.  Prints one JSON line.

    python scripts/track_bench.py [--frames 1200] [--rows 256] [--cols 301] [--tracks 10] [--batch-frames 100]

Workloads (config-2 maps, 256 x 301, from synth.track_maps):
  * the reference scripts' case: one sequence of --frames frames, multitarget_tracker (N_TRACKS = --tracks) and
    simple_target_tracker, from host arrays (the drop-ins, copies included) and device-resident (the C entry points
    on a caller stream, CUDA events);
  * a device-resident batch of 2 x SM-count sequences of --batch-frames frames, one call per tracker;
  * cfar_track: CFAR_2D of complex64 device maps, then the multi-target tracker;
  * the per-kernel times of the library's profile table (track_meas, track_multi, track_simple, and misc = CFAR).
The reference column runs the reference's multitarget_tracker and simple_target_tracker (oracle/_ref, placed there
by build()) on one host core over --ref-frames frames; np.float / np.int, which NumPy >= 1.24 removed, are aliased
in this process only.
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

EXTENT = [256.0, 200.0]


def card():
    """Name and power limit of GPU 0, read now (nvidia-smi query only)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": q[0].strip(), "power_limit": q[1].strip()}
    except Exception as exc:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({exc.__class__.__name__})"}


def reference_frames_per_s(data, tracks):
    """The reference's trackers on one host core: frames/s of each, or None without oracle/_ref."""
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref_dir, "passiveRadar")):
        return None
    np.float = np.float64
    np.int = np.int_
    sys.path.insert(0, ref_dir)
    try:
        from passiveRadar import target_detection as td
    finally:
        sys.path.remove(ref_dir)
    T = data.shape[2]
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):            # the reference prints when candidates run out
        t0 = time.perf_counter()
        td.multitarget_tracker(data, EXTENT, tracks)
        t1 = time.perf_counter()
        td.simple_target_tracker(data, EXTENT[1], EXTENT[0])
        t2 = time.perf_counter()
    return {"frames": T, "multitarget_frames_per_s": round(T / (t1 - t0), 1),
            "simple_frames_per_s": round(T / (t2 - t1), 1)}


def timed(stream, fn, reps):
    fn()
    stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        fn()
    e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1200, help="the reference scripts' num_frames")
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--cols", type=int, default=301)
    ap.add_argument("--tracks", type=int, default=10)
    ap.add_argument("--batch-frames", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-frames", type=int, default=40)
    args = ap.parse_args()

    lib = _lib.load()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    stream = torch.cuda.Stream(dev)
    T, rows, cols, N = args.frames, args.rows, args.cols, args.tracks
    n = rows * cols
    maps = synth.track_maps(2024, rows, cols, T, 10)          # (T, rows, cols) float32
    data = np.moveaxis(maps, 0, 2)                             # the reference's layout: frames on the last axis
    res = {"what": "Kalman trackers (target_detection.py:164-681)", "map": [rows, cols], "n_tracks": N, **card(),
           "sms": nsm}

    # one sequence from host arrays: the drop-ins, copies included
    prb.multitarget_tracker(data[:, :, :8], EXTENT, N)
    t0 = time.perf_counter()
    hm = prb.multitarget_tracker(data, EXTENT, N)
    t1 = time.perf_counter()
    hs = prb.simple_target_tracker(data, EXTENT[1], EXTENT[0])
    t2 = time.perf_counter()
    res["one_sequence_host"] = {"frames": T, "multitarget_frames_per_s": round(T / (t1 - t0), 1),
                                "simple_frames_per_s": round(T / (t2 - t1), 1)}

    # one sequence device-resident, device history, caller stream
    with torch.cuda.stream(stream):
        dmaps = torch.from_numpy(maps).to(dev)
        dhm = torch.empty(T * N * 880, dtype=torch.uint8, device=dev)
        dhs = torch.empty(T * 768, dtype=torch.uint8, device=dev)
    stream.synchronize()
    sp = C.c_void_p(stream.cuda_stream)

    def multi(ptr, S, Tn, ss, out):
        _lib.check(lib.prc_multitarget_track_frames(ptr, rows, cols, S, Tn, ss, n, EXTENT[0], EXTENT[1], N, out,
                                                    _lib.MEM_DEVICE, 0, sp, _lib.FLAG_ASYNC))

    def simple(ptr, S, Tn, ss, out):
        _lib.check(lib.prc_simple_track_frames(ptr, rows, cols, S, Tn, ss, n, EXTENT[1], EXTENT[0], out,
                                               _lib.MEM_DEVICE, 0, sp, _lib.FLAG_ASYNC))

    _lib.profile_reset()
    _lib.profile(True)
    ms_m = timed(stream, lambda: multi(dmaps.data_ptr(), 1, T, T * n, dhm.data_ptr()), args.reps)
    ms_s = timed(stream, lambda: simple(dmaps.data_ptr(), 1, T, T * n, dhs.data_ptr()), args.reps)
    prof = _lib.profile_read()
    _lib.profile(False)
    same = (dhm.cpu().numpy().tobytes() == hm.tobytes()) and (dhs.cpu().numpy().tobytes() == hs.tobytes())
    res["one_sequence_device"] = {"frames": T, "multitarget_ms": round(ms_m, 3),
                                  "multitarget_frames_per_s": round(T / (ms_m * 1e-3), 1),
                                  "simple_ms": round(ms_s, 3), "simple_frames_per_s": round(T / (ms_s * 1e-3), 1),
                                  "matches_host_call": same,
                                  "kernel_ms_per_sequence": {k: round(v[0] / (args.reps + 1), 3) for k, v in prof.items()
                                                             if k.startswith("track_")}}

    # a batch of sequences filling the GPU: overlapping windows of the device maps, seq_stride = 4 frames
    S, Tb = 2 * nsm, min(args.batch_frames, T)
    step = max(1, (T - Tb) // max(1, S - 1))
    with torch.cuda.stream(stream):
        bhm = torch.empty(S * Tb * N * 880, dtype=torch.uint8, device=dev)
        bhs = torch.empty(S * Tb * 768, dtype=torch.uint8, device=dev)
    _lib.profile_reset()
    _lib.profile(True)
    ms_bm = timed(stream, lambda: multi(dmaps.data_ptr(), S, Tb, step * n, bhm.data_ptr()), args.reps)
    ms_bs = timed(stream, lambda: simple(dmaps.data_ptr(), S, Tb, step * n, bhs.data_ptr()), args.reps)
    prof_b = _lib.profile_read()
    _lib.profile(False)
    last = np.frombuffer(bhm[-Tb * N * 880:].cpu().numpy().tobytes(), dtype=prb.target_track_dtype).reshape(Tb, N)
    want = prb.multitarget_tracker_frames(maps[None, (S - 1) * step:(S - 1) * step + Tb], EXTENT, N)[0]
    res["batch_device"] = {"sequences": S, "frames_per_sequence": Tb, "seq_stride_frames": step,
                           "multitarget_frames_per_s": round(S * Tb / (ms_bm * 1e-3), 1),
                           "simple_frames_per_s": round(S * Tb / (ms_bs * 1e-3), 1),
                           "last_sequence_matches_single_call": last.tobytes() == want.tobytes(),
                           "kernel_ms_per_batch": {k: round(v[0] / (args.reps + 1), 3) for k, v in prof_b.items()
                                                   if k.startswith("track_")}}

    # cfar_track: complex64 device maps -> CFAR_2D -> multi-target tracker
    with torch.cuda.stream(stream):
        cmaps = dmaps.to(torch.complex64)
    stream.synchronize()
    with torch.cuda.stream(stream):
        prb.cfar_track(cmaps[:8], 18, 4, EXTENT, N)
        _lib.profile_reset()
        _lib.profile(True)
        t0 = time.perf_counter()
        prb.cfar_track(cmaps, 18, 4, EXTENT, N)
        t1 = time.perf_counter()
        prof_c = _lib.profile_read()
        _lib.profile(False)
    res["cfar_track"] = {"frames": T, "frames_per_s": round(T / (t1 - t0), 1),
                         "kernel_ms": {k: round(v[0], 3) for k, v in prof_c.items() if v[1]}}

    ref = reference_frames_per_s(data[:, :, :args.ref_frames].astype(np.float64), N)
    if ref is not None:
        ref["host_cores_used"] = 1
        res["reference_cpu"] = ref
        res["speedup_one_sequence_device"] = {
            "multitarget": round(res["one_sequence_device"]["multitarget_frames_per_s"] / ref["multitarget_frames_per_s"], 1),
            "simple": round(res["one_sequence_device"]["simple_frames_per_s"] / ref["simple_frames_per_s"], 1)}
    print(json.dumps(res))
    if not (same and res["batch_device"]["last_sequence_matches_single_call"]):
        sys.exit(1)


if __name__ == "__main__":
    main()
