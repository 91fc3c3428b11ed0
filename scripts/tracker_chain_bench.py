#!/usr/bin/env python
"""The tracker scripts' chain on the GPU (passiveradar_b200.TrackerPipeline): one JSON line.

    python scripts/tracker_chain_bench.py [--frames 1200] [--host-frames 240] [--ref-frames 20]

Per map size (256 x 301 and the shipped config's 1024 x 176), per tracker (multi-target with 10 tracks, simple) and
with and without rendering: frames/s of run_device on a device-resident complex64 stack of --frames maps, once with
the whole stack in one call and once one map per call (the live case, the host loop included); the per-kernel times
of one profiled whole-stack pass (prc_profile_*); and the host-array run path over --host-frames maps.  The maps are
synth.track_maps magnitudes (Rayleigh background, moving point targets) with seeded phases.  The reference column
runs the scripts' own chain on one host core over --ref-frames maps: the CFAR_2D loop into a float64 stack, then
multitarget_tracker or simple_target_tracker, with the reference's modules when oracle/_ref holds them (np.float /
np.int, which NumPy >= 1.24 removed, aliased in this process only) and the NumPy oracles otherwise; the line says
which.  The card's name and power limit are read in the same run.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = ((256, 301), (1024, 176))
MAX_RANGE, MAX_DOPPLER, N_TRACKS = 200.0, 256.0, 10
KERNELS = ("cfar_frames", "track_meas", "track_multi", "track_simple", "persistence", "percentile")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power}
    except Exception as exc:              # the line still says what could not be read
        return {"name": None, "power_limit": None, "error": str(exc)}


def reference_chain():
    """(label, CFAR_2D, multitarget_tracker, simple_target_tracker) of the reference when installed, else the oracles."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if os.path.exists(os.path.join(ref, "passiveRadar", "target_detection.py")):
        np.float = np.float64              # the aliases the reference's target_detection.py needs (this process only)
        np.int = np.int_
        sys.path.insert(0, ref)
        from passiveRadar.target_detection import CFAR_2D, multitarget_tracker, simple_target_tracker
        return "reference", CFAR_2D, multitarget_tracker, simple_target_tracker
    from oracle.frontend_oracle import cfar_2d_oracle
    from oracle.track_oracle import multitarget_tracker, simple_target_tracker
    return "oracle", cfar_2d_oracle, multitarget_tracker, simple_target_tracker


def wall(torch, fn):
    """Seconds of fn(), from a synchronised start to a synchronised end (host loop included)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1200)
    ap.add_argument("--host-frames", type=int, default=240)
    ap.add_argument("--ref-frames", type=int, default=20)
    args = ap.parse_args()
    import torch
    from passiveradar_b200 import _lib, synth
    from passiveradar_b200.target_detection import TrackerPipeline
    label, ref_cfar, ref_multi, ref_simple = reference_chain()
    _lib.load()
    T = args.frames
    result = {"bench": "tracker_chain", "card": card(), "frames": T, "n_tracks": N_TRACKS,
              "reference_chain": label, "shapes": {}}
    for F, R1 in SHAPES:
        mag = synth.track_maps(2024, F, R1, T, 10)
        g = torch.Generator(device="cuda").manual_seed(1)
        phase = torch.rand((T, F, R1), dtype=torch.float32, device="cuda", generator=g) * (2 * np.pi)
        maps = torch.from_numpy(mag).cuda() * torch.exp(1j * phase)
        del phase
        shape = {}
        for tracker in ("multi", "simple"):
            for render in (True, False):
                pipe = TrackerPipeline(MAX_RANGE, MAX_DOPPLER, tracker=tracker, n_tracks=N_TRACKS, render=render)

                def whole():
                    pipe.reset()
                    pipe.run_device(maps)

                def live():
                    pipe.reset()
                    for t in range(T):
                        pipe.run_device(maps[t:t + 1])

                pipe.run_device(maps[:2])                                   # warm every launch of both modes
                pipe.run_device(maps[2:3])
                s_whole = min(wall(torch, whole) for _ in range(2))
                s_live = wall(torch, live)
                _lib.profile_reset()
                _lib.profile(True)
                whole()
                prof = _lib.profile_read()
                _lib.profile(False)
                _lib.profile_reset()
                shape[f"{tracker}{'' if render else '_norender'}"] = {
                    "whole_stack_ms": round(1e3 * s_whole, 2), "whole_stack_frames_per_s": round(T / s_whole, 1),
                    "batch1_ms": round(1e3 * s_live, 1), "batch1_frames_per_s": round(T / s_live, 1),
                    "kernel_ms": {k: round(prof[k][0], 3) for k in KERNELS if k in prof and prof[k][1]}}
            H = min(args.host_frames, T)
            host = np.ascontiguousarray(maps[:H].cpu().numpy().transpose(1, 2, 0))
            pipe = TrackerPipeline(MAX_RANGE, MAX_DOPPLER, tracker=tracker, n_tracks=N_TRACKS, batch=64)
            pipe.run(host[:, :, :2])
            t0 = time.perf_counter()
            pipe.run(host)
            s_host = time.perf_counter() - t0
            shape[f"{tracker}_host_run"] = {"frames": H, "seconds": round(s_host, 3),
                                            "frames_per_s": round(H / s_host, 1)}
        # the scripts' chain on one host core: the CFAR_2D loop, then each tracker
        K = min(args.ref_frames, T)
        xambg = np.abs(np.ascontiguousarray(maps[:K].cpu().numpy().transpose(1, 2, 0)))
        t0 = time.perf_counter()
        CF = np.zeros(xambg.shape)
        for i in range(K):
            CF[:, :, i] = ref_cfar(xambg[:, :, i], 18, 4)
        t_cfar = time.perf_counter() - t0
        with contextlib.redirect_stdout(io.StringIO()):          # the reference prints when candidates run out
            t0 = time.perf_counter()
            ref_multi(CF, [MAX_DOPPLER, MAX_RANGE], N_TRACKS)
            t_multi = time.perf_counter() - t0
            t0 = time.perf_counter()
            ref_simple(CF, MAX_RANGE, MAX_DOPPLER)
            t_simple = time.perf_counter() - t0
        shape["host_reference"] = {"frames": K, "cfar_ms_per_frame": round(1e3 * t_cfar / K, 2),
                                   "multi_chain_frames_per_s": round(K / (t_cfar + t_multi), 2),
                                   "simple_chain_frames_per_s": round(K / (t_cfar + t_simple), 2)}
        result["shapes"][f"{F}x{R1}"] = shape
        del maps
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
