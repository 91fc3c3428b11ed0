#!/usr/bin/env python
"""Frame chain of range_doppler_plot.py:45-85 on the GPU (passiveradar_b200.RenderPipeline): one JSON line.

    python scripts/render_bench.py [--frames 1200] [--host-frames 240] [--ref-frames 24]

Per map size (256 x 301 and the shipped 1024 x 176): frames/s of run_device on device-resident complex64 maps, the
per-kernel times of one profiled pass (prc_profile_*), the host-array run path, the same maps through one
prc_cfar2d_f32 call per frame, and the reference chain on the host over a sample of frames (the reference's own
CFAR_2D and persistence when oracle/_ref holds them, else oracle/plot_oracle.py; the line says which).  The card's
name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = ((256, 301), (1024, 176))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power}
    except Exception as exc:              # the line still says what could not be read
        return {"name": None, "power_limit": None, "error": str(exc)}


def reference_chain():
    """(label, cfar(frame), persistence(CF, k, hold, decay)) of the reference when installed, else of the oracle."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if os.path.exists(os.path.join(ref, "passiveRadar", "plotting_tools.py")) and \
            os.path.exists(os.path.join(ref, "passiveRadar", "target_detection.py")):
        np.float = np.float64              # the aliases the reference's target_detection.py needs (this process only)
        np.int = np.int_
        try:
            import matplotlib.pyplot       # noqa: F401
        except ImportError:               # plotting_tools imports it and persistence does not use it
            mpl = types.ModuleType("matplotlib")
            mpl.pyplot = types.ModuleType("matplotlib.pyplot")
            sys.modules.setdefault("matplotlib", mpl)
            sys.modules.setdefault("matplotlib.pyplot", mpl.pyplot)
        sys.path.insert(0, ref)
        from passiveRadar.plotting_tools import persistence
        from passiveRadar.target_detection import CFAR_2D
        return "reference", CFAR_2D, persistence
    from oracle.frontend_oracle import cfar_2d_oracle
    from oracle.plot_oracle import persistence_oracle
    return "oracle", cfar_2d_oracle, persistence_oracle


def timed(torch, fn, reps=1):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1200)
    ap.add_argument("--host-frames", type=int, default=240)
    ap.add_argument("--ref-frames", type=int, default=24)
    args = ap.parse_args()
    import torch
    from passiveradar_b200 import _lib
    from passiveradar_b200.plotting_tools import RenderPipeline
    label, ref_cfar, ref_persistence = reference_chain()
    lib = _lib.load()
    result = {"bench": "render", "card": card(), "frames": args.frames, "reference_chain": label, "shapes": {}}
    g = torch.Generator(device="cuda").manual_seed(1)
    for F, R1 in SHAPES:
        T = args.frames
        maps = torch.randn((T, F, R1), dtype=torch.complex64, device="cuda", generator=g)
        pipe = RenderPipeline()

        def device_run():
            pipe.reset()
            pipe.run_device(maps)

        ms = timed(torch, device_run, reps=3)
        _lib.profile_reset()
        _lib.profile(True)
        device_run()
        prof = _lib.profile_read()
        _lib.profile(False)
        _lib.profile_reset()
        kern = {k: round(prof[k][0], 4) for k in ("cfar_frames", "persistence", "percentile")}
        cr = torch.empty((F, R1), dtype=torch.float32, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream or 1       # the legacy default stream (cudaStreamLegacy)

        def per_frame():
            for t in range(T):
                _lib.check(lib.prc_cfar2d_f32(maps[t].data_ptr(), F, R1, 18, 4, None, cr.data_ptr(), None,
                                              _lib.MEM_DEVICE, 0, stream, _lib.FLAG_ABS_C64 | _lib.FLAG_ASYNC))

        ms_single = timed(torch, per_frame)
        H = min(args.host_frames, T)
        host = np.ascontiguousarray(maps[:H].cpu().numpy().transpose(1, 2, 0))
        t0 = time.perf_counter()
        RenderPipeline(batch=64).run(host)
        host_s = time.perf_counter() - t0
        # the reference chain on the host: CFAR_2D per frame, persistence and the two percentiles of the last frame
        K = min(args.ref_frames, H)
        mag = np.abs(host[:, :, :K])
        t0 = time.perf_counter()
        CF = np.zeros(mag.shape)
        for i in range(K):
            CF[:, :, i] = ref_cfar(mag[:, :, i], 18, 4)
        t_cfar = time.perf_counter() - t0
        t0 = time.perf_counter()
        for kk in range(K):
            data = np.fliplr(ref_persistence(CF, kk, 20, 0.90).T)
        t_pers = time.perf_counter() - t0
        t0 = time.perf_counter()
        for kk in range(K):
            np.percentile(data.flatten(), 35), 1.5 * np.percentile(data.flatten(), 99)
        t_pct = time.perf_counter() - t0
        result["shapes"][f"{F}x{R1}"] = {
            "device_ms": round(ms, 3), "device_frames_per_s": round(T / (ms / 1e3), 1), "kernel_ms": kern,
            "per_frame_cfar2d_f32_ms": round(ms_single, 3),
            "host_run": {"frames": H, "seconds": round(host_s, 3), "frames_per_s": round(H / host_s, 1)},
            "host_chain_ms_per_frame": {"frames": K, "cfar": round(1e3 * t_cfar / K, 2),
                                        "persistence": round(1e3 * t_pers / K, 2),
                                        "percentiles": round(1e3 * t_pct / K, 2)},
        }
        del maps
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
