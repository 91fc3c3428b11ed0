"""Time the recording chain (passiveradar_b200.recording) on a synthetic recording.

    python scripts/recording_bench.py [--config shipped|fast] [--chunks 16] [--batch 8]

Prints one JSON line with
  * frames/s of RecordingPipeline.run from raw data in pinned host memory,
  * frames/s of RecordingPipeline.run_device from device-resident raw data,
  * frames/s of main.py's per-chunk composition of the drop-ins (what install() gives main.py: every stage of every
    chunk a host -> device -> host call, one thread, no dask),
  * per-stage kernel time per frame from prc_profile_* in a separate profiled run,
  * the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import passiveradar_b200 as prb                                   # noqa: E402
from passiveradar_b200 import _lib                                # noqa: E402
from passiveradar_b200.recording import RecordingPipeline        # noqa: E402
from passiveradar_b200 import synth                               # noqa: E402
from oracle.recording_oracle import dropin_composition            # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as exc:                 # the card name is part of the result: say that it is missing
        return f"unknown ({exc})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="shipped", choices=["shipped", "fast"])
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--composition-chunks", type=int, default=4)
    args = ap.parse_args()
    import torch
    if _lib.device_count() < 1:
        raise SystemExit("recording_bench.py needs a CUDA device")
    config = synth.RECORDING_CONFIGS[args.config]
    ref, srv, _, _ = synth.recording_for(config, args.chunks, seed=1)
    pipe = RecordingPipeline.from_config(config, batch=args.batch)
    pipe.run(ref[:len(ref) // 3], srv[:len(srv) // 3], offset=0)            # warm-up: modules, tables, allocations
    t0 = time.perf_counter()
    pipe.run(ref, srv, offset=0)
    host_fps = pipe.nframes / (time.perf_counter() - t0)
    rd, sd = torch.from_numpy(ref).cuda(), torch.from_numpy(srv).cuda()
    pipe.run_device(rd, sd, offset=0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pipe.run_device(rd, sd, offset=0)
    torch.cuda.synchronize()
    dev_fps = pipe.nframes / (time.perf_counter() - t0)
    cut = args.composition_chunks * config["input_chunk_length"] + 16       # main.py makes that many chunks of it
    dropin_composition(config, ref[:cut], srv[:cut], 0)                      # warm-up
    t0 = time.perf_counter()
    comp_maps, _ = dropin_composition(config, ref[:cut], srv[:cut], 0)
    comp_fps = comp_maps.shape[2] / (time.perf_counter() - t0)
    _lib.profile(True)
    _lib.profile_reset()
    pipe.run_device(rd, sd, offset=0)
    prof = _lib.profile_read()
    _lib.profile(False)
    stages = {k: round(1e3 * ms / pipe.nframes, 1) for k, (ms, cnt) in prof.items() if cnt}
    name, power = card()
    print(json.dumps({"config": args.config, "frames": pipe.nframes, "batch": args.batch,
                      "pipeline_host_fps": round(host_fps, 2), "pipeline_device_fps": round(dev_fps, 2),
                      "composition_fps": round(comp_fps, 3), "composition_frames": comp_maps.shape[2], "stage_us_per_frame": stages,
                      "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
