"""Time the recording chain (passiveradar_b200.recording) on a synthetic recording.

    python scripts/recording_bench.py [--config shipped|fast] [--chunks 16] [--batch 8] [--interleaved]

Prints one JSON line with
  * frames/s of RecordingPipeline.run from raw data in pinned host memory,
  * frames/s of RecordingPipeline.run_device from device-resident raw data,
  * frames/s of main.py's per-chunk composition of the drop-ins (what install() gives main.py: every stage of every
    chunk a host -> device -> host call, one thread, no dask),
  * per-stage kernel time per frame from prc_profile_* in a separate profiled run,
  * the card's name and power limit read in the same run.
With --interleaved, the same recording is also stored as one interleaved two-channel stream (PRconfig.yaml's
interleaved_input_channels) and the line gains an ``interleaved`` entry: run and run_device frames/s of both layouts,
measured alternately in this call (``--rounds`` times each), and the front end's kernel time per frame
(``frontend_chunks``) of both layouts from a profiled run of each.
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
    ap.add_argument("--interleaved", action="store_true", help="also time the interleaved two-channel layout")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of the two layouts (--interleaved)")
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
    result = {"config": args.config, "frames": pipe.nframes, "batch": args.batch,
              "pipeline_host_fps": round(host_fps, 2), "pipeline_device_fps": round(dev_fps, 2),
              "composition_fps": round(comp_fps, 3), "composition_frames": comp_maps.shape[2], "stage_us_per_frame": stages,
              "card": name, "power_limit": power}
    if args.interleaved:
        result["interleaved"] = interleaved(args, config, ref, srv, pipe, rd, sd)
    print(json.dumps(result))


def interleaved(args, config, ref, srv, sep, rd, sd):
    """Both layouts of one recording, timed alternately: the separate channels (ref, srv) and the stream
    synth.interleave_channels(ref, srv), both at offset 0, where they make the same frames."""
    import torch
    stream = synth.interleave_channels(ref, srv)
    inter = RecordingPipeline.from_config(dict(config, interleaved_input_channels=True), batch=args.batch,
                                          interleaved_chunking="separate")
    streamd = torch.from_numpy(stream).cuda()
    inter.run(stream[:len(stream) // 3], offset=0)                             # warm-up
    inter.run_device(streamd, offset=0)
    runs = {"separate_run": lambda: sep.run(ref, srv, offset=0), "interleaved_run": lambda: inter.run(stream, offset=0),
            "separate_run_device": lambda: sep.run_device(rd, sd, offset=0),
            "interleaved_run_device": lambda: inter.run_device(streamd, offset=0)}
    fps = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, f in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            fps[k].append(round(sep.nframes / (time.perf_counter() - t0), 2))
    assert inter.nframes == sep.nframes
    front = {}
    for k, (pipe, call) in {"separate": (sep, lambda: sep.run_device(rd, sd, offset=0)),
                            "interleaved": (inter, lambda: inter.run_device(streamd, offset=0))}.items():
        _lib.profile(True)
        _lib.profile_reset()
        call()
        ms, _ = _lib.profile_read()["frontend_chunks"]
        _lib.profile(False)
        front[k] = round(1e3 * ms / pipe.nframes, 1)
    return {"frames": inter.nframes, "fps": fps, "frontend_chunks_us_per_frame": front}


if __name__ == "__main__":
    main()
