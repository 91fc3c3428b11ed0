#!/usr/bin/env python
"""Beamscan of K channels' maps (prc_beamscan_frames, csrc/beamscan.cuh) on the GPU: one JSON line.

    python scripts/beamscan_bench.py [--frames 1200] [--rounds 3] [--chunk 8]

Per map size (256 x 301 and the shipped 1024 x 176), K = 2, 3, 4, and grid (181 angles of a half-wave ULA over a
sector, or 360 angles of a 0.3-wavelength UCA with wrap), on --frames device-resident complex64 frames:
  * kernel time per frame from prc_profile_* in a profiled run of its own;
  * frames/s of beamscan_frames with the profiler off, and of the torch composition einsum -> abs()**2 -> max over
    angles (--chunk frames per einsum), timed alternately over --rounds rounds; the two are checked to agree;
  * the lane instructions and HBM bytes of a frame from the shapes (DESIGN.md section 21), the time each would take at
    the card's maximum SM clock and 3.35 TB/s, and the share of the larger of those bounds the kernel reaches.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = ((256, 301), (1024, 176))
CHANNELS = (2, 3, 4)
SMS, LANES_PER_SM, HBM = 132, 128, 3.35e12          # H100 SXM: FP32 lanes per SM per clock, data-sheet bandwidth


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:
        return {"name": None, "power_limit": None, "max_sm_clock": None, "error": str(exc)}


def model(cells, K, A):
    """(lane instructions, bytes) of one frame: per cell and angle 4K FMAs for the complex dot, 2 for the power and
    about 6 for the scan; per cell K complex64 maps read and two float32 results written."""
    return cells * A * (4 * K + 8), cells * (8 * K + 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--chunk", type=int, default=8)
    a = ap.parse_args()
    import numpy as np
    import torch
    from passiveradar_b200 import _lib
    from passiveradar_b200.beamforming import beamscan_frames, steering_vectors, uca_positions, ula_positions

    if not torch.cuda.is_available():
        raise SystemExit("beamscan_bench needs a CUDA device")
    cd = card()
    try:
        clock_hz = float(cd["max_sm_clock"].split()[0]) * 1e6
    except Exception:
        clock_hz = 1.98e9
    res = {"bench": "beamscan", "frames": a.frames, "rounds": a.rounds, "card": cd, "cases": []}

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / 1e3, out

    for rows, cols in SHAPES:
        cells = rows * cols
        for K in CHANNELS:
            g = torch.Generator(device="cuda").manual_seed(rows + cols + K)
            maps = torch.complex(torch.randn((K, a.frames, rows, cols), generator=g, device="cuda"),
                                 torch.randn((K, a.frames, rows, cols), generator=g, device="cuda"))
            for A, wrap in ((181, False), (360, True)):
                S = (steering_vectors(uca_positions(K, 0.3), np.arange(360.0)) if wrap else
                     steering_vectors(ula_positions(K, 0.5), np.arange(181.0)))
                St = torch.from_numpy(S).cuda()

                def kernel():
                    return beamscan_frames(maps, S, wrap=wrap)

                def composition():
                    amp = torch.empty((a.frames, rows, cols), device="cuda")
                    idx = torch.empty((a.frames, rows, cols), dtype=torch.int64, device="cuda")
                    for t0 in range(0, a.frames, a.chunk):
                        cube = torch.einsum("ak,ktrc->tarc", St, maps[:, t0:t0 + a.chunk])
                        p, i = (cube.abs() ** 2).max(dim=1)
                        amp[t0:t0 + a.chunk] = p.sqrt()
                        idx[t0:t0 + a.chunk] = i
                    return amp, idx

                kernel(), composition()                  # warm-up of every shape
                torch.cuda.synchronize()
                _lib.profile_reset()
                _lib.profile(True)
                kernel()
                torch.cuda.synchronize()
                ms, n = _lib.profile_read()["beamscan"]
                _lib.profile(False)
                k_rates, t_rates = [], []
                for _ in range(a.rounds):
                    tk, (amp, pos) = timed(kernel)
                    tt, (amp_t, idx_t) = timed(composition)
                    k_rates.append(a.frames / tk)
                    t_rates.append(a.frames / tt)
                rel = float(((amp.double() ** 2 - amp_t.double() ** 2).abs().max() / (amp_t.double() ** 2).max()))
                same = float((torch.floor(pos + 0.5).long() % A == idx_t).double().mean())
                assert rel <= 1e-5 and same >= 0.99, (rows, cols, K, A, rel, same)
                instr, nbytes = model(cells, K, A)
                t_issue, t_mem = instr / (SMS * LANES_PER_SM * clock_hz), nbytes / HBM
                kt = ms / 1e3 / a.frames
                res["cases"].append({
                    "shape": [rows, cols], "K": K, "A": A, "wrap": wrap,
                    "kernel_us_per_frame": round(kt * 1e6, 3), "launches": n,
                    "kernel_frames_per_s": [round(r, 1) for r in k_rates],
                    "torch_frames_per_s": [round(r, 1) for r in t_rates],
                    "speedup": round(float(np.median(k_rates) / np.median(t_rates)), 2),
                    "lane_instructions": instr, "bytes": nbytes,
                    "issue_bound_us": round(t_issue * 1e6, 3), "hbm_bound_us": round(t_mem * 1e6, 3),
                    "bound": "issue" if t_issue >= t_mem else "hbm",
                    "share_of_bound": round(max(t_issue, t_mem) / kt, 3),
                    "amp2_rel_diff_vs_torch": rel, "same_beam_fraction": same,
                })
            del maps
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
