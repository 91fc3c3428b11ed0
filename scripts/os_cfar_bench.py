#!/usr/bin/env python
"""Ordered-statistic CFAR (prc_os_cfar2d_frames, csrc/oscfar.cuh) against CFAR_2D on the GPU: one JSON line.

    python scripts/os_cfar_bench.py [--frames 1200] [--render-frames 240] [--rounds 3] [--host-frames 4]

Per map size (256 x 301 and the shipped 1024 x 176), fw = 18, gw = 4, k = ceil(3N / 4) = 225:
  * OS and CA kernel time per frame (the mean-sum kernel included in both) over --frames device-resident complex64
    maps, from prc_profile_* in a profiled run of its own;
  * RenderPipeline frames/s with cfar="ca" and cfar="os" on the same maps, timed alternately, --rounds each;
  * scipy.ndimage.rank_filter on the host (the same window and rank on |map|) over --host-frames frames.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from render_bench import card  # noqa: E402

SHAPES = ((256, 301), (1024, 176))
FW, GW = 18, 4


def maps_for(torch, rows, cols, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    re = torch.randn((T, rows, cols), generator=g, device="cuda")
    im = torch.randn((T, rows, cols), generator=g, device="cuda")
    return torch.complex(re, im)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1200)
    ap.add_argument("--render-frames", type=int, default=240)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-frames", type=int, default=4)
    a = ap.parse_args()
    import torch
    from scipy import ndimage
    from passiveradar_b200 import _lib
    from passiveradar_b200.plotting_tools import RenderPipeline
    from passiveradar_b200.target_detection import os_rank

    if not torch.cuda.is_available():
        raise SystemExit("os_cfar_bench needs a CUDA device")
    lib = _lib.load()
    k = os_rank(FW, GW)
    res = {"bench": "os_cfar", "fw": FW, "gw": GW, "k": k, "frames": a.frames, "card": card(), "shapes": {}}
    for rows, cols in SHAPES:
        cells = rows * cols
        md = maps_for(torch, rows, cols, a.frames, rows + cols)
        cf = torch.empty((a.frames, rows, cols), dtype=torch.float64, device="cuda")
        flags = _lib.FLAG_CR_F64 | _lib.FLAG_ABS_C64

        def ca():
            _lib.check(lib.prc_cfar2d_frames(md.data_ptr(), rows, cols, a.frames, cells, FW, GW, cf.data_ptr(), cells,
                                             _lib.MEM_DEVICE, 0, None, flags))

        def os_():
            _lib.check(lib.prc_os_cfar2d_frames(md.data_ptr(), rows, cols, a.frames, cells, FW, GW, k, cf.data_ptr(),
                                                cells, 0, None, flags))

        ca(), os_()                                     # warm-up
        _lib.profile_reset()
        _lib.profile(True)
        for _ in range(3):
            ca()
            os_()
        prof = _lib.profile_read()
        _lib.profile(False)
        kern = {name: round(1e3 * prof[key][0] / (prof[key][1] * a.frames), 3)
                for name, key in (("ca_us_per_frame", "cfar_frames"), ("os_us_per_frame", "os_cfar"))}

        # the chain, timed alternately on the same maps
        rm = md[:a.render_frames]
        pipes = {"ca": RenderPipeline(), "os": RenderPipeline(cfar="os")}
        for p in pipes.values():
            p.run_device(rm)
        torch.cuda.synchronize()
        fps = {name: [] for name in pipes}
        for _ in range(a.rounds):
            for name, p in pipes.items():
                p.reset()
                t0 = time.perf_counter()
                p.run_device(rm)
                torch.cuda.synchronize()
                fps[name].append(rm.shape[0] / (time.perf_counter() - t0))

        # the host rank filter on |map| over a sample of frames
        host = np.abs(md[:a.host_frames].cpu().numpy())
        fp = np.ones((FW, FW), bool)
        e1 = (FW - GW) // 2
        fp[e1:FW - e1 + 1, e1:FW - e1 + 1] = False
        t0 = time.perf_counter()
        for f in host:
            ndimage.rank_filter(f, k - 1, footprint=fp[::-1, ::-1], mode="wrap", origin=0)
        host_ms = 1e3 * (time.perf_counter() - t0) / len(host)

        res["shapes"][f"{rows}x{cols}"] = {
            **kern,
            "os_over_ca_kernel": round(kern["os_us_per_frame"] / kern["ca_us_per_frame"], 2),
            "render_fps_ca": [round(v, 1) for v in fps["ca"]],
            "render_fps_os": [round(v, 1) for v in fps["os"]],
            "render_frames": int(rm.shape[0]),
            "scipy_rank_filter_ms_per_frame": round(host_ms, 2),
            "host_frames": len(host),
        }
        del md, cf
    print(json.dumps(res))


if __name__ == "__main__":
    main()
