#!/usr/bin/env python
"""Generate the tracker golden vectors under tests/golden/ by EXECUTING THE REFERENCE.

    PR_REFERENCE=<reference checkout> python tests/golden/make_track_golden.py [--only NAME]

Every output written here comes from the reference's own ``passiveRadar.target_detection`` (get_measurements,
multitarget_tracker, simple_target_tracker) imported from the reference checkout.  That module uses ``np.float`` and
``np.int``, which NumPy >= 1.24 removed, so this process aliases them to float64 / int64 before importing it; the
reference files are not touched.  Inputs come from the seeded generator ``passiveradar_b200.synth.track_maps`` and are
not stored: each .npz keeps the generator's seed and parameters and the sha256 of the maps it produced.
tests/golden/track_reference_digests.json holds the sha256 of every stored array as this script produced them.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
if not os.environ.get("PR_REFERENCE"):
    raise SystemExit("set PR_REFERENCE to a checkout of the reference (Max-Manning/passiveRadar)")
sys.path.insert(0, os.environ["PR_REFERENCE"])
np.float = np.float64          # the aliases the reference's target_detection.py needs (NumPy < 1.24)
np.int = np.int_

from passiveRadar import target_detection as td                       # noqa: E402  (the reference)
from passiveradar_b200 import synth                                    # noqa: E402

OUT_DIR = os.environ.get("PR_GOLDEN_OUT", HERE)
EXTENT = (256.0, 200.0)        # frame_extent = [Doppler Hz, range km]

# (row0, col0, row_rate, col_rate, amplitude, t_on, t_off) per target; row = Doppler bin, col = range bin
SMALL_TARGETS = [
    (12.0, 30.0, 0.05, 0.25, 30.0, 0, 120),        # long-lived: promoted to confirmed
    (50.0, 80.0, -0.05, -0.3, 25.0, 5, 60),        # vanishes at frame 60: its track is killed
    (20.0, 70.0, 0.1, -0.2, 20.0, 30, 120),        # crosses the first one
    (45.0, 20.0, 0.0, 0.0, 18.0, 70, 100),         # stationary: repeated measurements, zero R scaling
    (5.0, 50.0, 0.3, 0.1, 35.0, 90, 110),          # appears late, moves fast
]
BIG_TARGETS = [
    (60.0, 100.0, 0.2, 0.4, 30.0, 0, 100),
    (200.0, 250.0, -0.3, -0.5, 25.0, 10, 80),
    (100.0, 150.0, 0.5, 0.0, 20.0, 20, 100),
    (180.0, 60.0, 0.0, 0.3, 22.0, 40, 70),
]
EDGE_TARGETS = [                                   # the strongest target sits near the range edge for a while
    (140.0, 15.0, 0.1, 0.05, 60.0, 0, 40),
    (90.0, 200.0, 0.2, -0.5, 30.0, 0, 100),
    (30.0, 120.0, -0.2, 0.3, 25.0, 30, 100),
]

CASES = [
    ("track_meas_256x301", dict(kind="meas", seed=101, rows=256, cols=301, T=1, targets=12)),
    ("track_meas_64x101", dict(kind="meas", seed=102, rows=64, cols=101, T=1, targets=3)),
    ("track_multi_small_n10", dict(kind="multi", seed=103, rows=64, cols=101, T=120, targets=SMALL_TARGETS, n_tracks=10)),
    ("track_multi_small_n1", dict(kind="multi", seed=103, rows=64, cols=101, T=120, targets=SMALL_TARGETS, n_tracks=1)),
    ("track_multi_small_n32", dict(kind="multi", seed=103, rows=64, cols=101, T=120, targets=SMALL_TARGETS, n_tracks=32)),
    ("track_multi_256x301", dict(kind="multi", seed=104, rows=256, cols=301, T=100, targets=BIG_TARGETS, n_tracks=10)),
    ("track_simple_256x301", dict(kind="simple", seed=105, rows=256, cols=301, T=100, targets=EDGE_TARGETS)),
]


def maps_sha256(maps):
    return hashlib.sha256(np.ascontiguousarray(maps).tobytes()).hexdigest()


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def case(name, kind, seed, rows, cols, T, targets, n_tracks=0):
    maps = synth.track_maps(seed, rows, cols, T, targets)              # (T, rows, cols) float32
    data = np.moveaxis(maps, 0, 2).astype(np.float64)                  # what the reference's scripts feed it
    spec = np.asarray(targets if not isinstance(targets, int) else [], dtype=np.float64).reshape(-1, 7)
    t0 = time.time()
    if kind == "meas":
        out = dict(meas=td.get_measurements(data[:, :, 0], 99.8, list(EXTENT)))
    elif kind == "multi":
        out = dict(history=td.multitarget_tracker(data, list(EXTENT), n_tracks))
    else:
        out = dict(history=td.simple_target_tracker(data, EXTENT[1], EXTENT[0]))
    dt = time.time() - t0
    arrays = dict(kind=kind, seed=seed, rows=rows, cols=cols, T=T, n_targets=targets if isinstance(targets, int) else -1,
                  targets=spec, n_tracks=n_tracks, extent=np.array(EXTENT), maps_sha256=maps_sha256(maps), **out)
    path = os.path.join(OUT_DIR, name + ".npz")
    np.savez_compressed(path, seconds=dt, **arrays)
    print(f"{name}: {kind} {rows}x{cols}x{T} {dt:.2f}s -> {os.path.getsize(path) / 1024:.1f} KiB")
    return {k: digest(v) for k, v in arrays.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    args = ap.parse_args()
    dpath = os.path.join(OUT_DIR, "track_reference_digests.json")
    digests = json.load(open(dpath)) if os.path.exists(dpath) else {}
    for name, kw in CASES:
        if args.only is None or args.only in name:
            digests[name] = case(name, **kw)
    with open(dpath, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
