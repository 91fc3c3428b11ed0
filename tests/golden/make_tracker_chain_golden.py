#!/usr/bin/env python
"""Generate the tracker-chain golden vector under tests/golden/ by EXECUTING THE REFERENCE.

    PR_REFERENCE=<reference checkout> python tests/golden/make_tracker_chain_golden.py

Every output written here comes from the reference's own ``passiveRadar.target_detection`` (CFAR_2D,
multitarget_tracker, simple_target_tracker) and ``passiveRadar.plotting_tools.persistence`` imported from the reference
checkout, composed as the lines of multitarget_kalman_tracker.py / simple_kalman_tracker.py do: np.abs of the stack,
the CFAR loop into a float64 stack, the tracker, the scripts' masks of the estimates, and the phosphor frames with
their colour limits.  target_detection uses ``np.float`` and ``np.int``, which NumPy >= 1.24 removed, so this process
aliases them to float64 / int64; plotting_tools imports matplotlib.pyplot, which persistence does not use, so an empty
stub stands in for it.  The reference files are not touched.

tracker_chain.npz: a seeded complex64 stack of 60 frames of 64 x 101 (magnitudes synth.track_maps(seed, ...), phases
from default_rng(seed); its sha256 is stored, not the stack): both trackers' histories, the masked estimates, the
colour limits of every frame and the phosphor frames listed in data_frames.
tests/golden/tracker_chain_reference_digests.json holds the sha256 of every stored array as this script produced them.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
if not os.environ.get("PR_REFERENCE"):
    raise SystemExit("set PR_REFERENCE to a checkout of the reference (Max-Manning/passiveRadar)")
sys.path.insert(0, os.environ["PR_REFERENCE"])
np.float = np.float64          # the aliases the reference's target_detection.py needs (NumPy < 1.24)
np.int = np.int_
_mpl = types.ModuleType("matplotlib")
_mpl.pyplot = types.ModuleType("matplotlib.pyplot")
sys.modules.setdefault("matplotlib", _mpl)
sys.modules.setdefault("matplotlib.pyplot", _mpl.pyplot)

from passiveRadar.plotting_tools import persistence                                        # noqa: E402
from passiveRadar.target_detection import CFAR_2D, multitarget_tracker, simple_target_tracker  # noqa: E402
from passiveradar_b200 import synth                                                         # noqa: E402

OUT_DIR = os.environ.get("PR_GOLDEN_OUT", HERE)
CASE = dict(seed=233, rows=64, cols=101, T=60, targets=4, fw=18, gw=4, hold=20, decay=0.90, n_tracks=10,
            max_range=200.0, max_doppler=256.0)
DATA_FRAMES = (0, 1, 18, 19, 20, 59)


def complex_maps(seed, rows, cols, T, targets):
    """(T, rows, cols) complex64: the tracker maps as magnitudes, seeded phases."""
    rng = np.random.default_rng(seed)
    mag = synth.track_maps(seed, rows, cols, T, targets)
    return (mag * np.exp(1j * rng.uniform(0, 2 * np.pi, mag.shape))).astype(np.complex64)


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def chain_case():
    c = CASE
    maps = complex_maps(c["seed"], c["rows"], c["cols"], c["T"], c["targets"])
    xambg = np.abs(np.moveaxis(maps, 0, 2))                   # the scripts: xambg = np.abs(f['/xambg'])
    Nframes = xambg.shape[2]
    CF = np.zeros(xambg.shape)
    for i in range(Nframes):
        CF[:, :, i] = CFAR_2D(xambg[:, :, i], c["fw"], c["gw"])
    # multitarget_kalman_tracker.py:60-75
    tracker_history = multitarget_tracker(CF, [c["max_doppler"], c["max_range"]], c["n_tracks"])
    tracker_status = tracker_history['status']
    tracker_status_confirmed_idx = np.nonzero(tracker_status != 2)
    tracker_range = np.squeeze(tracker_history['estimate'][:, :, 0]).copy()
    tracker_doppler = np.squeeze(tracker_history['estimate'][:, :, 1]).copy()
    tracker_range[tracker_status_confirmed_idx] = np.nan
    tracker_doppler[tracker_status_confirmed_idx] = np.nan
    # simple_kalman_tracker.py:210-222
    history = simple_target_tracker(CF, c["max_range"], c["max_doppler"])
    estimate = history['estimate']
    lockMode = history['lock_mode']
    unlocked = lockMode[:, 0].astype(bool)
    estimate_locked = estimate.copy()
    estimate_locked[unlocked, 0] = np.nan
    estimate_locked[unlocked, 1] = np.nan
    estimate_unlocked = estimate.copy()
    estimate_unlocked[~unlocked, 0] = np.nan
    estimate_unlocked[~unlocked, 1] = np.nan
    # the rendering loop of both scripts
    data, limits = [], []
    for kk in range(Nframes):
        d = np.fliplr(persistence(CF, kk, c["hold"], c["decay"]).T)
        limits.append((np.percentile(d.flatten(), 35), 1.5 * np.percentile(d.flatten(), 99)))
        if kk in DATA_FRAMES:
            data.append(d)
    return dict(maps_sha256=hashlib.sha256(maps.tobytes()).hexdigest(), multi_history=tracker_history,
                track_range=tracker_range, track_doppler=tracker_doppler, simple_history=history,
                estimate_locked=estimate_locked, estimate_unlocked=estimate_unlocked, limits=np.array(limits),
                data_frames=np.array(DATA_FRAMES), data=np.stack(data), **{k: np.asarray(v) for k, v in c.items()})


def main():
    arrays = chain_case()
    st = arrays["multi_history"]["status"]
    print(f"confirmed track-frames: {(st == 2).sum()}, locked frames: {(arrays['simple_history']['lock_mode'][:, 0] == 0).sum()}")
    path = os.path.join(OUT_DIR, "tracker_chain.npz")
    np.savez_compressed(path, **arrays)
    print(f"tracker_chain: {len(arrays)} arrays -> {os.path.getsize(path) / 1024:.1f} KiB")
    with open(os.path.join(OUT_DIR, "tracker_chain_reference_digests.json"), "w") as f:
        json.dump({"tracker_chain": {k: digest(v) for k, v in arrays.items()}}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
