#!/usr/bin/env python
"""Generate the frame-chain golden vectors under tests/golden/ by EXECUTING THE REFERENCE.

    PR_REFERENCE=<reference checkout> python tests/golden/make_render_golden.py

Every output written here comes from the reference's own ``passiveRadar.plotting_tools.persistence`` and
``passiveRadar.target_detection.CFAR_2D`` imported from the reference checkout, composed as range_doppler_plot.py:45-85
does.  plotting_tools imports matplotlib.pyplot, which it does not use for persistence: this process puts an empty
stub module in its place.  target_detection uses ``np.float`` and ``np.int``, which NumPy >= 1.24 removed, so this
process aliases them to float64 / int64 before importing it.  The reference files are not touched.

render_persistence.npz: two seeded (5, 7, 25) stacks (float64 and float32) holding -0.0, NaN, +inf and -inf cells, and
persistence(X, k, hold, decay) for every k < 25, for decays given as Python floats, np.float32 and np.float64, and
hold in {1, 2, 20, 30}; plus the edge calls k = -1, k = -2 and hold = 0.
render_chain.npz: the chain on the seeded maps synth.track_maps(seed, rows, cols, T) (their sha256 is stored, not the
maps): data / vmin / vmax of every frame.
tests/golden/render_reference_digests.json holds the sha256 of every stored array as this script produced them.
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

from passiveRadar.plotting_tools import persistence                  # noqa: E402  (the reference)
from passiveRadar.target_detection import CFAR_2D                    # noqa: E402  (the reference)
from passiveradar_b200 import synth                                   # noqa: E402

OUT_DIR = os.environ.get("PR_GOLDEN_OUT", HERE)
SHAPE = (5, 7, 25)
HOLDS = (1, 2, 20, 30)
DECAYS = {"py0.9": 0.9, "f32_0.9": np.float32(0.9), "f64_0.9": np.float64(0.9), "py0.0": 0.0, "py1.0": 1.0,
          "py1.5": 1.5}
CHAIN = dict(seed=151, rows=32, cols=45, T=24, targets=3, fw=18, gw=4, hold=20, decay=0.90)


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def stack(dtype, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal(SHAPE).astype(dtype)
    X[0, 0, :] = -0.0                   # a cell that is -0.0 in every frame
    X[1, 2, 3] = np.nan
    X[2, 3, 10] = np.inf
    X[3, 4, 12] = -np.inf
    X[4, 6, 0] = -0.0
    X[0, 1, 24] = np.inf
    return X


def persistence_cases():
    out = {}
    for tag, dtype, seed in (("f64", np.float64, 11), ("f32", np.float32, 12)):
        X = stack(dtype, seed)
        out[f"stack_{tag}"] = X
        for dname, decay in DECAYS.items():
            for hold in HOLDS:
                with np.errstate(invalid="ignore", over="ignore"):
                    out[f"out_{tag}_{dname}_h{hold}"] = np.stack([persistence(X, k, hold, decay) for k in range(SHAPE[2])])
        out[f"edge_{tag}_km1"] = persistence(X, -1, 20, 0.9)
        out[f"edge_{tag}_km2"] = persistence(X, -2, 20, 0.9)
        out[f"edge_{tag}_h0"] = persistence(X, 5, 0, 0.9)
    return out


def chain_case():
    c = CHAIN
    maps = synth.track_maps(c["seed"], c["rows"], c["cols"], c["T"], c["targets"])   # (T, rows, cols) float32 >= 0
    xambg = np.abs(np.moveaxis(maps, 0, 2))                                            # (F, R+1, nframes)
    CF = np.zeros(xambg.shape)
    for i in range(xambg.shape[2]):
        CF[:, :, i] = CFAR_2D(xambg[:, :, i], c["fw"], c["gw"])
    data, vmin, vmax = [], [], []
    for kk in range(xambg.shape[2]):
        d = np.fliplr(persistence(CF, kk, c["hold"], c["decay"]).T)
        data.append(d)
        vmin.append(np.percentile(d.flatten(), 35))
        vmax.append(1.5 * np.percentile(d.flatten(), 99))
    return dict(maps_sha256=hashlib.sha256(maps.tobytes()).hexdigest(), data=np.stack(data),
                vmin=np.array(vmin), vmax=np.array(vmax), **{k: np.asarray(v) for k, v in c.items()})


def main():
    digests = {}
    for name, arrays in (("render_persistence", persistence_cases()), ("render_chain", chain_case())):
        path = os.path.join(OUT_DIR, name + ".npz")
        np.savez_compressed(path, **arrays)
        print(f"{name}: {len(arrays)} arrays -> {os.path.getsize(path) / 1024:.1f} KiB")
        digests[name] = {k: digest(v) for k, v in arrays.items()}
    with open(os.path.join(OUT_DIR, "render_reference_digests.json"), "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
