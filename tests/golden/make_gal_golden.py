#!/usr/bin/env python
"""Generate the GAL_JPE golden vectors under tests/golden/ by EXECUTING THE REFERENCE.

    PR_REFERENCE=<reference checkout> python tests/golden/make_gal_golden.py [--only NAME]

Every array written here is an output of the reference's own ``passiveRadar.clutter_removal.GAL_JPE`` imported from
the reference checkout, on inputs from the seeded generator ``passiveradar_b200.synth``; nothing from ``oracle/`` or
``passiveradar_b200/csrc`` is involved.  tests/golden/gal_reference_digests.json holds the sha256 of every array (dtype,
shape and bytes; the wall-time entry excluded) as this script produced them; the tests read only the .npz files and
that digest file.
"""
from __future__ import annotations

import argparse
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

from passiveRadar.clutter_removal import GAL_JPE                      # noqa: E402  (the reference)
from passiveradar_b200 import synth                                    # noqa: E402

OUT_DIR = os.environ.get("PR_GOLDEN_OUT", HERE)

CASES = [
    ("gal_full", dict(n=6000, lattice_len=16, delay_line_len=16, mu1=1e-3, mu2=1e-2, peek=10, profile="P1")),
    ("gal_partial", dict(n=6000, lattice_len=8, delay_line_len=24, mu1=1e-3, mu2=1e-2, peek=10, profile="P1")),
    # mu1 = 2e-2 is above the 5e-3 clamp: min() picks the Python float on the first step
    ("gal_clamp", dict(n=4000, lattice_len=8, delay_line_len=12, mu1=2e-2, mu2=1e-2, peek=3, profile="P1")),
    ("gal_peek0", dict(n=3000, lattice_len=4, delay_line_len=17, mu1=1e-3, mu2=1e-2, peek=0, profile="P0")),
    ("gal_lattice1", dict(n=3000, lattice_len=1, delay_line_len=9, mu1=1e-3, mu2=1e-2, peek=10, profile="P1")),
    ("gal_mid", dict(n=20_000, lattice_len=32, delay_line_len=32, mu1=1e-3, mu2=1e-2, peek=10, profile="P1")),
]


def gal_case(name, n, lattice_len, delay_line_len, mu1, mu2, peek, profile, frame=0):
    ref, srv = synth.make_frame(n, profile, frame)
    t0 = time.time()
    out, k, h = GAL_JPE(ref, srv, lattice_len, delay_line_len, mu1, mu2, peek, True)
    dt = time.time() - t0
    path = os.path.join(OUT_DIR, name + ".npz")
    np.savez_compressed(path, n=n, lattice_len=lattice_len, delay_line_len=delay_line_len, mu1=mu1, mu2=mu2,
                        peek=peek, profile=profile, frame=frame, ref=ref, srv=srv, out=out, k=k, h=h, seconds=dt)
    print(f"{name}: n={n} latticeLen={lattice_len} delayLineLen={delay_line_len} mu1={mu1} mu2={mu2} peek={peek} "
          f"{profile} {dt:.2f}s -> {os.path.getsize(path) / 1024:.1f} KiB")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    args = ap.parse_args()
    for name, kw in CASES:
        if args.only is None or args.only in name:
            gal_case(name, **kw)


if __name__ == "__main__":
    main()
