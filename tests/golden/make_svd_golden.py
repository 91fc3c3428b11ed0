#!/usr/bin/env python
"""Generate the LS_Filter_SVD golden vectors under tests/golden/ by EXECUTING THE REFERENCE.

    PR_REFERENCE=<reference checkout> python tests/golden/make_svd_golden.py [--only NAME]

Every ``out`` / ``taps`` written here is an output of the reference's own ``passiveRadar.clutter_removal.LS_Filter_SVD``
imported from the reference checkout.  Frames of ``synth.make_frame`` are not stored (the .npz keeps their seed and
``synth.frame_digest``); the hand-made inputs (a short frame, a zero and a periodic reference, complex128 and float32
channels) are stored.  tests/golden/svd_reference_digests.json holds the sha256 of every array (dtype, shape and bytes;
the wall-time entry excluded) as this script produced them.
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

from passiveRadar.clutter_removal import LS_Filter_SVD                 # noqa: E402  (the reference)
from passiveradar_b200 import synth                                    # noqa: E402

OUT_DIR = os.environ.get("PR_GOLDEN_OUT", HERE)


def periodic(n, period, seed):
    """A reference that repeats every `period` samples (n a multiple of it, so every circular shift repeats too) and a
    surveillance channel of two delayed copies plus noise: the data matrix has rank exactly `period`."""
    rng = np.random.default_rng(seed)
    base = (rng.standard_normal(period) + 1j * rng.standard_normal(period)).astype(np.complex64)
    ref = np.tile(base, n // period)
    noise = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    srv = (0.8 * np.roll(ref, 3) - 0.3j * np.roll(ref, -2) + 0.1 * noise).astype(np.complex64)
    return ref, srv


def random_pair(n, dtype, seed):
    rng = np.random.default_rng(seed)
    cplx = np.dtype(dtype).kind == "c"

    def one():
        x = rng.standard_normal(n) + (1j * rng.standard_normal(n) if cplx else 0)
        return x.astype(dtype)
    ref = one()
    srv = (0.7 * np.roll(ref, 2) + 0.2 * one()).astype(dtype)
    return ref, srv


# name -> (filter_len, peek, input spec): ("synth", n, profile, frame) or ("stored", maker)
CASES = [
    ("ls_svd_p0", 40, 10, ("synth", 8192, "P0", 0)),
    ("ls_svd_p1", 40, 10, ("synth", 8192, "P1", 0)),
    ("ls_svd_peek0", 30, 0, ("synth", 4000, "P1", 2)),
    ("ls_svd_short", 30, 10, ("stored", lambda: synth.make_frame(24, "P0", 3))),
    ("ls_svd_zero", 20, 5, ("stored", lambda: (np.zeros(2000, np.complex64), synth.make_frame(2000, "P1", 4)[1]))),
    ("ls_svd_periodic", 30, 10, ("stored", lambda: periodic(8190, 13, 7))),
    ("ls_svd_c128", 20, 10, ("stored", lambda: random_pair(3000, np.complex128, 8))),
    ("ls_svd_f32", 20, 10, ("stored", lambda: random_pair(3000, np.float32, 9))),
    ("ls_svd_c4", 175, 10, ("synth", 32768, "P1", 5)),
]


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def case(name, filter_len, peek, spec):
    arrays = dict(filter_len=filter_len, peek=peek)
    if spec[0] == "synth":
        _, n, profile, frame = spec
        ref, srv = synth.make_frame(n, profile, frame)
        arrays.update(n=n, profile=profile, frame=frame, digest=synth.frame_digest(ref, srv))
    else:
        ref, srv = spec[1]()
        arrays.update(n=ref.shape[0], ref=ref, srv=srv)
    t0 = time.time()
    out, taps = LS_Filter_SVD(ref, srv, filter_len, peek, True)
    dt = time.time() - t0
    arrays.update(out=out, taps=taps, srv_absmax=np.float64(np.abs(srv).max()))
    path = os.path.join(OUT_DIR, name + ".npz")
    np.savez_compressed(path, seconds=dt, **arrays)
    print(f"{name}: n={ref.shape[0]} filterLen={filter_len} peek={peek} {srv.dtype} {dt:.2f}s "
          f"-> {os.path.getsize(path) / 1024:.1f} KiB")
    return {k: digest(np.asarray(v)) for k, v in arrays.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    args = ap.parse_args()
    dpath = os.path.join(OUT_DIR, "svd_reference_digests.json")
    digests = json.load(open(dpath)) if os.path.exists(dpath) else {}
    for name, fl, peek, spec in CASES:
        if args.only is None or args.only in name:
            digests[name] = case(name, fl, peek, spec)
    with open(dpath, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
