#!/usr/bin/env python
"""Generate the channel-offset goldens under tests/golden/ by EXECUTING THE REFERENCE.

    PR_REFERENCE=<reference checkout> python tests/golden/make_offset_golden.py

Every output here comes from the reference's own ``passiveRadar.signal_utils.find_channel_offset`` imported from the
reference checkout; the lags come from the same SciPy calls it makes (decimate, pad, correlate), since the reference
returns only the offset.  Inputs come from the seeded ``passiveradar_b200.synth.offset_pair`` and are not stored: each
case keeps the generator's arguments and the sha256 of both inputs.  |xc| is stored in full when it has at most 4096
lags, otherwise as a window of 129 lags around the peak plus 256 seeded lags.  Everything goes into
tests/golden/offset_goldens.npz.
"""
from __future__ import annotations

import hashlib
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

from passiveRadar import signal_utils as su                            # noqa: E402  (the reference)
from passiveradar_b200 import synth                                    # noqa: E402
from oracle import offset_oracle as oo                                  # noqa: E402

# name: (kind, n1, n2, nd, nl, planted delay, seed)
CASES = {
    "i8_pos": ("int8", 20000, 20000, 1, 500, 123, 1),
    "i8_neg_nd2": ("int8", 20000, 20000, 2, 400, -250, 2),
    "i8_edge_neg": ("int8", 20000, 20000, 1, 300, -300, 3),
    "u8_zero_nd3": ("uint8", 18000, 18000, 3, 300, 0, 4),
    "c64_edge_nd8": ("complex64", 40000, 40000, 8, 100, 800, 5),
    "c64_outside": ("complex64", 20000, 20000, 1, 50, 300, 6),
    "c64_b1_longer": ("complex64", 30000, 5000, 1, 100, 4000, 7),
    "i8_unequal_nd64": ("int8", 200000, 150000, 64, 200, -640, 8),
    "i8_main": ("int8", 5242880, 5242880, 1, 5000000, 1234, 9),
}
FULL_MAX = 4096


def digest(a):
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def main():
    out = {}
    for name, (kind, n1, n2, nd, nl, delay, seed) in CASES.items():
        s1, s2 = synth.offset_pair(n1, n2, kind, delay, seed)
        t = time.time()
        off = su.find_channel_offset(s1, s2, nd, nl)
        sec = time.time() - t
        o_off, xc = oo.find_channel_offset_oracle(s1, s2, nd, nl)
        assert o_off == off
        rng = np.random.default_rng(seed)
        if xc.shape[0] <= FULL_MAX:
            lags = np.arange(xc.shape[0])
        else:
            k = int(np.argmax(xc))
            win = np.arange(max(0, k - 64), min(xc.shape[0], k + 65))
            lags = np.unique(np.concatenate([win, rng.integers(0, xc.shape[0], 256), [0, xc.shape[0] - 1]]))
        p = name + "/"
        out[p + "args"] = np.array([n1, n2, nd, nl, delay, seed], dtype=np.int64)
        out[p + "kind"] = np.array(kind)
        out[p + "offset"] = np.array(off, dtype=np.int64)
        out[p + "nvalid"] = np.array(xc.shape[0], dtype=np.int64)
        out[p + "lags"] = lags.astype(np.int64)
        out[p + "xc"] = xc[lags]
        out[p + "digest"] = np.array([digest(s1), digest(s2)])
        out[p + "seconds"] = np.array(sec)
        print(f"{name}: offset {off} (planted {delay}), {xc.shape[0]} lags, stored {lags.shape[0]}, reference {sec:.2f} s")
    np.savez_compressed(os.path.join(os.environ.get("PR_GOLDEN_OUT", HERE), "offset_goldens.npz"), **out)


if __name__ == "__main__":
    main()
