#!/usr/bin/env python
"""Generate the signal-preview goldens under tests/golden/ by EXECUTING THE REFERENCE.

    python tests/golden/make_preview_golden.py        (after build() has placed the reference's modules in oracle/_ref)

Each case is a small seeded ``synth.recording`` preview with a planted channel delay, in one of signal_preview.py's two
branches (separate channels, or one source whose complex samples alternate between the channels), for int8 or int16.
Inputs are not stored: each case keeps the generator's arguments and the sha256 of its raw sources.  What comes from
the reference's own functions (oracle/_ref: deinterleave_IQ, find_channel_offset, frequency_shift, resample, xcorr):
the offset, both resampled channels (complex64, in full) and |xcorr| (float32 around its peak, sha256 of all of it).
The spectra are not stored: plt.psd is matplotlib, not reference code, and tests take them from
oracle.spectrum_oracle.psd_oracle.  preview_reference_digests.json records which is which and the sha256 of every
array written.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from passiveradar_b200 import synth                                    # noqa: E402
from oracle import spectrum_oracle as so                                # noqa: E402

BASE = {"input_sample_rate": 2400000, "input_center_freq": 102000000, "offset_freq": 100000, "resamp_up": 13,
        "resamp_dn": 119, "channel_bandwidth": 200000, "channel_freq": 101900000}
# name: (kind, interleaved, complex samples per channel, channel_delay, seed, input_chunk_length)
CASES = {
    "i8_split": ("int8", False, 20040, 8, 31, 40000),
    "i16_split": ("int16", False, 20040, -12, 32, 40000),
    "i8_inter": ("int8", True, 10040, 4, 33, 40002),
    "i16_inter": ("int16", True, 10040, -8, 34, 40000),
}
PEAK = 64


def config(name):
    kind, inter, n, delay, seed, icl = CASES[name]
    return dict(BASE, input_chunk_length=icl, interleaved_input_channels=inter)


def sources(name):
    """The case's raw sources: (ref_raw, srv_raw) or (interleaved, None)."""
    kind, inter, n, delay, seed, icl = CASES[name]
    c = config(name)
    ref, srv = synth.recording(n, c["input_sample_rate"], c["offset_freq"], c["resamp_up"], c["resamp_dn"],
                               delay=3 * c["resamp_up"], fd=20.0, channel_delay=delay, kind=kind, seed=seed)
    return (synth.interleave_channels(ref, srv), None) if inter else (ref, srv)


def digest(a):
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def main():
    out_dir = os.environ.get("PR_GOLDEN_OUT", HERE)
    table = {"from_reference": ["offset", "ref_resampled", "srv_resampled", "xcorr_peak", "xcorr_digest"],
             "from_oracle": ["input_psd and channel_psd: oracle.spectrum_oracle.psd_oracle (mlab.psd restated), "
                             "computed by the tests, not stored"],
             "cases": {}}
    for name in CASES:
        a, b = sources(name)
        r = so.preview_reference(config(name), a, b)
        xa = np.abs(r["xcorr"])
        k = int(np.argmax(xa))
        lo, hi = max(0, k - PEAK), min(xa.shape[0], k + PEAK + 1)
        arrays = {"args": np.array(CASES[name][2:5] + (CASES[name][5],), dtype=np.int64),
                  "kind": np.array(CASES[name][0]), "interleaved": np.array(CASES[name][1]),
                  "source_digest": np.array([digest(s) for s in (a, b) if s is not None]),
                  "offset": np.array(r["offset"], dtype=np.int64),
                  "ref_resampled": r["ref_resampled"].astype(np.complex64),
                  "srv_resampled": r["srv_resampled"].astype(np.complex64),
                  "xcorr_peak_lo": np.array(lo, dtype=np.int64), "xcorr_peak": xa[lo:hi].astype(np.float32),
                  "xcorr_len": np.array(xa.shape[0], dtype=np.int64), "xcorr_digest": np.array(digest(r["xcorr"]))}
        path = os.path.join(out_dir, f"preview_{name}.npz")
        np.savez_compressed(path, **arrays)
        table["cases"][name] = {k: digest(v) for k, v in arrays.items()}
        print(f"{name}: offset {r['offset']} (planted channel delay {CASES[name][3]}), resampled "
              f"{r['ref_resampled'].shape[0]} / {r['srv_resampled'].shape[0]}, xcorr {xa.shape[0]} lags, "
              f"{os.path.getsize(path)} bytes")
    with open(os.path.join(out_dir, "preview_reference_digests.json"), "w") as f:
        json.dump(table, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
