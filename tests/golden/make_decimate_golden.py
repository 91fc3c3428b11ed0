#!/usr/bin/env python
"""Generate the decimate / channel_preprocessing / normalize goldens under tests/golden/ by EXECUTING THE REFERENCE.

    PR_REFERENCE=<reference checkout> python tests/golden/make_decimate_golden.py

Every output comes from the reference's own ``passiveRadar.signal_utils.decimate``, ``channel_preprocessing`` and
``normalize`` imported from the reference checkout.  Inputs come from the seeded ``passiveradar_b200.synth.raw_iq``
(``signal`` below) and are not stored: each case keeps its arguments and the sha256 of its input.  Outputs of more than
4096 values are stored as 512 seeded samples.  Everything goes into tests/golden/decimate_goldens.npz, and the sha256 of
every stored array into decimate_reference_digests.json.
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

# decimate: name -> (dtype, n, k columns (0: one-dimensional), q, seed)
DECIMATE = {
    "dec_c64_q12": ("complex64", 5000, 0, 12, 1),
    "dec_c64_q96": ("complex64", 9000, 0, 96, 2),
    "dec_f32_q7_k3": ("float32", 2000, 3, 7, 3),
    "dec_i8_q2": ("int8", 1501, 0, 2, 4),
    "dec_c128_q173": ("complex128", 4000, 0, 173, 5),
    "dec_f64_q90": ("float64", 1801, 0, 90, 6),
    "dec_i16_q3_k8": ("int16", 999, 8, 3, 7),
    "dec_u8_q13": ("uint8", 700, 0, 13, 8),
    "dec_c64_q1000": ("complex64", 30001, 0, 1000, 9),
}
# channel_preprocessing: name -> (raw kind, complex samples, dec, fc, Fs, which of fc / Fs is a NumPy float64, seed)
CHANNEL = {
    "chan_i8_c64": ("int8", 20000, 12, -3.0e4, 2.4e5, "", 11),
    "chan_i16_f64": ("int16", 12000, 96, 1.0e4, 2.4e5, "fc", 12),
    "chan_f32_fs64": ("float32", 8001, 7, 5.0e3, 1.0e5, "Fs", 13),
    "chan_i8_q100": ("int8", 30000, 100, 2.0e5, 2.0e6, "", 14),
}
# normalize: name -> (dtype, shape, seed)
NORMALIZE = {
    "norm_i8": ("int8", (300, 2), 21),
    "norm_u8": ("uint8", (257,), 22),
    "norm_i16": ("int16", (40, 5), 23),
    "norm_f32": ("float32", (1000,), 24),
    "norm_f64": ("float64", (33, 3), 25),
    "norm_c64": ("complex64", (1200,), 26),
    "norm_c128": ("complex128", (17, 4), 27),
}
SAMPLE_ABOVE, SAMPLES = 4096, 512


def signal(dtype, n, seed):
    """Seeded samples of one dtype from synth.raw_iq: integers as drawn, floats and complex values from its float32
    I/Q; int8 includes -128."""
    dt = np.dtype(dtype)
    if dt in (np.int8, np.uint8):
        return synth.raw_iq(n, "int8", seed)[:n].view(dt)
    if dt == np.int16:
        return synth.raw_iq(n, "int16", seed)[:n]
    iq = synth.raw_iq(n, "float32", seed)
    if dt.kind == "c":
        return iq.view(np.complex64).astype(dt)
    return iq[:n].astype(dt)


def decimate_input(dtype, n, k, seed):
    x = signal(dtype, n * max(k, 1), seed)
    return x.reshape(n, k) if k else x


def channel_args(kind, n, dec, fc, Fs, strong, seed):
    sig = synth.raw_iq(n, kind, seed)
    fc = np.float64(fc) if strong == "fc" else fc
    Fs = np.float64(Fs) if strong == "Fs" else Fs
    return sig, dec, fc, Fs


def normalize_input(dtype, shape, seed):
    x = signal(dtype, int(np.prod(shape)), seed).reshape(shape)
    if x.dtype == np.int8:
        x.reshape(-1)[:3] = -128                     # numpy's abs wraps there
    return x


def digest(a):
    a = np.asarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def sampled(y, seed):
    """(flat indices, values) of y: all of it when small, else SAMPLES seeded positions plus both ends."""
    flat = np.asarray(y).reshape(-1)
    if flat.size <= SAMPLE_ABOVE:
        idx = np.arange(flat.size)
    else:
        rng = np.random.default_rng(seed)
        idx = np.unique(np.concatenate([rng.integers(0, flat.size, SAMPLES), [0, flat.size - 1]]))
    return idx.astype(np.int64), flat[idx]


def main():
    if not os.environ.get("PR_REFERENCE"):
        raise SystemExit("set PR_REFERENCE to a checkout of the reference (Max-Manning/passiveRadar)")
    sys.path.insert(0, os.environ["PR_REFERENCE"])
    from passiveRadar import signal_utils as su                        # the reference

    out = {}
    for name, (dtype, n, k, q, seed) in DECIMATE.items():
        x = decimate_input(dtype, n, k, seed)
        y = su.decimate(x, q)
        idx, vals = sampled(y, seed)
        out.update({name + "/args": np.array([n, k, q, seed], np.int64), name + "/dtype": np.array(dtype),
                    name + "/input": np.array(digest(x)), name + "/shape": np.array(y.shape, np.int64),
                    name + "/idx": idx, name + "/y": vals})
        print(f"{name}: {x.shape} {x.dtype} q={q} -> {y.shape} {y.dtype}, stored {idx.size}")
    for name, (kind, n, dec, fc, Fs, strong, seed) in CHANNEL.items():
        sig, dec_, fc_, Fs_ = channel_args(kind, n, dec, fc, Fs, strong, seed)
        y = su.channel_preprocessing(sig, dec_, fc_, Fs_)
        idx, vals = sampled(y, seed)
        out.update({name + "/args": np.array([n, dec, seed], np.int64), name + "/freqs": np.array([fc, Fs]),
                    name + "/kind": np.array(kind), name + "/strong": np.array(strong),
                    name + "/input": np.array(digest(sig)), name + "/shape": np.array(y.shape, np.int64),
                    name + "/idx": idx, name + "/y": vals})
        print(f"{name}: {sig.dtype} n={n} dec={dec} -> {y.shape} {y.dtype}, stored {idx.size}")
    for name, (dtype, shape, seed) in NORMALIZE.items():
        x = normalize_input(dtype, shape, seed)
        y = su.normalize(x)
        out.update({name + "/args": np.array([seed], np.int64), name + "/dtype": np.array(dtype),
                    name + "/in_shape": np.array(shape, np.int64), name + "/input": np.array(digest(x)),
                    name + "/y": y})
        print(f"{name}: {x.shape} {x.dtype} -> {y.dtype}")
    dest = os.environ.get("PR_GOLDEN_OUT", HERE)
    np.savez_compressed(os.path.join(dest, "decimate_goldens.npz"), **out)
    cases = {}
    for key, v in out.items():
        case, field = key.split("/")
        cases.setdefault(case, {})[field] = digest(v)
    with open(os.path.join(dest, "decimate_reference_digests.json"), "w") as f:
        json.dump({"generator": "tests/golden/make_decimate_golden.py", "cases": cases}, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
