#!/usr/bin/env python
"""Time the Welch PSD and signal_preview.py's chain and print one JSON line.

    python scripts/preview_bench.py [--reps 5] [--no-reference]

Rows: SignalPreview.run from host int8 arrays and run_device at the shipped PRconfig.yaml (each with per-kernel times
from the library's event profiler); psd alone at (2 399 625 complex64, NFFT 8192) and (262 144, NFFT 2048); psd_frames
on 1 200 device-resident frames of 2^19 complex64 at NFFT 2048 and 8192, in frames/s, with the kernel's algorithmic
bytes and FP64 flops (5 pad_to log2 pad_to per segment) and its share of whichever bound is larger (bytes / 3.35 TB/s,
flops / 34 TFLOP/s, the H100 SXM data sheet's HBM3 bandwidth and non-tensor FP64 rate); on the host,
scipy.signal.welch with mlab's parameters standing in for mlab.psd (matplotlib.mlab itself where it imports), and the
reference's preview functions (oracle/_ref) composed as the script composes them.  Every shape is warmed up; times are
medians of --reps repetitions.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import passiveradar_b200 as prb                                    # noqa: E402
from passiveradar_b200 import _lib, synth                          # noqa: E402
from offset_bench import card                                      # noqa: E402

HBM_BPS, FP64_FLOPS = 3.35e12, 34e12
SHIPPED = dict(synth.RECORDING_CONFIGS["shipped"], input_center_freq=102000000, channel_freq=101900000,
               channel_bandwidth=200000)


def timed(fn, reps, sync=None):
    fn()                                             # warm-up of this shape
    if sync:
        sync()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        if sync:
            sync()
        ts.append(time.perf_counter() - t)
    return {"median_ms": 1e3 * statistics.median(ts), "min_ms": 1e3 * min(ts), "max_ms": 1e3 * max(ts)}


def profiled(fn, sync):
    _lib.profile_reset()
    _lib.profile(True)
    fn()
    sync()
    prof = _lib.profile_read()
    _lib.profile(False)
    return {k: {"ms": v[0], "launches": v[1]} for k, v in prof.items() if v[1]}


def psd_work(frames, n, nfft):
    """Algorithmic bytes (complex64 frames read once, float64 spectra written once) and FP64 flops (5 P log2 P per
    segment transform) of psd_frames at noverlap 0, and the bytes the kernels' partial spectra add on top (written by
    spec_segments, read by spec_finish)."""
    nseg = n // nfft
    per_cta = -(-nseg // 64)
    nchunk = -(-nseg // per_cta)
    b = frames * (n * 8 + nfft * 8)
    f = frames * nseg * 5 * nfft * np.log2(nfft)
    return b, f, frames * 2 * nchunk * nfft * 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    import torch
    assert _lib.device_count() >= 1, "preview_bench.py needs a CUDA device"
    sync = torch.cuda.synchronize
    out = {"bench": "signal_preview", "card": card(), "reps": args.reps, "rows": {}}
    rows = out["rows"]

    ref, srv, _, _ = synth.recording_for(SHIPPED, 1, channel_delay=12, seed=4)
    pre = prb.SignalPreview.from_config(SHIPPED)
    r = pre.run(ref, srv)
    rows["preview_run_host_int8"] = dict(timed(lambda: pre.run(ref, srv), args.reps), offset=r["offset"],
                                         kernels=profiled(lambda: pre.run(ref, srv), sync))
    icl = SHIPPED["input_chunk_length"]
    dref, dsrv = torch.from_numpy(ref[:icl]).cuda(), torch.from_numpy(srv[:icl]).cuda()
    rows["preview_run_device"] = dict(timed(lambda: pre.run_device(dref, dsrv), args.reps, sync),
                                      kernels=profiled(lambda: pre.run_device(dref, dsrv), sync))

    rng = np.random.default_rng(3)
    for n, nfft in ((2399625, 8192), (262144, 2048)):
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        xd = torch.from_numpy(x).cuda()
        rows[f"psd_host_{n}_nfft{nfft}"] = timed(lambda: prb.psd(x, NFFT=nfft), args.reps)
        rows[f"psd_device_{n}_nfft{nfft}"] = timed(lambda: prb.psd(xd, NFFT=nfft), args.reps, sync)

    B, n = 1200, 1 << 19
    frames = torch.randn(B, n, dtype=torch.complex64, device="cuda")
    for nfft in (2048, 8192):
        t = timed(lambda: prb.psd_frames(frames, nfft), args.reps, sync)
        kern = profiled(lambda: prb.psd_frames(frames, nfft), sync)
        b, f, partial = psd_work(B, n, nfft)
        kms = kern.get("psd_segments", {}).get("ms", 0.0) + kern.get("psd_finish", {}).get("ms", 0.0)
        bound = max(b / HBM_BPS, f / FP64_FLOPS)
        rows[f"psd_frames_1200x2^19_nfft{nfft}"] = dict(
            t, frames_per_s=B / (t["median_ms"] * 1e-3), kernels=kern, algorithmic_bytes=int(b), partial_spectra_bytes=int(partial),
            fp64_flops=float(f),
            bound="bytes" if b / HBM_BPS >= f / FP64_FLOPS else "fp64",
            kernel_share_of_bound=(bound / (kms * 1e-3)) if kms else None)
    del frames
    torch.cuda.empty_cache()

    # host: what the script's spectra cost with NumPy / SciPy, and the reference's own preview functions
    xs = (rng.standard_normal(2399625) + 1j * rng.standard_normal(2399625)).astype(np.complex64)
    try:
        from matplotlib import mlab
        rows["host_mlab_psd_2399625_nfft8192"] = timed(lambda: mlab.psd(xs, NFFT=8192, Fs=2400000), args.reps)
    except Exception:
        import scipy.signal as signal
        rows["host_welch_2399625_nfft8192"] = timed(
            lambda: signal.welch(xs, fs=2400000, window=np.hanning(8192), nperseg=8192, noverlap=0, nfft=8192,
                                 detrend=False, return_onesided=False), args.reps)
    if args.no_reference:
        rows["host_reference_preview"] = "not measured (--no-reference)"
    else:
        try:
            from oracle import spectrum_oracle as so
            so.reference_signal_utils()
            rows["host_reference_preview"] = timed(lambda: so.preview_reference(SHIPPED, ref, srv), 1)
        except ImportError:
            rows["host_reference_preview"] = "not measured (no oracle/_ref)"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
