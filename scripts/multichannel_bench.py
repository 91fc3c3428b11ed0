#!/usr/bin/env python
"""Several surveillance channels against one reference: prc_frames_multi_c64 against K prc_frames_c64 calls, one JSON line.

    python scripts/multichannel_bench.py [--cpis 16] [--calls 10] [--rounds 5]

Device-resident, float32 Kaiser window, for K = 1 .. 4 channels at two shapes:
  * config 2 (2^20 samples, 256 x 300, filter_len 300, peek 10): the one-pass plan is on, so K >= FM_MIN_SHARED_K
    channels take the shared pass (csrc/framemulti.cuh);
  * 2^20 samples, 256 x 1300, filter_len 310: the one-pass plan is off (R + M leave segments under L / 4), so every K
    runs prc_frames_c64's two-pass FFT path channel by channel.
For each (shape, K): channel-CPIs per second (--cpis CPIs per call, all K channels counted) of the multi-channel call and
of K single-channel calls on the same data, timed alternately over --rounds rounds of --calls calls each; per-kernel
milliseconds per call of both from a profiled run of its own; and the transform counts of the plan (transforms()).
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

L = 2048
SHAPES = {
    "config2": dict(n=2 ** 20, F=256, R=300, filter_len=300, peek=10),
    "onepass_off": dict(n=2 ** 20, F=256, R=1300, filter_len=310, peek=10),
}


def decimator_offset(ntaps, D):
    half = (ntaps - 1) // 2
    pre_pad = D - half % D
    return (half + pre_pad) // D * D - pre_pad


def transforms(n, F, R, filter_len, peek, K, nf, slots):
    """Length-L transforms of nf frames' K channels as K single-channel one-pass frames and as the shared pass, with
    ``slots`` CTAs of frame_pass_kernel in one wave, from the one-pass partition (prcore_corr.cu: onepass_plan;
    whether the plan is on is left to the caller): (single, shared)."""
    M = filter_len + peek
    bls = L - 2 * M + 2
    bmax = min(bls, L - M - R - peek + 1)
    D = n // F
    ntaps = D + 1
    c0 = decimator_offset(ntaps, D)
    seg = 0
    for j in range(F):
        lo, hi = max(j * D + c0 - (ntaps - 1), 0), min(j * D + c0 + 1, n)
        seg += -(-max(hi - lo, 0) // bmax)
    tail_lo = min((F - 1) * D + c0 + 1, n)
    ntail = -(-(n - tail_lo) // bls)
    ncta = max(1, min(F + ntail, slots // nf))
    single = K * (4 * seg + 3 * ntail + 2 * ncta + F)
    shared = (3 + K) * seg + (2 + K) * ntail + (1 + K) * ncta + K * F
    return nf * single, nf * shared


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cpis", type=int, default=16)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    import scipy.signal as signal
    import torch
    from passiveradar_b200 import _lib

    if not torch.cuda.is_available():
        raise SystemExit("multichannel_bench needs a CUDA device")
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    nsm = torch.cuda.get_device_properties(dev).multi_processor_count
    res = {"bench": "multichannel", "cpis_per_call": a.cpis, "calls": a.calls, "rounds": a.rounds, "card": card(),
           "unit": "channel-CPIs/s", "shapes": {}}
    nf = a.cpis
    for label, s in SHAPES.items():
        n, F, R, fl, peek = s["n"], s["F"], s["R"], s["filter_len"], s["peek"]
        g = torch.Generator(device=dev).manual_seed(n + R)
        ref = torch.complex(torch.randn((nf, n), generator=g, device=dev), torch.randn((nf, n), generator=g, device=dev))
        srv = torch.complex(torch.randn((4, nf, n), generator=g, device=dev), torch.randn((4, nf, n), generator=g, device=dev))
        srv += 0.5 * ref                  # clutter: the reference leaks into every channel
        w = torch.from_numpy(signal.get_window(("kaiser", 5.0), n).astype(np.float32)).to(dev)
        maps_m = torch.empty((4, nf, F, R + 1), dtype=torch.complex64, device=dev)
        maps_s = torch.empty((4, nf, F, R + 1), dtype=torch.complex64, device=dev)
        flags = _lib.FLAG_ASYNC | _lib.FLAG_WINDOW_F32
        out = {}
        for K in range(1, 5):
            def multi():
                _lib.check(lib.prc_frames_multi_c64(ref.data_ptr(), srv.data_ptr(), n, nf, n, K, nf * n, fl, peek, 1.0,
                                                    R, F, w.data_ptr(), maps_m.data_ptr(), None, 0, None, flags))

            def single():
                for k in range(K):
                    _lib.check(lib.prc_frames_c64(ref.data_ptr(), srv[k].data_ptr(), n, nf, n, fl, peek, 1.0, R, F,
                                                  w.data_ptr(), maps_s[k].data_ptr(), None, None, _lib.MEM_DEVICE, 0,
                                                  None, flags))

            arms = {"multi": multi, "single": single}
            for f in arms.values():              # warm-up
                f()
            _lib.check(lib.prc_sync(0, None))
            same = bool(torch.equal(maps_m[:K], maps_s[:K]))
            rate = {name: [] for name in arms}
            for _ in range(a.rounds):
                for name, f in arms.items():
                    _lib.check(lib.prc_sync(0, None))
                    t0 = time.perf_counter()
                    for _ in range(a.calls):
                        f()
                    _lib.check(lib.prc_sync(0, None))
                    rate[name].append(K * nf * a.calls / (time.perf_counter() - t0))
            kern = {}
            for name, f in arms.items():
                _lib.profile_reset()
                _lib.profile(True)
                f()
                prof = _lib.profile_read()
                _lib.profile(False)
                kern[name] = {k: round(v[0], 4) for k, v in prof.items() if v[1] > 0}
            counts = None
            if label == "config2":
                single_t, shared_t = transforms(n, F, R, fl, peek, K, nf, _lib.get_option("fft_ctas_frame") * nsm)
                counts = {"single": single_t, "shared": shared_t}
            out[f"K={K}"] = {
                "multi": [round(v, 1) for v in rate["multi"]],
                "single": [round(v, 1) for v in rate["single"]],
                "multi_over_single_median": round(float(np.median(rate["multi"]) / np.median(rate["single"])), 4),
                "multi_spread": round(float((max(rate["multi"]) - min(rate["multi"])) / np.median(rate["multi"])), 4),
                "single_spread": round(float((max(rate["single"]) - min(rate["single"])) / np.median(rate["single"])), 4),
                "maps_bit_identical": same,
                "kernel_ms_per_call": kern,
                "transforms_per_call": counts,
            }
        res["shapes"][label] = {**s, **out}
        del ref, srv, maps_m, maps_s
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
