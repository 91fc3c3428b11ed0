"""Seeded synthetic two-channel IQ used by the tests, the goldens and bench.py.

The reference ships no recordings (its README points at a 6 GB Google-Drive
file), so every measurement in this repo runs on synthetic complex64 IQ with
the shapes BASELINE.json names.  Two profiles (SURVEY.md section 8d):

* ``P0``  reference and surveillance channels are independent unit-power white
  noise.  Strict-parity profile: nothing cancels, so float32 round-off of the
  reference implementation itself stays at the 1e-7 level.
* ``P1``  surveillance = direct-path + multipath clutter (delayed, scaled copies
  of the illuminator) + one weak Doppler-shifted target + receiver noise.  This
  is what a passive radar actually sees and what the LS / NLMS cancellers are
  for.

Pure host-side numpy; nothing here is on the timed path.
"""
from __future__ import annotations

import numpy as np

BASE_SEED = 20260924

# (delay in samples, complex amplitude) of the static clutter taps of profile P1
P1_CLUTTER = ((0, 1.0 + 0.0j), (3, 0.5j), (17, -0.2 + 0.0j), (60, 0.05 + 0.05j))
P1_TARGET = dict(delay=40, doppler_hz=37.0, amplitude=1e-3)
P1_NOISE_SIGMA = 1e-3
P1_SAMPLE_RATE = float(2 ** 19)


def white_iq(rng: np.random.Generator, n: int) -> np.ndarray:
    """Unit-power circular white noise, complex64."""
    re = rng.standard_normal(n, dtype=np.float32)
    im = rng.standard_normal(n, dtype=np.float32)
    out = np.empty(n, dtype=np.complex64)
    out.real = re
    out.imag = im
    out *= np.float32(1.0 / np.sqrt(2.0))
    return out


def make_frame(n: int, profile: str = "P1", frame: int = 0, seed: int = BASE_SEED):
    """Return ``(ref, srv)`` complex64 arrays of length ``n`` for CPI frame ``frame``."""
    rng = np.random.default_rng(seed + frame)
    ref = white_iq(rng, n)
    if profile == "P0":
        srv = white_iq(rng, n)
        return ref, srv
    if profile != "P1":
        raise ValueError(f"unknown profile {profile!r}")
    noise = white_iq(rng, n)
    acc = np.zeros(n, dtype=np.complex128)
    for delay, amp in P1_CLUTTER:
        acc += amp * np.roll(ref, delay % n if n else 0)
    t = P1_TARGET
    phase = 2.0 * np.pi * t["doppler_hz"] * np.arange(n, dtype=np.float64) / P1_SAMPLE_RATE
    acc += t["amplitude"] * np.roll(ref, t["delay"] % n if n else 0) * np.exp(1j * phase)
    acc += P1_NOISE_SIGMA * noise
    return ref, acc.astype(np.complex64)


def frame_digest(ref: np.ndarray, srv: np.ndarray) -> np.ndarray:
    """Small fingerprint stored next to goldens to detect RNG-stream drift."""
    n = ref.shape[0]
    picks = np.unique(np.clip(np.array([0, 1, n // 3, n // 2, n - 1]), 0, max(n - 1, 0)))
    return np.concatenate([
        ref[picks], srv[picks],
        np.array([ref.astype(np.complex128).sum(), srv.astype(np.complex128).sum()]).astype(np.complex64),
    ])


def raw_iq(n, kind="int8", seed=11):
    """Seeded interleaved I/Q block of ``n`` complex samples as a receiver would deliver it
    (``int8``: HackRF-style, ``int16``, or ``float32``); input of the front-end chain."""
    rng = np.random.default_rng(seed)
    if kind == "int8":
        return rng.integers(-128, 128, size=2 * n, dtype=np.int8)
    if kind == "int16":
        return rng.integers(-2048, 2048, size=2 * n, dtype=np.int16)
    if kind == "float32":
        return rng.standard_normal(2 * n).astype(np.float32)
    raise ValueError(f"unknown raw IQ kind {kind!r}")


def track_maps(seed, rows, cols, T, targets=4):
    """Seeded (T, rows, cols) float32 maps of the detector-output kind for the trackers: a Rayleigh(1) background
    plus point targets.  ``targets`` is a count (drawn from the seed) or a sequence of
    (row0, col0, row_rate, col_rate, amplitude, t_on, t_off): a target at (row0 + row_rate t, col0 + col_rate t)
    (row = Doppler bin, wrapped; col = range bin, dropped outside the map) with a half-amplitude cross around it,
    present for t_on <= t < t_off.  Targets move, cross, appear and vanish."""
    rng = np.random.default_rng(seed)
    maps = rng.rayleigh(1.0, size=(T, rows, cols)).astype(np.float32)
    if isinstance(targets, (int, np.integer)):
        spec = []
        for _ in range(int(targets)):
            on = int(rng.integers(0, max(1, T // 3)))
            spec.append((rng.uniform(0, rows), rng.uniform(10, max(11, cols - 10)), rng.uniform(-0.4, 0.4),
                         rng.uniform(-0.3, 0.3), rng.uniform(12, 40), on, int(rng.integers(on + 1, T + 1))))
        targets = spec
    for r0, c0, vr, vc, amp, on, off in targets:
        for t in range(int(on), min(int(off), T)):
            r = int(np.floor(r0 + vr * t + 0.5)) % rows
            c = int(np.floor(c0 + vc * t + 0.5))
            if not 0 <= c < cols:
                continue
            maps[t, r, c] += np.float32(amp)
            for dr, dc in ((1, 0), (-1, 0), (0, 1), (0, -1)):
                if 0 <= c + dc < cols:
                    maps[t, (r + dr) % rows, c + dc] += np.float32(0.5 * amp)
    return maps


def offset_pair(n1, n2, kind="int8", delay=0, seed=5):
    """Seeded two-channel capture of one illuminator for the channel-offset estimator: s2[j] = s1[j + delay] (same
    source, ``delay`` samples apart; independent receiver noise on each channel), as ``int8`` raw samples, ``uint8``
    offset-binary samples or ``complex64`` IQ, of n1 and n2 samples."""
    rng = np.random.default_rng(seed)
    a = max(0, -delay)
    total = a + max(n1, delay + n2) + 1
    if kind == "complex64":
        u = white_iq(rng, total)
        s1 = u[a:a + n1] + np.complex64(0.1) * white_iq(rng, n1)
        s2 = u[a + delay:a + delay + n2] + np.complex64(0.1) * white_iq(rng, n2)
        return s1.astype(np.complex64), s2.astype(np.complex64)
    u = rng.integers(-96, 96, size=total)
    s1 = u[a:a + n1] + rng.integers(-16, 17, size=n1)
    s2 = u[a + delay:a + delay + n2] + rng.integers(-16, 17, size=n2)
    if kind == "int8":
        return s1.astype(np.int8), s2.astype(np.int8)
    if kind == "uint8":
        return (s1 + 128).astype(np.uint8), (s2 + 128).astype(np.uint8)
    raise ValueError(f"unknown offset-pair kind {kind!r}")
