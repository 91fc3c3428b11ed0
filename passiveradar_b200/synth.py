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


def recording(n, fs, fo, up, dn, *, delay, fd, channel_delay=0, multipath=0.3, clutter=True, kind="int8", seed=23):
    """Seeded two-channel raw recording of one FM-like illuminator for the recording chain (main.py:44-194): ``(ref,
    srv)`` interleaved I/Q of ``n`` complex samples each at the input rate ``fs``.

    The illuminator is complex noise low-passed to 0.4 of the IF rate ``fs * up / dn`` and sits at ``-fo``, where
    ``frequency_shift(x, fo, fs)`` brings it to 0 Hz.  ``srv`` holds the direct path (gain 1), one zero-Doppler multipath
    echo of gain ``multipath`` ``up / gcd(up, dn)`` IF samples late and one target ``delay`` IF samples late with Doppler ``fd`` Hz
    (gain 0.05), plus independent receiver noise on each channel.  Delays are whole input samples, so ``delay`` must be a multiple of ``up / gcd(up, dn)``.  ``srv`` lags ``ref`` by ``channel_delay`` input
    samples (``ref[j]`` and ``srv[j + channel_delay]`` see the same instant; find_channel_offset on the raw arrays gives
    ``-2 * channel_delay``).  ``clutter=False`` leaves the direct path and the multipath out of ``srv``.  ``kind`` is
    ``int8`` or ``int16``."""
    from scipy.signal import fftconvolve, firwin
    g = np.gcd(up, dn)
    up, dn = up // g, dn // g
    if delay % up:
        raise ValueError(f"delay must be a multiple of {up} IF samples")
    d_in, m_in = delay // up * dn, dn
    rng = np.random.default_rng(seed)
    lead = d_in + m_in + abs(channel_delay) + 1
    total = n + lead + abs(channel_delay)
    h = firwin(257, 0.4 * up / dn)
    u = fftconvolve(white_iq(rng, total + 256).astype(np.complex128), h, mode="valid")[:total]
    u *= np.exp(-2j * np.pi * (fo / fs) * np.arange(total))
    t = np.arange(total)
    echo = np.zeros(total, np.complex128)
    echo[m_in:] += multipath * u[:total - m_in]
    tgt = np.zeros(total, np.complex128)
    tgt[d_in:] = 0.05 * u[:total - d_in]
    scene = (u + echo if clutter else 0) + tgt * np.exp(2j * np.pi * (fd / fs) * t)
    r0 = lead
    s0 = lead - channel_delay
    ref = u[r0:r0 + n] + 0.02 * white_iq(rng, n)
    srv = scene[s0:s0 + n] + 0.02 * white_iq(rng, n)
    scale, top = (24.0, 127) if kind == "int8" else (2000.0, 32767)
    dt = {"int8": np.int8, "int16": np.int16}[kind]

    def raw(x):
        x = x / np.sqrt(np.mean(np.abs(u) ** 2)) * scale
        iq = np.empty(2 * n)
        iq[0::2], iq[1::2] = x.real, x.imag
        return np.clip(np.round(iq), -top, top).astype(dt)

    return raw(ref), raw(srv)


# main.py geometries for the recording chain: what the reference's getConfiguration derives from PRconfig.yaml
# ("shipped"), and from it with channel_bandwidth 50 kHz, cpi_seconds_nominal 1, max_doppler_nominal 64 and
# max_range_nominal 300 ("fast")
RECORDING_CONFIGS = {
    "shipped": {'cpi_samples': 524288, 'resamp_up': 13, 'resamp_dn': 119, 'input_sample_rate': 2400000,
                'offset_freq': 100000, 'IF_sample_rate': 262184.87394957984, 'input_chunk_length': 4799250,
                'window_overlap': 131072, 'num_range_cells': 175, 'num_doppler_cells': 1024, 'num_frames': 1200,
                'overlap_cpi': True, 'interleaved_input_channels': False, 'frame_interval': 0.9998441025641025,
                'range_cell_width': 1.1434679487179487, 'doppler_cell_width': 0.5000779608718487},
    "fast": {'cpi_samples': 65536, 'resamp_up': 8, 'resamp_dn': 293, 'input_sample_rate': 2400000,
             'offset_freq': 100000, 'IF_sample_rate': 65529.01023890785, 'input_chunk_length': 2400256,
             'window_overlap': 16384, 'num_range_cells': 66, 'num_doppler_cells': 128, 'num_frames': 1200,
             'overlap_cpi': True, 'interleaved_input_channels': False, 'frame_interval': 0.5000533333333333,
             'range_cell_width': 4.575072916666667, 'doppler_cell_width': 0.9998933447098975},
}


def recording_for(config, nchunks, channel_delay=0, clutter=True, seed=1):
    """``recording`` sized so that main.py makes exactly ``nchunks`` chunks of ``config`` from it (no channel offset),
    with the target 3 * resamp_up IF samples late at 40 Doppler cells.  Returns (ref, srv, delay, doppler_cells)."""
    icl = config["input_chunk_length"]
    up, dn = config["resamp_up"], config["resamp_dn"]
    n = nchunks * icl // 2 + 40 + abs(channel_delay)
    fd = 40 * config["doppler_cell_width"]
    ref, srv = recording(n, config["input_sample_rate"], config["offset_freq"], up, dn, delay=3 * up, fd=fd,
                         channel_delay=channel_delay, clutter=clutter, seed=seed)
    return ref, srv, 3 * up, 40


def interleave_channels(ref, srv):
    """One raw source of two channels' interleaved IQ (``ref``, ``srv`` as ``recording`` returns them): complex
    samples alternate between the channels, ``[ref_I[0], ref_Q[0], srv_I[0], srv_Q[0], ref_I[1], ...]``, the layout
    PRconfig.yaml's ``interleaved_input_channels: True`` describes."""
    out = np.empty(ref.shape[0] + srv.shape[0], dtype=ref.dtype)
    out.reshape(-1, 4)[:, 0:2] = ref.reshape(-1, 2)
    out.reshape(-1, 4)[:, 2:4] = srv.reshape(-1, 2)
    return out
