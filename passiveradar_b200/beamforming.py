"""Beamscan of several surveillance channels' range-Doppler maps (prc_beamscan_frames, csrc/beamscan.cuh).

``FramePipeline(channels=K)`` gives K complex maps per CPI, one per surveillance antenna, laid out (K, T, F, R+1).
``beamscan_frames`` combines them against a steering table into one float32 amplitude map per frame, which the CFAR,
render and tracker chains take as they are, and a fractional grid index of the best beam per cell, which ``bearing``
turns into degrees::

    S = steering_vectors(ula_positions(3, 0.5), np.arange(0.0, 181.0))      # (181, 3)
    amp, pos = beamscan_frames(maps_d, S)                                     # (T, F, R+1) each
    deg = bearing(pos, np.arange(0.0, 181.0))

Convention: element k at (x_k, y_k) wavelengths, azimuth theta from the x axis, a_k(theta) = exp(+j 2 pi (x_k cos theta +
y_k sin theta)).  A line array along x is broadside at theta = 90 degrees, where every a_k is 1.  The CAF conjugates the
surveillance channel, so an echo from theta appears as m_k = conj(a_k(theta)) * c, and the table is used as given.  The
channels are assumed calibrated; a caller who knows per-channel complex gains g_k folds them into the table as
S[a, k] / conj(g_k).
"""
from __future__ import annotations

import numpy as np

from . import _lib

MAX_BEAM_FRAMES = 65535        # frames of one prc_beamscan_frames call
MAX_ANGLES = 4096
MAX_CHANNELS = 4


def ula_positions(K, spacing=0.5):
    """(K, 2) positions in wavelengths of a uniform line array along x: element k at (k * spacing, 0)."""
    return np.stack([np.arange(int(K)) * float(spacing), np.zeros(int(K))], axis=1)


def uca_positions(K, radius):
    """(K, 2) positions in wavelengths of a uniform circular array: element k at angle 2 pi k / K."""
    phi = 2.0 * np.pi * np.arange(int(K)) / int(K)
    return float(radius) * np.stack([np.cos(phi), np.sin(phi)], axis=1)


def steering_vectors(positions, angles_deg):
    """(A, K) complex64 table a_k(theta_a) = exp(+j 2 pi (x_k cos theta_a + y_k sin theta_a)); positions (K, 2) or (K,)
    (x only) in wavelengths, angles in degrees of azimuth.  Entries are unit-modulus and not normalised."""
    pos = np.asarray(positions, dtype=np.float64)
    if pos.ndim == 1:
        pos = np.stack([pos, np.zeros_like(pos)], axis=1)
    if pos.ndim != 2 or pos.shape[1] != 2:
        raise ValueError(f"positions must be (K, 2) or (K,), got shape {pos.shape}")
    th = np.deg2rad(np.asarray(angles_deg, dtype=np.float64).reshape(-1))
    phase = 2.0 * np.pi * (np.cos(th)[:, None] * pos[None, :, 0] + np.sin(th)[:, None] * pos[None, :, 1])
    return np.exp(1j * phase).astype(np.complex64)


def beamscan_frames(maps, steering, *, wrap=False, device=None):
    '''Beamscan of K channels' maps: for every cell the power of each steering row, P[a] = |sum_k S[a, k] m_k|^2, its
    first maximum a*, amp = sqrt(P[a*]) and pos = a* + the three-point parabolic offset (DESIGN.md section 21).

    Parameters:
        maps: (K, T, F, R+1) complex64, FramePipeline(channels=K)'s layout; 1 <= K <= 4
        steering: (A, K) complex table, row a the array response of grid angle a; 1 <= A <= 4096
        wrap: the grid is a full circle (neighbours of a* mod A)

    Returns:
        (amp, pos), each (T, F, R+1) float32.  A CUDA tensor gives CUDA tensors, ordered on the current torch stream; a
        host array gives host arrays.  One launch per 65 535 frames.'''
    import torch
    host = not _lib.is_cuda_tensor(maps)
    S = np.ascontiguousarray(np.asarray(steering), dtype=np.complex64)
    if host:
        a = np.asarray(maps)
        if a.dtype != np.complex64:
            raise TypeError(f"maps must be complex64, got {a.dtype}")
        shape = a.shape
    else:
        if maps.dtype != torch.complex64:
            raise TypeError(f"maps must be complex64, got {maps.dtype}")
        shape = tuple(maps.shape)
    if len(shape) != 4:
        raise ValueError(f"maps must be four-dimensional (K, T, F, R+1), got {len(shape)} dimensions")
    K, T, rows, cols = shape
    if not 1 <= K <= MAX_CHANNELS:
        raise ValueError(f"maps has K={K} channels; 1 <= K <= {MAX_CHANNELS}")
    if S.ndim != 2 or S.shape[1] != K:
        raise ValueError(f"steering must have shape (A, {K}), got {S.shape}")
    if not 1 <= S.shape[0] <= MAX_ANGLES:
        raise ValueError(f"steering has A={S.shape[0]} angles; 1 <= A <= {MAX_ANGLES}")
    if rows < 1 or cols < 1:
        raise ValueError(f"maps of {rows} x {cols} cells")
    if wrap not in (True, False, 0, 1):
        raise ValueError(f"wrap must be a bool, got {wrap!r}")
    if host:
        dev = _lib.current_device(device)
        t = torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", dev))
    else:
        t = maps
        dev = t.device.index if device is None else int(device)
        if t.stride(3) != 1 or t.stride(2) != cols or (T > 1 and t.stride(1) < rows * cols):
            t = t.contiguous()
    cells = rows * cols
    amp = torch.empty((T, rows, cols), dtype=torch.float32, device=t.device)
    pos = torch.empty((T, rows, cols), dtype=torch.float32, device=t.device)
    lib = _lib.load()
    stream = _lib.stream_arg(t.device)
    for t0 in range(0, T, MAX_BEAM_FRAMES):
        nb = min(MAX_BEAM_FRAMES, T - t0)
        _lib.check(lib.prc_beamscan_frames(t[0, t0].data_ptr(), rows, cols, nb, t.stride(1), K, t.stride(0),
                                           S.ctypes.data, S.shape[0], 1 if wrap else 0, amp[t0].data_ptr(),
                                           pos[t0].data_ptr(), cells, dev, stream, _lib.FLAG_ASYNC))
    if host:
        return amp.cpu().numpy(), pos.cpu().numpy()
    return amp, pos


def bearing(pos, angles_deg, *, wrap=False):
    """Degrees of fractional grid indices: linear interpolation between the grid angles.  With ``wrap`` the grid must be
    uniform with a step of 360 / A, and the result is taken mod 360.  ``pos`` is a NumPy array or a torch tensor (the
    result is the same kind, float64 for NumPy, ``pos``'s dtype for torch)."""
    ang = np.asarray(angles_deg, dtype=np.float64).reshape(-1)
    A = ang.size
    if A < 1:
        raise ValueError("angles_deg is empty")
    is_torch = type(pos).__module__.startswith("torch")
    if wrap:
        step = 360.0 / A
        if A > 1 and not np.allclose(np.diff(ang), step, rtol=0, atol=1e-9 * 360):
            raise ValueError(f"with wrap the grid must be uniform with a step of 360 / A = {step:g} degrees")
        out = ang[0] + pos * step
        return out % 360.0
    if A == 1:
        return pos * 0.0 + ang[0]
    if is_torch:
        import torch
        g = torch.as_tensor(ang, dtype=pos.dtype, device=pos.device)
        i = torch.clamp(torch.floor(pos), 0, A - 2).long()
        return g[i] + (pos - i.to(pos.dtype)) * (g[i + 1] - g[i])
    return np.interp(np.asarray(pos, dtype=np.float64), np.arange(A, dtype=np.float64), ang)
