"""NumPy statement of the frame chain of the reference's range_doppler_plot.py:45-85 (no dask, no matplotlib): test
infrastructure for passiveradar_b200.plotting_tools, never imported by the package.

    CF[:, :, i] = CFAR_2D(|xambg[:, :, i]|, fw, gw)                      (float64 stack)
    data = fliplr(persistence(CF, kk, hold, decay).T)
    vmin, vmax = percentile(data, 35), 1.5 * percentile(data, 99)

``persistence`` is restated from its documented arithmetic (passiveRadar/plotting_tools.py:9-30): a float64 frame of
zeros to which X[:, :, k - i] * decay**i is added for i = 0 .. min(k + 1, hold) - 1, in that order, each product in
the precision NumPy's promotion gives it.
"""
import numpy as np

from .frontend_oracle import cfar_2d_oracle


def persistence_oracle(X, k, hold, decay):
    frame = np.zeros((X.shape[0], X.shape[1]))
    for i in range(min(k + 1, hold)):
        if k - i >= 0:
            frame = frame + X[:, :, k - i] * decay ** i
    return frame


def cfar_stack_oracle(xambg, fw=18, gw=4):
    """CF of range_doppler_plot.py:72-75 for an (F, R+1, nframes) stack (complex or magnitudes)."""
    mag = np.abs(xambg)
    CF = np.zeros(mag.shape)
    for i in range(mag.shape[2]):
        CF[:, :, i] = cfar_2d_oracle(mag[:, :, i], fw, gw)
    return CF


def render_frame_oracle(CF, kk, hold=20, decay=0.90):
    """(data, vmin, vmax) of frame kk (range_doppler_plot.py:79-96)."""
    data = np.fliplr(persistence_oracle(CF, kk, hold, decay).T)
    vmn = np.percentile(data.flatten(), 35)
    vmx = 1.5 * np.percentile(data.flatten(), 99)
    return data, vmn, vmx


def render_oracle(xambg, fw=18, gw=4, hold=20, decay=0.90):
    """Every frame: data (nframes, R+1, F) and limits (nframes, 2)."""
    CF = cfar_stack_oracle(xambg, fw, gw)
    n = CF.shape[2]
    data = np.empty((n, CF.shape[1], CF.shape[0]))
    limits = np.empty((n, 2))
    for kk in range(n):
        data[kk], limits[kk, 0], limits[kk, 1] = render_frame_oracle(CF, kk, hold, decay)
    return data, limits
