"""Target detection on the H100 -- ``CFAR_2D`` with the reference's call signature
(``passiveRadar/target_detection.py:683-703``).  No CPU fallback."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib


def CFAR_2D(X, fw, gw, thresh=None, *, device=None):
    '''constant false alarm rate target detection

    Parameters:
        fw: CFAR kernel width
        gw: number of guard cells
        thresh: detection threshold

    Returns:
        X with CFAR filter applied (float64 like the reference; bool array when ``thresh`` is given)'''
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError("X must be two-dimensional")
    if np.iscomplexobj(X):
        raise TypeError("CFAR_2D expects a real map (the reference is called with np.abs(xambg))")
    x = np.ascontiguousarray(X, dtype=np.float32)
    rows, cols = x.shape
    lib = _lib.load()
    dev = _lib.current_device() if device is None else int(device)
    if thresh is None:
        cr = np.empty((rows, cols), dtype=np.float32)
        _lib.check(lib.prc_cfar2d_f32(x.ctypes.data, rows, cols, int(fw), int(gw), None, cr.ctypes.data, None,
                                      _lib.MEM_HOST, dev, None, 0))
        return cr.astype(np.float64)
    t = C.c_float(float(thresh))
    det = np.empty((rows, cols), dtype=np.uint8)
    _lib.check(lib.prc_cfar2d_f32(x.ctypes.data, rows, cols, int(fw), int(gw), C.addressof(t), None, det.ctypes.data,
                                  _lib.MEM_HOST, dev, None, 0))
    return det.astype(bool)
