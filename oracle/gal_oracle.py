"""Oracle for ``GAL_JPE`` (TEST INFRASTRUCTURE ONLY, see oracle/__init__.py).

``gal_jpe_oracle_c``  follows ``GAL_JPE``, reference ``passiveRadar/clutter_removal.py:251-364``, in plain C
                      (oracle/gal_oracle.c) with the reference's complex64 rounding points and its mu1 type changes.
``gal_jpe_truth_c``   the same recurrence with every operation in float64.
``gal_jpe_truth_stats`` ``gal_jpe_truth_c`` (the same C code, the same bits) plus how mu1's clamp at 5e-3 went.

The C helper is compiled with gcc into oracle/_build/libgal_oracle.so on first use (``build()``).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build")
SRC = os.path.join(HERE, "gal_oracle.c")
LIB = os.path.join(OUT, "libgal_oracle.so")


def build(force: bool = False) -> str:
    if not os.path.exists(SRC):
        raise FileNotFoundError(SRC)
    os.makedirs(OUT, exist_ok=True)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        tmp = LIB + f".tmp{os.getpid()}"
        subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-o", tmp, SRC, "-lm"], check=True)
        os.replace(tmp, LIB)
    return LIB


def _gal_c(symbol, cdtype, ref, srv, lattice_len, delay_line_len, mu1, mu2, peek, stats=None):
    fn = getattr(C.CDLL(build()), symbol)
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int,
                   C.c_void_p, C.c_void_p, C.c_void_p] + ([C.c_void_p] if stats is not None else [])
    ref = np.ascontiguousarray(ref, dtype=np.complex64)
    srv = np.ascontiguousarray(srv, dtype=np.complex64)
    if ref.shape != srv.shape:
        raise ValueError('Input vectors must have the same length')
    out = np.empty(srv.shape[0], dtype=cdtype)
    k = np.empty(delay_line_len, dtype=cdtype)
    h = np.empty(delay_line_len, dtype=cdtype)
    st = fn(ref.ctypes.data, srv.ctypes.data, srv.shape[0], int(lattice_len), int(delay_line_len), float(mu1),
            float(mu2), int(peek), out.ctypes.data, k.ctypes.data, h.ctypes.data,
            *([stats.ctypes.data] if stats is not None else []))
    if st == -2:
        raise ValueError("GAL_JPE oracle: need 1 <= latticeLen <= delayLineLen and peek >= 0")
    if st != 0:
        raise MemoryError(f"{symbol} failed")
    return out, k, h


def gal_jpe_oracle_c(ref, srv, lattice_len, delay_line_len, mu1, mu2, peek=10):
    """``GAL_JPE`` of the reference in plain C, complex64 arithmetic with the reference's rounding points and its
    mu1 type changes.  Returns (out, k, h) as complex64."""
    return _gal_c("gal_oracle_c64", np.complex64, ref, srv, lattice_len, delay_line_len, mu1, mu2, peek)


def gal_jpe_truth_c(ref, srv, lattice_len, delay_line_len, mu1, mu2, peek=10):
    """The recurrence of ``gal_jpe_oracle_c`` with every operation in float64: how far the complex64 reference is
    from the exact recurrence.  Returns (out, k, h) as complex128."""
    return _gal_c("gal_truth_c128", np.complex128, ref, srv, lattice_len, delay_line_len, mu1, mu2, peek)



def gal_jpe_truth_stats(ref, srv, lattice_len, delay_line_len, mu1, mu2, peek=10):
    """``gal_jpe_truth_c``'s recurrence (the same C code: out, k, h are the same bits) that also reports how mu1's
    clamp ``min(0.999 mu1 + 1e-8 e**2, 5e-3)`` went.  Returns (out, k, h, stats) with stats a dict:

    ``clamps``   number of samples at which the clamp won (mu1 became the Python float 5e-3),
    ``margin``   the smallest |xr - 5e-3| / 5e-3 over all decisions, xr the real part compared with 5e-3 (inf when
                 there was no decision: n <= peek + 1),
    ``xr_max``   the largest |xr| over all decisions,
    ``mu1``      mu1 after the last sample (complex; imaginary part 0 when the clamp won last)."""
    stats = np.zeros(5, np.float64)
    out, k, h = _gal_c("gal_truth_stats_c128", np.complex128, ref, srv, lattice_len, delay_line_len, mu1, mu2, peek,
                       stats)
    return out, k, h, {"clamps": int(stats[0]), "margin": float(stats[1]), "xr_max": float(stats[2]),
                       "mu1": complex(stats[3], stats[4])}


if __name__ == "__main__":
    print(build(force=True))
