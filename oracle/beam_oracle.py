"""float64 oracle of the beamscan (prc_beamscan_frames, csrc/beamscan.cuh, DESIGN.md section 21).

For K co-registered complex maps m_k and a steering table S (A x K), per cell:

    P[a]  = | sum_k S[a, k] m_k |^2
    a*    = the first a with the largest P[a]
    amp   = sqrt(P[a*])
    den   = P[a*-1] - 2 P[a*] + P[a*+1]
    delta = clip(0.5 (P[a*-1] - P[a*+1]) / den, -0.5, 0.5) if den < 0 else 0
    pos   = a* + delta

With wrap the neighbours are taken mod A (a pos that lands on A - 0.5 is folded to -0.5); without it delta = 0 at
a* = 0 and a* = A - 1.  Test infrastructure only: the package never imports it.
"""
import numpy as np


def beam_powers(maps, steering):
    """P (A, ...) in float64 of maps (K, ...) against steering (A, K)."""
    m = np.asarray(maps).astype(np.complex128)
    S = np.asarray(steering).astype(np.complex128)
    return np.abs(np.tensordot(S, m, axes=([1], [0]))) ** 2


def peak_from_powers(P, wrap=False):
    """(amp, pos, a*, den) of powers P (A, ...) by the rules above, with broadcasting over the trailing axes."""
    P = np.asarray(P, dtype=np.float64)
    A = P.shape[0]
    a = np.argmax(P, axis=0)                       # the first maximum
    best = np.take_along_axis(P, a[None], 0)[0]
    lo, hi = a - 1, a + 1
    if wrap:
        lo, hi = lo % A, hi % A
        edge = np.zeros(a.shape, bool)
    else:
        edge = (a == 0) | (a == A - 1)
        lo, hi = np.clip(lo, 0, A - 1), np.clip(hi, 0, A - 1)
    left = np.take_along_axis(P, lo[None], 0)[0]
    right = np.take_along_axis(P, hi[None], 0)[0]
    den = left - 2.0 * best + right
    ok = ~edge & (den < 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        delta = np.where(ok, np.clip(0.5 * (left - right) / np.where(ok, den, -1.0), -0.5, 0.5), 0.0)
    pos = a + delta
    if wrap:
        pos = np.where(pos >= A - 0.5, pos - A, pos)
    return np.sqrt(best), pos, a, np.where(edge, 0.0, den)


def beamscan_oracle(maps, steering, wrap=False):
    """(amp, pos, a*, den, P) of maps (K, ...) against steering (A, K)."""
    P = beam_powers(maps, steering)
    amp, pos, a, den = peak_from_powers(P, wrap)
    return amp, pos, a, den, P


def delta_of_sequence(p, wrap=False):
    """(a*, delta) of one power sequence p[0 .. A-1], written out with explicit indices."""
    p = [float(v) for v in p]
    A = len(p)
    a = 0
    for i in range(1, A):
        if p[i] > p[a]:
            a = i
    if not wrap and (a == 0 or a == A - 1):
        return a, 0.0
    left, right = p[(a - 1) % A], p[(a + 1) % A]
    den = left - 2.0 * p[a] + right
    if not den < 0:
        return a, 0.0
    return a, min(0.5, max(-0.5, 0.5 * (left - right) / den))
