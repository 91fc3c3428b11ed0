"""Oracle for the SVD least-squares clutter filter (TEST INFRASTRUCTURE ONLY, see oracle/__init__.py).

``ls_filter_svd_oracle``     follows ``LS_Filter_SVD``, reference ``passiveRadar/clutter_removal.py:58-107``: the
                             complex64 data matrix of circularly delayed reference copies (:83-88), NumPy's thin SVD
                             in single precision (:91), reciprocals of the singular values with those below 1e-10
                             zeroed (:94-96), taps = V diag(1/S) U^H srv (:99), srv - A taps (:102).
``ls_filter_svd_truth``      the same least-squares problem in complex128 with the project's truncation rule (singular
                             values below max(1e-10, 1e-5 S_max) dropped, DESIGN.md section 13), on the explicit
                             data matrix; n <= 65536.
``ls_filter_svd_truth_gram`` the same solution from a float64 eigendecomposition of the circulant Gram matrix A^H A
                             (eigenvalues below max(1e-20, 1e-10 lambda_max) dropped), for any n.
The truths return (out, taps, rank) in complex128.
"""
from __future__ import annotations

import numpy as np

S_ABS = 1e-10
S_REL = 1e-5
TRUTH_MAX_N = 65536


def _delayed_copies(ref, ntaps, peek, dtype):
    """n x ntaps matrix whose column k is ``ref`` delayed circularly by k - peek samples."""
    n = ref.shape[0]
    rows = np.arange(n)[:, None]
    shifts = np.arange(ntaps)[None, :] - peek
    return np.asarray(ref)[(rows - shifts) % n].astype(dtype) if n else np.zeros((0, ntaps), dtype)


def ls_filter_svd_oracle(refChannel, srvChannel, filterLen, peek=10, return_filter=False):
    refChannel = np.asarray(refChannel)
    srvChannel = np.asarray(srvChannel)
    if refChannel.shape != srvChannel.shape:
        raise ValueError('Input vectors must have the same length')
    ntaps = filterLen + peek
    data = _delayed_copies(refChannel, ntaps, peek, np.complex64)
    u, sv, vh = np.linalg.svd(data, full_matrices=False)
    with np.errstate(divide="ignore"):
        inv = 1 / sv
    inv[sv < 1e-10] = 0.0
    pinv = (vh.conj().T * inv) @ u.conj().T                # the pseudo-inverse first, as the reference associates
    taps = pinv @ srvChannel
    cleaned = srvChannel - data @ taps
    return (cleaned, taps) if return_filter else cleaned


def ls_filter_svd_truth(ref, srv, filter_len, peek=10):
    ref = np.asarray(ref, dtype=np.complex128)
    srv = np.asarray(srv, dtype=np.complex128)
    if ref.shape[0] > TRUTH_MAX_N:
        raise ValueError(f"the explicit data matrix is limited to n <= {TRUTH_MAX_N}; use ls_filter_svd_truth_gram")
    data = _delayed_copies(ref, filter_len + peek, peek, np.complex128)
    u, sv, vh = np.linalg.svd(data, full_matrices=False)
    keep = sv >= max(S_ABS, S_REL * (sv.max() if sv.size else 0.0))
    taps = vh[keep].conj().T @ ((u[:, keep].conj().T @ srv) / sv[keep])
    return srv - data @ taps, taps, int(keep.sum())


def ls_filter_svd_truth_gram(ref, srv, filter_len, peek=10):
    ref = np.asarray(ref, dtype=np.complex128)
    srv = np.asarray(srv, dtype=np.complex128)
    n = ref.shape[0]
    m = filter_len + peek
    fr = np.fft.fft(ref)
    c = np.fft.ifft(np.conj(fr) * fr)                       # c[k] = sum_i conj(ref[i]) ref[(i + k) mod n]
    x = np.fft.ifft(np.conj(fr) * np.fft.fft(srv))          # x[k] = sum_i conj(ref[i]) srv[(i + k) mod n]
    lag = np.arange(m)[:, None] - np.arange(m)[None, :]     # Gram[a, b] = c[(a - b) mod n]
    gram = c[lag % n]
    gram = 0.5 * (gram + gram.conj().T)
    rhs = x[(np.arange(m) - peek) % n]
    lam, vec = np.linalg.eigh(gram)
    keep = lam >= max(S_ABS ** 2, S_REL ** 2 * lam.max())
    taps = vec[:, keep] @ ((vec[:, keep].conj().T @ rhs) / lam[keep])
    h = np.zeros(n, dtype=np.complex128)
    np.add.at(h, (np.arange(m) - peek) % n, taps)           # clutter[i] = sum_k taps[k] ref[(i - (k - peek)) mod n]
    return srv - np.fft.ifft(fr * np.fft.fft(h)), taps, int(keep.sum())
