"""Float64 NumPy statement of the ordered-statistic CFAR (Rohling) on CFAR_2D's window (test infrastructure for
``passiveradar_b200.target_detection.OS_CFAR_2D``; never imported by the package).

The window is built from the reference's ``Tfilt`` exactly as ``cfar_2d_oracle`` builds it, and its cells are read
through explicit modular index arrays, so a map smaller than the window wraps as ``convolve2d(boundary='wrap')`` does:

    cell (i, j) reads X[(i + c - a) mod rows, (j + c - b) mod cols] for every non-zero Tfilt[a, b], c = (fw - 1) // 2
    T  = the k-th smallest of those N values (np.partition)
    CR = (X * inv_mean) / (T + 1e-10),  inv_mean = rows*cols / sum|X|
"""
import numpy as np

CELLS_PER_CHUNK = 1 << 24          # window values gathered at once (128 MB of float64)


def tfilt(fw, gw):
    """CFAR_2D's kernel support: ones((fw, fw)) with the guard hole [e1:e2, e1:e2] zeroed, NumPy slice rules."""
    T = np.ones((fw, fw))
    e1 = (fw - gw) // 2
    e2 = fw - e1 + 1
    T[e1:e2, e1:e2] = 0
    return T


def window_cells(fw, gw):
    """N, the number of cells of the window."""
    return int(tfilt(fw, gw).sum())


def default_rank(n):
    """ceil(3N / 4)."""
    return -(-3 * n // 4)


def os_window(X, fw, gw, r0=0, r1=None):
    """The window values of rows r0 .. r1 - 1 of X: a (r1 - r0, cols, N) float64 array."""
    X = np.asarray(X, dtype=np.float64)
    rows, cols = X.shape
    r1 = rows if r1 is None else r1
    A, B = np.nonzero(tfilt(fw, gw))
    c = (fw - 1) // 2
    I = (np.arange(r0, r1)[:, None, None] + c - A[None, None, :]) % rows
    J = (np.arange(cols)[None, :, None] + c - B[None, None, :]) % cols
    return X[I, J]


def os_statistic(X, fw, gw, k=None):
    """T: the k-th smallest window value of every cell (k = ceil(3N / 4) by default)."""
    X = np.asarray(X, dtype=np.float64)
    rows, cols = X.shape
    n = window_cells(fw, gw)
    k = default_rank(n) if k is None else int(k)
    if not 1 <= k <= n:
        raise ValueError(f"k={k} outside [1, N = {n}]")
    T = np.empty((rows, cols))
    step = max(1, CELLS_PER_CHUNK // max(1, cols * n))
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        T[r0:r1] = np.partition(os_window(X, fw, gw, r0, r1), k - 1, axis=2)[:, :, k - 1]
    return T


def os_cfar_2d_oracle(X, fw, gw, k=None, thresh=None):
    """CR of the ordered-statistic CFAR; ``CR > thresh`` when thresh is given.  A complex X is used as np.abs(X)."""
    X = np.asarray(X)
    if np.iscomplexobj(X):
        X = np.abs(X)
    X = X.astype(np.float64)
    inv_mean = X.size / np.abs(X).sum()
    CR = (X * inv_mean) / (os_statistic(X, fw, gw, k) + 1e-10)
    return CR if thresh is None else CR > thresh
