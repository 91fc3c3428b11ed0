"""NumPy restatement of the reference's trackers (passiveRadar/target_detection.py:164-681) -- test infrastructure.

Written from the arithmetic DESIGN.md section 11 lists, with the documented tie rule for equal candidate strengths:
strength descending, then descending position in the transformed frame (np.flip(np.argsort(s, kind="stable"))).
Kalman products go through NumPy's matmul and np.linalg.inv, as in the reference.  ``pairwise_mean_twin`` is the host
twin of the measurement kernel's mean (csrc/track.cuh: the summation tree of prcore.cu's trk_plan).
"""
from __future__ import annotations

import numpy as np

from passiveradar_b200.target_detection import target_track_dtype, target_track_dtype_simple


# ------------------------------------------------------------------------------------------ mean|x|
def pairwise_plan(n):
    """NumPy's pairwise-summation tree of n elements, breadth-first: list of [off, len, left] and level starts."""
    nodes = [[0, n, -1]]
    level = [0]
    lo = 0
    while True:
        hi = len(nodes)
        for q in range(lo, hi):
            off, ln, _ = nodes[q]
            if ln <= 128:
                continue
            n2 = ln // 2 - (ln // 2) % 8
            nodes[q][2] = len(nodes)
            nodes.append([off, n2, -1])
            nodes.append([off + n2, ln - n2, -1])
        if len(nodes) == hi:
            break
        level.append(hi)
        lo = hi
    level.append(len(nodes))
    return nodes, level


def _leaf(a):
    a = [float(v) for v in a]
    if len(a) < 8:
        r = 0.0
        for v in a:
            r += v
        return r
    r = a[:8]
    i = 8
    while i < len(a) - len(a) % 8:
        for j in range(8):
            r[j] += a[i + j]
        i += 8
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for v in a[i:]:
        res += v
    return res


def pairwise_mean_twin(x):
    """mean|x| of a flattened float64 array evaluated the way track_meas_kernel does: leaves, then the inner nodes
    level by level from the deepest."""
    a = np.abs(np.asarray(x, dtype=np.float64).ravel())
    nodes, level = pairwise_plan(a.size)
    val = [0.0] * len(nodes)
    for q, (off, ln, left) in enumerate(nodes):
        if left < 0:
            val[q] = _leaf(a[off:off + ln])
    for lv in range(len(level) - 3, -1, -1):
        for q in range(level[lv], level[lv + 1]):
            if nodes[q][2] >= 0:
                val[q] = val[nodes[q][2]] + val[nodes[q][2] + 1]
    return val[0] / a.size


# ------------------------------------------------------------------------------------------ measurements
def _frame(data_frame):
    """The normalised frame in the reference's orientation: rows = range (row 0 <-> range_extent), columns = the
    flipped Doppler axis."""
    x = np.asarray(data_frame, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        y = x / np.mean(np.abs(x).ravel())
    return np.ascontiguousarray(y.T[:, ::-1])


def get_measurements(data_frame, p, frame_extent):
    """(3, M): range, Doppler, strength of the cells at or above the 99.8th percentile, strongest first."""
    rext, dext = float(frame_extent[1]), float(frame_extent[0])
    rows, cols = np.shape(data_frame)
    rpts = np.linspace(rext, 0, cols)
    dpts = np.linspace(-1 * dext, dext, rows)
    y = _frame(data_frame)
    y[:8, :] = 0
    y[-8:, :] = 0
    c = rows // 2
    y[:, c - 4:c + 4] = 0
    thr = np.percentile(y, 99.8)
    ri, di = np.nonzero(y >= thr)
    s = y[ri, di]
    order = np.flip(np.argsort(s, kind="stable"))
    return np.stack((rpts[ri][order], dpts[di][order], s[order]))


# ------------------------------------------------------------------------------------------ multi-target tracker
_F1 = np.array([[1, 0, -0.003, 0], [0, 0, -0.003, -0.003], [0, 0, 1, 1], [0, 0, 0, 1]], dtype=np.float64)
_F2 = np.array([[1, 1, 0, 0], [0, 1, 0, 0], [0, 0, 1, 1], [0, 0, 0, 1]], dtype=np.float64)
_H = np.array([[1, 0, 0, 0], [0, 0, 1, 0]], dtype=np.float64)


def new_track(meas):
    """A free track at (0, 0) without a measurement, a preliminary one at it with one."""
    t = np.zeros((), dtype=target_track_dtype)
    r, d = (0.0, 0.0) if meas is None else (float(meas[0]), float(meas[1]))
    t["status"] = 0 if meas is None else 1
    t["lifetime"] = 1
    t["measurement"] = (r, d)
    t["estimate"] = (r, d)
    t["measurement_history"][[0, 5, 6, 7, 8, 9]] = 1
    k = t["kalman_state"]
    k["x"] = (r, 0.0, d, -1.0)
    k["P"] = np.diag([5.0, 0.0225, 0.04, 0.1])
    k["F1"] = _F1
    k["F2"] = _F2
    k["Q"] = np.diag([4.0, 0.03, 0.2, 0.08])
    k["H"] = _H
    k["R"] = np.diag([5.0, 2.0])
    k["S"] = np.eye(2)
    return t


def kalman_step(k, z=None, z_last=None):
    """Predict (and, with a measurement z, correct with R scaled by |z - z_last|^2).  Returns (estimate, state)."""
    out = k.copy()
    x = k["F1"] @ k["x"]
    P = k["F2"] @ k["P"] @ k["F2"].T + k["Q"]
    H = k["H"]
    if z is None:
        S = H @ P @ H.T + k["R"]
    else:
        dz = np.asarray(z) - np.asarray(z_last)
        S = H @ P @ H.T + k["R"] * (dz[0] ** 2 + dz[1] ** 2)
        K = P @ H.T @ np.linalg.inv(S)
        x = x + K @ (np.asarray(z) - H @ x)
        P = (np.eye(4) - K @ H) @ P
    out["x"], out["P"], out["S"] = x, P, S
    return H @ x, out


def associate(track, cand):
    """The measurement this track takes from the candidate list (or None) and the list that remains."""
    st = int(track["status"])
    r, d, s = cand
    if st == 0:
        gate = np.ones(r.shape, bool)
    elif st == 1:
        gate = (np.abs(r - track["measurement"][0]) < 5) & (np.abs(d - track["measurement"][1]) < 24)
    else:
        gate = (np.abs(r - track["estimate"][0]) < 4) & (np.abs(d - track["estimate"][1]) < 20)
    idx = np.flatnonzero(gate)
    if st == 2:
        inv_s = np.linalg.inv(track["kalman_state"]["S"])
        ok = []
        for q in idx:
            z = np.array([track["measurement"][0] - r[q], track["measurement"][1] - d[q]])
            ok.append(z.T @ inv_s @ z < 6)
        idx = idx[np.array(ok, dtype=bool)] if len(idx) else idx
    if idx.size == 0:
        return None, cand
    if idx.size == 1:
        pick = idx[0]
    elif st == 0:
        pick = 0
        gate = (np.abs(r - r[0]) < 10) & (np.abs(d - d[0]) < 12)
    elif st == 1:
        pick = idx[np.argmin(np.sqrt(r[idx] ** 2 + d[idx] ** 2))]
    else:
        pick = idx[0]
    return np.array([r[pick], d[pick]]), cand[:, ~gate]


def update(track, meas):
    out = track.copy()
    st, life = int(track["status"]), int(track["lifetime"])
    hist = track["measurement_history"].copy()
    if meas is None:
        est, k = kalman_step(track["kalman_state"])
        new_meas = track["measurement"].copy()
    else:
        est, k = kalman_step(track["kalman_state"], meas, track["measurement"])
        new_meas = meas
    if st == 1:
        if life > 4 and hist[:10].sum() < 6:
            st = 0
        if life > 4 and hist[:10].sum() > 8:
            st = 2
    elif st == 2 and life > 4 and hist.sum() < 4:
        st = 0
    out["status"], out["lifetime"] = st, life + 1
    out["measurement"], out["estimate"] = new_meas, est
    out["measurement_history"] = np.concatenate(([0.0 if meas is None else 1.0], hist[:-1]))
    out["kalman_state"] = k
    return out


def multitarget_tracker(data, frame_extent, N_TRACKS):
    """(Nframes, N_TRACKS) target_track_dtype history; data has frames on its last axis."""
    data = np.asarray(data)
    T = data.shape[2]
    tracks = np.array([new_track(None) for _ in range(N_TRACKS)], dtype=target_track_dtype)
    hist = np.zeros((T, N_TRACKS), dtype=target_track_dtype)
    for i in range(T):
        cand = get_measurements(data[:, :, i], 99.8, frame_extent)
        st = tracks["status"].copy()
        for t in list(np.flatnonzero(st == 2)) + list(np.flatnonzero(st == 1)):
            m, cand = associate(tracks[t], cand)
            tracks[t] = update(tracks[t], m)
        for t in np.flatnonzero(st == 0):
            if cand.shape[1] == 0:
                break
            m, cand = associate(tracks[t], cand)
            tracks[t] = new_track(m)
        hist[i] = tracks
    return hist


# ------------------------------------------------------------------------------------------ simple tracker
def _py_slice(start, stop, n):
    return slice(start, stop).indices(n)[:2]


def simple_target_tracker(data, rangeExtent, dopplerExtent):
    data = np.asarray(data)
    T = data.shape[2]
    s = np.zeros((), dtype=target_track_dtype_simple)
    s["lock_mode"] = (1, 0, 0, 0)
    s["measurement"] = (30.0, -20.0)          # H x: the reference fills its fields positionally, out of order
    s["measurement_idx"] = (35, -30)
    s["estimate"] = (50.0, 50.0)
    s["range_extent"], s["doppler_extent"] = rangeExtent, dopplerExtent
    k = s["kalman_state"]
    k["x"] = (30.0, 2.0, -20.0, -1.0)
    k["P"] = np.diag([5.0, 0.0225, 0.04, 0.1])
    k["F1"] = np.array([[1, 0, -0.003, 0], [0, 0, -0.003, -0.03], [0, 0, 1, 1], [0, 0, 0, 1]])
    k["F2"] = _F2
    k["Q"] = np.diag([2.0, 0.02, 0.2, 0.05])
    k["H"] = _H
    k["R"] = np.diag([5.0, 5.0])
    k["S"] = np.eye(2)
    found_m = np.array([[0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 1, 0], [0, 0, 1, 0]]).T
    lost_m = np.array([[1, 0, 0, 0], [1, 0, 0, 0], [0, 0, 0, 1], [1, 0, 0, 0]]).T
    hist = np.zeros((T,), dtype=target_track_dtype_simple)
    for i in range(T):
        y = _frame(data[:, :, i])
        y[:8, :] = 0
        y[-8:, :] = 0
        y[:, 250:260] = 0
        lm = s["lock_mode"]
        ly, lx = int(s["measurement_idx"][0]), int(s["measurement_idx"][1])
        half = (24, 48) if (lm[1] == 1 or (lm[2] != 1 and lm[3] == 1)) else (16, 32)
        if lm[1] == 1 or lm[2] == 1 or lm[3] == 1:
            gate = np.zeros(y.shape)
            y0, y1 = _py_slice(ly - half[0], ly + half[0], y.shape[0])
            x0, x1 = _py_slice(lx - half[1], lx + half[1], y.shape[1])
            gate[y0:max(y0, y1), x0:max(x0, x1)] = 1.0
            y = y * gate
        i0, i1 = np.unravel_index(np.argmax(y), y.shape)
        meas = np.array([rangeExtent * (1 - i0 / y.shape[0]), dopplerExtent * (2 * i1 / y.shape[1] - 1)])
        surprise = meas - s["estimate"]
        found = (surprise[0] ** 2 + (0.5 * surprise[1]) ** 2) ** 0.5 < 12
        new = s.copy()
        new["lock_mode"] = (found_m if found else lost_m) @ lm
        est, new["kalman_state"] = kalman_step(s["kalman_state"], meas, s["measurement"])
        new["measurement"], new["measurement_idx"], new["estimate"] = meas, (i0, i1), est
        s = new
        hist[i] = s
    return hist
