"""numpy model of the FFT-domain kernels (fftcorr.cuh): pins the algebra (block partition, aliasing margins, shifts,
conjugation conventions) against direct float64 sums before the CUDA transliteration is trusted.  Run: python scripts/fft/model.py"""
import numpy as np

rng = np.random.default_rng(7)


def direct_lags(x, s, lags, n, linear=False):
    """C[l] = sum_i x[i] conj(s[i + l]) (circular mod n, or zero outside [0, n) when linear)"""
    out = np.zeros(len(lags), complex)
    for q, l in enumerate(lags):
        if linear:
            sh = np.zeros(n, complex)
            if l >= 0:
                sh[:n - l] = s[l:]
            else:
                sh[-l:] = s[:n + l]
        else:
            sh = np.roll(s, -l)
        out[q] = np.sum(x * np.conj(sh))
    return out


def model_lscorr(ref, srv, M, peek, L, linear=False):
    """segments of Bs <= L - M + 1 samples; X = zero-padded reference segment, Yr / Ys = the L reference / surveillance
    samples that start with it (surveillance shifted by -peek); sum over segments of X conj(Y) is the spectrum of the lag sums"""
    n = len(ref)
    bmax = L - M + 1
    nseg = -(-n // bmax)
    Bs = -(-n // nseg)
    nseg = -(-n // Bs)

    def take(sig, base, ln):
        idx = base + np.arange(L)
        if linear:
            v = np.where((idx >= 0) & (idx < n), sig[np.clip(idx, 0, n - 1)], 0)
        else:
            v = sig[idx % n]
        v = v.astype(complex)
        v[ln:] = 0
        return np.fft.fft(v)

    accC = np.zeros(L, complex)
    accX = np.zeros(L, complex)
    for q in range(nseg):
        i0 = q * Bs
        ln = min(Bs, n - i0)
        X = take(ref, i0, ln)
        accC += X * np.conj(take(ref, i0, L))
        accX += X * np.conj(take(srv, i0 - peek, L))
    return np.fft.fft(accC)[:M] / L, np.fft.fft(accX)[:M] / L


def taps_spectrum(w, L):
    M = len(w)
    h = np.zeros(L, complex)
    h[(np.arange(M) - (M - 1)) % L] = w
    return np.fft.fft(h)


def model_fir(ref, srv, w, peek, L, linear=False):
    n, M = len(ref), len(w)
    Wp = taps_spectrum(w, L)
    Bf = L - M + 1
    out = np.zeros(n, complex)
    for p0 in range(0, n, Bf):
        idx = p0 + peek - (M - 1) + np.arange(L)
        r = np.where((idx >= 0) & (idx < n), ref[np.clip(idx, 0, n - 1)], 0) if linear else ref[idx % n]
        Y = np.fft.fft(r) * Wp
        yc = np.fft.fft(np.conj(Y))          # = L conj(y)
        y = np.conj(yc) / L
        m = min(Bf, n - p0)
        out[p0:p0 + m] = srv[p0:p0 + m] - y[:m]
    return out


def model_caf(ref, srv, win, R, F, L, w=None, peek=0):
    """block sums P[j, d], d = 0..R, optionally with the clutter FIR fused in the frequency domain"""
    n = len(ref)
    D = n // F
    ntaps = D + 1 if D > 1 else 1
    half = (ntaps - 1) // 2
    pre_pad = D - half % D
    pre_rem = (half + pre_pad) // D
    c0 = pre_rem * D - pre_pad if D > 1 else 0
    M = len(w) if w is not None else 1
    Bmax = L - R - (M - 1 if w is not None else 0)
    Wp = taps_spectrum(w, L) if w is not None else None
    xw = ref * (win if win is not None else 1.0)
    P = np.zeros((F, R + 1), complex)
    for j in range(F):
        lo = j * D + c0 - (ntaps - 1)
        hi = j * D + c0 + 1            # exclusive
        lo, hi = max(lo, 0), min(hi, n)
        if hi <= lo:
            continue
        nseg = -(-(hi - lo) // Bmax)
        Bs = -(-(hi - lo) // nseg)
        acc = np.zeros(L, complex)
        for q in range(nseg):
            i0 = lo + q * Bs
            ln = min(Bs, hi - i0)
            x = np.zeros(L, complex)
            x[:ln] = xw[i0:i0 + ln]
            S = np.fft.fft(srv[(i0 + np.arange(L)) % n])
            if w is not None:
                Rr = np.fft.fft(ref[(i0 + peek - (M - 1) + np.arange(L)) % n])
                S = S - Rr * Wp
            acc += np.fft.fft(x) * np.conj(S)
        P[j] = np.fft.fft(acc)[:R + 1] / L
    return P


def onepass_limits(L, M, R, peek):
    """segment limits of the one-pass frame (framepass.cuh): LS-only segments (lags M-1 .. 2M-2 of X_ls conj(Yr')) and
    block segments (also the CAF lags peek .. R + peek of the cleaned window, whose W' wrap starts past L - M)"""
    bls = L - 2 * M + 2
    return bls, min(bls, L - M - R - peek + 1)


def onepass_partition(n, F, M, R, peek, L, limits=None):
    """The segments of the one-pass frame: per Doppler block (lo, hi, ls_end, nseg, Bs) -- samples [lo, hi) in nseg
    segments of Bs, X_ls takes [lo, ls_end) -- and the LS-only tail (tail_lo, ntail, Bt)."""
    D = n // F
    ntaps = D + 1
    half = (ntaps - 1) // 2
    pre_pad = D - half % D
    c0 = ((half + pre_pad) // D) * D - pre_pad
    assert c0 - (ntaps - 1) <= 0, "no samples before the first block"
    bls, bmax = limits or onepass_limits(L, M, R, peek)
    assert bmax >= 1
    blocks = []
    for j in range(F):
        lo = max(j * D + c0 - (ntaps - 1), 0)
        hi = min(j * D + c0 + 1, n)
        ls_end = min(hi, max((j + 1) * D + c0 - (ntaps - 1), 0)) if j + 1 < F else hi
        nseg = -(-(hi - lo) // bmax)
        blocks.append((lo, hi, ls_end, nseg, -(-(hi - lo) // nseg) if nseg else 0))
    tail_lo = min((F - 1) * D + c0 + 1, n)
    ntail = -(-(n - tail_lo) // bls)
    return blocks, (tail_lo, ntail, -(-(n - tail_lo) // ntail) if ntail else 0)


def model_onepass(ref, srv, win, w, R, F, peek, L, limits=None):
    """framepass.cuh in numpy: per Doppler-block segment Ys' (srv from i0 - peek), Yr' (ref from i0 - (M-1)), X_ls and
    X_caf; LS sums from X_ls, AccP / AccQ per block from X_caf, then AccP - AccQ conj(W') and lags peek .. R + peek.
    The sample two blocks share goes to the first block's X_ls only; samples after the last block are LS-only
    segments.  Returns (c, x, P)."""
    n, M = len(ref), len(w)
    blocks, (tail_lo, ntail, Bt) = onepass_partition(n, F, M, R, peek, L, limits)
    Wp = taps_spectrum(w, L)
    xw = ref * (win if win is not None else 1.0)

    def spec(sig, base):
        return np.fft.fft(sig[(base + np.arange(L)) % n])

    def seg(sig, i0, ln, lo_off=0):
        x = np.zeros(L, complex)
        x[lo_off:ln] = sig[i0 + lo_off:i0 + ln]
        return np.fft.fft(x)

    accC = np.zeros(L, complex)
    accX = np.zeros(L, complex)
    P = np.zeros((F, R + 1), complex)
    covered = np.zeros(n, int)
    for j, (lo, hi, ls_end, nseg, Bs) in enumerate(blocks):
        accP = np.zeros(L, complex)
        accQ = np.zeros(L, complex)
        for q in range(nseg):
            i0 = lo + q * Bs
            ln = min(Bs, hi - i0)
            lx = max(0, min(ln, ls_end - i0))
            covered[i0:i0 + lx] += 1
            Ys = spec(srv, i0 - peek)
            Yr = spec(ref, i0 - (M - 1))
            Xls = seg(ref, i0, lx)
            Xcaf = seg(xw, i0, ln)
            accC += Xls * np.conj(Yr)
            accX += Xls * np.conj(Ys)
            accQ += Xcaf * np.conj(Yr)
            accP += Xcaf * np.conj(Ys)
        P[j] = np.fft.fft(accP - accQ * np.conj(Wp))[peek:peek + R + 1] / L
    for k in range(ntail):
        i0 = tail_lo + k * Bt
        ln = min(Bt, n - i0)
        covered[i0:i0 + ln] += 1
        Xls = seg(ref, i0, ln)
        accC += Xls * np.conj(spec(ref, i0 - (M - 1)))
        accX += Xls * np.conj(spec(srv, i0 - peek))
    assert (covered == 1).all(), "every sample in exactly one X_ls"
    c = np.fft.fft(accC)[M - 1:2 * M - 1] / L
    x = np.fft.fft(accX)[:M] / L
    return c, x, P


def onepass_truth(ref, srv, win, w, R, F, peek):
    """float64 direct sums of what the one-pass frame computes: LS lag sums and the CAF block sums of the cleaned channel"""
    n, M = len(ref), len(w)
    c = direct_lags(ref, ref, range(M), n)
    x = direct_lags(ref, srv, range(-peek, M - peek), n)
    s_eff = srv - sum(w[k] * np.roll(ref, k - peek) for k in range(M))
    xw = ref * (win if win is not None else 1.0)
    D = n // F
    ntaps = D + 1
    half = (ntaps - 1) // 2
    pre_pad = D - half % D
    c0 = ((half + pre_pad) // D) * D - pre_pad
    P = np.zeros((F, R + 1), complex)
    for d in range(R + 1):
        prod = xw * np.conj(np.roll(s_eff, -d))
        for j in range(F):
            P[j, d] = prod[max(j * D + c0 - (ntaps - 1), 0):min(j * D + c0 + 1, n)].sum()
    return c, x, P


def check(name, a, b, den=None, tol=1e-9):
    e = np.abs(a - b).max() / (den if den else np.abs(b).max())
    print(f"{name:56s} {e:.2e}")
    assert e < tol, name


# the one-pass frame: the headline shape (c2) and the planner's edges -- M = 1, 2, 1023, 1024 with peek 0 and M - 1, D = 32,
# F = 1, n not a multiple of F, R + M near L (the CAF limit below the LS one), no window and a float window
ONEPASS = [
    # n, F, R, M, peek, L, window
    (2 ** 20, 256, 300, 310, 10, 2048, True),
    (20000, 16, 100, 1, 0, 2048, True),
    (20000, 16, 100, 2, 0, 2048, False),
    (20000, 16, 100, 2, 1, 2048, True),
    (30000, 8, 200, 1023, 0, 4096, True),
    (30000, 8, 200, 1024, 1023, 4096, False),
    (32 * 128 + 17, 128, 40, 50, 10, 1024, True),
    (10000, 1, 100, 60, 10, 1024, True),
    (20011, 7, 60, 40, 39, 1024, True),
    (12000, 10, 600, 200, 5, 1024, False),
]


def main():
    for n, M, peek, L in [(8192, 110, 10, 2048), (20000, 310, 10, 2048), (5000, 64, 0, 1024), (12345, 300, 7, 2048)]:
        ref = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        srv = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        for linear in (False, True):
            C, X = model_lscorr(ref, srv, M, peek, L, linear)
            check(f"lscorr n={n} M={M} L={L} linear={linear} autocorr", C, direct_lags(ref, ref, range(M), n, linear))
            check(f"lscorr n={n} M={M} L={L} linear={linear} xcorr", X, direct_lags(ref, srv, range(-peek, M - peek), n, linear))
        w = (rng.standard_normal(M) + 1j * rng.standard_normal(M)) / M
        for linear in (False, True):
            got = model_fir(ref, srv, w, peek, L, linear)
            want = srv.copy()
            for k in range(M):
                sh = np.roll(ref, k - peek)
                if linear:
                    d = k - peek
                    sh = np.zeros(n, complex)
                    if d >= 0:
                        sh[d:] = ref[:n - d]
                    else:
                        sh[:n + d] = ref[-d:]
                want = want - w[k] * sh
            check(f"fir n={n} M={M} linear={linear}", got, want)

    for n, F, R, M, peek, L in [(16384, 8, 40, 50, 10, 2048), (20000, 16, 100, 110, 10, 2048), (8192, 32, 20, 30, 10, 1024), (10000, 7, 33, 0, 0, 1024)]:
        ref = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        srv = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        win = np.kaiser(n, 5.0)
        D = n // F
        ntaps = D + 1
        half = (ntaps - 1) // 2
        pre_pad = D - half % D
        c0 = ((half + pre_pad) // D) * D - pre_pad
        w = (rng.standard_normal(M) + 1j * rng.standard_normal(M)) / M if M else None
        s_eff = srv if w is None else srv - sum(w[k] * np.roll(ref, k - peek) for k in range(M))
        want = np.zeros((F, R + 1), complex)
        xw = ref * win
        for j in range(F):
            for m in range(ntaps):
                i = j * D + c0 - m
                if 0 <= i < n:
                    want[j] += xw[i] * np.conj(s_eff[(i + np.arange(R + 1)) % n])
        got = model_caf(ref, srv, win, R, F, L, w, peek)
        check(f"caf n={n} F={F} R={R} M={M} L={L}", got, want)
    for n, F, R, M, peek, L, use_win in ONEPASS:
        ref = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        srv = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        win = np.kaiser(n, 5.0) if use_win else None
        w = (rng.standard_normal(M) + 1j * rng.standard_normal(M)) / M
        tc, tx, tP = onepass_truth(ref, srv, win, w, R, F, peek)
        c, x, P = model_onepass(ref, srv, win, w, R, F, peek, L)
        tag = f"onepass n={n} F={F} R={R} M={M} peek={peek} L={L}"
        check(tag + " c", c, tc, tol=1e-12)
        check(tag + " x", x, tx, tol=1e-12)
        check(tag + " P", P, tP, tol=1e-12)
    # the headline shape: Bmax = 1429, three segments per block, a 2047-sample LS-only tail
    assert onepass_limits(2048, 310, 300, 10) == (1430, 1429)
    print("model OK")


if __name__ == "__main__":
    main()
