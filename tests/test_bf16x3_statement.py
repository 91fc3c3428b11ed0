"""CPU statement of the two numerical ideas behind the tensor-core (wgmma) kernels (csrc/toepcorr.cuh, csrc/firtc.cuh):
(1) a float32 value split into three BF16 numbers and the six products of order <= 2 reproduce a float32
product to ~2^-23; (2) the lag correlation of complex signals is the sum over the real diagonals of a GEMM on
interleaved real data (the "Toeplitz GEMM").  Pure numpy, no GPU: it documents WHY the kernels can be exact."""
import numpy as np


def bf16_round(x):
    """round-to-nearest-even to BF16 (8 significand bits), returned as float32"""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def split3(x):
    b0 = bf16_round(x)
    r1 = (x - b0).astype(np.float32)
    b1 = bf16_round(r1)
    b2 = bf16_round((r1 - b1).astype(np.float32))
    return b0, b1, b2


def test_three_way_split_is_exact_to_24_bits_and_six_products_suffice():
    rng = np.random.default_rng(0)
    x = rng.standard_normal(200000).astype(np.float32)
    y = rng.standard_normal(200000).astype(np.float32)
    xs, ys = split3(x), split3(y)
    assert np.max(np.abs((xs[0].astype(np.float64) + xs[1] + xs[2]) - x) / np.abs(x)) <= 2.0 ** -23
    exact = x.astype(np.float64) * y.astype(np.float64)
    six = sum(xs[i].astype(np.float64) * ys[j].astype(np.float64) for i, j in [(0, 0), (0, 1), (1, 0), (0, 2), (2, 0), (1, 1)])
    three = sum(xs[i].astype(np.float64) * ys[j].astype(np.float64) for i, j in [(0, 0), (0, 1), (1, 0)])
    scale = np.abs(x.astype(np.float64)) * np.abs(y.astype(np.float64))
    assert np.max(np.abs(six - exact) / scale) <= 2.0 ** -21            # dropped terms are b1*b2, b2*b1, b2*b2 (~2^-24)
    assert np.max(np.abs(three - exact) / scale) >= 2.0 ** -18          # three products (a "BF16x2") are NOT enough for 1e-5 on short sums
    # a long dot product: the six-product form is at float32 accuracy
    d6 = six.sum()
    assert abs(d6 - exact.sum()) <= 1e-7 * np.sqrt((exact ** 2).sum())


def test_toeplitz_gemm_diagonals_are_the_lag_correlation():
    """D[u][v] = sum_a zx[128 a + u] * zs[128 a + v] on interleaved reals; diagonal delta = v - u collects
    re/im parts of C[l] = sum_i x[i] conj(s[i + l]) exactly as the epilogue of toepcorr_kernel sums them."""
    rng = np.random.default_rng(1)
    nrows, nlag = 6, 40
    n = 64 * nrows
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    s = (rng.standard_normal(n + 64 + nlag) + 1j * rng.standard_normal(n + 64 + nlag))
    zx = np.stack([x.real, x.imag], axis=1).reshape(-1)
    zs = np.stack([s.real, s.imag], axis=1).reshape(-1)
    ncol = 2 * (64 + nlag)
    X = np.stack([zx[128 * a: 128 * a + 128] for a in range(nrows)])            # K x M
    S = np.stack([zs[128 * a: 128 * a + ncol] for a in range(nrows)])           # K x N (overlapping rows)
    D = X.T @ S                                                                 # 128 x ncol
    C = np.zeros(nlag, dtype=np.complex128)
    for u in range(128):
        for v in range(ncol):
            delta = v - u
            if delta % 2 == 0:
                l = delta // 2
                if 0 <= l < nlag:
                    C[l] += D[u, v]                                             # re*re + im*im
            elif u % 2 == 1:
                l = (delta + 1) // 2
                if 0 <= l < nlag:
                    C[l] += 1j * D[u, v]                                        # im(x) * re(s)
            else:
                l = (delta - 1) // 2
                if 0 <= l < nlag:
                    C[l] -= 1j * D[u, v]                                        # re(x) * im(s)
    want = np.array([np.sum(x * np.conj(s[l: l + n])) for l in range(nlag)])
    assert np.max(np.abs(C - want)) <= 1e-10 * np.abs(want).max()


def test_fir_as_gemm_with_a_taps_matrix():
    """firtc_kernel: out block a (64 samples = 128 reals) = window of the interleaved signal times Wm, with
    Wm[v'][u'] built from the taps as fir_bmat_kernel does (k = io + shift - iq; [[wr, -wi], [wi, wr]])."""
    rng = np.random.default_rng(2)
    M, peek = 23, 4
    pre = -(-(M - 1 - peek) // 4) * 4
    shift = peek + pre
    kv = 2 * (64 + peek + pre)
    w = rng.standard_normal(M) + 1j * rng.standard_normal(M)
    n = 64 * 5
    ref = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    Wm = np.zeros((kv, 128))
    for up in range(128):
        io, ao = up >> 1, up & 1
        for vp in range(kv):
            iq, bq = vp >> 1, vp & 1
            k = io + shift - iq
            if 0 <= k < M:
                Wm[vp, up] = (w[k].real if ao == bq else (w[k].imag if ao else -w[k].imag))
    out = np.zeros(n, dtype=np.complex128)
    for a in range(n // 64):
        idx = (64 * a - pre + np.arange(kv // 2)) % n                 # circular window starting `pre` samples early
        z = np.stack([ref[idx].real, ref[idx].imag], axis=1).reshape(-1)
        o = z @ Wm
        out[64 * a: 64 * a + 64] = o[0::2] + 1j * o[1::2]
    want = np.array([sum(w[k] * ref[(i + peek - k) % n] for k in range(M)) for i in range(n)])
    assert np.max(np.abs(out - want)) <= 1e-10 * np.abs(want).max()
