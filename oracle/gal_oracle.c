/* gal_oracle.c -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
 *
 * Plain-C restatement of the reference's GAL_JPE (passiveRadar/clutter_removal.py:251-364): a
 * gradient-adaptive lattice of `L` stages followed by an NLMS transversal filter over the D backward
 * prediction errors.  The Python loop needs 40-160 us per sample; this runs the same recurrence with
 * the reference's complex64 rounding points in well under a microsecond per stage, so a 2^19-sample
 * CPI can be checked in seconds.  Pinned against the reference's own output by tests/test_gal_jpe.py.
 *
 * Rounding points of the reference (NumPy 2, complex64 state), per sample n < N - peek - 1:
 *   f[0] = b[0] = ref[n+peek];  f[m] = f[m-1] - conj(k[m]) bo[m-1];  b[m] = bo[m-1] - k[m] f[m-1]
 *   P[m-1] = 0.9f P[m-1] + fl32(1 - 0.9^2) (|f[m-1]|^2 + |bo[m-1]|^2)        (|.| = hypotf)
 *   k[m]  += (mu1 * grad) * (1 / (P[m-1] + 1e-10f))   complex64 / real-valued complex64 is a reciprocal multiply
 *   b[m]   = bo[m-1] (m >= L);  e = srv[n] - h^H b;  h += ((mu2 conj(e)) b) * (1 / (b^H b + 1e-10f))
 *   mu1    = min(0.999 mu1 + 1e-8 e^2, 5e-3)
 * mu1 starts as a Python float (0.999 mu1 in float64, rounded to float32 when it meets complex64), becomes
 * complex64 after the first step, and min() compares complex64 against 5e-3 lexicographically (real part,
 * then imaginary part); when the clamp wins mu1 is the Python float 5e-3 again.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float re, im; } c64;
typedef struct { double re, im; } c128;

static c64 cmul(c64 a, c64 b) { c64 r = {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; return r; }
static c64 cconj(c64 a) { c64 r = {a.re, -a.im}; return r; }
static c64 csub(c64 a, c64 b) { c64 r = {a.re - b.re, a.im - b.im}; return r; }
static c64 cadd(c64 a, c64 b) { c64 r = {a.re + b.re, a.im + b.im}; return r; }

int gal_oracle_c64(const c64* ref, const c64* srv, long n, int L, int D, double mu1, double mu2, int peek,
                   c64* out, c64* k_out, c64* h_out)
{
    if (L < 1 || D < L || peek < 0) return -2;
    c64* st = (c64*)calloc((size_t)D * 5, sizeof(c64));
    float* P = (float*)malloc((size_t)D * sizeof(float));
    if (!st || !P) { free(st); free(P); return -1; }
    c64 *f = st, *b = st + D, *bo = st + 2 * D, *k = st + 3 * D, *h = st + 4 * D;
    for (int m = 0; m < D; ++m) P[m] = 1e-8f;
    const float beta = 0.9f, omb2 = (float)(1.0 - 0.9 * 0.9), gammaf = 0.999f, deltaf = 1e-8f, mu2f = (float)mu2;
    int mu_py = 1;              /* mu1 is a Python float (value mu_d) or a complex64 (mu_c) */
    double mu_d = mu1;
    c64 mu_c = {0.f, 0.f};
    memset(out, 0, (size_t)n * sizeof(c64));
    for (long t = 0; t < n - peek - 1; ++t) {
        memcpy(bo, b, (size_t)D * sizeof(c64));
        f[0] = b[0] = ref[t + peek];
        for (int m = 1; m < L; ++m) {
            f[m] = csub(f[m - 1], cmul(cconj(k[m]), bo[m - 1]));
            b[m] = csub(bo[m - 1], cmul(k[m], f[m - 1]));
        }
        for (int m = 1; m < L; ++m) {
            const float af = hypotf(f[m - 1].re, f[m - 1].im), ab = hypotf(bo[m - 1].re, bo[m - 1].im);
            const float Em = af * af + ab * ab;
            P[m - 1] = beta * P[m - 1] + omb2 * Em;
            const c64 grad = cadd(cmul(cconj(f[m - 1]), b[m]), cmul(bo[m - 1], cconj(f[m])));
            c64 q;
            if (mu_py) { const float mf = (float)mu_d; q.re = mf * grad.re; q.im = mf * grad.im; }
            else q = cmul(mu_c, grad);
            const float r = 1.0f / (P[m - 1] + 1e-10f);
            k[m].re += q.re * r;
            k[m].im += q.im * r;
        }
        for (int m = L; m < D; ++m) b[m] = bo[m - 1];
        c64 hb = {0.f, 0.f};
        float bb = 0.f;
        for (int m = 0; m < D; ++m) {
            hb = cadd(hb, cmul(cconj(h[m]), b[m]));
            bb += b[m].re * b[m].re + b[m].im * b[m].im;
        }
        const c64 e = csub(srv[t], hb);
        const float r2 = 1.0f / (bb + 1e-10f);
        const c64 c = {mu2f * e.re, mu2f * -e.im};
        for (int m = 0; m < D; ++m) {
            const c64 u = cmul(c, b[m]);
            h[m].re += u.re * r2;
            h[m].im += u.im * r2;
        }
        out[t] = e;
        const c64 e2 = cmul(e, e);
        float xr, xi;
        if (mu_py) { xr = (float)(0.999 * mu_d) + deltaf * e2.re; xi = 0.0f + deltaf * e2.im; }
        else { xr = gammaf * mu_c.re + deltaf * e2.re; xi = gammaf * mu_c.im + deltaf * e2.im; }
        if (xr > 5e-3f || (xr == 5e-3f && xi > 0.f)) { mu_py = 1; mu_d = 5e-3; }
        else { mu_py = 0; mu_c.re = xr; mu_c.im = xi; }
    }
    if (k_out) memcpy(k_out, k, (size_t)D * sizeof(c64));
    if (h_out) memcpy(h_out, h, (size_t)D * sizeof(c64));
    free(st); free(P);
    return 0;
}

/* The same recurrence with every operation in double (inputs are the complex64 samples): the float64 "truth" that
 * tells how far the complex64 reference itself is from the exact recurrence.  mu1 keeps the reference's type rules
 * (a real start value, complex afterwards, the lexicographic clamp), evaluated in double. */
static c128 zmul(c128 a, c128 b) { c128 r = {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; return r; }
static c128 zconj(c128 a) { c128 r = {a.re, -a.im}; return r; }
static c128 zsub(c128 a, c128 b) { c128 r = {a.re - b.re, a.im - b.im}; return r; }
static c128 zadd(c128 a, c128 b) { c128 r = {a.re + b.re, a.im + b.im}; return r; }

static int gal_truth_run(const c64* ref, const c64* srv, long n, int L, int D, double mu1, double mu2, int peek,
                         c128* out, c128* k_out, c128* h_out, double* stats)
{
    if (L < 1 || D < L || peek < 0) return -2;
    c128* st = (c128*)calloc((size_t)D * 5, sizeof(c128));
    double* P = (double*)malloc((size_t)D * sizeof(double));
    if (!st || !P) { free(st); free(P); return -1; }
    c128 *f = st, *b = st + D, *bo = st + 2 * D, *k = st + 3 * D, *h = st + 4 * D;
    for (int m = 0; m < D; ++m) P[m] = 1e-8;
    int mu_py = 1;
    double mu_d = mu1;
    c128 mu_c = {0.0, 0.0};
    long clamps = 0;
    double margin = INFINITY, xr_max = 0.0;
    memset(out, 0, (size_t)n * sizeof(c128));
    for (long t = 0; t < n - peek - 1; ++t) {
        memcpy(bo, b, (size_t)D * sizeof(c128));
        f[0].re = b[0].re = ref[t + peek].re;
        f[0].im = b[0].im = ref[t + peek].im;
        for (int m = 1; m < L; ++m) {
            f[m] = zsub(f[m - 1], zmul(zconj(k[m]), bo[m - 1]));
            b[m] = zsub(bo[m - 1], zmul(k[m], f[m - 1]));
        }
        for (int m = 1; m < L; ++m) {
            const double Em = f[m - 1].re * f[m - 1].re + f[m - 1].im * f[m - 1].im
                            + bo[m - 1].re * bo[m - 1].re + bo[m - 1].im * bo[m - 1].im;
            P[m - 1] = 0.9 * P[m - 1] + (1.0 - 0.9 * 0.9) * Em;
            const c128 grad = zadd(zmul(zconj(f[m - 1]), b[m]), zmul(bo[m - 1], zconj(f[m])));
            c128 q;
            if (mu_py) { q.re = mu_d * grad.re; q.im = mu_d * grad.im; }
            else q = zmul(mu_c, grad);
            const double den = P[m - 1] + 1e-10;
            k[m].re += q.re / den;
            k[m].im += q.im / den;
        }
        for (int m = L; m < D; ++m) b[m] = bo[m - 1];
        c128 hb = {0.0, 0.0};
        double bb = 0.0;
        for (int m = 0; m < D; ++m) {
            hb = zadd(hb, zmul(zconj(h[m]), b[m]));
            bb += b[m].re * b[m].re + b[m].im * b[m].im;
        }
        const c128 s = {srv[t].re, srv[t].im};
        const c128 e = zsub(s, hb);
        const double den2 = bb + 1e-10;
        const c128 c = {mu2 * e.re, mu2 * -e.im};
        for (int m = 0; m < D; ++m) {
            const c128 u = zmul(c, b[m]);
            h[m].re += u.re / den2;
            h[m].im += u.im / den2;
        }
        out[t] = e;
        const c128 e2 = zmul(e, e);
        double xr, xi;
        if (mu_py) { xr = 0.999 * mu_d + 1e-8 * e2.re; xi = 1e-8 * e2.im; }
        else { xr = 0.999 * mu_c.re + 1e-8 * e2.re; xi = 0.999 * mu_c.im + 1e-8 * e2.im; }
        const double mg = fabs(xr - 5e-3) / 5e-3;
        if (mg < margin) margin = mg;
        if (fabs(xr) > xr_max) xr_max = fabs(xr);
        if (xr > 5e-3 || (xr == 5e-3 && xi > 0.0)) { mu_py = 1; mu_d = 5e-3; ++clamps; }
        else { mu_py = 0; mu_c.re = xr; mu_c.im = xi; }
    }
    if (stats) {
        stats[0] = (double)clamps;
        stats[1] = margin;
        stats[2] = xr_max;
        stats[3] = mu_py ? mu_d : mu_c.re;
        stats[4] = mu_py ? 0.0 : mu_c.im;
    }
    if (k_out) memcpy(k_out, k, (size_t)D * sizeof(c128));
    if (h_out) memcpy(h_out, h, (size_t)D * sizeof(c128));
    free(st); free(P);
    return 0;
}

int gal_truth_c128(const c64* ref, const c64* srv, long n, int L, int D, double mu1, double mu2, int peek,
                   c128* out, c128* k_out, c128* h_out)
{
    return gal_truth_run(ref, srv, n, L, D, mu1, mu2, peek, out, k_out, h_out, NULL);
}

/* gal_truth_c128 (the same code path, so the same bits) that also reports on mu1's clamp, in stats[5]: the number of
 * samples at which the clamp at 5e-3 won, the smallest |xr - 5e-3| / 5e-3 over all clamp decisions (INFINITY when
 * there were none), the largest |xr|, and mu1 after the last sample (real and imaginary part; a real value when the
 * clamp won last).  xr is the real part min() compares with 5e-3.  A complex64 evaluation of a decision whose margin
 * is below its own rounding error can go the other way. */
int gal_truth_stats_c128(const c64* ref, const c64* srv, long n, int L, int D, double mu1, double mu2, int peek,
                         c128* out, c128* k_out, c128* h_out, double* stats)
{
    return gal_truth_run(ref, srv, n, L, D, mu1, mu2, peek, out, k_out, h_out, stats);
}
