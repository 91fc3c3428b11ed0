/* nlms_oracle.c -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
 *
 * Plain-C restatement of the reference's NLMS_filter
 * (passiveRadar/clutter_removal.py:189-249, update rule :211-215)
 * extended with the block_NLMS definition of oracle/clutter_oracle.py, so that the
 * 2M-sample BASELINE config can be checked in seconds instead of the ~18 s/frame the
 * Python loop needs.  Arithmetic is complex float (as numpy's complex64 path), with the
 * dot products accumulated in 8 interleaved partial sums the way a SIMD BLAS cdotc does.
 * Pinned against the reference's own output by tests/test_oracle_golden.py.
 *
 *   u_k[j] = ref[M + k - j],  e_k = srv[k+L] - w^H u_k,
 *   w += mu * sum_{k in block} u_k conj(e_k) / (u_k^H u_k)   at each block end.
 */
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float re, im; } c64;

int nlms_oracle_c64(const c64* ref, const c64* srv, long n, int filter_len, int peek, float mu,
                    int block_len, const c64* init, c64* out, c64* taps_out)
{
    const int M = filter_len + peek;
    const long nsteps = n - M;
    c64* w = (c64*)calloc((size_t)(M > 0 ? M : 1), sizeof(c64));
    c64* grad = (c64*)calloc((size_t)(M > 0 ? M : 1), sizeof(c64));
    if (!w || !grad) { free(w); free(grad); return -1; }
    if (init) memcpy(w, init, (size_t)M * sizeof(c64));
    memset(out, 0, (size_t)n * sizeof(c64));
    int in_block = 0;
    for (long k = 0; k < nsteps; ++k) {
        const c64* top = ref + M + k;            /* u[j] = top[-j] */
        float ar[8] = {0}, ai[8] = {0}, nn[8] = {0};
        for (int j = 0; j < M; ++j) {
            const c64 u = top[-j];
            const int s = j & 7;
            ar[s] += w[j].re * u.re + w[j].im * u.im;      /* conj(w) * u */
            ai[s] += w[j].re * u.im - w[j].im * u.re;
            nn[s] += u.re * u.re + u.im * u.im;
        }
        const float dr = ((ar[0] + ar[4]) + (ar[2] + ar[6])) + ((ar[1] + ar[5]) + (ar[3] + ar[7]));
        const float di = ((ai[0] + ai[4]) + (ai[2] + ai[6])) + ((ai[1] + ai[5]) + (ai[3] + ai[7]));
        const float nrm = ((nn[0] + nn[4]) + (nn[2] + nn[6])) + ((nn[1] + nn[5]) + (nn[3] + nn[7]));
        const float er = srv[k + filter_len].re - dr;
        const float ei = srv[k + filter_len].im - di;
        out[k + filter_len].re = er;
        out[k + filter_len].im = ei;
        for (int j = 0; j < M; ++j) {
            const c64 u = top[-j];
            /* mu * u * conj(e) / nrm */
            const float mr = mu * u.re, mi = mu * u.im;
            const float pr = mr * er + mi * ei;
            const float pi = mi * er - mr * ei;
            grad[j].re += pr / nrm;
            grad[j].im += pi / nrm;
        }
        if (++in_block == block_len || k == nsteps - 1) {
            for (int j = 0; j < M; ++j) {
                w[j].re += grad[j].re; w[j].im += grad[j].im;
                grad[j].re = 0.f; grad[j].im = 0.f;
            }
            in_block = 0;
        }
    }
    if (taps_out) memcpy(taps_out, w, (size_t)M * sizeof(c64));
    free(w); free(grad);
    return 0;
}

/* The same recurrence with every operation in double (inputs are the complex64 samples): the float64
 * "truth" that tells how far the complex64 reference itself is from the exact recurrence. */
typedef struct { double re, im; } c128;

int nlms_truth_c128(const c64* ref, const c64* srv, long n, int filter_len, int peek, double mu,
                    int block_len, const c64* init, c128* out, c128* taps_out)
{
    const int M = filter_len + peek;
    const long nsteps = n - M;
    c128* w = (c128*)calloc((size_t)(M > 0 ? M : 1), sizeof(c128));
    c128* grad = (c128*)calloc((size_t)(M > 0 ? M : 1), sizeof(c128));
    if (!w || !grad) { free(w); free(grad); return -1; }
    if (init) for (int j = 0; j < M; ++j) { w[j].re = init[j].re; w[j].im = init[j].im; }
    memset(out, 0, (size_t)n * sizeof(c128));
    int in_block = 0;
    for (long k = 0; k < nsteps; ++k) {
        const c64* top = ref + M + k;
        double dr = 0.0, di = 0.0, nrm = 0.0;
        for (int j = 0; j < M; ++j) {
            const double ur = top[-j].re, ui = top[-j].im;
            dr += w[j].re * ur + w[j].im * ui;
            di += w[j].re * ui - w[j].im * ur;
            nrm += ur * ur + ui * ui;
        }
        const double er = (double)srv[k + filter_len].re - dr;
        const double ei = (double)srv[k + filter_len].im - di;
        out[k + filter_len].re = er;
        out[k + filter_len].im = ei;
        for (int j = 0; j < M; ++j) {
            const double ur = top[-j].re, ui = top[-j].im;
            grad[j].re += mu * (ur * er + ui * ei) / nrm;
            grad[j].im += mu * (ui * er - ur * ei) / nrm;
        }
        if (++in_block == block_len || k == nsteps - 1) {
            for (int j = 0; j < M; ++j) {
                w[j].re += grad[j].re; w[j].im += grad[j].im;
                grad[j].re = 0.0; grad[j].im = 0.0;
            }
            in_block = 0;
        }
    }
    if (taps_out) memcpy(taps_out, w, (size_t)M * sizeof(c128));
    free(w); free(grad);
    return 0;
}
