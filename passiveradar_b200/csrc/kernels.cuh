// kernels.cuh -- sm_90a device code of libprcore (passive-radar hot path).
//
// Four kernels carry the frame  LS_Filter -> fast_xambg  (DESIGN.md section 3):
//
//   lagcorr_kernel   partial lag-correlation sums  C[d] = sum_i x[i] conj(s[i+d])
//                    used three times: Gram column + right-hand side of the LS
//                    normal equations (clutter_removal.py:39,45) and the per-Doppler-
//                    block lag products of the CAF (range_doppler_processing.py:81-86)
//   levinson_kernel  (T + reg I) w = rhs for the Hermitian Toeplitz Gram matrix, fp64
//                    (replaces np.linalg.solve, clutter_removal.py:42-45)
//   fir_apply_kernel out = srv - circular FIR(ref, w)              (clutter_removal.py:51)
//   doppler_fft_*    chunk sum + FFT along Doppler + fftshift  (range_doppler_processing.py:89)
//
// lagcorr, fir_apply and lagstream_kernel (lagstream.cuh) share one inner loop, a register-tiled
// sliding-window complex multiply-accumulate on (re, im) register pairs (slide_mac2 / slide_mac2n).
// A thread owns TD accumulator pairs per component and a ring of TI+TD window samples; every step
// it pulls TI fresh window samples (128-bit LDS, lane stride TD*8 B = an odd multiple of 16 B,
// hence bank-conflict free) and TI broadcast operands, and issues TI*TD complex MACs (4 FFMA
// each): the loop is FP32-pipe bound by design.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace prc {

// stream decomposition used by lagstream_kernel and its consumers: block `blk` of length blk_len
// starts at stream position blk*blk_len; CTA c owns [c*per_cta, (c+1)*per_cta)
__host__ __device__ inline long long stream_first_cta(long long blk, int blk_len, long long per_cta) {
    return (blk * (long long)blk_len) / per_cta;
}
__host__ __device__ inline int stream_pieces(long long blk, int blk_len, long long per_cta) {
    const long long a = (blk * (long long)blk_len) / per_cta;
    const long long b = ((blk + 1) * (long long)blk_len - 1) / per_cta;
    return (int)(b - a + 1);
}

// (a.x * b.x + c.x, a.y * b.y + c.y) with one rounding each.  Hopper has no packed FP32x2 FMA, so this is two
// scalar fma.rn: the register pairs stay aligned 64-bit operands and the roundings are those of the packed form.
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

template <int A, int B> struct Gcd { static constexpr int v = Gcd<B, A % B>::v; };
template <int A> struct Gcd<A, 0> { static constexpr int v = A; };

// Sliding-window MAC on (re, im) register pairs (ffma2_rn):
//   A1[v] += sum_{t<nsteps, u<TI} (xr, xr)[t*TI+u] * (wr, wi)[t*TI+u+v]      A2[v]: the same with (xi, xi)
// v = 0..TD-1; every operand is an aligned 64-bit register pair (on sm_90a each pair is two scalar FFMAs).
// xs4: operand shared by the lanes of a group, xs4[i] = (xr, xr, xi, xi) of sample i (one broadcast 128-bit
// load per sample); ws: this thread's window.  Both must be 16-byte aligned; ws must be readable up to index
// nsteps*TI + TD - 1.  The caller combines
//   x*conj(w): re = A1.x + A2.y, im = A2.x - A1.y        x*w: re = A1.x - A2.y, im = A1.y + A2.x
template <int TI, int TD>
__device__ __forceinline__ void slide_mac2(float2 (&A1)[TD], float2 (&A2)[TD], const float4* __restrict__ xs4,
                                           const float2* __restrict__ ws, int nsteps) {
    static_assert(TI % 2 == 0 && TD % 2 == 0, "128-bit shared loads need even tile sizes");
    constexpr int RS = TI + TD;                       // ring size
    constexpr int PERIOD = RS / Gcd<RS, TI>::v;       // steps after which ring slots repeat
    static_assert(PERIOD <= 4, "unroll factor too large for the instruction cache");
    float2 W[RS];
#pragma unroll
    for (int q = 0; q < TD; q += 2) {
        const float4 v = *reinterpret_cast<const float4*>(ws + q);
        W[q] = make_float2(v.x, v.y);
        W[q + 1] = make_float2(v.z, v.w);
    }
    for (int t0 = 0; t0 < nsteps; t0 += PERIOD) {
#pragma unroll
        for (int p = 0; p < PERIOD; ++p) {
            if (t0 + p < nsteps) {
                const float2* wp = ws + (t0 + p) * TI + TD;
                const float4* xp = xs4 + (t0 + p) * TI;
#pragma unroll
                for (int q = 0; q < TI; q += 2) {
                    const float4 v = *reinterpret_cast<const float4*>(wp + q);
                    W[(p * TI + TD + q) % RS] = make_float2(v.x, v.y);
                    W[(p * TI + TD + q + 1) % RS] = make_float2(v.z, v.w);
                }
#pragma unroll
                for (int u = 0; u < TI; ++u) {
                    const float4 xv = xp[u];
                    const float2 xr2 = make_float2(xv.x, xv.y);
                    const float2 xi2 = make_float2(xv.z, xv.w);
#pragma unroll
                    for (int v = 0; v < TD; ++v) A1[v] = ffma2_rn(xr2, W[(p * TI + u + v) % RS], A1[v]);
#pragma unroll
                    for (int v = 0; v < TD; ++v) A2[v] = ffma2_rn(xi2, W[(p * TI + u + v) % RS], A2[v]);
                }
            }
        }
    }
}

// FFMA2 sliding MAC with x in its natural (re, im) layout; the (xr, xr) / (xi, xi) operand pairs
// are built in registers (moves go to the ALU pipe, whose issue slots the half-rate FFMA2 stream
// leaves free).  Otherwise identical to slide_mac2.
template <int TI, int TD>
__device__ __forceinline__ void slide_mac2n(float2 (&A1)[TD], float2 (&A2)[TD], const float2* __restrict__ xs,
                                            const float2* __restrict__ ws, int nsteps) {
    static_assert(TI % 2 == 0 && TD % 2 == 0, "128-bit shared loads need even tile sizes");
    constexpr int RS = TI + TD;
    constexpr int PERIOD = RS / Gcd<RS, TI>::v;
    static_assert(PERIOD <= 4, "unroll factor too large for the instruction cache");
    float2 W[RS];
#pragma unroll
    for (int q = 0; q < TD; q += 2) {
        const float4 v = *reinterpret_cast<const float4*>(ws + q);
        W[q] = make_float2(v.x, v.y);
        W[q + 1] = make_float2(v.z, v.w);
    }
    for (int t0 = 0; t0 < nsteps; t0 += PERIOD) {
#pragma unroll
        for (int p = 0; p < PERIOD; ++p) {
            if (t0 + p < nsteps) {
                const float2* wp = ws + (t0 + p) * TI + TD;
                const float2* xp = xs + (t0 + p) * TI;
#pragma unroll
                for (int q = 0; q < TI; q += 2) {
                    const float4 v = *reinterpret_cast<const float4*>(wp + q);
                    W[(p * TI + TD + q) % RS] = make_float2(v.x, v.y);
                    W[(p * TI + TD + q + 1) % RS] = make_float2(v.z, v.w);
                }
#pragma unroll
                for (int u = 0; u < TI; u += 2) {
                    const float4 xv = *reinterpret_cast<const float4*>(xp + u);
#pragma unroll
                    for (int uu = 0; uu < 2; ++uu) {
                        const float2 xr2 = uu ? make_float2(xv.z, xv.z) : make_float2(xv.x, xv.x);
                        const float2 xi2 = uu ? make_float2(xv.w, xv.w) : make_float2(xv.y, xv.y);
#pragma unroll
                        for (int v = 0; v < TD; ++v) A1[v] = ffma2_rn(xr2, W[(p * TI + u + uu + v) % RS], A1[v]);
#pragma unroll
                        for (int v = 0; v < TD; ++v) A2[v] = ffma2_rn(xi2, W[(p * TI + u + uu + v) % RS], A2[v]);
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// lagcorr: partial[prob][blk][chunk][l] = sum_{i in chunk of block blk} xw[i] * conj(s[(i + dmin + l) mod n])
//   xw[i] = x[i] * win[i] * taps[blk_hi - i]   (either factor optional), 0 outside [0, n)
// One CTA per (block, chunk, problem).  Threads = H lag groups (TD lags each) x G sample groups.
// ------------------------------------------------------------------------------------------
struct LagCorrParams {
    const float2* x;
    const float2* s[2];
    int dmin[2];
    const float* win;
    const float* taps;
    int n;
    long long blk_first_lo;
    long long blk_stride;
    int blk_len;
    int nblk;
    int nchunk;
    int chunk_len;
    int H;        // lag groups; padded lag count = H*TD
    int G;        // sample groups
    int steps;    // TI-sample steps per sample group
    float2* partial;
};

// x is staged as (xr, xr, xi, xi) float4 and the MACs are FFMA2 (slide_mac2)
template <int TI, int TD>
__global__ void __launch_bounds__(512) lagcorr_kernel(const __grid_constant__ LagCorrParams p) {
    extern __shared__ __align__(16) float2 smem[];
    const int tid = threadIdx.x;
    const int nthr = blockDim.x;
    const int blk = blockIdx.x / p.nchunk;
    const int chunk = blockIdx.x - blk * p.nchunk;
    const int prob = blockIdx.y;
    const int Sg = p.steps * TI;
    const int Lpad = p.G * Sg;
    const int HT = p.H * TD;
    constexpr int XW = 2;                   // float2 slots per staged x sample
    float2* xs = smem;
    float2* ss = smem + XW * Lpad;

    const long long blk_lo = p.blk_first_lo + (long long)blk * p.blk_stride;
    const long long blk_hi = blk_lo + p.blk_len - 1;
    const long long chunk_lo = blk_lo + (long long)chunk * p.chunk_len;
    int len = p.blk_len - chunk * p.chunk_len;
    if (len > p.chunk_len) len = p.chunk_len;

    // Staging issues STAGE_BATCH independent global loads per thread before the first store:
    // a one-load-per-iteration loop would serialise ~16 DRAM latencies per CTA.
    constexpr int STAGE_BATCH = 8;
    // ---- stage the weighted x chunk (zero outside the block / the signal)
    const float2* __restrict__ x = p.x;
    for (int base = 0; base < Lpad; base += nthr * STAGE_BATCH) {
        float2 v[STAGE_BATCH];
        float w[STAGE_BATCH];
#pragma unroll
        for (int b = 0; b < STAGE_BATCH; ++b) {
            const int q = base + b * nthr + tid;
            const long long i = chunk_lo + q;
            const bool ok = q < len && i >= 0 && i < p.n;
            v[b] = ok ? x[i] : make_float2(0.f, 0.f);
            w[b] = 1.f;
            if (p.win && ok) w[b] = p.win[i];
            if (p.taps && ok) w[b] *= p.taps[blk_hi - i];
        }
#pragma unroll
        for (int b = 0; b < STAGE_BATCH; ++b) {
            const int q = base + b * nthr + tid;
            if (q < Lpad) {
                float2 t = v[b];
                if (p.win || p.taps) { t.x *= w[b]; t.y *= w[b]; }
                reinterpret_cast<float4*>(xs)[q] = make_float4(t.x, t.x, t.y, t.y);
            }
        }
    }
    // ---- stage the circular window of s that the chunk's lags touch
    const float2* __restrict__ s = p.s[prob];
    {
        long long s0 = (chunk_lo + p.dmin[prob]) % p.n;
        if (s0 < 0) s0 += p.n;
        const unsigned start = (unsigned)s0;
        const unsigned n = (unsigned)p.n;
        const int cnt = Lpad + HT;
        for (int base = 0; base < cnt; base += nthr * STAGE_BATCH) {
            float2 v[STAGE_BATCH];
#pragma unroll
            for (int b = 0; b < STAGE_BATCH; ++b) {
                const int q = base + b * nthr + tid;
                unsigned idx = start + (unsigned)q;
                if (idx >= n) { idx -= n; if (idx >= n) idx %= n; }
                v[b] = (q < cnt) ? s[idx] : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int b = 0; b < STAGE_BATCH; ++b) {
                const int q = base + b * nthr + tid;
                if (q < cnt) ss[q] = v[b];
            }
        }
    }
    __syncthreads();

    float2 acc[TD];
#pragma unroll
    for (int v = 0; v < TD; ++v) acc[v] = make_float2(0.f, 0.f);
    const int h = tid % p.H;
    const int g = tid / p.H;
    const bool active = g < p.G;
    if (active) {
        float2 A1[TD], A2[TD];
#pragma unroll
        for (int v = 0; v < TD; ++v) { A1[v] = make_float2(0.f, 0.f); A2[v] = make_float2(0.f, 0.f); }
        slide_mac2<TI, TD>(A1, A2, reinterpret_cast<const float4*>(xs) + g * Sg, ss + g * Sg + h * TD, p.steps);
#pragma unroll
        for (int v = 0; v < TD; ++v) acc[v] = make_float2(A1[v].x + A2[v].y, A2[v].x - A1[v].y);
    }
    __syncthreads();

    // ---- reduce the G sample groups in a fixed order (deterministic), write the partial row
    float2* red = smem;
    if (active) {
#pragma unroll
        for (int v = 0; v < TD; ++v) red[g * HT + h * TD + v] = acc[v];
    }
    __syncthreads();
    float2* out = p.partial + (((size_t)prob * p.nblk + blk) * p.nchunk + chunk) * (size_t)HT;
    for (int l = tid; l < HT; l += nthr) {
        float2 sum = red[l];
        for (int gg = 1; gg < p.G; ++gg) {
            const float2 t = red[gg * HT + l];
            sum.x += t.x;
            sum.y += t.y;
        }
        out[l] = sum;
    }
}

// ------------------------------------------------------------------------------------------
// fir_apply: out[i] = srv[i] - sum_{k<M} taps[k] * ref[(i + peek - k) mod n]
// One CTA per LO = blockDim*TO consecutive outputs; taps reversed and zero-padded to Mpad.
// ------------------------------------------------------------------------------------------
struct FirParams {
    const float2* ref;
    const float2* srv;
    const float2* taps;
    float2* out;
    int n;
    int M;
    int Mpad;     // multiple of TK
    int peek;
    int linear;   // 1: ref[j] = 0 for j < 0 instead of wrapping (np.convolve of LS_Filter_Toeplitz)
};

// FFMA2 with the (t, t) operand pairs built in registers (slide_mac2n: fewest shared-memory bytes per MAC)
template <int TK, int TO>
__global__ void __launch_bounds__(512) fir_apply_kernel(const __grid_constant__ FirParams p) {
    extern __shared__ __align__(16) float2 smem[];
    const int tid = threadIdx.x;
    const int nthr = blockDim.x;
    const int LO = nthr * TO;
    float2* tr = smem;                   // Mpad reversed taps
    float2* rs = smem + p.Mpad;          // LO + Mpad window of ref
    const long long I0 = (long long)blockIdx.x * LO;

    for (int q = tid; q < p.Mpad; q += nthr) {
        const int k = p.Mpad - 1 - q;
        tr[q] = (k < p.M) ? p.taps[k] : make_float2(0.f, 0.f);
    }
    {
        long long r0 = (I0 + p.peek - (p.Mpad - 1)) % p.n;
        if (r0 < 0) r0 += p.n;
        const unsigned start = (unsigned)r0;
        const unsigned n = (unsigned)p.n;
        const float2* __restrict__ ref = p.ref;
        constexpr int STAGE_BATCH = 8;          // independent loads in flight per thread
        const int cnt = LO + p.Mpad;
        const long long lin0 = I0 + p.peek - (p.Mpad - 1);
        for (int base = 0; base < cnt; base += nthr * STAGE_BATCH) {
            float2 v[STAGE_BATCH];
#pragma unroll
            for (int b = 0; b < STAGE_BATCH; ++b) {
                const int q = base + b * nthr + tid;
                unsigned idx = start + (unsigned)q;
                if (idx >= n) { idx -= n; if (idx >= n) idx %= n; }
                const bool ok = q < cnt && (!p.linear || lin0 + q >= 0);
                v[b] = ok ? ref[idx] : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int b = 0; b < STAGE_BATCH; ++b) {
                const int q = base + b * nthr + tid;
                if (q < cnt) rs[q] = v[b];
            }
        }
    }
    __syncthreads();

    float2 acc[TO];
    float2 A1[TO], A2[TO];
#pragma unroll
    for (int v = 0; v < TO; ++v) { A1[v] = make_float2(0.f, 0.f); A2[v] = make_float2(0.f, 0.f); }
    slide_mac2n<TK, TO>(A1, A2, tr, rs + tid * TO, p.Mpad / TK);
#pragma unroll
    for (int v = 0; v < TO; ++v) acc[v] = make_float2(A1[v].x - A2[v].y, A1[v].y + A2[v].x);

    const long long i0 = I0 + (long long)tid * TO;
#pragma unroll
    for (int v = 0; v < TO; ++v) {
        const long long i = i0 + v;
        if (i < p.n) {
            const float2 d = p.srv[i];
            p.out[i] = make_float2(d.x - acc[v].x, d.y - acc[v].y);
        }
    }
}

// ------------------------------------------------------------------------------------------
// levinson: reduce the chunk partials of the two LS correlations in fp64, then solve the
// Hermitian Toeplitz system (T + reg I) w = rhs by Levinson recursion (fp64, one warp).
//   t[m]   = conj( sum_c partial[0][c][m] )          m = 0..M-1   (first column of A^H A)
//   rhs[a] = conj( sum_c partial[1][c][a] )          a = 0..M-1   (A^H srv)
// status: 0 ok, 1 = not positive definite / non-finite pivot.
// ------------------------------------------------------------------------------------------
struct LevinsonParams {
    const float2* partial;   // [2][nchunk][HT]
    int nchunk;
    int HT;
    int M;
    double reg;
    float2* taps;            // M
    int* status;
};

__device__ __forceinline__ double2 zmul(double2 a, double2 b) {
    return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ double2 zmulc(double2 a, double2 b) {   // a * conj(b)
    return make_double2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y);
}
// Inner-product-free (Schur-type) Levinson: besides the forward vector f and the solution w it
// carries P = T[f;0], Q = T[b;0] (b = conj(reverse(f))) and the residual rho = rhs - T[w;0], so the
// reflection coefficient of order n is simply P[n] and the solution increment is rho[n]; every
// step is element-wise plus a one-element shift (DESIGN.md section 3.3).  Thread tid owns elements
// tid*E .. tid*E+E-1 in registers; one named-barrier sync per step; fp64 throughout.
//   E = 1: blockDim 1024, M <= 1024        E = 4: blockDim 512, M <= 2048
constexpr int LEV_SCRATCH = 4 + 2 * 32 * 2;     // double2: pivot[2][2] + edge[2][32][2]

__host__ __device__ inline int levinson_nparts(int M, int threads) {
    const int q = threads / (2 * M);
    return q > 3 ? 3 : q;
}
__host__ __device__ inline size_t levinson_smem(int M, int threads) {
    const int np = levinson_nparts(M, threads);
    const int scratch = np * 2 * M > LEV_SCRATCH ? np * 2 * M : LEV_SCRATCH;
    return (size_t)(2 * M + scratch) * sizeof(double2);
}

template <int E>
__global__ void __launch_bounds__(E == 1 ? 1024 : 512) levinson_kernel(const __grid_constant__ LevinsonParams p) {
    extern __shared__ __align__(16) double2 zs[];
    const int M = p.M;
    double2* t = zs;                  // M   Toeplitz first column (t[0] real, + reg)
    double2* r = zs + M;              // M   right-hand side
    double2* part = zs + 2 * M;       // phase-A partial sums, then reused as:
    double2* pivot = part;            //   [2][2]      (P[n], rho[n]) double buffered
    double2* edge = part + 4;         //   [2][32][2]  last (newQ, newb) of every warp
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    // one CTA per frame of a batch: [frame][2][nchunk][HT] partials, [frame][M] taps, [frame] status
    const float2* const gpartial = p.partial + (size_t)blockIdx.x * 2 * p.nchunk * p.HT;

    // ---- phase A: fp64 sum of the chunk partials in a fixed order, conjugate
    {
        const int nval = 2 * M;
        const int nparts = levinson_nparts(M, blockDim.x);
        if (nparts > 0) {
            const int pt = tid / nval, v = tid - pt * nval;
            if (pt < nparts) {
                const int prob = v / M, l = v - prob * M;
                const float2* src = gpartial + (size_t)prob * p.nchunk * p.HT + l;
                double sx = 0.0, sy = 0.0;
#pragma unroll 8
                for (int c = pt; c < p.nchunk; c += nparts) {
                    const float2 q = src[(size_t)c * p.HT];
                    sx += (double)q.x;
                    sy += (double)q.y;
                }
                part[pt * nval + v] = make_double2(sx, sy);
            }
            __syncthreads();
        }
        double2 tot[(E == 1) ? 2 : 8];
        int cnt = 0;
        for (int v2 = tid; v2 < nval; v2 += blockDim.x, ++cnt) {
            double sx = 0.0, sy = 0.0;
            if (nparts > 0) {
                for (int k = 0; k < nparts; ++k) { sx += part[k * nval + v2].x; sy += part[k * nval + v2].y; }
            } else {
                const int prob = v2 / M, l = v2 - prob * M;
                const float2* src = gpartial + (size_t)prob * p.nchunk * p.HT + l;
#pragma unroll 8
                for (int c = 0; c < p.nchunk; ++c) {
                    const float2 q = src[(size_t)c * p.HT];
                    sx += (double)q.x;
                    sy += (double)q.y;
                }
            }
            tot[cnt] = make_double2(sx, -sy);
        }
        __syncthreads();                 // everyone is done reading `part` before t/r/pivot/edge are written
        cnt = 0;
        for (int v2 = tid; v2 < nval; v2 += blockDim.x, ++cnt) {
            if (v2 < M) t[v2] = tot[cnt];
            else r[v2 - M] = tot[cnt];
        }
        __syncthreads();
    }

    const int nact = ((M + E - 1) / E + 31) & ~31;      // threads taking part in the recursion
    if (tid >= nact) return;
    const double t0 = t[0].x + p.reg;
    int bad = !(t0 > 0.0) || !isfinite(t0);
    const double it0 = 1.0 / t0;

    double2 P[E], Qs[E], rho[E], f[E], bs[E], x[E];
    const double2 x0 = make_double2(r[0].x * it0, r[0].y * it0);
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int j = tid * E + e;
        const double2 zero = make_double2(0.0, 0.0);
        const double2 tj = (j < M) ? (j == 0 ? make_double2(t0, 0.0) : t[j]) : zero;
        const double2 tjm = (j >= 1 && j <= M) ? (j == 1 ? make_double2(t0, 0.0) : t[j - 1]) : zero;
        const double2 rj = (j < M) ? r[j] : zero;
        P[e] = make_double2(tj.x * it0, tj.y * it0);              // T[f;0],  f = [1/t0]
        Qs[e] = make_double2(tjm.x * it0, tjm.y * it0);           // (T[b;0]) shifted down by one
        f[e] = (j == 0) ? make_double2(it0, 0.0) : zero;
        bs[e] = (j == 1) ? make_double2(it0, 0.0) : zero;         // b shifted down by one
        x[e] = (j == 0) ? x0 : zero;
        const double2 xt = zmul(x0, tj);
        rho[e] = make_double2(rj.x - xt.x, rj.y - xt.y);          // rhs - T[x;0]
        if (j == 1) { pivot[2] = P[e]; pivot[3] = rho[e]; }       // step n reads buffer n & 1
    }
    asm volatile("bar.sync 1, %0;" ::"r"(nact));

    for (int n = 1; n < M; ++n) {
        const int buf = n & 1;
        const double2 ef = pivot[buf * 2 + 0];
        const double2 d = pivot[buf * 2 + 1];
        const double den = 1.0 - (ef.x * ef.x + ef.y * ef.y);
        if (!(den > 0.0) || !isfinite(den)) bad = 1;
        // The recursion is a chain of dependent fp64 operations (~40 cycles each on this part), so
        // everything that does not need 1/den is computed while the reciprocal is in flight, and the
        // reciprocal itself is a float seed + two Newton steps instead of the IEEE division routine.
        double al;
        {
            const double y0 = (double)__frcp_rn((float)den);
            const double e0 = fma(-den, y0, 1.0);
            const double y1 = fma(y0, e0, y0);
            const double e1 = fma(-den, y1, 1.0);
            al = fma(y1, e1, y1);
            if (!isfinite(al)) bad = 1;
        }
        double2 nQ[E], nb[E];
        // Only half of the state matters at step n: (f, b, x) live on elements j <= n, (P, Q, rho) on
        // j >= n.  Threads are ordered by j, so at most one warp diverges.
        // warp-uniform guards: a warp whose elements are all below / above n skips the other half
        // entirely (per-thread conditions alone are turned into predication and save nothing)
        const int wlo = (tid & ~31) * E, whi = wlo + 32 * E - 1;
        const bool warp_has_P = whi >= n, warp_has_F = wlo <= n;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int j = tid * E + e;
            nQ[e] = make_double2(0.0, 0.0);
            nb[e] = make_double2(0.0, 0.0);
            if (warp_has_P && j >= n) {
                const double2 q0 = (j == 0) ? make_double2(ef.x, -ef.y) : Qs[e];
                const double2 a = zmul(ef, q0);
                const double2 b = zmulc(P[e], ef);        // conj(ef) * P
                const double2 tp = make_double2(P[e].x - a.x, P[e].y - a.y);      // P' / al
                const double2 tq = make_double2(q0.x - b.x, q0.y - b.y);          // Q' / al
                const double2 dq = zmul(d, tq);                                   // d * Q' / al
                const double2 np = make_double2(al * tp.x, al * tp.y);
                nQ[e] = make_double2(al * tq.x, al * tq.y);
                rho[e] = make_double2(fma(-al, dq.x, rho[e].x), fma(-al, dq.y, rho[e].y));
                P[e] = np;
                if (j == n + 1) { pivot[(buf ^ 1) * 2 + 0] = np; pivot[(buf ^ 1) * 2 + 1] = rho[e]; }
            }
            if (warp_has_F && j <= n) {
                const double2 c = zmul(ef, bs[e]);
                const double2 g = zmulc(f[e], ef);        // conj(ef) * f
                const double2 tf = make_double2(f[e].x - c.x, f[e].y - c.y);
                const double2 tb = make_double2(bs[e].x - g.x, bs[e].y - g.y);
                const double2 dx = zmul(d, tb);
                nb[e] = make_double2(al * tb.x, al * tb.y);
                x[e] = make_double2(fma(al, dx.x, x[e].x), fma(al, dx.y, x[e].y));
                f[e] = make_double2(al * tf.x, al * tf.y);
            }
        }
        // shift by one element: (Qs, bs)[j] <- (nQ, nb)[j-1]
        double2 inQ, inB;
        inQ.x = __shfl_up_sync(0xffffffffu, nQ[E - 1].x, 1);
        inQ.y = __shfl_up_sync(0xffffffffu, nQ[E - 1].y, 1);
        inB.x = __shfl_up_sync(0xffffffffu, nb[E - 1].x, 1);
        inB.y = __shfl_up_sync(0xffffffffu, nb[E - 1].y, 1);
        if (lane == 31) {
            edge[(buf * 32 + warp) * 2 + 0] = nQ[E - 1];
            edge[(buf * 32 + warp) * 2 + 1] = nb[E - 1];
        }
        asm volatile("bar.sync 1, %0;" ::"r"(nact));
        if (lane == 0) {
            if (warp == 0) {
                inQ = make_double2(0.0, 0.0);
                inB = make_double2(0.0, 0.0);
            } else {
                inQ = edge[(buf * 32 + warp - 1) * 2 + 0];
                inB = edge[(buf * 32 + warp - 1) * 2 + 1];
            }
        }
#pragma unroll
        for (int e = E - 1; e >= 1; --e) { Qs[e] = nQ[e - 1]; bs[e] = nb[e - 1]; }
        Qs[0] = inQ;
        bs[0] = inB;
    }
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int j = tid * E + e;
        if (j < M) p.taps[(size_t)blockIdx.x * M + j] = make_float2((float)x[e].x, (float)x[e].y);
    }
    if (tid == 0) p.status[blockIdx.x] = bad;
}

// ------------------------------------------------------------------------------------------
// Doppler stage: P[j][lag] = sum_chunks partial[j][c][lag];  X = FFT_j(P);  out[(f+F/2)%F][R-lag]
// ------------------------------------------------------------------------------------------
__global__ void twiddle_kernel(float2* tw, int F) {      // tw[m] = exp(-2 pi i m / F), m < F
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m < F) {
        double s, c;
        sincospi(-2.0 * (double)m / (double)F, &s, &c);
        tw[m] = make_float2((float)c, (float)s);
    }
}

struct DopplerParams {
    const float2* partial;   // [F][nchunk][HT]
    const float2* tw;        // [F]
    float2* out;             // [F][R+1]
    int F;
    int logF;
    int R;
    int nchunk;              // partial rows reserved per Doppler block
    int HT;
    int blk_len;             // stream layout (lagstream_kernel): rows actually written for block j =
    long long per_cta;       //   stream_pieces(j, blk_len, per_cta); per_cta == 0: all nchunk rows
    // optional boundary sample of every Doppler block, i = j*bstride + boff, added to its lag sums
    // (bx == nullptr: none; every launch in prcore_corr.cu leaves it null)
    const float2* bx;
    const float2* bs;
    const float* bwin;       // optional: bx is the unweighted reference, multiply by bwin[i]
    long long bstride, boff;
    int n;
    long long partial_fstride, out_fstride;   // batch of frames in blockIdx.y (float2 elements; 0 for a single frame)
};

__device__ __forceinline__ float2 doppler_boundary(const DopplerParams& p, int j, int k) {
    const long long i = (long long)j * p.bstride + p.boff;
    if (p.bx == nullptr || i < 0 || i >= p.n) return make_float2(0.f, 0.f);
    float2 xv = p.bx[i];
    if (p.bwin) {                                  // x = ref * window formed here (no complex64 copy of it exists)
        const float w = p.bwin[i];
        xv.x *= w;
        xv.y *= w;
    }
    const float2 sv = p.bs[(i + (p.R - k)) % p.n];
    return make_float2(xv.x * sv.x + xv.y * sv.y, xv.y * sv.x - xv.x * sv.y);      // x * conj(s)
}

__device__ __forceinline__ int doppler_rows(const DopplerParams& p, int j) {
    return p.per_cta > 0 ? stream_pieces(j, p.blk_len, p.per_cta) : p.nchunk;
}

// power-of-two F: radix-2 Stockham autosort in shared memory, CT range columns per CTA
template <int CT>
__global__ void __launch_bounds__(256) doppler_fft_pow2_kernel(const __grid_constant__ DopplerParams p) {
    extern __shared__ __align__(16) float2 smem[];
    const int F = p.F;
    float2* a = smem;
    float2* b = smem + (size_t)F * CT;
    const int k0 = blockIdx.x * CT;
    const int tid = threadIdx.x;
    for (int idx = tid; idx < F * CT; idx += blockDim.x) {
        const int j = idx / CT, c = idx - j * CT;
        const int k = k0 + c;
        float2 sum = make_float2(0.f, 0.f);
        if (k <= p.R) {
            const float2* src = p.partial + (size_t)blockIdx.y * p.partial_fstride + (size_t)j * p.nchunk * p.HT + (p.R - k);
            const int rows = doppler_rows(p, j);
            for (int ch = 0; ch < rows; ++ch) {
                const float2 v = src[(size_t)ch * p.HT];
                sum.x += v.x;
                sum.y += v.y;
            }
            const float2 bv = doppler_boundary(p, j, k);
            sum.x += bv.x;
            sum.y += bv.y;
        }
        a[idx] = sum;
    }
    __syncthreads();
    const int half = F >> 1;
    for (int st = 0; st < p.logF; ++st) {
        const int Ns = 1 << st;
        for (int idx = tid; idx < half * CT; idx += blockDim.x) {
            const int bf = idx / CT, c = idx - bf * CT;
            const int kk = bf & (Ns - 1);
            const float2 w = p.tw[kk * (half >> st)];          // exp(-2 pi i kk / (2 Ns))
            const float2 u = a[bf * CT + c];
            const float2 v0 = a[(bf + half) * CT + c];
            const float2 v = make_float2(v0.x * w.x - v0.y * w.y, v0.x * w.y + v0.y * w.x);
            const int j0 = ((bf - kk) << 1) + kk;
            b[j0 * CT + c] = make_float2(u.x + v.x, u.y + v.y);
            b[(j0 + Ns) * CT + c] = make_float2(u.x - v.x, u.y - v.y);
        }
        __syncthreads();
        float2* tmp = a; a = b; b = tmp;
    }
    for (int idx = tid; idx < F * CT; idx += blockDim.x) {
        const int fp = idx / CT, c = idx - fp * CT;
        const int k = k0 + c;
        if (k <= p.R) {
            const int f = (fp + half) & (F - 1);
            p.out[(size_t)blockIdx.y * p.out_fstride + (size_t)f * (p.R + 1) + k] = a[idx];
        }
    }
}

// any F: chunk-sum into a compact [F][R+1] buffer, then a direct DFT with an exact twiddle table
__global__ void chunk_sum_kernel(const float2* __restrict__ partial, float2* __restrict__ P,
                                 int F, int R, int nchunk, int HT, int blk_len, long long per_cta,
                                 const __grid_constant__ DopplerParams bp) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= F * (R + 1)) return;
    const int j = idx / (R + 1), k = idx - j * (R + 1);
    const float2* src = partial + (size_t)j * nchunk * HT + (R - k);
    float2 sum = make_float2(0.f, 0.f);
    const int rows = per_cta > 0 ? stream_pieces(j, blk_len, per_cta) : nchunk;
    for (int ch = 0; ch < rows; ++ch) {
        const float2 v = src[(size_t)ch * HT];
        sum.x += v.x;
        sum.y += v.y;
    }
    const float2 bv = doppler_boundary(bp, j, k);
    P[idx] = make_float2(sum.x + bv.x, sum.y + bv.y);
}

__global__ void doppler_dft_kernel(const float2* __restrict__ P, const float2* __restrict__ tw,
                                   float2* __restrict__ out, int F, int R) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int fp = blockIdx.y;
    if (k > R) return;
    float ax = 0.f, ay = 0.f;
    int m = 0;
    for (int j = 0; j < F; ++j) {
        const float2 v = P[(size_t)j * (R + 1) + k];
        const float2 w = tw[m];
        ax = fmaf(v.x, w.x, ax); ax = fmaf(-v.y, w.y, ax);
        ay = fmaf(v.x, w.y, ay); ay = fmaf(v.y, w.x, ay);
        m += fp;
        if (m >= F) m -= F;
    }
    const int f = (fp + F / 2) % F;
    out[(size_t)f * (R + 1) + k] = make_float2(ax, ay);
}

// ------------------------------------------------------------------------------------------
// small element-wise helpers
// ------------------------------------------------------------------------------------------
// rs[i] = ref[(i + peek) mod n] * exp(i theta_j), j = (i + peek) mod n, theta_j = fl32(fl32(B * j) * fl32(1/Fs))
// (numpy divides a complex64 array by a real scalar as a multiplication by the float32 reciprocal):
// np.roll(frequency_shift(ref, fc, Fs), -peek) with the reference's float32 phase ramp
// (signal_utils.py:24-27: arange(..., dtype=complex64)); shift == 0 is a plain roll.
__global__ void shift_roll_kernel(const float2* __restrict__ ref, float2* __restrict__ rs, int n, int peek,
                                  int shift, float B, float rFs, long long frame_stride = 0) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ref += (size_t)blockIdx.y * frame_stride;          // a batch of frames in blockIdx.y
    rs += (size_t)blockIdx.y * frame_stride;
    int j = i + peek;
    if (j >= n) j %= n;
    float2 v = ref[j];
    if (shift) {
        const float th = __fmul_rn(__fmul_rn(B, (float)j), rFs);
        float sn, cs;
        sincosf(th, &sn, &cs);
        v = make_float2(__fmaf_rn(v.x, cs, -__fmul_rn(v.y, sn)), __fmaf_rn(v.x, sn, __fmul_rn(v.y, cs)));
    }
    rs[i] = v;
}

__global__ void f64_to_f32_kernel(const double* __restrict__ in, float* __restrict__ out, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)in[i];
}

}  // namespace prc
