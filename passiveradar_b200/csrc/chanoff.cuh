// chanoff.cuh -- channel-offset estimator (reference passiveRadar/signal_utils.py:29-78): zero-phase Chebyshev
// decimator (scipy.signal.decimate = sosfiltfilt + stride), a large float64 FFT correlation and the argmax of |xc|.
// Everything is float64 / complex128 whatever the input dtype (DESIGN.md section 11).
//
//   chanoff_iir      one pass of the order-8 (4 biquad) IIR cascade, chunked: one chunk per thread, every chunk
//                    but the first of a pass starts from a zero state W samples before its own start
//   chanoff_load     raw input widened to complex128 into a transform buffer (xcorr: no filter)
//   chanoff_twiddle  two-level float64 twiddle table exp(-2 pi i e / L) = hi[e >> TW_LO_BITS] * lo[e & mask]
//   chanoff_fft      one pass (<= 11 radix-2 stages) of the in-place transform in shared memory: forward
//                    decimation in frequency (natural in, bit-reversed out), inverse decimation in time
//                    (bit-reversed in, natural out); the first inverse pass multiplies X * conj(Y) on load
//   chanoff_argmax   the valid lags: |xc| (optionally written out) with a first-index argmax, or the lags themselves
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace prc {
namespace chanoff {

// input dtypes (include/prcore.h PRC_DT_*)
enum Dtype { DT_I8 = 0, DT_U8 = 1, DT_I16 = 2, DT_F32 = 3, DT_F64 = 4, DT_C64 = 5, DT_C128 = 6 };
inline bool dt_complex(int dt) { return dt == DT_C64 || dt == DT_C128; }
inline size_t dt_size(int dt) {
    switch (dt) {
        case DT_I8: case DT_U8: return 1;
        case DT_I16: return 2;
        case DT_F32: return 4;
        case DT_F64: case DT_C64: return 8;
        default: return 16;
    }
}

constexpr int PADLEN = 27;              // sosfiltfilt's default 3 * (2 * n_sections + 1)
constexpr int NSEC = 4;                 // cheby1(8, ...) as second-order sections
constexpr int IIR_THREADS = 128;
constexpr int FFT_THREADS = 256;
constexpr int FFT_TILE_BITS = 11;       // 2048 complex128 = 32 KB of shared memory per CTA
constexpr int TW_LO_BITS = 11;
constexpr int ARG_THREADS = 256;
constexpr int ARG_MAX_BLOCKS = 1024;

struct Sos { double s[NSEC][6]; double zi[NSEC][2]; };

// element i of the input widened to double (component `im` of a complex sample)
__device__ __forceinline__ double load_raw(const void* p, int dt, long long i, int im) {
    switch (dt) {
        case DT_I8: return (double)static_cast<const int8_t*>(p)[i];
        case DT_U8: return (double)static_cast<const uint8_t*>(p)[i];
        case DT_I16: return (double)static_cast<const int16_t*>(p)[i];
        case DT_F32: return (double)static_cast<const float*>(p)[i];
        case DT_F64: return static_cast<const double*>(p)[i];
        case DT_C64: return (double)static_cast<const float*>(p)[2 * i + im];
        default: return static_cast<const double*>(p)[2 * i + im];
    }
}

// 2 * x[a] - x[b] of odd_ext, in the input's own arithmetic: NumPy evaluates it in the integer dtype, wrapping
// (int8 2 * 100 - (-100) is -56); for float inputs the double evaluation is exact
__device__ __forceinline__ double odd_ext(const void* p, int dt, long long a, long long b, int im) {
    switch (dt) {
        case DT_I8: {
            const int8_t* q = static_cast<const int8_t*>(p);
            return (double)(int8_t)(2 * (int)q[a] - (int)q[b]);
        }
        case DT_U8: {
            const uint8_t* q = static_cast<const uint8_t*>(p);
            return (double)(uint8_t)(2 * (int)q[a] - (int)q[b]);
        }
        case DT_I16: {
            const int16_t* q = static_cast<const int16_t*>(p);
            return (double)(int16_t)(2 * (int)q[a] - (int)q[b]);
        }
        default: return 2.0 * load_raw(p, dt, a, im) - load_raw(p, dt, b, im);
    }
}

struct IirParams {
    Sos f;
    const void* x;          // forward: the raw input (dtype dt); backward: the forward pass output (double / double2)
    int dt;
    long long n;            // input samples
    long long next;         // n + 2 * PADLEN
    long long chunk;        // samples per thread
    long long warm;         // W: warm-up samples of a chunk that does not start the pass
    void* y;                // forward: next samples (double / double2); backward: decimated output (double2)
    int nd;
};

// ext[i] of sosfiltfilt's odd extension, component im
__device__ __forceinline__ double ext_at(const IirParams& p, long long i, int im) {
    if (i < PADLEN) return odd_ext(p.x, p.dt, 0, PADLEN - i, im);
    if (i < PADLEN + p.n) return load_raw(p.x, p.dt, i - PADLEN, im);
    const long long j = i - PADLEN - p.n;                    // 0 .. PADLEN-1
    return odd_ext(p.x, p.dt, p.n - 1, p.n - 2 - j, im);
}

template <bool CPLX>
struct Val { double v[CPLX ? 2 : 1]; };

// one sample through the cascade (scipy's _sosfilt: transposed direct form II per section)
template <bool CPLX>
__device__ __forceinline__ Val<CPLX> sos_step(const Sos& f, double (&z)[NSEC][2][CPLX ? 2 : 1], Val<CPLX> x) {
#pragma unroll
    for (int s = 0; s < NSEC; ++s) {
        Val<CPLX> y;
#pragma unroll
        for (int c = 0; c < (CPLX ? 2 : 1); ++c) {
            const double xc = x.v[c];
            const double yc = fma(f.s[s][0], xc, z[s][0][c]);
            z[s][0][c] = fma(f.s[s][1], xc, fma(-f.s[s][4], yc, z[s][1][c]));
            z[s][1][c] = fma(f.s[s][2], xc, -f.s[s][5] * yc);
            y.v[c] = yc;
        }
        x = y;
    }
    return x;
}

// BACKWARD = false: y[i] = sosfilt(sos, ext, zi * ext[0])[i], i < next.
// BACKWARD = true : runs on the reversed forward output r[i'] = y[next - 1 - i'] from zi * r[0] and writes sample
//                   j = next - 1 - i' - PADLEN of the (stripped, zero-phase) result to out[j / nd] when j % nd == 0.
template <bool CPLX, bool BACKWARD>
__global__ void __launch_bounds__(IIR_THREADS) chanoff_iir_kernel(const IirParams p) {
    constexpr int NC = CPLX ? 2 : 1;
    const long long c = (long long)blockIdx.x * IIR_THREADS + threadIdx.x;
    const long long i0 = c * p.chunk;
    if (i0 >= p.next) return;
    const long long i1 = min(i0 + p.chunk, p.next);
    long long i = i0 - p.warm;
    double z[NSEC][2][NC];
    auto in = [&](long long q) {
        Val<CPLX> v;
        if (BACKWARD) {
            const double* f = static_cast<const double*>(p.x) + (p.next - 1 - q) * NC;
#pragma unroll
            for (int k = 0; k < NC; ++k) v.v[k] = f[k];
        } else {
#pragma unroll
            for (int k = 0; k < NC; ++k) v.v[k] = ext_at(p, q, k);
        }
        return v;
    };
    if (i <= 0) {                   // this chunk starts the pass: the exact initial state
        i = 0;
        const Val<CPLX> x0 = in(0);
#pragma unroll
        for (int s = 0; s < NSEC; ++s)
#pragma unroll
            for (int k = 0; k < NC; ++k) { z[s][0][k] = p.f.zi[s][0] * x0.v[k]; z[s][1][k] = p.f.zi[s][1] * x0.v[k]; }
    } else {
#pragma unroll
        for (int s = 0; s < NSEC; ++s)
#pragma unroll
            for (int k = 0; k < NC; ++k) { z[s][0][k] = 0.0; z[s][1][k] = 0.0; }
    }
    for (; i < i0; ++i) sos_step<CPLX>(p.f, z, in(i));
    if (!BACKWARD) {
        double* y = static_cast<double*>(p.y);
        for (; i < i1; ++i) {
            const Val<CPLX> v = sos_step<CPLX>(p.f, z, in(i));
#pragma unroll
            for (int k = 0; k < NC; ++k) y[i * NC + k] = v.v[k];
        }
    } else {
        double2* out = static_cast<double2*>(p.y);
        long long j = p.next - 1 - i - PADLEN;                 // output sample of reversed position i
        long long rem = j >= 0 ? j % p.nd : 0;
        for (; i < i1; ++i, --j) {
            const Val<CPLX> v = sos_step<CPLX>(p.f, z, in(i));
            if (j >= 0 && j < p.n && rem == 0) out[j / p.nd] = make_double2(v.v[0], CPLX ? v.v[NC - 1] : 0.0);
            rem = rem == 0 ? p.nd - 1 : rem - 1;
        }
    }
}

// x (dtype dt, n samples) -> dst[0 .. n) complex128
__global__ void chanoff_load_kernel(const void* x, int dt, long long n, double2* dst) {
    const bool cplx = dt == DT_C64 || dt == DT_C128;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        dst[i] = make_double2(load_raw(x, dt, i, 0), cplx ? load_raw(x, dt, i, 1) : 0.0);
}

// lo[k] = exp(-2 pi i k / L), k < 2^TW_LO_BITS;  hi[k] = exp(-2 pi i k 2^TW_LO_BITS / L), k < nhi
__global__ void chanoff_twiddle_kernel(double2* lo, double2* hi, int nhi, int m) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const double inv = ldexp(-2.0, -m);                     // -2 / L: sincospi takes multiples of pi
    double s, c;
    if (k < (1 << TW_LO_BITS)) { sincospi(inv * k, &s, &c); lo[k] = make_double2(c, s); }
    if (k < nhi) { sincospi(inv * ((double)k * (1 << TW_LO_BITS)), &s, &c); hi[k] = make_double2(c, s); }
}

struct FftParams {
    double2* buf[2];            // forward: blockIdx.y picks X or Y; inverse: buf[0] = X (in/out), buf[1] = Y
    const double2* tw_lo;
    const double2* tw_hi;
    int m;                      // L = 2^m
    int lo, nb, c;              // the pass works on index bits [lo, lo + nb), 2^c consecutive columns per tile
    int s0;                     // global stage index of the pass's first (highest-span) stage
    int product;                // inverse only: load X * conj(Y)
};

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
    return make_double2(fma(a.x, b.x, -a.y * b.y), fma(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ double2 cmulc(double2 a, double2 b) {      // a * conj(b)
    return make_double2(fma(a.x, b.x, a.y * b.y), fma(a.y, b.x, -a.x * b.y));
}

template <bool INVERSE>
__global__ void __launch_bounds__(FFT_THREADS) chanoff_fft_kernel(const FftParams p) {
    __shared__ double2 sm[1 << FFT_TILE_BITS];
    double2* g = (!INVERSE && blockIdx.y) ? p.buf[1] : p.buf[0];
    const int S = 1 << (p.nb + p.c);
    const int ucols = 1 << p.c;
    const long long tile = blockIdx.x;
    const int tshift = p.lo - p.c;                          // tiles per high part = 2^(lo - c)
    const long long hi = tile >> tshift;
    const long long u0 = (tile & ((1ll << tshift) - 1)) << p.c;
    auto gidx = [&](int e) {
        const long long t = e >> p.c, u = e & (ucols - 1);
        return (hi << (p.lo + p.nb)) | (t << p.lo) | (u0 + u);
    };
    for (int e = threadIdx.x; e < S; e += FFT_THREADS) {
        const long long q = gidx(e);
        sm[e] = (INVERSE && p.product) ? cmulc(g[q], p.buf[1][q]) : g[q];
    }
    __syncthreads();
    const int half_tiles = S >> 1;
    const long long twmask = (1ll << TW_LO_BITS) - 1;
    for (int rr = 0; rr < p.nb; ++rr) {
        const int r = INVERSE ? p.nb - 1 - rr : rr;         // local stage; span 2^(nb - 1 - r) rows
        const int half = 1 << (p.nb - 1 - r);
        const int s = p.s0 + r;
        for (int b = threadIdx.x; b < half_tiles; b += FFT_THREADS) {
            const int u = b & (ucols - 1), bt = b >> p.c;
            const int tt = (bt / half) * 2 * half + (bt % half);
            const int e1 = (tt << p.c) | u, e2 = ((tt + half) << p.c) | u;
            const long long ex = ((((long long)(tt % half)) << p.lo) | (u0 + u)) << s;   // (i mod h) * 2^s < L / 2
            double2 w = cmul(p.tw_hi[ex >> TW_LO_BITS], p.tw_lo[ex & twmask]);
            const double2 a = sm[e1], bb = sm[e2];
            if (!INVERSE) {
                sm[e1] = make_double2(a.x + bb.x, a.y + bb.y);
                sm[e2] = cmul(make_double2(a.x - bb.x, a.y - bb.y), w);
            } else {
                w.y = -w.y;
                const double2 t = cmul(bb, w);
                sm[e1] = make_double2(a.x + t.x, a.y + t.y);
                sm[e2] = make_double2(a.x - t.x, a.y - t.y);
            }
        }
        __syncthreads();
    }
    for (int e = threadIdx.x; e < S; e += FFT_THREADS) g[gidx(e)] = sm[e];
}

enum ArgMode { ARG_ABS = 0, ARG_COMPLEX = 1, ARG_REAL = 2 };

struct ArgParams {
    const double2* cc;          // L-point circular correlation times L (natural order)
    long long L, nvalid, p0;    // valid lag k reads cc[(k + p0) mod L]
    double scale;               // 1 / L
    int mode;
    void* out;                  // ARG_ABS: |xc| (double, optional); else the lags (double2 / double)
    double* part_v;             // per-block maximum of |xc| and its first index
    long long* part_k;
};

__device__ __forceinline__ void arg_take(double& bv, long long& bk, double v, long long k) {
    if (v > bv || (v == bv && k < bk)) { bv = v; bk = k; }
}

__device__ __forceinline__ void arg_block(double& bv, long long& bk) {
    __shared__ double sv[ARG_THREADS / 32];
    __shared__ long long sk[ARG_THREADS / 32];
    for (int o = 16; o; o >>= 1) arg_take(bv, bk, __shfl_down_sync(0xffffffffu, bv, o), __shfl_down_sync(0xffffffffu, bk, o));
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = bv; sk[threadIdx.x >> 5] = bk; }
    __syncthreads();
    if (threadIdx.x < 32) {
        bv = threadIdx.x < ARG_THREADS / 32 ? sv[threadIdx.x] : -1.0;
        bk = threadIdx.x < ARG_THREADS / 32 ? sk[threadIdx.x] : (long long)INT64_MAX;
        for (int o = 16; o; o >>= 1) arg_take(bv, bk, __shfl_down_sync(0xffffffffu, bv, o), __shfl_down_sync(0xffffffffu, bk, o));
    }
}

__global__ void __launch_bounds__(ARG_THREADS) chanoff_argmax_kernel(const ArgParams p) {
    double bv = -1.0;
    long long bk = INT64_MAX;
    for (long long k = (long long)blockIdx.x * ARG_THREADS + threadIdx.x; k < p.nvalid; k += (long long)gridDim.x * ARG_THREADS) {
        const double2 v0 = p.cc[(k + p.p0) & (p.L - 1)];
        const double2 v = make_double2(v0.x * p.scale, v0.y * p.scale);
        if (p.mode == ARG_ABS) {
            const double a = hypot(v.x, v.y);
            if (p.out) static_cast<double*>(p.out)[k] = a;
            if (a > bv) { bv = a; bk = k; }                  // a thread's k increase: strict > keeps the first
        } else if (p.mode == ARG_COMPLEX) {
            static_cast<double2*>(p.out)[k] = v;
        } else {
            static_cast<double*>(p.out)[k] = v.x;
        }
    }
    if (p.mode != ARG_ABS) return;
    arg_block(bv, bk);
    if (threadIdx.x == 0) { p.part_v[blockIdx.x] = bv; p.part_k[blockIdx.x] = bk; }
}

// res[0] = first argmax, res[1] = (argmax - nl) * nd
__global__ void __launch_bounds__(ARG_THREADS) chanoff_argmax_final_kernel(const double* part_v, const long long* part_k,
                                                                        int nparts, long long nl, long long nd,
                                                                        long long* res) {
    double bv = -1.0;
    long long bk = INT64_MAX;
    for (int q = threadIdx.x; q < nparts; q += ARG_THREADS) arg_take(bv, bk, part_v[q], part_k[q]);
    arg_block(bv, bk);
    if (threadIdx.x == 0) { res[0] = bk; res[1] = (bk - nl) * nd; }
}

// ---- launches (host side; prcore.cu brackets them with its profiling scopes and checks the launch) ----------------
template <bool CPLX, bool BACKWARD>
inline void launch_iir_t(const IirParams& p, cudaStream_t st) {
    const long long nchunk = (p.next + p.chunk - 1) / p.chunk;
    chanoff_iir_kernel<CPLX, BACKWARD><<<(unsigned)((nchunk + IIR_THREADS - 1) / IIR_THREADS), IIR_THREADS, 0, st>>>(p);
}

inline void launch_iir(const IirParams& p, bool cplx, bool backward, cudaStream_t st) {
    if (cplx) { if (backward) launch_iir_t<true, true>(p, st); else launch_iir_t<true, false>(p, st); }
    else { if (backward) launch_iir_t<false, true>(p, st); else launch_iir_t<false, false>(p, st); }
}

inline void launch_load(const void* x, int dt, long long n, double2* dst, int nsm, cudaStream_t st) {
    const long long want = (n + 255) / 256;
    chanoff_load_kernel<<<(unsigned)(want < 8ll * nsm ? (want > 0 ? want : 1) : 8ll * nsm), 256, 0, st>>>(x, dt, n, dst);
}

inline void launch_twiddle(double2* lo, double2* hi, int nhi, int m, cudaStream_t st) {
    const int n = nhi > (1 << TW_LO_BITS) ? nhi : (1 << TW_LO_BITS);
    chanoff_twiddle_kernel<<<(n + 255) / 256, 256, 0, st>>>(lo, hi, nhi, m);
}

inline void launch_fft_pass(const FftParams& p, bool inverse, cudaStream_t st) {
    const unsigned tiles = (unsigned)(1ll << (p.m - p.nb - p.c));
    if (inverse) chanoff_fft_kernel<true><<<tiles, FFT_THREADS, 0, st>>>(p);
    else chanoff_fft_kernel<false><<<dim3(tiles, 2), FFT_THREADS, 0, st>>>(p);
}

inline int argmax_blocks(long long nvalid) {
    const long long b = (nvalid + ARG_THREADS * 8 - 1) / (ARG_THREADS * 8);
    return (int)(b < 1 ? 1 : (b > ARG_MAX_BLOCKS ? ARG_MAX_BLOCKS : b));
}

inline void launch_argmax(const ArgParams& p, int nblocks, cudaStream_t st) {
    chanoff_argmax_kernel<<<nblocks, ARG_THREADS, 0, st>>>(p);
}

inline void launch_argmax_final(const double* pv, const long long* pk, int nparts, long long nl, long long nd,
                                long long* res, cudaStream_t st) {
    chanoff_argmax_final_kernel<<<1, ARG_THREADS, 0, st>>>(pv, pk, nparts, nl, nd, res);
}

}  // namespace chanoff
}  // namespace prc
