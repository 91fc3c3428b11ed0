// decimate.cuh -- scipy.signal.decimate(x, q, 20q, ftype='fir', axis=0) on rows of samples, the same decimator fed from
// raw interleaved I/Q (channel_preprocessing: deinterleave, frequency_shift, decimate in one pass), and normalize
// (x / mean|x|).  DESIGN.md section 18.
//
//   y[m] = sum_{j=0}^{20q} b[j] x[m q + 10 q - j],   x = 0 outside [0, n),   m = 0 .. ceil(n / q) - 1
//
// Write j = p + q t (p < q, t = 0 .. 20) and X_u[p] = x[u q - p]: y[m] = sum_t sum_p b[p + q t] X_{m+10-t}[p].  A CTA owns
// MT consecutive outputs, so it reads the MT + 20 input blocks u = m0 - 10 .. m0 + MT + 9 and the 21 tap rows b[. + q t].
// Both are staged in slabs of KS columns p (KS <= 4 G), so shared memory does not grow with q.  A group of G lanes owns
// R = 4 consecutive outputs: lane l takes the columns p = l, l + G, ... of every slab, keeps the 21 taps of its column in
// registers and slides over the R + 20 input rows the group's outputs read, so each staged sample feeds up to 4 MACs.
// After the last slab the G partial sums of each output are added with shuffles in a fixed tree.  Nothing depends on
// the row count or on where a row sits in the batch, so a row of a batch is bit-identical to a one-row call on it.
//
// G grows with q (4 at q < 16, up to 32 at q >= 64): every lane has at least two columns of work and the input a CTA
// stages is (MT + 20) / MT of its own share: 1.08x at G = 4, 1.6x at G = 32.  The staged rows are padded to a stride
// that makes a warp's loads conflict-free (ksp below).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "frontend.cuh"

namespace prc {
namespace dec {

// sources (include/prcore.h): PRC_DT_* of a typed row, or SRC_RAW + PRC_IQ_* for raw interleaved I/Q that is mixed on load
enum Src { DT_I8 = 0, DT_U8 = 1, DT_I16 = 2, DT_F32 = 3, DT_F64 = 4, DT_C64 = 5, DT_C128 = 6, SRC_RAW = 16 };

constexpr int THREADS = 256;
constexpr int R = 4;                    // consecutive outputs per lane group
constexpr int NT = 21;                  // tap rows t = 0 .. 20
constexpr int MIN_Q = 2;
constexpr int MAX_Q = 1 << 16;          // 20 q + 1 = 1 310 721 taps at most

struct DecParams {
    const void* x;          // row b at x + b * row_stride elements (complex samples for raw I/Q)
    int src;                // Src
    MixParams mix;          // SRC_RAW: kind, mode and ramp constants (mix.in is replaced by the row's start)
    long long n;            // samples per row
    long long row_stride;
    int q;
    int G;                  // lanes per output group: 4, 8, 16 or 32
    int ks, ksp;            // columns per slab (a multiple of G), padded row stride of the staged input
    int nslab;              // ceil(q / ks)
    long long nout;         // ceil(n / q)
    const void* taps;       // 20 q + 1 taps, float or double as the accumulator
    void* y;                // row b at y + b * out_stride outputs
    long long out_stride;
    int row0;               // first row of the launch
};

// ---- the work split: every quantity depends on q alone ----------------------------------------------------------------
inline int group_lanes(int q) {
    int p2 = 1;
    while (p2 * 2 <= q) p2 *= 2;                       // largest power of two <= q
    const int g = p2 / 2;
    return g < 4 ? 4 : g > 32 ? 32 : g;
}
inline int outputs_per_cta(int G) { return THREADS / G * R; }
// slab: at most 4 G columns, the fewest slabs, columns a multiple of G
inline void slab_geometry(int q, int G, int* ks, int* ksp, int* nslab) {
    const int ns = (q + 4 * G - 1) / (4 * G);
    const int per = (q + ns - 1) / ns;
    *ks = (per + G - 1) / G * G;
    *nslab = (q + *ks - 1) / *ks;
    // rows g R apart must fall in distinct banks for the G lanes of each group: ksp / (G / R) odd
    const int c = G / R;
    int k = (*ks + c - 1) / c;
    if (!(k & 1)) ++k;
    *ksp = k * c;
}

template <class V> struct VT;
template <> struct VT<float> { using S = float; };
template <> struct VT<float2> { using S = float; };
template <> struct VT<double> { using S = double; };
template <> struct VT<double2> { using S = double; };

template <class V> size_t smem_bytes(int G, int ks, int ksp) {
    using S = typename VT<V>::S;
    const size_t tb = ((size_t)NT * ks * sizeof(S) + 15) & ~(size_t)15;
    return tb + (size_t)(outputs_per_cta(G) + NT - 1) * ksp * sizeof(V);
}

__device__ __forceinline__ void zero(float& a) { a = 0.f; }
__device__ __forceinline__ void zero(double& a) { a = 0.0; }
__device__ __forceinline__ void zero(float2& a) { a = make_float2(0.f, 0.f); }
__device__ __forceinline__ void zero(double2& a) { a = make_double2(0.0, 0.0); }
__device__ __forceinline__ void mac(float& a, float b, float x) { a = fmaf(b, x, a); }
__device__ __forceinline__ void mac(double& a, double b, double x) { a = fma(b, x, a); }
__device__ __forceinline__ void mac(float2& a, float b, float2 x) { a.x = fmaf(b, x.x, a.x); a.y = fmaf(b, x.y, a.y); }
__device__ __forceinline__ void mac(double2& a, double b, double2 x) { a.x = fma(b, x.x, a.x); a.y = fma(b, x.y, a.y); }
__device__ __forceinline__ void add_down(float& a, int off, int G) { a += __shfl_down_sync(0xffffffffu, a, off, G); }
__device__ __forceinline__ void add_down(double& a, int off, int G) { a += __shfl_down_sync(0xffffffffu, a, off, G); }
__device__ __forceinline__ void add_down(float2& a, int off, int G) {
    a.x += __shfl_down_sync(0xffffffffu, a.x, off, G);
    a.y += __shfl_down_sync(0xffffffffu, a.y, off, G);
}
__device__ __forceinline__ void add_down(double2& a, int off, int G) {
    a.x += __shfl_down_sync(0xffffffffu, a.x, off, G);
    a.y += __shfl_down_sync(0xffffffffu, a.y, off, G);
}

// sample i of row b, in the accumulator's type
// (mix_sample reads the grid constants in place: a local copy of MixParams would be kept in the stack frame)
__device__ __forceinline__ float2 raw_sample(const DecParams& p, int b, long long i) {
    const int kind = p.mix.kind;
    const void* in = static_cast<const char*>(p.x) + (size_t)b * p.row_stride * (kind == IQ_I8 ? 2 : kind == IQ_I16 ? 4 : 8);
    return mix_sample(p.mix, iq_load_scalar(in, kind, i), i);
}
template <class V> __device__ V load(const DecParams& p, int b, long long i);
template <> __device__ __forceinline__ float load<float>(const DecParams& p, int b, long long i) {
    return static_cast<const float*>(p.x)[b * p.row_stride + i];
}
template <> __device__ __forceinline__ float2 load<float2>(const DecParams& p, int b, long long i) {
    if (p.src >= SRC_RAW) return raw_sample(p, b, i);
    return static_cast<const float2*>(p.x)[b * p.row_stride + i];
}
template <> __device__ __forceinline__ double load<double>(const DecParams& p, int b, long long i) {
    const long long k = b * p.row_stride + i;
    if (p.src == DT_I8) return (double)static_cast<const signed char*>(p.x)[k];
    if (p.src == DT_U8) return (double)static_cast<const unsigned char*>(p.x)[k];
    if (p.src == DT_I16) return (double)static_cast<const short*>(p.x)[k];
    return static_cast<const double*>(p.x)[k];
}
template <> __device__ __forceinline__ double2 load<double2>(const DecParams& p, int b, long long i) {
    if (p.src >= SRC_RAW) {
        const float2 v = raw_sample(p, b, i);           // the reference's float64 modes: a complex64 sample widened
        return make_double2((double)v.x, (double)v.y);
    }
    return static_cast<const double2*>(p.x)[b * p.row_stride + i];
}

template <class V>
__global__ void __launch_bounds__(THREADS, sizeof(V) == 16 ? 2 : 4) dec_kernel(const __grid_constant__ DecParams p) {
    using S = typename VT<V>::S;
    extern __shared__ __align__(16) unsigned char dec_smem[];
    S* bs = reinterpret_cast<S*>(dec_smem);                                                  // [NT][ks]
    V* xs = reinterpret_cast<V*>(dec_smem + (((size_t)NT * p.ks * sizeof(S) + 15) & ~(size_t)15));   // [rows][ksp]
    const int G = p.G, ks = p.ks, ksp = p.ksp, q = p.q;
    const int mt = THREADS / G * R, rows = mt + NT - 1;
    const int b = p.row0 + blockIdx.y;
    const long long m0 = (long long)blockIdx.x * mt;
    const long long u0 = m0 - 10;                       // input block of staged row 0
    const int lane = threadIdx.x & (G - 1), g = threadIdx.x / G;
    const S* taps = static_cast<const S*>(p.taps);
    V acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) zero(acc[r]);
    for (int sl = 0; sl < p.nslab; ++sl) {
        const int p0 = sl * ks;
        if (sl) __syncthreads();                        // the previous slab has been consumed
        for (int e = threadIdx.x; e < NT * ks; e += THREADS) {
            const int t = e / ks, pc = p0 + (e - t * ks);
            const long long j = (long long)pc + (long long)q * t;
            bs[e] = (pc < q && j <= 20ll * q) ? taps[j] : (S)0;
        }
        // element e = s ks + pl of the slab, walked by the whole CTA with (s, pl) stepped without a division
        const int ds = THREADS / ks, dp = THREADS - ds * ks;
        int s = threadIdx.x / ks, pl = threadIdx.x - s * ks;
#pragma unroll 4
        for (; s < rows; s += ds, pl += dp) {
            if (pl >= ks) { pl -= ks; ++s; if (s >= rows) break; }
            const long long i = (u0 + s) * q - (p0 + pl);       // X_u[p] = x[u q - p]
            V v;
            zero(v);
            if (p0 + pl < q && i >= 0 && i < p.n) v = load<V>(p, b, i);
            xs[s * ksp + pl] = v;
        }
        __syncthreads();
        for (int pl = lane; pl < ks; pl += G) {
            S bt[NT];
#pragma unroll
            for (int t = 0; t < NT; ++t) bt[t] = bs[t * ks + pl];
            const bool last_row = p0 + pl == 0;         // b[p + 20 q] exists for p = 0 only
            const V* xr = xs + (size_t)g * R * ksp + pl;
#pragma unroll
            for (int s = 0; s < R + NT - 1; ++s) {      // output r of the group reads row r + 20 - t
                const V xv = xr[s * ksp];
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const int t = r + NT - 1 - s;
                    if (t >= 0 && t < NT - 1) mac(acc[r], bt[t], xv);
                    else if (t == NT - 1 && last_row) mac(acc[r], bt[t], xv);
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
        for (int off = G >> 1; off >= 1; off >>= 1) add_down(acc[r], off, G);
    if (lane == 0) {
        V* y = static_cast<V*>(p.y) + (size_t)b * p.out_stride;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const long long m = m0 + (long long)g * R + r;
            if (m < p.nout) y[m] = acc[r];
        }
    }
}

// ---- normalize: x / mean(|x|) -----------------------------------------------------------------------------------------
// norm_sum: CTA c adds |x| over its fixed share [c per_cta, (c + 1) per_cta) in float64 (thread-strided, then a tree in
// shared memory) and writes one partial.  norm_scale: every CTA adds the partials in one fixed order, divides by n and
// writes x / mean in NumPy's result dtype.  No atomics: the result is the same on every run.
constexpr int NORM_THREADS = 256;
constexpr int NORM_MAX_CTAS = 1024;

struct NormParams {
    const void* x;
    int dt;                 // PRC_DT_*
    long long n, per_cta;
    int nctas;
    double* part;           // nctas partial sums
    void* y;
};

// numpy's abs: integers keep their width, so abs(-128) of int8 and abs(-32768) of int16 wrap to themselves
__device__ __forceinline__ double abs_elem(const void* x, int dt, long long i) {
    switch (dt) {
        case DT_I8: { const int v = static_cast<const signed char*>(x)[i]; return (double)(signed char)(v < 0 ? -v : v); }
        case DT_U8: return (double)static_cast<const unsigned char*>(x)[i];
        case DT_I16: { const int v = static_cast<const short*>(x)[i]; return (double)(short)(v < 0 ? -v : v); }
        case DT_F32: return (double)fabsf(static_cast<const float*>(x)[i]);
        case DT_F64: return fabs(static_cast<const double*>(x)[i]);
        case DT_C64: {                                  // |z| of complex64 is float32: rounded from the exact value
            const float2 v = static_cast<const float2*>(x)[i];
            return (double)(float)hypot((double)v.x, (double)v.y);
        }
        default: { const double2 v = static_cast<const double2*>(x)[i]; return hypot(v.x, v.y); }
    }
}

__global__ void __launch_bounds__(NORM_THREADS) norm_sum_kernel(const NormParams p) {
    __shared__ double red[NORM_THREADS];
    const long long lo = (long long)blockIdx.x * p.per_cta;
    const long long hi = min(lo + p.per_cta, p.n);
    double s = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += NORM_THREADS) s += abs_elem(p.x, p.dt, i);
    red[threadIdx.x] = s;
    __syncthreads();
    for (int h = NORM_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) p.part[blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(NORM_THREADS) norm_scale_kernel(const NormParams p) {
    __shared__ double total;
    if (threadIdx.x < 32) {
        double s = 0.0;
        for (int c = threadIdx.x; c < p.nctas; c += 32) s += p.part[c];
        for (int off = 16; off >= 1; off >>= 1) s += __shfl_down_sync(0xffffffffu, s, off);
        if (threadIdx.x == 0) total = s;
    }
    __syncthreads();
    const double mean = total / (double)p.n;
    const long long stride = (long long)gridDim.x * NORM_THREADS;
    for (long long i = (long long)blockIdx.x * NORM_THREADS + threadIdx.x; i < p.n; i += stride) {
        switch (p.dt) {
            case DT_F32: {                              // float32 / float32(mean)
                static_cast<float*>(p.y)[i] = __fdiv_rn(static_cast<const float*>(p.x)[i], (float)mean);
                break;
            }
            case DT_C64: {                              // numpy divides complex by real as a product with 1 / d
                const float scl = __fdiv_rn(1.0f, (float)mean);
                const float2 v = static_cast<const float2*>(p.x)[i];
                static_cast<float2*>(p.y)[i] = make_float2(__fmul_rn(v.x, scl), __fmul_rn(v.y, scl));
                break;
            }
            case DT_C128: {
                const double scl = 1.0 / mean;
                const double2 v = static_cast<const double2*>(p.x)[i];
                static_cast<double2*>(p.y)[i] = make_double2(v.x * scl, v.y * scl);
                break;
            }
            case DT_F64: static_cast<double*>(p.y)[i] = static_cast<const double*>(p.x)[i] / mean; break;
            case DT_I8: static_cast<double*>(p.y)[i] = (double)static_cast<const signed char*>(p.x)[i] / mean; break;
            case DT_U8: static_cast<double*>(p.y)[i] = (double)static_cast<const unsigned char*>(p.x)[i] / mean; break;
            default: static_cast<double*>(p.y)[i] = (double)static_cast<const short*>(p.x)[i] / mean; break;
        }
    }
}

// ---- launches (host side; prcore.cu brackets them with its profiling scopes and checks the launch) --------------------
template <class V> inline cudaError_t set_attr_t(int lim) {
    return cudaFuncSetAttribute(dec_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim);
}
inline cudaError_t set_attrs(int lim) {
    const cudaError_t e[4] = {set_attr_t<float>(lim), set_attr_t<float2>(lim), set_attr_t<double>(lim),
                              set_attr_t<double2>(lim)};
    for (cudaError_t x : e)
        if (x != cudaSuccess) return x;
    return cudaSuccess;
}

// rows [row0, row0 + nrows) of one launch (nrows <= 65535)
template <class V> inline void launch_decimate_t(DecParams p, int row0, int nrows, cudaStream_t st) {
    p.row0 = row0;
    const int mt = outputs_per_cta(p.G);
    const dim3 grid((unsigned)((p.nout + mt - 1) / mt), (unsigned)nrows);
    dec_kernel<V><<<grid, THREADS, smem_bytes<V>(p.G, p.ks, p.ksp), st>>>(p);
}

// the accumulator a source decimates in: 0 float, 1 float2, 2 double, 3 double2
inline int acc_kind(int src, int mode) {
    if (src >= SRC_RAW) return (mode == MIX_NONE || mode == MIX_C64) ? 1 : 3;
    if (src == DT_F32) return 0;
    if (src == DT_C64) return 1;
    if (src == DT_C128) return 3;
    return 2;
}

inline size_t decimate_smem(int acc, int G, int ks, int ksp) {
    switch (acc) {
        case 0: return smem_bytes<float>(G, ks, ksp);
        case 1: return smem_bytes<float2>(G, ks, ksp);
        case 2: return smem_bytes<double>(G, ks, ksp);
        default: return smem_bytes<double2>(G, ks, ksp);
    }
}

inline void launch_decimate(const DecParams& p, int acc, int row0, int nrows, cudaStream_t st) {
    switch (acc) {
        case 0: launch_decimate_t<float>(p, row0, nrows, st); break;
        case 1: launch_decimate_t<float2>(p, row0, nrows, st); break;
        case 2: launch_decimate_t<double>(p, row0, nrows, st); break;
        default: launch_decimate_t<double2>(p, row0, nrows, st); break;
    }
}

inline int norm_ctas(long long n) {
    const long long c = (n + 4095) / 4096;
    return (int)(c < 1 ? 1 : c > NORM_MAX_CTAS ? NORM_MAX_CTAS : c);
}

inline void launch_norm_sum(const NormParams& p, cudaStream_t st) {
    norm_sum_kernel<<<p.nctas, NORM_THREADS, 0, st>>>(p);
}

inline void launch_norm_scale(const NormParams& p, int nsm, cudaStream_t st) {
    const long long need = (p.n + NORM_THREADS - 1) / NORM_THREADS;
    const long long grid = need < 8ll * nsm ? need : 8ll * nsm;
    norm_scale_kernel<<<(unsigned)(grid < 1 ? 1 : grid), NORM_THREADS, 0, st>>>(p);
}

}  // namespace dec
}  // namespace prc
