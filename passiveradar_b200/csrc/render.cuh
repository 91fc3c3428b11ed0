// render.cuh -- the frame chain of range_doppler_plot.py:45-85 (DESIGN.md section 15) after CFAR_2D of every frame
// (detect.cuh): the reference's persistence (passiveRadar/plotting_tools.py:9-30) along the frame axis, and the two
// per-frame percentiles that set the colour limits.
//
// pst_kernel: out[k] = sum_{i < min(k + 1, hold)} X[k - i] * w[i], summed from +0.0 in the order i = 0, 1, ... with
//   separate multiplies and adds (no contraction), the products in float32 when NumPy's promotion makes them so.  One
//   thread per cell walks the frames in order and keeps the last PST_RING inputs of its cell in shared memory, so an
//   input is read once per call (older ones, when hold > PST_RING, are read again, from L2).  The oriented output
//   fliplr(P.T) goes through a shared tile so that its stores stay contiguous.
// pct_kernel: one CTA per frame, NumPy's linear-method percentiles by track.cuh's radix select over order-preserving
//   keys; the radix passes of all the requested percentiles share one read of the frame.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "track.cuh"

namespace prc {
namespace rdr {

// ---- persistence -------------------------------------------------------------------------------------------------
constexpr int PST_TX = 32, PST_TY = 8;
constexpr int PST_RING = 20;                 // inputs of a cell kept in shared memory: the reference script's hold

struct PersistParams {
    const void* x;             // n_carry + nframes frames (float, or double with f64), frame f at x + f * frame_stride
    long long frame_stride;
    int f64;
    int f32prod;               // products float32(x) * float32(w) (NumPy promotion of a float32 stack), else float64
    int oriented;              // out frames are fliplr(P.T), (cols, rows); else P, (rows, cols)
    int rows, cols;
    int n_carry, nframes, hold;
    const double* w;           // hold weights decay**i
    double* out;               // nframes frames of rows * cols doubles
};

__device__ __forceinline__ double pst_load(const PersistParams& p, int f, long long o) {
    const long long e = (long long)f * p.frame_stride + o;
    return p.f64 ? __ldg(static_cast<const double*>(p.x) + e) : (double)__ldg(static_cast<const float*>(p.x) + e);
}

__global__ void __launch_bounds__(PST_TX * PST_TY) pst_kernel(const __grid_constant__ PersistParams p) {
    __shared__ double ring[PST_RING][PST_TX * PST_TY];
    __shared__ double tile[PST_TY][PST_TX + 1];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * PST_TX + tx;
    const int r0 = blockIdx.y * PST_TY, c0 = blockIdx.x * PST_TX;
    const int r = r0 + ty, c = c0 + tx;
    const bool in = r < p.rows && c < p.cols;
    const long long o = (long long)r * p.cols + c;
    const long long fsz = (long long)p.rows * p.cols;
    const int total = p.n_carry + p.nframes;
    for (int f = 0; f < total; ++f) {
        if (in) ring[f % PST_RING][tid] = pst_load(p, f, o);
        if (f < p.n_carry) continue;
        double s = 0.0;                                // np.zeros, then frame = frame + X[k - i] * decay**i
        if (in) {
            const int nt = min(f + 1, p.hold);
            for (int i = 0; i < nt; ++i) {
                const double xv = i < PST_RING ? ring[(f - i) % PST_RING][tid] : pst_load(p, f - i, o);
                const double wv = __ldg(p.w + i);
                const double prod = p.f32prod ? (double)__fmul_rn((float)xv, __double2float_rn(wv)) : __dmul_rn(xv, wv);
                s = __dadd_rn(s, prod);
            }
        }
        double* out = p.out + (long long)(f - p.n_carry) * fsz;
        if (!p.oriented) {
            if (in) out[o] = s;
            continue;
        }
        // fliplr(P.T)[c][rows - 1 - r] = P[r][c]: each of the tile's 32 columns becomes 8 contiguous outputs
        __syncthreads();                               // the previous frame's tile has been read
        tile[ty][tx] = s;
        __syncthreads();
        const int oc = c0 + tid / PST_TY, e = tid % PST_TY;
        const int orr = r0 + (PST_TY - 1 - e);
        if (oc < p.cols && orr < p.rows) out[(long long)oc * p.rows + (p.rows - 1 - orr)] = tile[PST_TY - 1 - e][tid / PST_TY];
    }
}

// ---- per-frame percentiles ---------------------------------------------------------------------------------------
constexpr int PCT_THREADS = 512;
constexpr int PCT_MAX_Q = 4;
constexpr int PCT_MAX_N = 0x7fffffff - PCT_THREADS;   // largest frame: its int indices stay below INT_MAX

struct PctParams {
    const double* x;           // frame f at x + f * frame_stride
    long long frame_stride;
    int n, nq;
    int k[PCT_MAX_Q];          // order statistics k and k + 1 (both n - 1 when the virtual index reaches it) ...
    double g[PCT_MAX_Q];       // ... and NumPy's gamma between them
    double scale[PCT_MAX_Q];   // result * scale (__dmul_rn) when has_scale
    int has_scale;
    double* out;               // [nframes][nq]
};

__global__ void __launch_bounds__(PCT_THREADS) pct_kernel(const __grid_constant__ PctParams p) {
    __shared__ unsigned int s_hist[PCT_MAX_Q][TRK_HIST];
    __shared__ unsigned long long s_red[32];
    __shared__ int s_ired[32];
    __shared__ int s_sel[PCT_MAX_Q][2];
    __shared__ int s_nan;
    const double* __restrict__ x = p.x + (long long)blockIdx.x * p.frame_stride;
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31, warp = tid >> 5;
    const int n = p.n, nq = p.nq;
    double* out = p.out + (long long)blockIdx.x * nq;
    unsigned long long prefix[PCT_MAX_Q];
    int rank[PCT_MAX_Q];
#pragma unroll
    for (int q = 0; q < PCT_MAX_Q; ++q) { prefix[q] = 0; rank[q] = p.k[q]; }
    if (tid == 0) s_nan = 0;
    // radix select of every k, 8 bits per pass; one read of the frame per pass serves all of them
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int q = tid; q < PCT_MAX_Q * TRK_HIST; q += nthr) (&s_hist[0][0])[q] = 0;
        __syncthreads();
        const unsigned long long hmask = shift == 56 ? 0ull : (~0ull << (shift + 8));
        bool nan = false;
        for (int base = 0; base < n; base += nthr) {            // n <= PCT_MAX_N: base + nthr cannot overflow
            const int o = base + tid;
            unsigned long long key = 0;
            if (o < n) {
                const double v = __ldg(x + o);
                nan |= isnan(v);
                key = trk_key(v);
            }
#pragma unroll
            for (int q = 0; q < PCT_MAX_Q; ++q) {
                if (q >= nq) break;
                int bin = TRK_HIST + lane;                      // no bin
                if (o < n && (key & hmask) == prefix[q]) bin = (int)((key >> shift) & 255);
                const unsigned peers = __match_any_sync(0xffffffffu, bin);
                if (bin < TRK_HIST && lane == __ffs(peers) - 1) atomicAdd(&s_hist[q][bin], (unsigned)__popc(peers));
            }
        }
        if (nan) s_nan = 1;
        __syncthreads();
        if (s_nan) break;                                       // np.percentile of a frame holding NaN is NaN
        if (warp < nq) {                                        // warp q: the bin holding rank q
            const unsigned int* h = s_hist[warp];
            unsigned cnt[8], tot = 0;
#pragma unroll
            for (int b = 0; b < 8; ++b) { cnt[b] = h[lane * 8 + b]; tot += cnt[b]; }
            unsigned inc = tot;
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned u = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= d) inc += u;
            }
            const unsigned exc = inc - tot;
            int rk = 0;
#pragma unroll
            for (int q = 0; q < PCT_MAX_Q; ++q)
                if (q == warp) rk = rank[q];
            if ((unsigned)rk >= exc && (unsigned)rk < inc) {
                unsigned below = exc;
                int b = 0;
                while (below + h[lane * 8 + b] <= (unsigned)rk) { below += h[lane * 8 + b]; ++b; }
                s_sel[warp][0] = lane * 8 + b;
                s_sel[warp][1] = (int)below;
            }
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < PCT_MAX_Q; ++q) {
            if (q >= nq) break;
            prefix[q] |= (unsigned long long)s_sel[q][0] << shift;
            rank[q] -= s_sel[q][1];
        }
        __syncthreads();
    }
    if (s_nan) {
        if (tid < nq) out[tid] = __longlong_as_double(0x7ff8000000000000ll);
        return;
    }
    // order statistic k + 1: the same value when more than k + 1 keys are <= it, else the smallest key above it
    int le[PCT_MAX_Q];
    unsigned long long above[PCT_MAX_Q];
#pragma unroll
    for (int q = 0; q < PCT_MAX_Q; ++q) { le[q] = 0; above[q] = ~0ull; }
    for (int o = tid; o < n; o += nthr) {
        const unsigned long long key = trk_key(__ldg(x + o));
#pragma unroll
        for (int q = 0; q < PCT_MAX_Q; ++q) {
            if (key <= prefix[q]) ++le[q];
            else if (key < above[q]) above[q] = key;
        }
    }
#pragma unroll
    for (int q = 0; q < PCT_MAX_Q; ++q) {
        if (q >= nq) break;
        const int cnt = trk_block_sum(le[q], s_ired);
        const unsigned long long ab = trk_block_ext<false>(above[q], s_red);
        if (tid == 0) {
            const double a = trk_unkey(prefix[q]);
            const double b = (cnt >= p.k[q] + 2 || p.k[q] + 1 > n - 1) ? a : trk_unkey(ab);
            // numpy _lerp: a + (b - a) g, or b - (b - a)(1 - g) when g >= 0.5
            const double d = __dsub_rn(b, a);
            const double g = p.g[q];
            double v = g >= 0.5 ? __dsub_rn(b, __dmul_rn(d, __dsub_rn(1.0, g))) : __dadd_rn(a, __dmul_rn(d, g));
            if (p.has_scale) v = __dmul_rn(v, p.scale[q]);
            out[q] = v;
        }
    }
}

// ---- launches (host side; prcore_detect.cu brackets them with its profiling scope and checks the launch) ----------------
inline void launch_persistence(const PersistParams& p, cudaStream_t st) {
    const dim3 grid((unsigned)((p.cols + PST_TX - 1) / PST_TX), (unsigned)((p.rows + PST_TY - 1) / PST_TY));
    pst_kernel<<<grid, dim3(PST_TX, PST_TY), 0, st>>>(p);
}

inline void launch_percentiles(const PctParams& p, int nframes, cudaStream_t st) {
    pct_kernel<<<(unsigned)nframes, PCT_THREADS, 0, st>>>(p);
}

}  // namespace rdr
}  // namespace prc
