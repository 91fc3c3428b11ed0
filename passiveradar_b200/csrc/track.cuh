// track.cuh -- the reference's Kalman target trackers (passiveRadar/target_detection.py:164-681): measurement
// extraction (get_measurements), the multi-target tracker (multitarget_tracker with associate_measurements,
// initialize_track, update_track, adaptive_kalman_update, kalman_extrapolate) and the simple tracker
// (simple_target_tracker).  DESIGN.md section 11 lists the reference behaviour reproduced here.
//
// A map is rows x cols (the reference's data[:, :, i]: rows = Doppler bins, cols = range bins), float32 or float64,
// always evaluated in float64.  The reference works on the transformed frame fliplr((x / mean|x|).T): its element
// (i, j) (i = range row, j = flipped Doppler column) is x[rows - 1 - j][i] / mean, and its row-major position is
// p = i * rows + j.  Nothing is transformed in memory: every pass reads the map in its own order and carries p.
//
// track_meas_kernel (one CTA per frame, every frame of every sequence in one launch):
//   1. mean|x| in NumPy's pairwise order: the host builds the summation tree of n (pw_plan), the leaves (<= 128
//      elements, 8 partial sums) are summed in parallel, the inner nodes level by level;
//   2. np.percentile(frame, 99.8): order statistics k and k + 1 by a radix select over order-preserving 64-bit keys,
//      then NumPy's _lerp;
//   3. candidates frame >= thr, collected in shared memory and sorted by (strength desc, p desc) -- the documented
//      tie rule (what np.flip(np.argsort(s, kind="stable")) gives).  When more candidates than fit in shared memory
//      tie (constant or mostly-zero maps), MODE_MEAS emits them level by level, each level in descending p.
// track_multi_kernel (one warp per sequence) walks the frames in order; each frame's candidate list comes from the
//   slot the measurement kernel filled, or -- when the frame had more candidates than a slot holds -- is enumerated
//   from the map itself.  Removal from the list is recorded as the gates that removed candidates.
// track_simple_kernel (one CTA per sequence) walks the frames in order: a CTA-wide argmax over the gated frame, then
//   a scalar Kalman update.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "prcore.h"

namespace prc {

constexpr int TRK_THREADS = 512;             // measurement kernel
constexpr int TRK_SIMPLE_THREADS = 256;      // simple tracker (one CTA per sequence)
constexpr int TRK_MAX_TRACKS = 64;           // largest n_tracks of the multi-target tracker
constexpr long long TRK_MAX_CELLS = 1 << 19; // largest map (rows * cols): the summation tree lives in shared memory
constexpr int TRK_MAX_CAP = 4096;            // largest candidate list sorted in shared memory
constexpr int TRK_HIST = 256;                // radix-select digit: 8 bits

enum { TRK_MODE_MEAN = 0, TRK_MODE_SLOTS = 1, TRK_MODE_MEAS = 2 };

struct PwNode { int off, len, left, pad; };  // pairwise-sum tree node, breadth-first; left child index, -1 for a leaf

struct TrkMapParams {
    const void* maps;
    long long seq_stride, frame_stride;      // elements
    int rows, cols, n;                       // n = rows * cols
    int nframes;                             // frames per sequence (stats index s * nframes + f)
    int f0;                                  // frame of blockIdx.x == 0
    const PwNode* plan;
    const int* level;                        // level[l] = first node of depth l, level[nlevels] = nnodes
    int nnodes, nlevels;
    int k;                                   // percentile: order statistics k and k + 1 ...
    double g;                                // ... and the fraction between them
    int dlo, dhi;                            // zeroed (transformed) Doppler columns [dlo, dhi)
    int n_unbanded;                          // cells outside the zeroed bands
    double rng_start, dop_start, dop_stop;   // linspace(range_extent, 0, cols), linspace(-doppler_extent, doppler_extent, rows)
    int cap;                                 // candidates sorted in shared memory
    double* mean;                            // [nseq * nframes]
    double* thr;
    int* count;
    double* out;                             // frame (s, f): out + (s * out_nf + f - f0) * 3 * out_cap: range, Doppler, strength rows
    long long out_cap;
    int out_nf;
};

__device__ __forceinline__ unsigned long long trk_key(double v) {
    if (v == 0.0) v = 0.0;                   // -0 and +0 are the same value
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// np.linspace(start, stop, num)[k], NumPy 2: k * step + start (k / div * delta when step == 0), last point = stop
__device__ __forceinline__ double trk_linspace(double start, double stop, int num, int k) {
    const int div = num - 1;
    const double delta = __dsub_rn(stop, start);
    double y;
    if (div > 0) {
        const double step = __ddiv_rn(delta, (double)div);
        y = step == 0.0 ? __dmul_rn(__ddiv_rn((double)k, (double)div), delta) : __dmul_rn((double)k, step);
    } else {
        y = __dmul_rn((double)k, delta);
    }
    y = __dadd_rn(y, start);
    if (div > 0 && k == div) y = stop;
    return y;
}

template <class T>
__device__ __forceinline__ double trk_ld(const T* x, long long o) { return (double)x[o]; }

// one leaf of NumPy's pairwise sum of |x| (numpy/_core/src/umath/loops_utils.h.src)
template <class T>
__device__ double trk_leaf(const T* __restrict__ x, int len) {
    if (len < 8) {
        double r = 0.0;
        for (int i = 0; i < len; ++i) r = __dadd_rn(r, fabs(trk_ld(x, i)));
        return r;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = fabs(trk_ld(x, j));
    int i = 8;
    for (; i < len - (len % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], fabs(trk_ld(x, i + j)));
    }
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                           __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < len; ++i) res = __dadd_rn(res, fabs(trk_ld(x, i)));
    return res;
}

// mean|x| in NumPy's order; nv: nnodes doubles of shared memory.  Every thread returns the mean.
template <class T>
__device__ double trk_mean(const TrkMapParams& p, const T* __restrict__ x, double* nv) {
    for (int q = threadIdx.x; q < p.nnodes; q += blockDim.x) {
        const PwNode nd = p.plan[q];
        if (nd.left < 0) nv[q] = trk_leaf(x + nd.off, nd.len);
    }
    __syncthreads();
    for (int l = p.nlevels - 2; l >= 0; --l) {
        for (int q = p.level[l] + threadIdx.x; q < p.level[l + 1]; q += blockDim.x) {
            const int c = p.plan[q].left;
            if (c >= 0) nv[q] = __dadd_rn(nv[c], nv[c + 1]);
        }
        __syncthreads();
    }
    const double m = __ddiv_rn(nv[0], (double)p.n);
    __syncthreads();
    return m;
}

// value of the transformed, normalised, band-zeroed frame at map index o; i, j, pos: its coordinates
template <class T>
__device__ __forceinline__ double trk_value(const TrkMapParams& p, const T* __restrict__ x, int o, double mean,
                                            int& i, int& j, int& pos) {
    const int r = o / p.cols;
    i = o - r * p.cols;
    j = p.rows - 1 - r;
    pos = i * p.rows + j;
    const bool banded = i < 8 || i >= p.cols - 8 || (j >= p.dlo && j < p.dhi);
    return banded ? 0.0 : __ddiv_rn(trk_ld(x, o), mean);
}

__device__ __forceinline__ unsigned long long trk_shfl_u64(unsigned long long v, int src) {
    return (unsigned long long)__shfl_sync(0xffffffffu, (long long)v, src);
}

// block-wide sum of an int (every thread gets it); red: >= 32 ints of shared memory
__device__ __forceinline__ int trk_block_sum(int v, int* red) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    int t = 0;
    for (int q = 0; q < nw; ++q) t += red[q];
    __syncthreads();
    return t;
}

// block-wide max / min of a 64-bit key (every thread gets it); red: >= 32 u64 of shared memory
template <bool MAX>
__device__ __forceinline__ unsigned long long trk_block_ext(unsigned long long v, unsigned long long* red) {
    for (int o = 16; o; o >>= 1) {
        const unsigned long long u = trk_shfl_u64(v, (threadIdx.x & 31) ^ o);
        v = MAX ? (u > v ? u : v) : (u < v ? u : v);
    }
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if ((threadIdx.x & 31) == 0) red[w] = v;
    __syncthreads();
    unsigned long long t = red[0];
    for (int q = 1; q < nw; ++q) t = MAX ? (red[q] > t ? red[q] : t) : (red[q] < t ? red[q] : t);
    __syncthreads();
    return t;
}

__device__ __forceinline__ double trk_unkey(unsigned long long k) {
    const unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    return __longlong_as_double((long long)u);
}

template <class T>
__device__ __forceinline__ void trk_write_cand(const TrkMapParams& p, const T* __restrict__ x, double mean,
                                               double* out, long long e, int pos) {
    const int i = pos / p.rows, j = pos - (pos / p.rows) * p.rows;
    int ii, jj, pp;
    const double s = trk_value(p, x, (p.rows - 1 - j) * p.cols + i, mean, ii, jj, pp);
    out[e] = trk_linspace(p.rng_start, 0.0, p.cols, i);
    out[p.out_cap + e] = trk_linspace(p.dop_start, p.dop_stop, p.rows, j);
    out[2 * p.out_cap + e] = s;
}

// dynamic shared memory: nnodes doubles | cap keys (u64) | cap positions (int)
template <class T, int MODE>
__global__ void __launch_bounds__(TRK_THREADS) track_meas_kernel(const __grid_constant__ TrkMapParams p) {
    extern __shared__ __align__(16) unsigned char trk_dyn[];
    __shared__ unsigned int s_hist[TRK_HIST];
    __shared__ unsigned long long s_red[32];
    __shared__ int s_ired[32];
    __shared__ int s_sel[2];
    __shared__ int s_m;
    const int s = blockIdx.y, f = p.f0 + blockIdx.x;
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
    const T* __restrict__ x = static_cast<const T*>(p.maps) + s * p.seq_stride + f * p.frame_stride;
    const long long sidx = (long long)s * p.nframes + f;
    double* nv = reinterpret_cast<double*>(trk_dyn);
    const double mean = trk_mean(p, x, nv);
    if (MODE == TRK_MODE_MEAN) {
        if (tid == 0) p.mean[sidx] = mean;
        return;
    }
    unsigned long long* skey = reinterpret_cast<unsigned long long*>(trk_dyn + (((size_t)p.nnodes * 8 + 15) & ~(size_t)15));
    int* spos = reinterpret_cast<int*>(skey + p.cap);
    double* out = p.out + ((long long)s * p.out_nf + (f - p.f0)) * 3 * p.out_cap;
    const int n = p.n;
    double thr;
    if (mean == 0.0 && p.n_unbanded > 0) {
        thr = __longlong_as_double(0x7ff8000000000000ll);      // 0 / 0 in the frame: np.percentile is NaN, nothing passes
    } else {
        // radix select of order statistic k (ascending) over the keys, 8 bits per pass
        unsigned long long prefix = 0;
        int rank = p.k;
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (int q = tid; q < TRK_HIST; q += nthr) s_hist[q] = 0;
            __syncthreads();
            const unsigned long long hmask = shift == 56 ? 0ull : (~0ull << (shift + 8));
            for (int base = 0; base < n; base += nthr) {
                const int o = base + tid;
                int bin = TRK_HIST + lane;                    // no bin
                if (o < n) {
                    int i, j, pos;
                    const unsigned long long key = trk_key(trk_value(p, x, o, mean, i, j, pos));
                    if ((key & hmask) == prefix) bin = (int)((key >> shift) & 255);
                }
                const unsigned peers = __match_any_sync(0xffffffffu, bin);
                if (bin < TRK_HIST && lane == __ffs(peers) - 1) atomicAdd(&s_hist[bin], (unsigned)__popc(peers));
            }
            __syncthreads();
            if (tid < 32) {                                   // warp 0: find the bin holding rank
                unsigned c[8], tot = 0;
#pragma unroll
                for (int q = 0; q < 8; ++q) { c[q] = s_hist[lane * 8 + q]; tot += c[q]; }
                unsigned inc = tot;
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
                    if (lane >= o) inc += u;
                }
                const unsigned exc = inc - tot;
                if ((unsigned)rank >= exc && (unsigned)rank < inc) {
                    unsigned below = exc;
                    int b = 0;
                    while (below + s_hist[lane * 8 + b] <= (unsigned)rank) { below += s_hist[lane * 8 + b]; ++b; }
                    s_sel[0] = lane * 8 + b;
                    s_sel[1] = (int)below;
                }
            }
            __syncthreads();
            prefix |= (unsigned long long)s_sel[0] << shift;
            rank -= s_sel[1];
            __syncthreads();
        }
        // order statistic k + 1: the same value when more than k + 1 keys are <= it, else the smallest key above it
        int le = 0;
        unsigned long long above = ~0ull;
        for (int o = tid; o < n; o += nthr) {
            int i, j, pos;
            const unsigned long long key = trk_key(trk_value(p, x, o, mean, i, j, pos));
            if (key <= prefix) ++le;
            else if (key < above) above = key;
        }
        le = trk_block_sum(le, s_ired);
        above = trk_block_ext<false>(above, s_red);
        const double a = trk_unkey(prefix);
        const double b = (le >= p.k + 2 || p.k + 1 > n - 1) ? a : trk_unkey(above);
        // numpy _lerp: a + (b - a) g, or b - (b - a)(1 - g) when g >= 0.5
        const double d = __dsub_rn(b, a);
        thr = p.g >= 0.5 ? __dsub_rn(b, __dmul_rn(d, __dsub_rn(1.0, p.g))) : __dadd_rn(a, __dmul_rn(d, p.g));
    }
    // candidates: collect (key, p) in shared memory (up to cap) and count them
    if (tid == 0) s_m = 0;
    __syncthreads();
    for (int base = 0; base < n; base += nthr) {
        const int o = base + tid;
        bool cand = false;
        unsigned long long key = 0;
        int pos = 0;
        if (o < n) {
            int i, j;
            const double v = trk_value(p, x, o, mean, i, j, pos);
            cand = v >= thr;
            key = trk_key(v);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, cand);
        int at = 0;
        if (bal) {
            if (lane == __ffs(bal) - 1) at = atomicAdd(&s_m, __popc(bal));
            at = __shfl_sync(0xffffffffu, at, __ffs(bal) - 1) + __popc(bal & ((1u << lane) - 1u));
            if (cand && at < p.cap) { skey[at] = key; spos[at] = pos; }
        }
    }
    __syncthreads();
    const int M = s_m;
    if (tid == 0) { p.mean[sidx] = mean; p.thr[sidx] = thr; p.count[sidx] = M; }
    if (M <= p.cap) {
        int sz = 2;
        while (sz < M) sz <<= 1;
        for (int q = M + tid; q < sz; q += nthr) { skey[q] = 0; spos[q] = -1; }
        __syncthreads();
        // bitonic sort, descending in (key, pos)
        for (int kk = 2; kk <= sz; kk <<= 1) {
            for (int jj = kk >> 1; jj > 0; jj >>= 1) {
                for (int q = tid; q < sz; q += nthr) {
                    const int r = q ^ jj;
                    if (r > q) {
                        const unsigned long long ka = skey[q], kb = skey[r];
                        const int pa = spos[q], pb = spos[r];
                        const bool a_first = ka > kb || (ka == kb && pa > pb);
                        const bool desc = (q & kk) == 0;
                        if (desc ? !a_first : a_first) { skey[q] = kb; skey[r] = ka; spos[q] = pb; spos[r] = pa; }
                    }
                }
                __syncthreads();
            }
        }
        const long long lim = M < p.out_cap ? M : p.out_cap;
        for (int e = tid; e < lim; e += nthr) trk_write_cand(p, x, mean, out, e, spos[e]);
        return;
    }
    if (MODE != TRK_MODE_MEAS) return;       // the tracker enumerates such a frame from the map itself
    // more candidates than shared memory holds: they tie at few values.  Emit level by level (largest first), each
    // level in descending p.
    const long long lim = M < p.out_cap ? M : p.out_cap;
    long long emitted = 0;
    unsigned long long hi = ~0ull;
    int* wtot = s_ired;
    while (emitted < lim) {
        unsigned long long lv = 0;
        for (int o = tid; o < n; o += nthr) {
            int i, j, pos;
            const double v = trk_value(p, x, o, mean, i, j, pos);
            const unsigned long long key = trk_key(v);
            if (v >= thr && key < hi && key > lv) lv = key;
        }
        lv = trk_block_ext<true>(lv, s_red);
        long long run = 0;
        for (int base = n - 1; base >= 0; base -= nthr) {
            const int q = base - tid;
            bool hit = false;
            if (q >= 0) {
                const int i = q / p.rows, j = q - i * p.rows;
                int ii, jj, pos;
                const double v = trk_value(p, x, (p.rows - 1 - j) * p.cols + i, mean, ii, jj, pos);
                hit = v >= thr && trk_key(v) == lv;
            }
            const unsigned bal = __ballot_sync(0xffffffffu, hit);
            const int w = tid >> 5, nw = nthr >> 5;
            if (lane == 0) wtot[w] = __popc(bal);
            __syncthreads();
            int off = 0, tot = 0;
            for (int z = 0; z < nw; ++z) { if (z < w) off += wtot[z]; tot += wtot[z]; }
            const long long e = emitted + run + off + __popc(bal & ((1u << lane) - 1u));
            if (hit && e < lim) trk_write_cand(p, x, mean, out, e, q);
            run += tot;
            __syncthreads();
        }
        emitted += run;
        hi = lv;
    }
}

// ---------------------------------------------------------------------------------- Kalman filter (float64)
// x = F1 x;  P = F2 P F2^T + Q;  S = H P H^T + R * rs;  and with a measurement z:
// K = P H^T S^-1;  x += K (z - H x);  P = (I - K H) P.   est = H x.  (target_detection.py:63-148)
__device__ void trk_kalman(const prc_kalman& in, prc_kalman& out, bool update, double z0, double z1, double rs,
                           double est[2]) {
    double x[4], P[16], T[16];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc += in.F1[4 * i + k] * in.x[k];
        x[i] = acc;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc += in.F2[4 * i + k] * in.P[4 * k + j];
            T[4 * i + j] = acc;
        }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc += T[4 * i + k] * in.F2[4 * j + k];
            P[4 * i + j] = acc + in.Q[4 * i + j];
        }
    // PH = P H^T (4 x 2), S = H PH + R rs
    double PH[8], S[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc += P[4 * i + k] * in.H[4 * c + k];
            PH[2 * i + c] = acc;
        }
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc += in.H[4 * r + k] * PH[2 * k + c];
            S[2 * r + c] = acc + in.R[2 * r + c] * rs;
        }
    if (update) {
        const double det = S[0] * S[3] - S[1] * S[2];
        const double iS[4] = {S[3] / det, -S[1] / det, -S[2] / det, S[0] / det};
        double K[8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int c = 0; c < 2; ++c) K[2 * i + c] = PH[2 * i] * iS[c] + PH[2 * i + 1] * iS[2 + c];
        double y[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 4; ++k) acc += in.H[4 * r + k] * x[k];
            y[r] = (r == 0 ? z0 : z1) - acc;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) x[i] += K[2 * i] * y[0] + K[2 * i + 1] * y[1];
        // T = I - K H, then P = T P
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                T[4 * i + j] = (i == j ? 1.0 : 0.0) - (K[2 * i] * in.H[j] + K[2 * i + 1] * in.H[4 + j]);
        double Pn[16];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                double acc = 0.0;
#pragma unroll
                for (int k = 0; k < 4; ++k) acc += T[4 * i + k] * P[4 * k + j];
                Pn[4 * i + j] = acc;
            }
#pragma unroll
        for (int q = 0; q < 16; ++q) P[q] = Pn[q];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < 4; ++k) acc += in.H[4 * r + k] * x[k];
        est[r] = acc;
    }
    // in and out may alias: every read of `in` is above
#pragma unroll
    for (int q = 0; q < 16; ++q) {
        out.P[q] = P[q];
        out.F1[q] = in.F1[q];
        out.F2[q] = in.F2[q];
        out.Q[q] = in.Q[q];
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) out.H[q] = in.H[q];
#pragma unroll
    for (int q = 0; q < 4; ++q) { out.x[q] = x[q]; out.R[q] = in.R[q]; out.S[q] = S[q]; }
}

// ---------------------------------------------------------------------------------- multi-target tracker
struct TrkMultiParams {
    TrkMapParams m;                 // map geometry and the per-frame mean / thr / count of track_meas_kernel
    int f64;
    prc_track* hist;                // [nseq][nframes][n_tracks]
    int n_tracks;
    int f0, f1;                     // frames walked by this launch
    const double* slots;            // frame (s, f): slots + (s * fc + f - f0) * 3 * m.cap (range, Doppler, strength rows)
    int fc;
    int resume;                     // PRC_FLAG_TRACK_RESUME: frame 0 continues from the records already at hist[s][0]
};

// initialize_track (target_detection.py:350-396): free at (0, 0) without a measurement, preliminary at it with one
__device__ void trk_init_track(prc_track& t, bool have, double r, double d) {
    if (!have) { r = 0.0; d = 0.0; }
    t.status = have ? 1 : 0;
    t.lifetime = 1;
    // the record is built positionally against differently named fields: both hold (r, d)
    t.measurement[0] = r; t.measurement[1] = d;
    t.estimate[0] = r; t.estimate[1] = d;
    for (int q = 0; q < 20; ++q) t.measurement_history[q] = (q == 0 || (q >= 5 && q < 10)) ? 1.0 : 0.0;
    prc_kalman& k = t.kalman_state;
    k.x[0] = r; k.x[1] = 0.0; k.x[2] = d; k.x[3] = -1.0;
    const double P[4] = {5.0, 0.0225, 0.04, 0.1}, Q[4] = {4.0, 0.03, 0.2, 0.08};
    const double F1[16] = {1, 0, -0.003, 0, 0, 0, -0.003, -0.003, 0, 0, 1, 1, 0, 0, 0, 1};
    const double F2[16] = {1, 1, 0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1};
    for (int q = 0; q < 16; ++q) {
        k.P[q] = (q % 5 == 0) ? P[q / 5] : 0.0;
        k.Q[q] = (q % 5 == 0) ? Q[q / 5] : 0.0;
        k.F1[q] = F1[q];
        k.F2[q] = F2[q];
    }
    for (int q = 0; q < 8; ++q) k.H[q] = (q == 0 || q == 6) ? 1.0 : 0.0;
    k.R[0] = 5.0; k.R[1] = 0.0; k.R[2] = 0.0; k.R[3] = 2.0;
    k.S[0] = 1.0; k.S[1] = 0.0; k.S[2] = 0.0; k.S[3] = 1.0;
}

struct TrkBox { double r0, d0, hr, hd; };    // candidates with |r - r0| < hr and |d - d0| < hd have been removed

// what a pass over the candidate list looks for
enum { TRK_ANY = 0, TRK_PRELIM = 1, TRK_CONFIRMED = 2 };

struct TrkQuery {
    int kind;
    double r0, d0;                  // gate centre (last measurement or estimate)
    double mr, md;                  // last measurement (validation gate)
    double iS[4];                   // S^-1 (validation gate)
};

struct TrkBest {
    int count;
    double r, d;
};

// one warp: count the live candidates the query accepts and pick one -- the first in list order (strength desc,
// p desc), or for a preliminary track the one nearest the origin (ties: the first)
template <bool LIST>
__device__ TrkBest trk_scan(const TrkMultiParams& p, const double* slot, int M, const void* map, double mean,
                            double thr, const TrkBox* boxes, int nbox, const TrkQuery& q) {
    const int lane = threadIdx.x & 31;
    const int total = LIST ? M : p.m.n;
    int cnt = 0;
    unsigned long long oa = 0;                 // order: larger first
    int ob = -1;
    double dist = __longlong_as_double(0x7ff0000000000000ll);
    double br = 0.0, bd = 0.0;
    for (int e = lane; e < total; e += 32) {
        double r, d;
        unsigned long long ka;
        int kb;
        if (LIST) {
            r = slot[e];
            d = slot[p.m.cap + e];
            ka = (unsigned long long)(M - e);
            kb = 0;
        } else {
            int i, j, pos;
            const double v = p.f64 ? trk_value(p.m, static_cast<const double*>(map), e, mean, i, j, pos)
                                   : trk_value(p.m, static_cast<const float*>(map), e, mean, i, j, pos);
            if (!(v >= thr)) continue;
            r = trk_linspace(p.m.rng_start, 0.0, p.m.cols, i);
            d = trk_linspace(p.m.dop_start, p.m.dop_stop, p.m.rows, j);
            ka = trk_key(v);
            kb = pos;
        }
        bool live = true;
        for (int b = 0; b < nbox; ++b)
            if (fabs(__dsub_rn(r, boxes[b].r0)) < boxes[b].hr && fabs(__dsub_rn(d, boxes[b].d0)) < boxes[b].hd) live = false;
        if (!live) continue;
        double dd = 0.0;
        if (q.kind == TRK_PRELIM) {
            if (!(fabs(__dsub_rn(r, q.r0)) < 5.0 && fabs(__dsub_rn(d, q.d0)) < 24.0)) continue;
            dd = sqrt(__dadd_rn(__dmul_rn(r, r), __dmul_rn(d, d)));
        } else if (q.kind == TRK_CONFIRMED) {
            if (!(fabs(__dsub_rn(r, q.r0)) < 4.0 && fabs(__dsub_rn(d, q.d0)) < 20.0)) continue;
            const double z0 = __dsub_rn(q.mr, r), z1 = __dsub_rn(q.md, d);
            const double t0 = __dadd_rn(__dmul_rn(z0, q.iS[0]), __dmul_rn(z1, q.iS[2]));
            const double t1 = __dadd_rn(__dmul_rn(z0, q.iS[1]), __dmul_rn(z1, q.iS[3]));
            if (!(__dadd_rn(__dmul_rn(t0, z0), __dmul_rn(t1, z1)) < 6.0)) continue;
        }
        ++cnt;
        const bool better = q.kind == TRK_PRELIM ? (dd < dist || (dd == dist && (ka > oa || (ka == oa && kb > ob))))
                                                 : (ka > oa || (ka == oa && kb > ob));
        if (better) { dist = dd; oa = ka; ob = kb; br = r; bd = d; }
    }
    for (int o = 16; o; o >>= 1) {
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        const double dist2 = __shfl_xor_sync(0xffffffffu, dist, o);
        const unsigned long long oa2 = trk_shfl_u64(oa, lane ^ o);
        const int ob2 = __shfl_xor_sync(0xffffffffu, ob, o);
        const double br2 = __shfl_xor_sync(0xffffffffu, br, o), bd2 = __shfl_xor_sync(0xffffffffu, bd, o);
        const bool ord2 = oa2 > oa || (oa2 == oa && ob2 > ob);
        const bool better = q.kind == TRK_PRELIM ? (dist2 < dist || (dist2 == dist && ord2)) : ord2;
        if (better) { dist = dist2; oa = oa2; ob = ob2; br = br2; bd = bd2; }
    }
    return TrkBest{cnt, br, bd};
}

// one frame of multitarget_tracker (target_detection.py:485-524) for the warp's sequence.  prev and cur are the same
// records at frame 0, where tracks of every status run in place (free ones fresh, any when resuming): a track reads
// only its own record, every lane reads it before the __syncwarp that precedes lane 0's write, and trk_kalman reads
// all of its input before writing its output.
template <bool LIST>
__device__ void trk_multi_frame(const TrkMultiParams& p, const prc_track* prev, prc_track* cur, const double* slot,
                                int M, const void* map, double mean, double thr, TrkBox* boxes) {
    const int lane = threadIdx.x & 31;
    const int N = p.n_tracks;
    // the confirmed, preliminary and free lists are fixed at the start of the frame
    unsigned long long conf = 0, prel = 0;
    for (int t = lane; t < 64; t += 32) {
        const long long st = t < N ? prev[t].status : 0;
        const unsigned bc = __ballot_sync(0xffffffffu, st == 2), bp = __ballot_sync(0xffffffffu, st == 1);
        conf |= (unsigned long long)bc << (t - lane);
        prel |= (unsigned long long)bp << (t - lane);
    }
    int nbox = 0;
    bool all_gone = false;
    bool stopped = false;
    for (int pass = 2; pass >= 0; --pass) {
        for (int t = 0; t < N; ++t) {
            const bool c = (conf >> t) & 1, pr = (prel >> t) & 1;
            const int st = c ? 2 : (pr ? 1 : 0);
            if (st != pass) continue;
            const prc_track& in = prev[t];
            prc_track& o = cur[t];
            if (pass == 0 && stopped) {                   // the reference's `break`: the rest stay as they were
                if (prev != cur) {
                    const double* a = reinterpret_cast<const double*>(&in);
                    double* b = reinterpret_cast<double*>(&o);
                    for (int q = lane; q < (int)(sizeof(prc_track) / 8); q += 32) b[q] = a[q];
                }
                continue;
            }
            TrkQuery q{};
            q.kind = pass == 0 ? TRK_ANY : (pass == 1 ? TRK_PRELIM : TRK_CONFIRMED);
            q.mr = in.measurement[0];
            q.md = in.measurement[1];
            if (pass == 1) { q.r0 = q.mr; q.d0 = q.md; }
            if (pass == 2) {
                q.r0 = in.estimate[0];
                q.d0 = in.estimate[1];
                const double* S = in.kalman_state.S;
                const double det = S[0] * S[3] - S[1] * S[2];
                q.iS[0] = S[3] / det; q.iS[1] = -S[1] / det; q.iS[2] = -S[2] / det; q.iS[3] = S[0] / det;
            }
            TrkBest b{0, 0.0, 0.0};
            if (!all_gone) b = trk_scan<LIST>(p, slot, M, map, mean, thr, boxes, nbox, q);
            if (pass == 0 && b.count == 0) {              // no candidates left: `break`
                stopped = true;
                if (prev != cur) {
                    const double* a = reinterpret_cast<const double*>(&in);
                    double* d = reinterpret_cast<double*>(&o);
                    for (int z = lane; z < (int)(sizeof(prc_track) / 8); z += 32) d[z] = a[z];
                }
                continue;
            }
            const bool found = b.count > 0;
            // removal: a free track with one match takes the whole list; with several, everything within 10 km /
            // 12 Hz of the strongest; a preliminary track its early gate; a confirmed track its early gate
            if (found) {
                if (pass == 0 && b.count == 1) {
                    all_gone = true;
                } else if (nbox < TRK_MAX_TRACKS) {
                    TrkBox bx;
                    if (pass == 0) bx = TrkBox{b.r, b.d, 10.0, 12.0};
                    else if (pass == 1) bx = TrkBox{q.r0, q.d0, 5.0, 24.0};
                    else bx = TrkBox{q.r0, q.d0, 4.0, 20.0};
                    if (lane == 0) boxes[nbox] = bx;
                    ++nbox;
                }
            }
            __syncwarp();
            if (pass == 0) {
                if (lane == 0) trk_init_track(o, found, b.r, b.d);
            } else if (lane == 0) {
                // update_track (target_detection.py:398-453); the kill / promote tests use the history before the shift
                const long long life = in.lifetime;
                double h10 = 0.0, h20 = 0.0;
                for (int z = 0; z < 20; ++z) { h20 += in.measurement_history[z]; if (z < 10) h10 += in.measurement_history[z]; }
                long long nst = st;
                if (st == 1) {
                    if (life > 4 && h10 < 6) nst = 0;
                    if (life > 4 && h10 > 8) nst = 2;
                } else if (life > 4 && h20 < 4) {
                    nst = 0;
                }
                double rs = 0.0, mr = in.measurement[0], md = in.measurement[1];
                if (found) {
                    const double dr = b.r - in.measurement[0], dd = b.d - in.measurement[1];
                    rs = dr * dr + dd * dd;
                    mr = b.r;
                    md = b.d;
                }
                double hist[20];
                hist[0] = found ? 1.0 : 0.0;
                for (int z = 1; z < 20; ++z) hist[z] = in.measurement_history[z - 1];
                double est[2];
                trk_kalman(in.kalman_state, o.kalman_state, found, b.r, b.d, found ? rs : 1.0, est);
                o.status = nst;
                o.lifetime = life + 1;
                o.measurement[0] = mr; o.measurement[1] = md;
                o.estimate[0] = est[0]; o.estimate[1] = est[1];
                for (int z = 0; z < 20; ++z) o.measurement_history[z] = hist[z];
            }
            __syncwarp();
        }
    }
}

__global__ void __launch_bounds__(32) track_multi_kernel(const __grid_constant__ TrkMultiParams p) {
    __shared__ TrkBox boxes[TRK_MAX_TRACKS];
    const int s = blockIdx.x, lane = threadIdx.x & 31;
    const size_t per_seq = (size_t)p.m.nframes * p.n_tracks;
    for (int f = p.f0; f < p.f1; ++f) {
        prc_track* cur = p.hist + s * per_seq + (size_t)f * p.n_tracks;
        const prc_track* prev = cur - p.n_tracks;
        if (f == 0) {                                  // frame 0 runs in place: every track starts free, or resumes
            if (!p.resume) {
                for (int t = lane; t < p.n_tracks; t += 32) trk_init_track(cur[t], false, 0.0, 0.0);
                __syncwarp();
            }
            prev = cur;
        }
        const long long sidx = (long long)s * p.m.nframes + f;
        const int M = p.m.count[sidx];
        const double mean = p.m.mean[sidx], thr = p.m.thr[sidx];
        const void* map = static_cast<const char*>(p.m.maps) +
                          (s * p.m.seq_stride + f * p.m.frame_stride) * (p.f64 ? 8 : 4);
        if (M <= p.m.cap) {
            const double* slot = p.slots + ((size_t)s * p.fc + (f - p.f0)) * 3 * p.m.cap;
            trk_multi_frame<true>(p, prev, cur, slot, M, map, mean, thr, boxes);
        } else {
            trk_multi_frame<false>(p, prev, cur, nullptr, M, map, mean, thr, boxes);
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------- simple tracker
struct TrkSimpleParams {
    TrkMapParams m;                 // geometry and the per-frame means
    prc_track_simple* hist;         // [nseq][nframes]
    double range_extent, doppler_extent;
    int zlo, zhi;                   // zeroed columns [250:260], clipped to the frame
    int resume;                     // PRC_FLAG_TRACK_RESUME: frame 0 continues from the record already at hist[s][0]
};

// python slice [start:stop] of an axis of length len
__device__ __forceinline__ void trk_slice(long long start, long long stop, long long len, long long& lo, long long& hi) {
    if (start < 0) { start += len; if (start < 0) start = 0; } else if (start > len) start = len;
    if (stop < 0) { stop += len; if (stop < 0) stop = 0; } else if (stop > len) stop = len;
    lo = start;
    hi = stop;
}

template <class T>
__global__ void __launch_bounds__(TRK_SIMPLE_THREADS) track_simple_kernel(const __grid_constant__ TrkSimpleParams p) {
    __shared__ long long s_gate[5];          // gated, range rows [0, 1), Doppler columns [2, 3)
    __shared__ unsigned long long s_key[TRK_SIMPLE_THREADS / 32];
    __shared__ int s_pos[TRK_SIMPLE_THREADS / 32];
    __shared__ int s_best;
    const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int rows = p.m.rows, cols = p.m.cols, n = p.m.n;
    for (int f = 0; f < p.m.nframes; ++f) {
        prc_track_simple* cur = p.hist + (size_t)s * p.m.nframes + f;
        const prc_track_simple* prev = cur - 1;
        if (tid == 0) {
            if (f == 0 && !p.resume) {
                // simple_target_tracker's initial state (target_detection.py:634-653), built positionally against
                // differently ordered fields: measurement = H x = (30, -20), measurement_idx = (35, -30),
                // estimate = (50, 50)
                prc_track_simple& z = *cur;
                const double lm[4] = {1, 0, 0, 0};
                for (int q = 0; q < 4; ++q) z.lock_mode[q] = lm[q];
                z.measurement[0] = 30.0; z.measurement[1] = -20.0;
                z.measurement_idx[0] = 35; z.measurement_idx[1] = -30;
                z.estimate[0] = 50.0; z.estimate[1] = 50.0;
                z.range_extent = p.range_extent;
                z.doppler_extent = p.doppler_extent;
                prc_kalman& k = z.kalman_state;
                const double x[4] = {30, 2, -20, -1};
                const double F1[16] = {1, 0, -0.003, 0, 0, 0, -0.003, -0.03, 0, 0, 1, 1, 0, 0, 0, 1};
                const double F2[16] = {1, 1, 0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 0, 0, 0, 1};
                const double P[4] = {5.0, 0.0225, 0.04, 0.1}, Q[4] = {2.0, 0.02, 0.2, 0.05};
                for (int q = 0; q < 4; ++q) k.x[q] = x[q];
                for (int q = 0; q < 16; ++q) {
                    k.P[q] = (q % 5 == 0) ? P[q / 5] : 0.0;
                    k.Q[q] = (q % 5 == 0) ? Q[q / 5] : 0.0;
                    k.F1[q] = F1[q];
                    k.F2[q] = F2[q];
                }
                for (int q = 0; q < 8; ++q) k.H[q] = (q == 0 || q == 6) ? 1.0 : 0.0;
                k.R[0] = 5.0; k.R[1] = 0.0; k.R[2] = 0.0; k.R[3] = 5.0;
                k.S[0] = 1.0; k.S[1] = 0.0; k.S[2] = 0.0; k.S[3] = 1.0;
            }
            if (f == 0) prev = cur;                  // frame 0 runs in place
            const double* lm = prev->lock_mode;
            const long long ly = prev->measurement_idx[0], lx = prev->measurement_idx[1];
            long long gated = 0, half_y = 0, half_x = 0;
            if (lm[1] == 1.0) { gated = 1; half_y = 24; half_x = 48; }        // initial lock-on
            else if (lm[2] == 1.0) { gated = 1; half_y = 16; half_x = 32; }   // locked
            else if (lm[3] == 1.0) { gated = 1; half_y = 24; half_x = 48; }   // losing lock
            long long y0 = 0, y1 = 0, x0 = 0, x1 = 0;
            if (gated) {
                trk_slice(ly - half_y, ly + half_y, cols, y0, y1);
                trk_slice(lx - half_x, lx + half_x, rows, x0, x1);
            }
            s_gate[0] = gated; s_gate[1] = y0; s_gate[2] = y1; s_gate[3] = x0; s_gate[4] = x1;
        }
        __syncthreads();
        if (f == 0) prev = cur;
        const bool gated = s_gate[0] != 0;
        const long long y0 = s_gate[1], y1 = s_gate[2], x0 = s_gate[3], x1 = s_gate[4];
        const double mean = p.m.mean[(long long)s * p.m.nframes + f];
        const T* __restrict__ x = static_cast<const T*>(p.m.maps) + s * p.m.seq_stride + f * p.m.frame_stride;
        // np.argmax over frame * gate: the first maximum in row-major order, NaN above everything
        unsigned long long bk = 0;
        int bp = 0x7fffffff;
        for (int o = tid; o < n; o += blockDim.x) {
            const int r = o / cols, i = o - r * cols, j = rows - 1 - r;
            const bool banded = i < 8 || i >= cols - 8 || (j >= p.zlo && j < p.zhi);
            double v = banded ? 0.0 : __ddiv_rn((double)x[o], mean);
            if (gated) v = __dmul_rn(v, (i >= y0 && i < y1 && j >= x0 && j < x1) ? 1.0 : 0.0);
            const unsigned long long key = v != v ? ~0ull : trk_key(v);
            const int pos = i * rows + j;
            if (key > bk || (key == bk && pos < bp)) { bk = key; bp = pos; }
        }
        for (int o = 16; o; o >>= 1) {
            const unsigned long long k2 = trk_shfl_u64(bk, lane ^ o);
            const int p2 = __shfl_xor_sync(0xffffffffu, bp, o);
            if (k2 > bk || (k2 == bk && p2 < bp)) { bk = k2; bp = p2; }
        }
        if (lane == 0) { s_key[w] = bk; s_pos[w] = bp; }
        __syncthreads();
        if (tid == 0) {
            for (int q = 1; q < (int)(blockDim.x >> 5); ++q)
                if (s_key[q] > bk || (s_key[q] == bk && s_pos[q] < bp)) { bk = s_key[q]; bp = s_pos[q]; }
            s_best = bp;
            const long long i0 = bp / rows, i1 = bp - (bp / rows) * rows;
            const double rext = prev->range_extent, dext = prev->doppler_extent;
            // range = rext (1 - i0 / cols), Doppler = dext (2 i1 / rows - 1)
            const double rm = __dmul_rn(rext, __dsub_rn(1.0, __ddiv_rn((double)i0, (double)cols)));
            const double dm = __dmul_rn(dext, __dsub_rn(__ddiv_rn((double)(2 * i1), (double)rows), 1.0));
            const double s0 = __dsub_rn(rm, prev->estimate[0]), s1 = __dsub_rn(dm, prev->estimate[1]);
            const double h1 = __dmul_rn(0.5, s1);
            const bool found = sqrt(__dadd_rn(__dmul_rn(s0, s0), __dmul_rn(h1, h1))) < 12.0;
            const double* lm = prev->lock_mode;
            double nl[4];
            if (found) { nl[0] = 0.0; nl[1] = lm[0]; nl[2] = lm[1] + lm[2] + lm[3]; nl[3] = 0.0; }
            else { nl[0] = lm[0] + lm[1] + lm[3]; nl[1] = 0.0; nl[2] = 0.0; nl[3] = lm[2]; }
            const double dr = rm - prev->measurement[0], dd = dm - prev->measurement[1];
            double est[2];
            trk_kalman(prev->kalman_state, cur->kalman_state, true, rm, dm, dr * dr + dd * dd, est);
            for (int q = 0; q < 4; ++q) cur->lock_mode[q] = nl[q];
            cur->measurement[0] = rm; cur->measurement[1] = dm;
            cur->measurement_idx[0] = i0; cur->measurement_idx[1] = i1;
            cur->estimate[0] = est[0]; cur->estimate[1] = est[1];
            cur->range_extent = rext;
            cur->doppler_extent = dext;
        }
        __syncthreads();
    }
}

}  // namespace prc
