// oscfar.cuh -- ordered-statistic CFAR (Rohling) on CFAR_2D's window: the noise estimate of a cell is the k-th smallest
// of the N cells CFAR_2D sums (detect.cuh's header comment gives their placement), not their mean.
//   T(i, j) = k-th smallest of { X[(i + c - a) mod rows, (j + c - b) mod cols] : Tfilt[a, b] != 0 },  1 <= k <= N
//   CR      = (num * inv_mean) / (T + 1e-10)      in double
// where num, inv_mean = rows*cols / sum|X| and the sign of a real cell are formed exactly as cfar_frames_kernel forms
// them (the sum through cfar_frames_abssum_kernel's partition), so OS and CA differ only in the denominator.  Complex
// maps use hypotf(re, im), as cfar_load forms it.
//
// Selection: the CTA stages a wrapped tile of order-preserving uint32 keys of the float32 values in shared memory
// ((OS_ROWS + fw - 1) x (OS_TX + fw - 1) x 4 B, 30 020 B at fw = 64).  Each thread selects for two vertically adjacent
// cells at once: their windows share fw - 1 of their fw + 1 tile rows, so every key it loads is compared with both
// cells' candidates and the shared-memory traffic per cell is halved.  The key is found exactly by bisection on its
// bits: one pass takes the window's minimum and maximum, whose common leading bits the k-th key shares; then one pass
// per remaining bit counts the keys below the candidate prefix with that bit set.  Every pass is a compare and a
// predicated add per key, with no counter array, so nothing spills.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "detect.cuh"

namespace prc {
namespace oscfar {

constexpr int OS_TX = 32, OS_TY = 8;
constexpr int OS_CELLS = 2;                     // vertically adjacent cells per thread
constexpr int OS_ROWS = OS_TY * OS_CELLS;       // map rows of one CTA (CFAR_MAX_ROWS needs 32 768 CTA rows)

struct OsParams {
    CfarParams c;        // map, window geometry, partial sums and CR output, as cfar_frames_kernel reads them (det unused)
    int k;               // rank, 1 <= k <= N
    int h0, h1;          // guard hole: rows and columns [h0, h1) of the window (h1 = max(e1, e2))
};

// order-preserving float32 <-> uint32 keys: a < b as floats (with -0 < +0) iff key(a) < key(b) as unsigned
__device__ __forceinline__ uint32_t os_key(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float os_value(uint32_t key) {
    return __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}

// the two cells' passes over their windows: A / B say whether a key belongs to cell 0's / cell 1's window
struct OsMinMax {
    uint32_t mn0 = 0xffffffffu, mx0 = 0u, mn1 = 0xffffffffu, mx1 = 0u;
    template <bool A, bool B> __device__ __forceinline__ void at(uint32_t v) {
        if (A) { mn0 = min(mn0, v); mx0 = max(mx0, v); }
        if (B) { mn1 = min(mn1, v); mx1 = max(mx1, v); }
    }
};

struct OsCount {
    uint32_t t0, t1;
    int n0 = 0, n1 = 0;
    template <bool A, bool B> __device__ __forceinline__ void at(uint32_t v) {
        if (A) n0 += v < t0 ? 1 : 0;
        if (B) n1 += v < t1 ? 1 : 0;
    }
};

// columns [b0, b1) of one tile row (row[-b] is window column b); in0 / in1 are the same for every thread of the CTA
template <class Op>
__device__ __forceinline__ void os_segment(Op& op, const uint32_t* row, int b0, int b1, bool in0, bool in1) {
    if (in0 && in1) {
        for (int b = b0; b < b1; ++b) op.template at<true, true>(row[-b]);
    } else if (in0) {
        for (int b = b0; b < b1; ++b) op.template at<true, false>(row[-b]);
    } else if (in1) {
        for (int b = b0; b < b1; ++b) op.template at<false, true>(row[-b]);
    }
}

// Tile row u of the thread's fw + 1 rows is window row a0 = fw - 1 - u of cell 0 (u < fw) and a1 = fw - u of cell 1
// (u > 0).  A window row inside the hole skips columns [h0, h1).
template <class Op>
__device__ __forceinline__ void os_visit(Op& op, const uint32_t* rows, int tw, const OsParams& p) {
    const int fw = p.c.fw, h0 = p.h0, h1 = p.h1;
    for (int u = 0; u <= fw; ++u) {
        const int a0 = fw - 1 - u, a1 = fw - u;
        const bool v0 = u < fw, v1 = u > 0;
        const bool hole0 = a0 >= h0 && a0 < h1, hole1 = a1 >= h0 && a1 < h1;
        const uint32_t* row = rows + u * tw;
        os_segment(op, row, 0, h0, v0, v1);
        os_segment(op, row, h0, h1, v0 && !hole0, v1 && !hole1);
        os_segment(op, row, h1, fw, v0, v1);
    }
}

// the CR of frame blockIdx.z; thread (x, y) serves cells (i0 + 2y + s, j0 + x), s = 0, 1
__global__ void __launch_bounds__(OS_TX * OS_TY) os_select_kernel(const __grid_constant__ OsParams p) {
    extern __shared__ uint32_t os_tile[];             // [(OS_ROWS + fw - 1)][(OS_TX + fw - 1)]
    __shared__ double s_inv_mean;
    const CfarParams& q = p.c;
    const int b = blockIdx.z;
    const void* x = cfar_map(q, b);
    const int fw = q.fw;
    const int tw = OS_TX + fw - 1, th = OS_ROWS + fw - 1;
    const int i0 = blockIdx.y * OS_ROWS, j0 = blockIdx.x * OS_TX;
    const int tid = threadIdx.y * OS_TX + threadIdx.x;
    if (tid == 0) {                                   // cfar_frames_kernel's mean, summed in the same order
        const double* part = q.partial + (size_t)b * CFAR_MEAN_CTAS;
        double s = 0.0;
        for (int r = 0; r < CFAR_MEAN_CTAS; ++r) s += part[r];
        s_inv_mean = (double)q.rows * (double)q.cols / s;
    }
    // tile row t <-> map row (i0 + c - (fw - 1) + t) mod rows, as in cfar_frames_kernel
    const int rbase = i0 + q.c - (fw - 1), cbase = j0 + q.c - (fw - 1);
    for (int e = tid; e < tw * th; e += OS_TX * OS_TY) {
        const int tr = e / tw, tc = e - tr * tw;
        int r = (rbase + tr) % q.rows;
        if (r < 0) r += q.rows;
        int cc = (cbase + tc) % q.cols;
        if (cc < 0) cc += q.cols;
        os_tile[e] = os_key((float)cfar_load(q, x, r, cc));     // cfar_load widens a float32: exact
    }
    __syncthreads();
    const int i = i0 + OS_CELLS * threadIdx.y, j = j0 + threadIdx.x;
    if (i >= q.rows || j >= q.cols) return;
    // cell s's X[(i + s + c - a)][(j + c - bb)] = tile[OS_CELLS*y + s + fw - 1 - a][x + fw - 1 - bb]
    const uint32_t* rows = os_tile + (OS_CELLS * threadIdx.y) * tw + threadIdx.x + fw - 1;

    OsMinMax mm;
    os_visit(mm, rows, tw, p);
    // the k-th key lies in [min, max]: it shares their common leading bits, and the nb bits below are searched
    const uint32_t diff = (mm.mn0 ^ mm.mx0) | (mm.mn1 ^ mm.mx1);
    const int nb = 32 - __clz(diff);
    const uint32_t low = nb == 0 ? 0u : 0xffffffffu >> (32 - nb);
    uint32_t k0 = mm.mn0 & ~low, k1 = mm.mn1 & ~low;     // count(key < k_s) < k holds throughout
    for (int bit = nb - 1; bit >= 0; --bit) {
        OsCount cnt;
        cnt.t0 = k0 | (1u << bit);
        cnt.t1 = k1 | (1u << bit);
        os_visit(cnt, rows, tw, p);
        if (cnt.n0 < p.k) k0 = cnt.t0;
        if (cnt.n1 < p.k) k1 = cnt.t1;
    }

    const double inv_mean = s_inv_mean;
    for (int s = 0; s < OS_CELLS; ++s) {
        const int ii = i + s;
        if (ii >= q.rows) break;
        const double num = cfar_load(q, x, ii, j);      // the sign of a real cell kept; |x| of a complex one
        const double t = (double)os_value(s == 0 ? k0 : k1);
        const double cr = (num * inv_mean) / (t + 1e-10);
        const size_t o = (size_t)b * q.out_stride + (size_t)ii * q.cols + j;
        if (q.cr_f64) static_cast<double*>(q.cr)[o] = cr;
        else static_cast<float*>(q.cr)[o] = (float)cr;
    }
}

// ---- launches (host side; prcore_detect.cu brackets them with its profiling scope and checks the launch) ----------------
inline size_t os_smem(int fw) { return (size_t)(OS_TX + fw - 1) * (OS_ROWS + fw - 1) * sizeof(uint32_t); }

inline void launch_os_cfar(const OsParams& p, int nframes, cudaStream_t st) {
    cfar_frames_abssum_kernel<<<dim3(CFAR_MEAN_CTAS, (unsigned)nframes), 256, 0, st>>>(p.c);
    const dim3 grid((unsigned)((p.c.cols + OS_TX - 1) / OS_TX), (unsigned)((p.c.rows + OS_ROWS - 1) / OS_ROWS),
                    (unsigned)nframes);
    os_select_kernel<<<grid, dim3(OS_TX, OS_TY), os_smem(p.c.fw), st>>>(p);
}

}  // namespace oscfar
}  // namespace prc
