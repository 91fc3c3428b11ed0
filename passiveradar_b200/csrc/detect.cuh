// detect.cuh -- CFAR_2D (reference passiveRadar/target_detection.py:683-703), SURVEY.md section 8(f).3.
//   Tfilt = ones((fw, fw)) / (fw^2 - gw^2);  Tfilt[e1:e2, e1:e2] = 0,  e1 = (fw - gw) // 2, e2 = fw - e1 + 1
//   CR = (X / mean|X|) / (convolve2d(X, Tfilt, mode='same', boundary='wrap') + 1e-10)      [ > thresh ]
// 'same' centring of scipy for an even kernel: out[i] = sum_a T[a] X[(i + c - a) mod rows], c = (fw - 1) // 2
// (so the window is NOT symmetric: offsets -(fw - 1 - c) .. +c, and the guard hole is e2 - e1 = gw + 1 wide
// when fw - gw is even -- reproduced as is).  The map is 0.6 MB: one pass, tiles with a wrapped halo in
// shared memory; the mean is a fixed-order two-stage reduction (bit-reproducible).  The window sum and the
// denominator are formed in double, as the reference's float64 Tfilt makes convolve2d do: on a signed map the
// window sums cancel, and a float32 sum of up to fw^2 cells is then off by ~1e-3 of the result.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace prc {

constexpr int CFAR_TX = 32, CFAR_TY = 8;
constexpr int CFAR_MEAN_CTAS = 64;
constexpr int CFAR_MAX_FW = 64;
constexpr int CFAR_MAX_ROWS = 65535 * CFAR_TY;      // gridDim.y holds one CTA row of CFAR_TY map rows

struct CfarParams {
    const void* x;       // float [rows][cols], or float2 when is_complex (|x| is used)
    int is_complex;
    int rows, cols;
    int fw, e1, e2, c;   // kernel width, guard hole [e1, e2), centre offset
    double scale;        // 1 / (fw^2 - gw^2)
    int has_thresh;
    float thresh;
    const double* partial;   // [CFAR_MEAN_CTAS] partial sums of |x|
    float* cr;           // optional
    uint8_t* det;        // optional (needs has_thresh)
};

__device__ __forceinline__ double cfar_load(const CfarParams& p, int r, int cidx) {
    const size_t idx = (size_t)r * p.cols + cidx;
    if (p.is_complex) {
        const float2 v = reinterpret_cast<const float2*>(p.x)[idx];
        return (double)hypotf(v.x, v.y);
    }
    return (double)reinterpret_cast<const float*>(p.x)[idx];
}

__global__ void cfar_abssum_kernel(const __grid_constant__ CfarParams p, double* __restrict__ partial) {
    __shared__ double red[256];
    const long long total = (long long)p.rows * p.cols;
    const long long per = (total + gridDim.x - 1) / gridDim.x;
    const long long lo = blockIdx.x * per;
    long long hi = lo + per;
    if (hi > total) hi = total;
    double s = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        float v;
        if (p.is_complex) {
            const float2 z = reinterpret_cast<const float2*>(p.x)[i];
            v = hypotf(z.x, z.y);
        } else {
            v = fabsf(reinterpret_cast<const float*>(p.x)[i]);
        }
        s += (double)v;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int w = blockDim.x / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(CFAR_TX * CFAR_TY) cfar2d_kernel(const __grid_constant__ CfarParams p) {
    extern __shared__ double cfar_tile[];                // [(TY + fw - 1)][(TX + fw - 1)]
    __shared__ double s_inv_mean;
    const int fw = p.fw;
    const int tw = CFAR_TX + fw - 1, th = CFAR_TY + fw - 1;
    const int i0 = blockIdx.y * CFAR_TY, j0 = blockIdx.x * CFAR_TX;
    const int tid = threadIdx.y * CFAR_TX + threadIdx.x;
    if (tid == 0) {
        double s = 0.0;
        for (int q = 0; q < CFAR_MEAN_CTAS; ++q) s += p.partial[q];
        s_inv_mean = (double)p.rows * (double)p.cols / s;
    }
    // tile row t <-> map row (i0 + c - (fw - 1) + t) mod rows
    const int rbase = i0 + p.c - (fw - 1), cbase = j0 + p.c - (fw - 1);
    for (int q = tid; q < tw * th; q += CFAR_TX * CFAR_TY) {
        const int tr = q / tw, tc = q - tr * tw;
        int r = (rbase + tr) % p.rows;
        if (r < 0) r += p.rows;
        int cc = (cbase + tc) % p.cols;
        if (cc < 0) cc += p.cols;
        cfar_tile[q] = cfar_load(p, r, cc);
    }
    __syncthreads();
    const int i = i0 + threadIdx.y, j = j0 + threadIdx.x;
    if (i >= p.rows || j >= p.cols) return;
    // X[(i + c - a)] = tile[(i - i0) + (fw - 1) - a]
    double acc = 0.0;
    for (int a = 0; a < fw; ++a) {
        const double* row = cfar_tile + (threadIdx.y + fw - 1 - a) * tw + threadIdx.x + fw - 1;
        const bool hole_row = a >= p.e1 && a < p.e2;
        double racc = 0.0;
        for (int b = 0; b < fw; ++b) {
            if (hole_row && b >= p.e1 && b < p.e2) continue;
            racc += row[-b];
        }
        acc += racc;
    }
    const double xv = cfar_tile[(threadIdx.y + fw - 1 - p.c) * tw + threadIdx.x + fw - 1 - p.c];   // a = b = c: X[i][j]
    double num = xv;
    if (!p.is_complex) num = reinterpret_cast<const float*>(p.x)[(size_t)i * p.cols + j];          // keep the sign of a real X
    const double cr = (num * s_inv_mean) / (acc * p.scale + 1e-10);
    const size_t o = (size_t)i * p.cols + j;
    if (p.cr) p.cr[o] = (float)cr;
    if (p.det && p.has_thresh) p.det[o] = cr > (double)p.thresh ? 1 : 0;
}

// one row of direct_xambg: out[f][k] = sum over pieces of partial[piece][R - k]
__global__ void piece_sum_kernel(const float2* __restrict__ partial, int npieces, int HT, int R, float2* __restrict__ out_row) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > R) return;
    float2 s = make_float2(0.f, 0.f);
    for (int q = 0; q < npieces; ++q) {
        const float2 v = partial[(size_t)q * HT + (R - k)];
        s.x += v.x;
        s.y += v.y;
    }
    out_row[k] = s;
}

}  // namespace prc
