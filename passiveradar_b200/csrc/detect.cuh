// detect.cuh -- CFAR_2D (reference passiveRadar/target_detection.py:683-703), SURVEY.md section 8(f).3.
//   Tfilt = ones((fw, fw)) / (fw^2 - gw^2);  Tfilt[e1:e2, e1:e2] = 0,  e1 = (fw - gw) // 2, e2 = fw - e1 + 1
//   CR = (X / mean|X|) / (convolve2d(X, Tfilt, mode='same', boundary='wrap') + 1e-10)      [ > thresh ]
// 'same' centring of scipy for an even kernel: out[i] = sum_a T[a] X[(i + c - a) mod rows], c = (fw - 1) // 2
// (so the window is NOT symmetric: offsets -(fw - 1 - c) .. +c, and the guard hole is e2 - e1 = gw + 1 wide
// when fw - gw is even -- reproduced as is).  The map is 0.6 MB: one pass, tiles with a wrapped halo in
// shared memory; the mean is a fixed-order two-stage reduction (bit-reproducible).  The window sum and the
// denominator are formed in double, as the reference's float64 Tfilt makes convolve2d do: on a signed map the
// window sums cancel, and a float32 sum of up to fw^2 cells is then off by ~1e-3 of the result.
// One launch runs a stack of maps, the frame on a grid dimension: prc_cfar2d_f32 is a stack of one, and every frame of
// prc_cfar2d_frames is summed and tiled exactly as that call would treat it alone.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace prc {

constexpr int CFAR_TX = 32, CFAR_TY = 8;
constexpr int CFAR_MEAN_CTAS = 64;
constexpr int CFAR_MAX_FW = 64;
constexpr int CFAR_MAX_ROWS = 65535 * CFAR_TY;      // gridDim.y holds one CTA row of CFAR_TY map rows

struct CfarParams {
    const void* x;             // frame 0: float [rows][cols], or float2 when is_complex (|x| is used)
    long long frame_stride;    // elements (float, or float2 with is_complex) from one frame's map to the next
    int is_complex;
    int rows, cols;
    int fw, e1, e2, c;         // kernel width, guard hole [e1, e2), centre offset
    double scale;              // 1 / (fw^2 - gw^2)
    double* partial;           // [nframes][CFAR_MEAN_CTAS] partial sums of |x|
    void* cr;                  // optional: float, or double with cr_f64
    int cr_f64;
    uint8_t* det;              // optional: cr > thresh
    float thresh;
    long long out_stride;      // elements from one frame's CR (and detections) to the next
};

// frame b's map
__device__ __forceinline__ const char* cfar_map(const CfarParams& p, int b) {
    return static_cast<const char*>(p.x) + (size_t)b * p.frame_stride * (p.is_complex ? sizeof(float2) : sizeof(float));
}

__device__ __forceinline__ double cfar_load(const CfarParams& p, const void* x, int r, int cidx) {
    const size_t idx = (size_t)r * p.cols + cidx;
    if (p.is_complex) {
        const float2 v = reinterpret_cast<const float2*>(x)[idx];
        return (double)hypotf(v.x, v.y);
    }
    return (double)reinterpret_cast<const float*>(x)[idx];
}

// the partial sums of |x| of frame blockIdx.y, over a fixed 64-CTA partition
__global__ void cfar_frames_abssum_kernel(const __grid_constant__ CfarParams p) {
    __shared__ double red[256];
    const void* x = cfar_map(p, blockIdx.y);
    const long long total = (long long)p.rows * p.cols;
    const long long per = (total + gridDim.x - 1) / gridDim.x;
    const long long lo = blockIdx.x * per;
    long long hi = lo + per;
    if (hi > total) hi = total;
    double s = 0.0;
    for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        float v;
        if (p.is_complex) {
            const float2 z = reinterpret_cast<const float2*>(x)[i];
            v = hypotf(z.x, z.y);
        } else {
            v = fabsf(reinterpret_cast<const float*>(x)[i]);
        }
        s += (double)v;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int w = blockDim.x / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) p.partial[(size_t)blockIdx.y * CFAR_MEAN_CTAS + blockIdx.x] = red[0];
}

// the window sums and CR of frame blockIdx.z
__global__ void __launch_bounds__(CFAR_TX * CFAR_TY) cfar_frames_kernel(const __grid_constant__ CfarParams p) {
    extern __shared__ double cfar_tile[];                // [(TY + fw - 1)][(TX + fw - 1)]
    __shared__ double s_inv_mean;
    const int b = blockIdx.z;
    const void* x = cfar_map(p, b);
    const int fw = p.fw;
    const int tw = CFAR_TX + fw - 1, th = CFAR_TY + fw - 1;
    const int i0 = blockIdx.y * CFAR_TY, j0 = blockIdx.x * CFAR_TX;
    const int tid = threadIdx.y * CFAR_TX + threadIdx.x;
    if (tid == 0) {
        const double* part = p.partial + (size_t)b * CFAR_MEAN_CTAS;
        double s = 0.0;
        for (int q = 0; q < CFAR_MEAN_CTAS; ++q) s += part[q];
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
        cfar_tile[q] = cfar_load(p, x, r, cc);
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
        for (int bb = 0; bb < fw; ++bb) {
            if (hole_row && bb >= p.e1 && bb < p.e2) continue;
            racc += row[-bb];
        }
        acc += racc;
    }
    const double xv = cfar_tile[(threadIdx.y + fw - 1 - p.c) * tw + threadIdx.x + fw - 1 - p.c];   // a = b = c: X[i][j]
    double num = xv;
    if (!p.is_complex) num = reinterpret_cast<const float*>(x)[(size_t)i * p.cols + j];            // keep the sign of a real X
    const double cr = (num * s_inv_mean) / (acc * p.scale + 1e-10);
    const size_t o = (size_t)b * p.out_stride + (size_t)i * p.cols + j;
    if (p.cr) {
        if (p.cr_f64) static_cast<double*>(p.cr)[o] = cr;
        else static_cast<float*>(p.cr)[o] = (float)cr;
    }
    if (p.det) p.det[o] = cr > (double)p.thresh ? 1 : 0;
}

// ---- launches (host side; prcore_detect.cu brackets them with its profiling scope and checks the launch) ----------------
inline cudaError_t allow_cfar_smem(int bytes) {
    return cudaFuncSetAttribute(cfar_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

inline void launch_cfar(const CfarParams& p, int nframes, cudaStream_t st) {
    cfar_frames_abssum_kernel<<<dim3(CFAR_MEAN_CTAS, (unsigned)nframes), 256, 0, st>>>(p);
    const size_t smem = (size_t)(CFAR_TX + p.fw - 1) * (CFAR_TY + p.fw - 1) * sizeof(double);   // 53 960 B at fw = 64
    const dim3 grid((unsigned)((p.cols + CFAR_TX - 1) / CFAR_TX), (unsigned)((p.rows + CFAR_TY - 1) / CFAR_TY),
                    (unsigned)nframes);
    cfar_frames_kernel<<<grid, dim3(CFAR_TX, CFAR_TY), smem, st>>>(p);
}

}  // namespace prc
