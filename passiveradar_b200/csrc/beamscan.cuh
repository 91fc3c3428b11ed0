// beamscan.cuh -- conventional (Bartlett) beamscan of K co-registered range-Doppler maps: one amplitude map and one
// fractional bearing index per cell.
//   P[a] = | sum_k S[a, k] * m_k |^2                         a = 0 .. A-1, float32
//   a*   = the first a with the largest P[a]                  (strict ">" scanning a upwards)
//   amp  = sqrtf(P[a*])
//   den  = P[a*-1] - 2 P[a*] + P[a*+1];  delta = clamp(0.5 (P[a*-1] - P[a*+1]) / den, -0.5, 0.5) if den < 0, else 0
//   pos  = a* + delta
// The neighbours of a* wrap mod A with `wrap` (a full-circle grid); without it delta = 0 at a* = 0 and a* = A-1.  In
// wrap mode a pos that rounds to A - 0.5 is folded to -0.5, so pos lies in [-0.5, A - 0.5).
// The CAF conjugates the surveillance channel, so an echo from theta gives m_k = conj(a_k(theta)) * c and the table is
// used as given (DESIGN.md section 21).
//
// Work split: a thread holds the K complex values of BS_CPT cells in registers; the CTA stages the steering table in
// shared memory BS_TA angles at a time, and every entry a thread reads (a broadcast) serves all of its cells.  Per cell
// the scan keeps the running maximum, its index, its left neighbour, the value right after it, the previous value and
// P[0]; P[A-1] is the previous value when the scan ends.  No P array is stored.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace prc {
namespace beam {

constexpr int BS_THREADS = 256;
constexpr int BS_CPT = 4;                 // cells per thread (64 .. 96 registers at K = 1 .. 4: two CTAs per SM)
constexpr int BS_TA = 512;                // angles per staged tile: BS_TA * K * 8 B of shared memory (16 KB at K = 4)
constexpr int BS_MAX_ANGLES = 4096;
constexpr int BS_MAX_CHAN = 4;

struct BeamParams {
    const float2* maps;        // channel k of frame f at maps + k*chan_stride + f*frame_stride
    const float2* steer;       // [A][K], device copy of the caller's table
    float* amp;                // frame f at amp + f*out_stride, or NULL
    float* pos;                // frame f at pos + f*out_stride, or NULL
    long long cells;           // rows * cols
    long long frame_stride, chan_stride, out_stride;
    int nangles;
    int wrap;
};

// one cell's scan state
struct BeamCell {
    float best, left, right, prev, p0;
    int anext;                 // a* + 1
};

template <int K>
__device__ __forceinline__ float beam_power(const float2 (&m)[K], const float2* s) {
    float re = s[0].x * m[0].x, im = s[0].x * m[0].y;
    re = fmaf(-s[0].y, m[0].y, re);
    im = fmaf(s[0].y, m[0].x, im);
#pragma unroll
    for (int k = 1; k < K; ++k) {
        re = fmaf(s[k].x, m[k].x, re);
        re = fmaf(-s[k].y, m[k].y, re);
        im = fmaf(s[k].x, m[k].y, im);
        im = fmaf(s[k].y, m[k].x, im);
    }
    return fmaf(re, re, im * im);
}

// grid (ceil(cells / (BS_THREADS * BS_CPT)), nframes); thread t of CTA x serves cells x*BS_THREADS*BS_CPT + j*BS_THREADS + t
template <int K>
__global__ void __launch_bounds__(BS_THREADS, 2) beamscan_kernel(const __grid_constant__ BeamParams p) {
    __shared__ float2 s_steer[BS_TA * K];
    const int A = p.nangles;
    const long long f = blockIdx.y;
    const long long c0 = (long long)blockIdx.x * (BS_THREADS * BS_CPT) + threadIdx.x;
    const float2* frame = p.maps + f * p.frame_stride;

    float2 m[BS_CPT][K];
    BeamCell st[BS_CPT];
#pragma unroll
    for (int j = 0; j < BS_CPT; ++j) {
        const long long c = c0 + (long long)j * BS_THREADS;
#pragma unroll
        for (int k = 0; k < K; ++k) m[j][k] = c < p.cells ? frame[k * p.chan_stride + c] : make_float2(0.f, 0.f);
    }

    for (int t0 = 0; t0 < A; t0 += BS_TA) {
        const int na = min(BS_TA, A - t0);
        if (t0 > 0) __syncthreads();                      // the previous tile is no longer read
        for (int e = threadIdx.x; e < na * K; e += BS_THREADS) s_steer[e] = p.steer[(size_t)t0 * K + e];
        __syncthreads();
        int a0 = 0;
        if (t0 == 0) {                                    // angle 0 opens every cell's scan
#pragma unroll
            for (int j = 0; j < BS_CPT; ++j) {
                const float v = beam_power<K>(m[j], s_steer);
                st[j].best = st[j].left = st[j].right = st[j].prev = st[j].p0 = v;
                st[j].anext = 1;
            }
            a0 = 1;
        }
#pragma unroll 2
        for (int a = a0; a < na; ++a) {
            const float2* s = s_steer + a * K;
            const int ag = t0 + a;
#pragma unroll
            for (int j = 0; j < BS_CPT; ++j) {
                const float v = beam_power<K>(m[j], s);
                BeamCell& q = st[j];
                if (ag == q.anext) q.right = v;
                if (v > q.best) { q.best = v; q.left = q.prev; q.anext = ag + 1; }
                q.prev = v;
            }
        }
    }

    const long long ob = f * p.out_stride;
#pragma unroll
    for (int j = 0; j < BS_CPT; ++j) {
        const long long c = c0 + (long long)j * BS_THREADS;
        if (c >= p.cells) break;
        const BeamCell& q = st[j];
        const int as = q.anext - 1;
        if (p.amp) p.amp[ob + c] = sqrtf(q.best);
        if (!p.pos) continue;
        float left = q.left, right = q.right;
        bool edge = false;
        if (as == 0) { if (p.wrap) left = q.prev; else edge = true; }          // q.prev is P[A-1] now
        if (as == A - 1) { if (p.wrap) right = q.p0; else edge = true; }
        float delta = 0.f;
        const float den = (left - 2.f * q.best) + right;
        if (!edge && den < 0.f) delta = fminf(0.5f, fmaxf(-0.5f, 0.5f * (left - right) / den));
        float pos = (float)as + delta;
        if (p.wrap && pos >= (float)A - 0.5f) pos -= (float)A;
        p.pos[ob + c] = pos;
    }
}

// ---- launch (host side; prcore_array.cu brackets it with its profiling scope and checks the launch) -------------------
inline void launch_beamscan(const BeamParams& p, int nchan, int nframes, cudaStream_t st) {
    const dim3 grid((unsigned)((p.cells + BS_THREADS * BS_CPT - 1) / (BS_THREADS * BS_CPT)), (unsigned)nframes);
    switch (nchan) {
        case 1: beamscan_kernel<1><<<grid, BS_THREADS, 0, st>>>(p); break;
        case 2: beamscan_kernel<2><<<grid, BS_THREADS, 0, st>>>(p); break;
        case 3: beamscan_kernel<3><<<grid, BS_THREADS, 0, st>>>(p); break;
        default: beamscan_kernel<4><<<grid, BS_THREADS, 0, st>>>(p); break;
    }
}

}  // namespace beam
}  // namespace prc
