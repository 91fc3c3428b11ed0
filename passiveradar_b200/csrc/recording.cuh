// recording.cuh -- the front end of main.py:105-166 on one or many equal chunks of one channel in one launch: every
// chunk is deinterleaved, frequency-shifted with its own phase offset (main.py:122-149) and resampled with
// resample_poly's line extension taken from its own end points (main.py:151-166).  gridDim.y is the chunk.  These are
// the front end's only kernels: prc_iq_mix_c64 and prc_frontend_c64 run them on one chunk, so every chunk of
// prc_frontend_chunks_c64 is bit-identical to a single call on it.  I and Q are loaded as scalars: main.py slices the
// raw arrays by the channel offset (main.py:87-92), so a chunk may start at any raw element, odd ones included.  With
// PRC_FLAG_CHANNEL_PAIR the raw input is one channel of a two-channel stream (rs.mix.pitch = 4): complex sample i is
// raw elements 4i and 4i+1, and the other channel's samples in between are never read.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "frontend.cuh"

namespace prc {
namespace rec {

struct ChunkParams {
    ResampleParams rs;        // rs.mix describes chunk 0 (rs.mix.in, rs.mix.n); only the mix is read when up == down == 1
    long long chunk_bytes;    // raw bytes from one chunk's first sample to the next one's
    long long out_stride;     // complex samples between the outputs of consecutive chunks
    const double* po;         // device: phase offset of every chunk, or NULL: rs.mix.po (a single call)
    float2* ends;             // device: [nchunks][2] mixed end points x[0], x[n-1] of every chunk
    int nchunks;
};

constexpr int MIX_THREADS = 256;

// what chunk b's samples are mixed with: chunk 0's description moved to chunk b's raw samples and phase offset
__device__ __forceinline__ MixParams chunk_mix(const ChunkParams& p, int b) {
    MixParams m = p.rs.mix;
    m.in = static_cast<const char*>(p.rs.mix.in) + (size_t)b * p.chunk_bytes;
    if (p.po) m.po = p.po[b];
    return m;
}

__global__ void rec_ends_kernel(const __grid_constant__ ChunkParams p) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * p.nchunks) return;
    const MixParams m = chunk_mix(p, t >> 1);
    const long long i = (t & 1) ? m.n - 1 : 0;
    p.ends[t] = mix_sample(m, iq_load_scalar(m.in, m.kind, i, m.pitch), i);
}

__global__ void __launch_bounds__(RS_THREADS) rec_resample_kernel(const __grid_constant__ ChunkParams p,
                                                                  float2* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char rec_smem[];
    const ResampleParams& rp = p.rs;
    const int b = blockIdx.y;
    const long long n = rp.mix.n;
    float* hp = reinterpret_cast<float*>(rec_smem);                               // [up][tpp]
    float2* xs = reinterpret_cast<float2*>(rec_smem + rs_table_bytes(rp));
    // the polyphase table and the CTA's window xext[i_lo, i_lo + span) into shared memory
    const long long m0 = (long long)blockIdx.x * RS_THREADS;
    // input index range of this CTA: output m uses i = floor(T / up) - j, j = 0 .. tpp-1, T = (m + npr) * down
    const long long Tlo = (m0 + rp.n_pre_remove) * (long long)rp.down;
    const long long i_hi0 = Tlo / rp.up;                     // largest index of the first output
    const long long i_lo = i_hi0 - (rp.tpp - 1);             // smallest index any output of the CTA needs
    for (int q = threadIdx.x; q < rp.up * rp.tpp; q += RS_THREADS) hp[q] = rp.hp[q];
    const float2 x0 = p.ends[2 * b], x1 = p.ends[2 * b + 1];
    // n == 1 gives 0/0 = NaN, and every output NaN, as scipy's padtype='line' does
    const float2 slope = make_float2((x1.x - x0.x) / (float)(n - 1), (x1.y - x0.y) / (float)(n - 1));
    for (int q = threadIdx.x; q < rp.span; q += RS_THREADS) {
        const long long i = i_lo + q;
        float2 v;
        if (i < 0) v = make_float2(x0.x + (float)i * slope.x, x0.y + (float)i * slope.y);
        else if (i >= n) v = make_float2(x1.x + (float)(i - n + 1) * slope.x, x1.y + (float)(i - n + 1) * slope.y);
        else {
            // the chunk's MixParams are rebuilt per sample from the grid constants: a copy held across the staging
            // loop would be kept live over its 64-bit divisions and spill
            const MixParams m = chunk_mix(p, b);
            v = mix_sample(m, iq_load_scalar(m.in, m.kind, i, m.pitch), i);
        }
        xs[q] = v;
    }
    __syncthreads();
    const long long k = m0 + threadIdx.x;
    if (k >= rp.n_out) return;
    out[(size_t)b * p.out_stride + k] = rs_sum(rp, hp, xs, i_lo, k);
}

// up == down == 1: resample_poly returns its input, so only the mix runs
__global__ void rec_mix_kernel(const __grid_constant__ ChunkParams p, float2* __restrict__ out) {
    const int b = blockIdx.y;
    const long long i = (long long)blockIdx.x * MIX_THREADS + threadIdx.x;
    const MixParams m = chunk_mix(p, b);
    if (i >= m.n) return;
    out[(size_t)b * p.out_stride + i] = mix_sample(m, iq_load_scalar(m.in, m.kind, i, m.pitch), i);
}

// ---- launches (host side; prcore_signal.cu brackets them with its profiling scope and checks the launch) ----------------
inline cudaError_t allow_smem(int bytes) {
    return cudaFuncSetAttribute(rec_resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

inline void launch_resample(const ChunkParams& p, size_t smem, float2* out, cudaStream_t st) {
    rec_ends_kernel<<<(unsigned)((2 * p.nchunks + 255) / 256), 256, 0, st>>>(p);
    const dim3 grid((unsigned)((p.rs.n_out + RS_THREADS - 1) / RS_THREADS), (unsigned)p.nchunks);
    rec_resample_kernel<<<grid, RS_THREADS, smem, st>>>(p, out);
}

inline void launch_mix(const ChunkParams& p, float2* out, cudaStream_t st) {
    const dim3 grid((unsigned)((p.rs.mix.n + MIX_THREADS - 1) / MIX_THREADS), (unsigned)p.nchunks);
    rec_mix_kernel<<<grid, MIX_THREADS, 0, st>>>(p, out);
}

}  // namespace rec
}  // namespace prc
