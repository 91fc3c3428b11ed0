// recording.cuh -- the front end of main.py:105-166 on many equal chunks of one channel in one launch: every chunk is
// deinterleaved, frequency-shifted with its own phase offset (main.py:122-149) and resampled with resample_poly's
// line extension taken from its own end points (main.py:151-166), exactly as prc_frontend_c64 treats one chunk.
// gridDim.y is the chunk.  The staging and the polyphase sum are frontend.cuh's rs_stage / rs_sum, so every output
// is bit-identical to a per-chunk call.  I and Q are loaded as scalars: main.py slices the raw arrays by the channel
// offset (main.py:87-92), so a chunk may start at any raw element, odd ones included.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "frontend.cuh"

namespace prc {
namespace rec {

struct ChunkParams {
    ResampleParams rs;        // rs.mix describes chunk 0 (rs.mix.in, rs.mix.n); rs.mix.po and rs.ends are unused
    long long chunk_bytes;    // raw bytes from one chunk's first sample to the next one's
    long long out_stride;     // complex samples between the outputs of consecutive chunks
    const double* po;         // device: phase offset of every chunk
    float2* ends;             // device: [nchunks][2] mixed end points x[0], x[n-1] of every chunk
    int nchunks;
};

constexpr int MIX_THREADS = 256;

__device__ __forceinline__ float2 iq_load_scalar(const void* in, int kind, long long i) {
    if (kind == IQ_I8) {
        const signed char* x = static_cast<const signed char*>(in);
        return make_float2((float)x[2 * i], (float)x[2 * i + 1]);
    }
    if (kind == IQ_I16) {
        const short* x = static_cast<const short*>(in);
        return make_float2((float)x[2 * i], (float)x[2 * i + 1]);
    }
    const float* x = static_cast<const float*>(in);
    return make_float2(x[2 * i], x[2 * i + 1]);
}

// what chunk b's samples are mixed with: chunk 0's description moved to chunk b's raw samples and phase offset
__device__ __forceinline__ MixParams chunk_mix(const ChunkParams& p, int b) {
    MixParams m = p.rs.mix;
    m.in = static_cast<const char*>(p.rs.mix.in) + (size_t)b * p.chunk_bytes;
    m.po = p.po[b];
    return m;
}

__global__ void rec_ends_kernel(const __grid_constant__ ChunkParams p) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * p.nchunks) return;
    const MixParams m = chunk_mix(p, t >> 1);
    const long long i = (t & 1) ? m.n - 1 : 0;
    p.ends[t] = mix_sample(m, iq_load_scalar(m.in, m.kind, i), i);
}

__global__ void __launch_bounds__(RS_THREADS) rec_resample_kernel(const __grid_constant__ ChunkParams p,
                                                                  float2* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char rec_smem[];
    const int b = blockIdx.y;
    float* hp = reinterpret_cast<float*>(rec_smem);                              // [up][tpp]
    float2* xs = reinterpret_cast<float2*>(rec_smem + rs_table_bytes(p.rs));
    // the chunk's MixParams are rebuilt per sample from the grid constants: a copy held across the staging loop
    // would be kept live over its 64-bit divisions and spill
    const long long i_lo = rs_stage(p.rs, p.rs.mix.n, p.ends + 2 * b, hp, xs, [&p, b](long long i) {
        const MixParams m = chunk_mix(p, b);
        return mix_sample(m, iq_load_scalar(m.in, m.kind, i), i);
    });
    __syncthreads();
    const long long k = (long long)blockIdx.x * RS_THREADS + threadIdx.x;
    if (k >= p.rs.n_out) return;
    out[(size_t)b * p.out_stride + k] = rs_sum(p.rs, hp, xs, i_lo, k);
}

// up == down == 1: resample_poly returns its input, so only the mix runs (prc_frontend_c64 runs iq_mix_kernel then)
__global__ void rec_mix_kernel(const __grid_constant__ ChunkParams p, float2* __restrict__ out) {
    const int b = blockIdx.y;
    const long long i = (long long)blockIdx.x * MIX_THREADS + threadIdx.x;
    const MixParams m = chunk_mix(p, b);
    if (i >= m.n) return;
    out[(size_t)b * p.out_stride + i] = mix_sample(m, iq_load_scalar(m.in, m.kind, i), i);
}

// ---- launches (host side; prcore.cu brackets them with its profiling scope and checks the launch) ----------------
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
