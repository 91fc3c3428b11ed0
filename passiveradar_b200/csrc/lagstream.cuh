// lagstream.cuh -- persistent, software-pipelined lag-correlation kernel (sm_90a).
//
// Same arithmetic as lagcorr_kernel (kernels.cuh):
//     partial[prob][blk][piece][l] = sum_{i in piece of block blk} x[i] * conj(s[(i + dmin + l) mod n])
// but organised for the FP32 pipe instead of for simplicity:
//   * the blocks of one problem are laid end to end as one stream of nblk*blk_len samples and cut
//     into gridDim.x equal ranges, one per CTA ("stream-K"): every SM gets the same amount of work
//     whatever F, N and R are (256 Doppler blocks on 132 SMs lose 3 % to wave quantisation when a
//     CTA is tied to a block); a CTA that crosses a block boundary flushes one partial row per block
//     it touched ("piece");
//   * inside its range a CTA walks sub-chunks of <= G*steps*TI samples; sub-chunk k+1 is copied
//     global -> shared with cp.async (LDGSTS, zero-fill outside the signal) while sub-chunk k is in
//     the MAC loop: staging never leaves the math pipe idle;
//   * the register accumulators hold one sub-chunk (<= steps*TI samples per thread); after each
//     sub-chunk a thread folds them into its own slot of the reduction scratch with a compensated
//     (Kahan) sum, so the FP32 error does not grow with the length of a piece (a CTA's range can
//     span a whole 2**20-sample channel); the cross-group reduction and the partial row
//     are paid once per piece, not once per 1-2k samples.
// x must already carry its weights (ref, or ref*window written by weight_kernel); the tap-weighted
// decimator of fast_xambg(shortFilt=False) keeps using lagcorr_kernel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"

namespace prc {

struct LagStreamParams {
    const float2* x;
    const float2* s[2];
    int dmin[2];
    int n;
    long long blk_first_lo;
    long long blk_stride;
    int blk_len;
    int nblk;
    long long total;      // nblk * blk_len
    long long per_cta;    // samples of the stream per CTA
    int H, G, steps;      // lag groups, sample groups, max TI-steps per group and sub-chunk
    int maxpieces;        // partial rows reserved per block
    int s_linear;         // 1: s is zero outside [0, n) (LS_Filter_Toeplitz) instead of circular
    float2* partial;      // [prob][nblk][maxpieces][H*TD]
};

__device__ __forceinline__ void cp_async8(float2* dst, const float2* src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    const int bytes = valid ? 8 : 0;          // src-size 0 => the 8 bytes are zero-filled
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(d), "l"(src), "r"(bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// one sub-chunk of the CTA's walk through the stream
struct SubChunk {
    long long i0;     // first sample index (may be negative / beyond n: zero-filled)
    int len;          // samples (0 => end of range)
    int steps;        // TI-steps per sample group for this sub-chunk
    int blk;          // block it belongs to
    int flush;        // last sub-chunk of its piece: reduce + write the partial row afterwards
};

template <int TI>
__device__ __forceinline__ SubChunk next_subchunk(const LagStreamParams& p, long long q, long long q1) {
    SubChunk sc;
    if (q >= q1) {
        sc.i0 = 0; sc.len = 0; sc.steps = 0; sc.blk = 0; sc.flush = 0;
        return sc;
    }
    const long long blk = q / p.blk_len;
    const int off = (int)(q - blk * p.blk_len);
    long long seg_end = (blk + 1) * (long long)p.blk_len;
    if (seg_end > q1) seg_end = q1;
    const int lmax = p.G * p.steps * TI;
    long long len = seg_end - q;
    if (len > lmax) len = lmax;
    sc.i0 = p.blk_first_lo + blk * p.blk_stride + off;
    sc.len = (int)len;
    sc.steps = ((int)len + p.G * TI - 1) / (p.G * TI);
    sc.blk = (int)blk;
    sc.flush = (q + len == seg_end);
    return sc;
}

template <int TI, int TD>
__global__ void __launch_bounds__(512) lagstream_kernel(const __grid_constant__ LagStreamParams p) {
    extern __shared__ __align__(16) float2 smem[];
    const int tid = threadIdx.x;
    const int nthr = blockDim.x;
    const int prob = blockIdx.y;
    const int HT = p.H * TD;
    const int Lmax = p.G * p.steps * TI;
    // shared layout: two staging buffers {x[Lmax], s[Lmax + HT]}, the per-thread sums [G][HT] (thread (g, h) owns
    // entries g*HT + h*TD .. + TD - 1; the flush reduces them over g) and their Kahan compensations [G][HT]
    const int bufsz = 2 * Lmax + HT;
    float2* red = smem + 2 * bufsz;
    float2* comp = red + p.G * HT;

    const long long q0 = (long long)blockIdx.x * p.per_cta;
    long long q1 = q0 + p.per_cta;
    if (q1 > p.total) q1 = p.total;

    const float2* __restrict__ x = p.x;
    const float2* __restrict__ s = p.s[prob];
    const int dmin = p.dmin[prob];
    const unsigned n = (unsigned)p.n;

    auto stage = [&](const SubChunk& sc, float2* buf) {
        float2* xs = buf;
        float2* ss = buf + Lmax;
        const int Leff = p.G * sc.steps * TI;
        for (int q = tid; q < Leff; q += nthr) {
            const long long i = sc.i0 + q;
            const bool ok = q < sc.len && i >= 0 && i < (long long)n;
            cp_async8(xs + q, x + (ok ? i : 0), ok);
        }
        long long sb = (sc.i0 + dmin) % (long long)n;
        if (sb < 0) sb += n;
        const unsigned start = (unsigned)sb;
        const long long lin0 = sc.i0 + dmin;
        for (int q = tid; q < Leff + HT; q += nthr) {
            unsigned idx = start + (unsigned)q;
            if (idx >= n) { idx -= n; if (idx >= n) idx %= n; }
            const bool ok = !p.s_linear || (lin0 + q >= 0 && lin0 + q < (long long)n);
            cp_async8(ss + q, s + idx, ok);
        }
        cp_async_commit();
    };

    float2 A1[TD], A2[TD];
#pragma unroll
    for (int v = 0; v < TD; ++v) { A1[v] = make_float2(0.f, 0.f); A2[v] = make_float2(0.f, 0.f); }
    const int h = tid % p.H;
    const int g = tid / p.H;
    const bool active = g < p.G;
    const int own = g * HT + h * TD;       // this thread's slots of red / comp
    if (active) {
#pragma unroll
        for (int v = 0; v < TD; ++v) { red[own + v] = make_float2(0.f, 0.f); comp[own + v] = make_float2(0.f, 0.f); }
    }

    long long q = q0;
    SubChunk cur = next_subchunk<TI>(p, q, q1);
    if (cur.len > 0) stage(cur, smem);
    int b = 0;
    while (cur.len > 0) {
        q += cur.len;
        const SubChunk nxt = next_subchunk<TI>(p, q, q1);
        cp_async_wait_all();
        __syncthreads();      // sub-chunk `cur` is visible; everyone has left the buffer `nxt` will overwrite
        if (nxt.len > 0) stage(nxt, smem + (b ^ 1) * bufsz);
        if (active) {
            const float2* buf = smem + b * bufsz;
            const int Sg = cur.steps * TI;
            slide_mac2n<TI, TD>(A1, A2, buf + g * Sg, buf + Lmax + g * Sg + h * TD, cur.steps);
#pragma unroll
            for (int v = 0; v < TD; ++v) {      // red += sub-chunk sum, compensated (only this thread touches its slots)
                const float2 a = make_float2(A1[v].x + A2[v].y, A2[v].x - A1[v].y);
                const float2 sm = red[own + v], c = comp[own + v];
                const float2 y = make_float2(a.x - c.x, a.y - c.y);
                const float2 t = make_float2(sm.x + y.x, sm.y + y.y);
                comp[own + v] = make_float2((t.x - sm.x) - y.x, (t.y - sm.y) - y.y);
                red[own + v] = t;
                A1[v] = make_float2(0.f, 0.f);
                A2[v] = make_float2(0.f, 0.f);
            }
        }
        if (cur.flush) {
            __syncthreads();
            const long long piece = (long long)blockIdx.x - stream_first_cta(cur.blk, p.blk_len, p.per_cta);
            float2* out = p.partial + (((size_t)prob * p.nblk + cur.blk) * p.maxpieces + piece) * (size_t)HT;
            for (int l = tid; l < HT; l += nthr) {
                float2 sum = make_float2(red[l].x - comp[l].x, red[l].y - comp[l].y);
                for (int gg = 1; gg < p.G; ++gg) {
                    const float2 t = red[gg * HT + l], c = comp[gg * HT + l];
                    sum.x += t.x - c.x;
                    sum.y += t.y - c.y;
                }
                out[l] = sum;
            }
            __syncthreads();  // every thread has read the piece: the owners restart their sums
            if (active) {
#pragma unroll
                for (int v = 0; v < TD; ++v) { red[own + v] = make_float2(0.f, 0.f); comp[own + v] = make_float2(0.f, 0.f); }
            }
        }
        cur = nxt;
        b ^= 1;
    }
}

// xw[i] = x[i] * w[i]  (window folded into the reference channel once per frame)
__global__ void weight_kernel(const float2* __restrict__ x, const float* __restrict__ w, float2* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const float2 v = x[i];
        const float ww = w[i];
        out[i] = make_float2(v.x * ww, v.y * ww);
    }
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
