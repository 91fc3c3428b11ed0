// nlms_block.cuh -- NLMS_filter (reference clutter_removal.py:189-249) evaluated 32 samples at a time, exactly
// (and block_NLMS, whose taps are frozen inside a user block, with the same machinery minus the substitution).
//
// The reference recurrence
//     e_k = d_k - w_k^H u_k,   w_{k+1} = w_k + mu u_k conj(e_k) / (u_k^H u_k),   u_k[j] = ref[M + k - j]
// carries the whole tap vector from sample to sample, which makes a sample-serial kernel pay a block-wide
// reduction over the M taps per sample (~330 cycles).  Inside a block of L samples that starts with
// taps W the same numbers follow from a triangular system in the Gram matrix of the regressors:
//     r_k = d_k - W^H u_k                                     (L dot products, independent of each other)
//     e_k = r_k - mu * sum_{m<k} e_m g(m,k) / p_m,   g(m,k) = u_m^H u_k,  p_m = g(m,m)
//     W  <- W + mu * sum_m u_m conj(e_m) / p_m               (block end)
// g(m, m+delta) is a sliding window sum of conj(ref[q]) ref[q+delta]: one direct sum per lag and block, then a
// 31-step warp scan.  The serial part shrinks to one warp doing one shuffle broadcast + one complex FMA per
// (m, k) step; everything else is data-parallel over taps or lags.  Same arithmetic as the reference up to
// rounding order (numpy prototype against the sequential oracle: 5e-7, the oracle's own round-off level).
#pragma once
#include <cuda_runtime.h>

namespace prc {

struct NlmsParams {
    const float2* ref;
    const float2* srv;
    const float2* init;      // M initial taps or nullptr
    float2* out;             // n
    float2* taps_out;        // M or nullptr
    int n;
    int filter_len;
    int peek;
    float mu;
    int block_len;
    // a batch of independent frames, one CTA each (gridDim.x): frame f reads ref/srv + f * frame_stride, writes
    // out + f * frame_stride; init / taps_out advance by filter_len + peek taps per frame (init_shared: every frame
    // starts from the same init taps)
    long long frame_stride;
    int init_shared;
};

__device__ __forceinline__ NlmsParams nlms_frame_params(const NlmsParams& g) {
    NlmsParams p = g;
    const size_t f = blockIdx.x;
    const int M = g.filter_len + g.peek;
    p.ref += f * g.frame_stride;
    p.srv += f * g.frame_stride;
    p.out += f * g.frame_stride;
    if (p.init && !g.init_shared) p.init += f * M;
    if (p.taps_out) p.taps_out += f * M;
    return p;
}

constexpr int NLMS_TILE = 1024;      // samples staged per shared-memory tile
constexpr int NLMS_MAXT = 4;         // max taps per thread (M <= 4096)
constexpr int NB_L = 32;             // samples per exact block (one warp lane each)
constexpr int NB_THREADS = 1024;
constexpr int NB_PAD = 64;           // extra reference samples staged behind a tile (lag reach of the Gram)

// dynamic shared memory (float2 units):
//   tile  [NLMS_TILE + M + NB_PAD]   ref window,  tile[q] = ref[ts + 1 + q]
//   dtile [NLMS_TILE]                desired samples
//   Ws    [Mpad]                     taps (owners keep them in registers too)
//   P1    [32][NB_L]                 per-warp partial dot products
//   Gs    [NB_L][NB_L + 1]           g(m, m + delta)
//   es    [NB_L]                     mu conj(e_l) / p_l ;  invp [NB_L] floats (mu / p_m)
// NT threads (1024: lowest latency of one frame; 512: two CTAs fit on an SM, for batches of independent frames):
// NT / 32 warps share the 32 Gram lags and the tap segments, KT * NT >= M taps are owned by the threads
template <int KT, int NT = NB_THREADS>
__global__ void __launch_bounds__(NT, NT == 512 ? 3 : 1) nlms_block_kernel(const __grid_constant__ NlmsParams pg) {
    constexpr int NB_THREADS = NT;
    constexpr int NWARP = NT / 32;
    extern __shared__ __align__(16) float2 nbs[];
    const NlmsParams p = nlms_frame_params(pg);
    const int M = p.filter_len + p.peek;
    const int Mpad = (M + 1) & ~1;
    const int nsteps = p.n - M;
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    float2* tile = nbs;
    float2* dtile = tile + NLMS_TILE + Mpad + NB_PAD;
    float2* Ws = dtile + NLMS_TILE;
    float2* P1 = Ws + Mpad;
    float2* Gs = P1 + 32 * NB_L;
    float2* es = Gs + NB_L * (NB_L + 1);
    float* invp = reinterpret_cast<float*>(es + NB_L);

    for (int i = tid; i < p.n; i += NB_THREADS)
        if (i < p.filter_len || i >= p.filter_len + (nsteps > 0 ? nsteps : 0)) p.out[i] = make_float2(0.f, 0.f);

    float2 w[KT];
#pragma unroll
    for (int r = 0; r < KT; ++r) {
        const int j = tid + r * NB_THREADS;
        w[r] = (p.init && j < M) ? p.init[j] : make_float2(0.f, 0.f);
        if (j < Mpad) Ws[j] = (j < M) ? w[r] : make_float2(0.f, 0.f);
    }
    // block_NLMS (block_len > 1, DESIGN.md section 5): taps frozen inside a user block -- no substitution, the
    // increments are collected in `grad` and applied when the user block ends; sub-blocks never straddle one
    const bool frozen = p.block_len > 1;
    float2 grad[KT];
#pragma unroll
    for (int r = 0; r < KT; ++r) grad[r] = make_float2(0.f, 0.f);
    int in_block = 0;
    const int S = (M + NWARP - 1) / NWARP;            // taps per warp in the dot-product phase
    const long long nref = p.n;

    for (int ts = 0; ts < nsteps; ts += NLMS_TILE) {
        const int tl = min(NLMS_TILE, nsteps - ts);
        __syncthreads();
        for (int q = tid; q < tl + M - 1 + NB_PAD; q += NB_THREADS) {
            const long long i = (long long)ts + 1 + q;
            tile[q] = i < nref ? p.ref[i] : make_float2(0.f, 0.f);
        }
        for (int q = tid; q < tl; q += NB_THREADS) dtile[q] = p.srv[p.filter_len + ts + q];
        __syncthreads();
        int Lb = 0;
        for (int kk0 = 0; kk0 < tl; kk0 += Lb) {
            Lb = min(NB_L, tl - kk0);
            if (frozen) Lb = min(Lb, p.block_len - in_block);
            // ---- phase A1: partial dot products  sum_{j in warp's segment} conj(W[j]) * u_{kk0+lane}[j]
            {
                float ar = 0.f, ai = 0.f;
                const int j0 = warp * S, j1 = min(M, j0 + S);
                const float2* up = tile + (M - 1 + kk0 + lane);          // u_k[j] = up[-j]
                for (int j = j0; j < j1; ++j) {
                    const float2 wj = Ws[j];
                    const float2 u = up[-j];
                    ar = fmaf(wj.x, u.x, ar); ar = fmaf(wj.y, u.y, ar);
                    ai = fmaf(wj.x, u.y, ai); ai = fmaf(-wj.y, u.x, ai);
                }
                P1[warp * NB_L + lane] = make_float2(ar, ai);
            }
            // ---- phase A2: Gram lags delta = warp, warp + NWARP, ...: g(m, m + delta), m = lane
            for (int delta = warp; delta < 32; delta += NWARP) {
                const float2* t0 = tile + kk0;
                if (M < NB_L) {
                    // windows shorter than the block: the sliding increments below would telescope a window of a
                    // few samples out of differences of other samples' products, and a small p_m (one or two
                    // samples near zero) would be mostly their rounding.  Sum every window directly (< 32 MACs).
                    float gr = 0.f, gi = 0.f;
                    for (int q = 0; q < M; ++q) {
                        const float2 a = t0[lane + q], b = t0[lane + q + delta];
                        gr = fmaf(a.x, b.x, gr); gr = fmaf(a.y, b.y, gr);
                        gi = fmaf(a.x, b.y, gi); gi = fmaf(-a.y, b.x, gi);
                    }
                    Gs[lane * (NB_L + 1) + delta] = make_float2(gr, gi);
                    if (delta == 0) invp[lane] = p.mu / gr;
                    continue;
                }
                float cr = 0.f, ci = 0.f;
                for (int q = lane; q < M; q += 32) {                      // direct sum for m = 0
                    const float2 a = t0[q], b = t0[q + delta];
                    cr = fmaf(a.x, b.x, cr); cr = fmaf(a.y, b.y, cr);     // conj(a) * b
                    ci = fmaf(a.x, b.y, ci); ci = fmaf(-a.y, b.x, ci);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    cr += __shfl_xor_sync(0xffffffffu, cr, o);
                    ci += __shfl_xor_sync(0xffffffffu, ci, o);
                }
                // sliding increments: window [kk0 + m, kk0 + m + M) = previous window + new sample - dropped sample
                float ir = 0.f, ii = 0.f;
                if (lane > 0) {
                    const float2 a1 = t0[M - 1 + lane], b1 = t0[M - 1 + lane + delta];
                    const float2 a0 = t0[lane - 1], b0 = t0[lane - 1 + delta];
                    ir = (a1.x * b1.x + a1.y * b1.y) - (a0.x * b0.x + a0.y * b0.y);
                    ii = (a1.x * b1.y - a1.y * b1.x) - (a0.x * b0.y - a0.y * b0.x);
                }
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {                        // inclusive scan over lanes
                    const float tr = __shfl_up_sync(0xffffffffu, ir, o);
                    const float ti = __shfl_up_sync(0xffffffffu, ii, o);
                    if (lane >= o) { ir += tr; ii += ti; }
                }
                const float gr = cr + ir, gi = ci + ii;
                Gs[lane * (NB_L + 1) + delta] = make_float2(gr, gi);
                if (delta == 0) invp[lane] = p.mu / gr;
            }
            __syncthreads();
            // ---- phase B (warp 0): r_l, forward substitution, outputs, update coefficients
            if (warp == 0) {
                float sr = 0.f, si = 0.f;
#pragma unroll 8
                for (int q = 0; q < NWARP; ++q) {
                    const float2 v = P1[q * NB_L + lane];
                    sr += v.x; si += v.y;
                }
                const float2 d = lane < Lb ? dtile[kk0 + lane] : make_float2(0.f, 0.f);
                float rr = d.x - sr, ri = d.y - si;
                for (int m = 0; m < (frozen ? 0 : Lb - 1); ++m) {
                    // coefficient of e_m in sample `lane`: mu g(m, lane) / p_m  (independent of the chain: loads first)
                    const float ip = invp[m];
                    const float2 g = Gs[m * (NB_L + 1) + ((lane - m) & 31)];
                    const float er = __shfl_sync(0xffffffffu, rr, m);
                    const float ei = __shfl_sync(0xffffffffu, ri, m);
                    if (lane > m) {
                        const float gr = g.x * ip, gi = g.y * ip;
                        rr = fmaf(-er, gr, rr); rr = fmaf(ei, gi, rr);       // rr -= e * g
                        ri = fmaf(-er, gi, ri); ri = fmaf(-ei, gr, ri);
                    }
                }
                if (lane < Lb) {
                    p.out[p.filter_len + ts + kk0 + lane] = make_float2(rr, ri);
                    const float ip = invp[lane];
                    es[lane] = make_float2(rr * ip, -ri * ip);                // mu conj(e) / p
                } else {
                    es[lane] = make_float2(0.f, 0.f);
                }
            }
            __syncthreads();
            // ---- phase C: W += sum_l u_l[j] * es[l]  (tap owners), mirror to shared memory
#pragma unroll
            for (int r = 0; r < KT; ++r) {
                const int j = tid + r * NB_THREADS;
                if (j < M) {
                    const float2* up = tile + (M - 1 - j + kk0);             // u_{kk0+l}[j] = up[l]
                    // the block's 32 increments are summed on their own and added to the tap ONCE: adding them one by
                    // one rounds at the magnitude of the tap 32 times per block, and over 65 K blocks that random walk
                    // is what limits the accuracy (measured 1.0e-5 from the float64 recurrence against 2e-6 this way)
                    float sr = 0.f, si = 0.f, tr = 0.f, ti = 0.f;
#pragma unroll 8
                    for (int l = 0; l < NB_L; l += 2) {
                        const float2 u0 = up[l], u1 = up[l + 1];
                        const float2 c0 = es[l], c1 = es[l + 1];
                        sr = fmaf(u0.x, c0.x, sr); sr = fmaf(-u0.y, c0.y, sr);
                        si = fmaf(u0.x, c0.y, si); si = fmaf(u0.y, c0.x, si);
                        tr = fmaf(u1.x, c1.x, tr); tr = fmaf(-u1.y, c1.y, tr);
                        ti = fmaf(u1.x, c1.y, ti); ti = fmaf(u1.y, c1.x, ti);
                    }
                    if (!frozen) {
                        w[r] = make_float2(w[r].x + (sr + tr), w[r].y + (si + ti));
                        Ws[j] = w[r];
                    } else {
                        grad[r].x += sr + tr;
                        grad[r].y += si + ti;
                    }
                }
            }
            if (frozen) {
                in_block += Lb;
                if (in_block == p.block_len || ts + kk0 + Lb == nsteps) {     // user block complete: apply its gradient
#pragma unroll
                    for (int r = 0; r < KT; ++r) {
                        const int j = tid + r * NB_THREADS;
                        if (j < M) {
                            w[r].x += grad[r].x; w[r].y += grad[r].y;
                            Ws[j] = w[r];
                        }
                        grad[r] = make_float2(0.f, 0.f);
                    }
                    in_block = 0;
                }
            }
            __syncthreads();
        }
    }
    if (p.taps_out) {
#pragma unroll
        for (int r = 0; r < KT; ++r) {
            const int j = tid + r * NB_THREADS;
            if (j < M) p.taps_out[j] = w[r];
        }
    }
}

inline size_t nlms_block_smem(int M) {
    const int Mpad = (M + 1) & ~1;
    return (size_t)(NLMS_TILE + Mpad + NB_PAD + NLMS_TILE + Mpad + 32 * NB_L + NB_L * (NB_L + 1) + NB_L) * sizeof(float2) +
           NB_L * sizeof(float);
}

}  // namespace prc
