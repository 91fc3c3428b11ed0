// framemulti.cuh -- the one-pass frame (framepass.cuh) for K surveillance channels that share one reference channel.
//
// Of frame_pass_kernel's four transforms per block segment, three (Yr', X_ls, X_caf) and two of the four products
// (accC, AccQ) depend on the reference alone, and so does the Gram column c[m]: the Toeplitz matrix is the same for
// every channel.  One CTA therefore transforms the reference items once and then each channel's Ys':
//
//   frame_multi_pass_kernel<R3, K>   per block segment: Yr' (staged), X_ls and X_caf (both read Yr''s slots, as in
//                                    frame_pass_kernel), then Ys'_k of every channel k = 0 .. K-1 (staged);
//                                    accC += X_ls conj(Yr'), AccQ += X_caf conj(Yr') once per segment,
//                                    accX_k += X_ls conj(Ys'_k), AccP_k += X_caf conj(Ys'_k) once per channel.
//                                    LS-only tail segments: Yr', X_ls and the K Ys'.
//   caf_combine_multi_kernel<R3>     per block and channel AccP_k - AccQ conj(W'_k) and one transform back: the P rows
//                                    doppler_stage consumes.
//
// CTA c of a frame walks the same units as frame_pass_kernel's CTA c (the host launches both with the same grid for
// the same frames per launch), and each product is the same cmacc on the same operands in the same order, so every
// channel's lag sums, block spectra, taps and map are bit for bit those of frame_pass_kernel on (ref, srv_k).
//
// Registers hold accC, accX_0, the held spectra X_ls and h (Yr' until X_caf's AccQ product, X_caf after it) and the
// item being transformed: five 16-float2 arrays, as frame_pass_kernel.  Thread-private shared memory holds AccQ,
// AccP_0 .. AccP_{K-1} (per Doppler block, with frame_pass_kernel's first / middle / last discipline) and
// accX_1 .. accX_{K-1} (per CTA run): 2 K L float2 on top of frame_pass_kernel's layout without its AccP / AccQ slots,
// 60 544 + 32 768 K bytes at R3 = 8 (126 080 / 158 848 / 191 616 B for K = 2 / 3 / 4), one CTA per SM.
#pragma once
#include <cuda_runtime.h>

#include "fftcore.cuh"
#include "fftcorr.cuh"
#include "framepass.cuh"

namespace prc {
namespace fftc {

struct FrameMultiParams {
    FramePassParams fp;        // fp.srv: channel 0; fp.acc: [frame][F][1 + K][L] (AccQ, AccP_0 .. AccP_{K-1}, permuted
                               // order); fp.partial: [K][frame][2][gridDim.x][HT] (levinson_kernel's layout, one
                               // problem per (channel, frame); the c rows are the same for every channel)
    long long chan_stride;     // channel k of frame f at fp.srv + k chan_stride + f frame_stride
};

// shared memory: [FpSmem | staging L float2 | AccQ, AccP_0 .. AccP_{K-1}, accX_1 .. accX_{K-1}: 2 K L float2 |
// window staging L float]
template <int R3, int K> constexpr int framemulti_smem_float2() {
    return FpSmem<R3>::SMEM_FLOAT2 + (1 + 2 * K) * fft::Geo<R3>::L + fft::Geo<R3>::L / 2;
}

// Items of a block segment: 0 = Yr' (staged), 1 = X_ls, 2 = X_caf (1 and 2 read Yr''s slots, M - 1 further on,
// written by other threads: the barriers of Yr''s transform order those copies before the reads), 3 + k = Ys'_k
// (staged).  A tail segment has no X_caf: its items 2 .. K + 1 are kinds 3 .. K + 2.  The window is staged in X_ls's
// hook; Ys'_0's copies are issued in the hook of the segment's last reference item, when every thread has read the
// slots, and each other staged item's in the hook of the item before it.
template <int R3, int K>
__global__ void __launch_bounds__(16 * R3, 1) frame_multi_pass_kernel(const __grid_constant__ FrameMultiParams q) {
    using G = fft::Geo<R3>;
    const FramePassParams& p = q.fp;
    extern __shared__ __align__(16) float2 sm[];
    const int t = threadIdx.x;
    const FpSmem<R3> S(sm, p.tw, t);
    float2* stg = sm + FpSmem<R3>::SMEM_FLOAT2;
    float2* accs = stg + G::L;          // AccQ [r T + t], AccP_k [(1 + k) L + r T + t], accX_k [(K + k) L + r T + t]
    float* wst = reinterpret_cast<float*>(accs + 2 * K * G::L);
    const float2* ref = p.ref + (size_t)blockIdx.y * p.frame_stride;
    const float2* srv = p.srv + (size_t)blockIdx.y * p.frame_stride;
    const int U = p.F + p.ntail;
    const int u0 = (int)((long long)blockIdx.x * U / gridDim.x), u1 = (int)((long long)(blockIdx.x + 1) * U / gridDim.x);
    const int off = p.M - 1;
    auto items = [](const FpUnit& g) { return g.nk == 4 ? 3 + K : 2 + K; };
    auto kind_of = [](const FpUnit& g, int i) { return g.nk == 4 || i < 2 ? i : i + 1; };

    int cu = u0, cq = 0, ck = 0;
    FpUnit cg = fp_unit(p, cu);
    while (cu < u1 && cg.nseg == 0) { ++cu; if (cu < u1) cg = fp_unit(p, cu); }
    auto issue = [&](const FpUnit& g, int qs, int kind) {
        const int i0 = g.lo + qs * g.Bs;
        if (kind == 0) stage_sig<G::T, true>(stg, t, ref, i0 - off, G::L, p.n, 0);
        else if (kind >= 3) stage_sig<G::T, true>(stg, t, srv + (long long)(kind - 3) * q.chan_stride, i0 - p.peek, G::L, p.n, 0);
        else if (kind == 2 && p.win) {
            const int ln = min(g.Bs, g.hi - i0);
            const float* w0 = p.win + i0 + t;
#pragma unroll
            for (int n1 = 0; n1 < 16; ++n1)
                if (n1 * G::T < ln) cp_async4(wst + t + n1 * G::T, w0 + n1 * G::T, n1 * G::T + t < ln);
        }
        cp_async_commit();
    };
    if (cu < u1) issue(cg, 0, 0);
    fft::stage_tw2<R3, fft::Tw2Rows<R3>>(sm, p.tw, t);
#pragma unroll
    for (int k = 1; k < K; ++k)
#pragma unroll
        for (int r = 0; r < 16; ++r) accs[(K + k) * G::L + r * G::T + t] = make_float2(0.f, 0.f);
    __syncthreads();

    float2 accC[16], accX[16], x[16], h[16], v[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) accC[r] = accX[r] = x[r] = h[r] = make_float2(0.f, 0.f);
#pragma unroll 1
    while (cu < u1) {
        const int i0 = cg.lo + cq * cg.Bs;
        const int kind = kind_of(cg, ck);
        int nu = cu, nq = cq, nk = ck + 1;
        FpUnit ng = cg;
        if (nk == items(cg)) {
            nk = 0;
            if (++nq == cg.nseg) {
                nq = 0;
                do { ++nu; if (nu < u1) ng = fp_unit(p, nu); } while (nu < u1 && ng.nseg == 0);
            }
        }
        const int nkind = kind_of(ng, nk);
        if (kind == 1 || kind == 2) {
            const int ln = min(cg.Bs, cg.hi - i0);
            const int lx = kind == 1 ? max(0, min(ln, cg.ls_end - i0)) : ln;
            if (kind == 2) cp_async_wait_all();                          // the window
#pragma unroll
            for (int n1 = 0; n1 < 16; ++n1) {
                const int i = n1 * G::T + t;
                v[n1] = i < lx ? stg[i + off] : make_float2(0.f, 0.f);
            }
            if (kind == 2 && p.win) {
#pragma unroll
                for (int n1 = 0; n1 < 16; ++n1) {
                    if (n1 * G::T < lx) {
                        const float w = wst[t + n1 * G::T];
                        v[n1].x *= w;
                        v[n1].y *= w;
                    }
                }
            }
        } else {
            fetch_staged<G::T, true>(v, stg, t, G::L);
        }
        fft::fft_n2p<R3>(v, t, S, [&] { if (nu < u1 && nkind != 1) issue(ng, nq, nkind); });
        const bool first = cq == 0, last = cq + 1 == cg.nseg;
        float2* dst = p.acc + ((size_t)blockIdx.y * p.F + cu) * (1 + K) * G::L;
        if (kind == 1) {
#pragma unroll
            for (int r = 0; r < 16; ++r) cmacc(accC[r], v[r], h[r]);        // accC += X_ls conj(Yr')
        } else if (kind == 2) {
            // AccQ += X_caf conj(Yr'), from zero on the block's first segment; its last segment writes the sum out
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                float2 b = make_float2(0.f, 0.f);
                if (!first) b = accs[r * G::T + t];
                cmacc(b, v[r], h[r]);
                if (last) dst[r * G::T + t] = b;
                else accs[r * G::T + t] = b;
            }
        } else if (kind >= 3) {
            const int k = kind - 3;
            if (k == 0) {
#pragma unroll
                for (int r = 0; r < 16; ++r) cmacc(accX[r], x[r], v[r]);    // accX_0 += X_ls conj(Ys'_0)
            } else {
                float2* ax = accs + (K + k) * G::L + t;
#pragma unroll
                for (int r = 0; r < 16; ++r) {
                    float2 a = ax[r * G::T];
                    cmacc(a, x[r], v[r]);                                    // accX_k += X_ls conj(Ys'_k)
                    ax[r * G::T] = a;
                }
            }
            if (cg.nk == 4) {
                float2* ap = accs + (1 + k) * G::L + t;
                float2* dp = dst + (1 + k) * G::L + t;
#pragma unroll
                for (int r = 0; r < 16; ++r) {
                    float2 a = make_float2(0.f, 0.f);
                    if (!first) a = ap[r * G::T];
                    cmacc(a, h[r], v[r]);                                    // AccP_k += X_caf conj(Ys'_k)
                    if (last) dp[r * G::T] = a;
                    else ap[r * G::T] = a;
                }
            }
        }
        // the held spectra are updated in place (see frame_pass_kernel: assignments on separate branches make ptxas
        // keep each array in two register sets)
        if (kind < 3) {
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                h[r] = kind != 1 ? v[r] : h[r];
                x[r] = kind == 1 ? v[r] : x[r];
            }
        }
        if (nu != cu) cg = ng;
        cu = nu; cq = nq; ck = nk;
    }
    // LS lag sums: c[m] is lag m + M - 1 of accC, written for every channel's problem; x_k[m] lag m of accX_k
    const float inv = 1.0f / (float)G::L;
#pragma unroll 1
    for (int w = 0; w <= K; ++w) {
#pragma unroll
        for (int r = 0; r < 16; ++r) v[r] = w == 0 ? accC[r] : (w == 1 ? accX[r] : accs[(K + w - 1) * G::L + r * G::T + t]);
        fft::fft_p2n<R3>(v, t, S);
        const int sh = w ? 0 : off;
#pragma unroll 1
        for (int k = w ? w - 1 : 0; k < (w ? w : K); ++k) {
            float2* row = p.partial + (((size_t)(k * gridDim.y + blockIdx.y) * 2 + (w ? 1 : 0)) * gridDim.x + blockIdx.x) * p.HT;
#pragma unroll
            for (int n1 = 0; n1 < 16; ++n1) {
                const int m = n1 * G::T + t - sh;
                if (m >= 0 && m < p.M) row[m] = make_float2(v[n1].x * inv, v[n1].y * inv);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ combine
struct CafCombineMultiParams {
    const float2* acc;         // [frame][F][1 + nchan][L] from frame_multi_pass_kernel
    const float2* wp;          // [nchan][frame][L] taps spectra, permuted order
    int F, R, peek, nf, nchan;
    float2* P;                 // [nchan][frame][F][HT]; P[j][d], d = 0..R
    int HT;
    const float2* tw;
};

// problem blockIdx.y = k nf + f; CTA c walks blocks c, c + gridDim.x, ... of it (caf_combine_kernel's arithmetic)
template <int R3>
__global__ void __launch_bounds__(16 * R3) caf_combine_multi_kernel(const __grid_constant__ CafCombineMultiParams p) {
    using G = fft::Geo<R3>;
    extern __shared__ __align__(16) float2 sm[];
    const int t = threadIdx.x;
    const fft::Smem<R3> S(sm);
    fft::stage_twiddles<R3>(sm, p.tw, t);
    __syncthreads();
    const int k = blockIdx.y / p.nf, f = blockIdx.y - k * p.nf;
    const float2* wp = p.wp + (size_t)blockIdx.y * G::L;
    float2 w[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) w[r] = __ldg(wp + r * G::T + t);
    const float inv = 1.0f / (float)G::L;
#pragma unroll 1
    for (int j = blockIdx.x; j < p.F; j += gridDim.x) {
        const float2* accq = p.acc + ((size_t)f * p.F + j) * (1 + p.nchan) * G::L;
        const float2* accp = accq + (size_t)(1 + k) * G::L;
        float2 v[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const float2 a = __ldg(accp + r * G::T + t), qv = cmulc(__ldg(accq + r * G::T + t), w[r]);
            v[r] = make_float2(a.x - qv.x, a.y - qv.y);                  // AccP_k - AccQ conj(W'_k)
        }
        fft::fft_p2n<R3>(v, t, S);
        float2* row = p.P + ((size_t)blockIdx.y * p.F + j) * p.HT;
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int d = n1 * G::T + t - p.peek;
            if (d >= 0 && d <= p.R) row[d] = make_float2(v[n1].x * inv, v[n1].y * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------ host launchers
constexpr int FM_MAX_CHANNELS = 4;       // K = 2 .. 4 are instantiated

template <int K> inline size_t framemulti_smem_bytes() { return framemulti_smem_float2<FP_R3, K>() * sizeof(float2); }

inline cudaError_t framemulti_set_attrs(int smem_limit) {
    cudaError_t e = cudaFuncSetAttribute(frame_multi_pass_kernel<FP_R3, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(frame_multi_pass_kernel<FP_R3, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(frame_multi_pass_kernel<FP_R3, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(caf_combine_multi_kernel<FP_R3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit);
    return e;
}

template <int K> inline void launch_frame_multi_k(const FrameMultiParams& p, int ncta, int nf, cudaStream_t st) {
    frame_multi_pass_kernel<FP_R3, K><<<dim3(ncta, nf), 16 * FP_R3, framemulti_smem_bytes<K>(), st>>>(p);
}

// K = 2 .. FM_MAX_CHANNELS channels; the caller has checked K
inline void launch_frame_multi(const FrameMultiParams& p, int K, int ncta, int nf, cudaStream_t st) {
    if (K == 2) launch_frame_multi_k<2>(p, ncta, nf, st);
    else if (K == 3) launch_frame_multi_k<3>(p, ncta, nf, st);
    else launch_frame_multi_k<4>(p, ncta, nf, st);
}

// nprob = nchan x frames problems, gridDim.y
inline void launch_caf_combine_multi(const CafCombineMultiParams& p, int ncta, int nprob, cudaStream_t st) {
    caf_combine_multi_kernel<FP_R3><<<dim3(ncta, nprob), 16 * FP_R3, fft::Geo<FP_R3>::SMEM_FLOAT2 * sizeof(float2), st>>>(p);
}

}  // namespace fftc
}  // namespace prc
