// framepass.cuh -- the FFT-domain frame (LS_Filter -> fast_xambg) in one pass over each frame's channels.
//
// The fused CAF of fftcorr.cuh forms X conj(S - R_seg W') per segment.  By linearity
//
//     sum_seg X conj(S - R_seg W') = AccP - AccQ conj(W'),   AccP = sum_seg X conj(S),   AccQ = sum_seg X conj(R_seg)
//
// and W' (the taps spectrum) is one vector per frame, so AccP and AccQ can be accumulated BEFORE the Toeplitz solve, in
// the same pass that forms the LS lag sums, from the same reference and surveillance window transforms:
//
//   frame_pass_kernel   per segment of a Doppler block (segment start i0, ln <= Bmax samples) four transforms:
//                         Ys' = L surveillance samples from i0 - peek,   Yr' = L reference samples from i0 - (M-1),
//                         X_ls = the unwindowed reference segment,        X_caf = the windowed reference segment
//                       accC += X_ls conj(Yr') (lags M-1 .. 2M-2 of it are c[0 .. M-1]),  accX += X_ls conj(Ys') (x[m]),
//                       AccQ += X_caf conj(Yr'),  AccP += X_caf conj(Ys')  (written per Doppler block, permuted order).
//                       Samples outside every block (the tail after the last one) are LS-only segments: Ys', Yr', X_ls.
//                       The sample two neighbouring blocks share is in both blocks' X_caf and in the first one's X_ls
//                       only, so every sample of the channel is in exactly one X_ls.
//   caf_combine_kernel  per block AccP - AccQ conj(W') and one transform back: lag d + peek is P[j][d] (Ys' starts
//                       peek before the segment), the rows doppler_fft consumes.
//
// Segment limit (scripts/fft/model.py pins it against direct sums): lags M-1 .. 2M-2 of X_ls conj(Yr') stay inside the
// window, ln <= L - 2M + 2; the wrap of the circular convolution Yr' W' lands beyond position L - M, and CAF lags reach
// ln - 1 + R + peek, so ln <= L - M - R - peek + 1.  W' keeps taps_spectrum_kernel's placement: Yr' starts M - 1 - peek
// samples before Ys', exactly as R_seg starts before S in caf_fft_kernel.
//
// Registers: accC, accX (summed over the CTA's whole run) and the two held spectra Ys', Yr' stay in registers; AccP and
// AccQ (summed over one Doppler block) live in thread-private shared memory (2 x 16 KB at R3 = 8): a block's first
// segment stores its products there, the middle ones add to them, and the last one adds its products to what it reads
// and writes the sums to `acc` without storing them back, so a block of one segment never touches those slots.  (The
// other way round every X_ls item paid a read-modify-write of accC and accX; this way a block of nseg segments pays
// nseg - 1 reads and nseg - 1 writes.)  The shared-memory pipe bounds this kernel, so what it spares is what counts:
// the pass-1 / pass-3 twiddles come from five per-thread registers (fft::Tw1Seeds) instead of the tw1 table, and pass 2
// reads its twiddles two per load from padded rows (fft::Tw2Rows).  A CTA has 93 312 B of shared memory, and two fit in
// an SM.
#pragma once
#include <cuda_runtime.h>

#include "fftcore.cuh"
#include "fftcorr.cuh"

namespace prc {
namespace fftc {

struct FramePassParams {
    const float2* ref;
    const float2* srv;
    long long frame_stride;
    const float* win;          // n floats shared by all frames, or NULL
    int n, M, peek, F;
    long long D;               // Doppler block j = samples [j D + c0 - (ntaps - 1), j D + c0] inside [0, n)
    int c0, ntaps;
    int Bmax;                  // segment limit of block segments: min(L - 2M + 2, L - M - R - peek + 1)
    int tail_lo;               // LS-only samples [tail_lo, n): ntail segments of Bt samples (the last one shorter)
    int ntail, Bt;
    float2* acc;               // [frame][F][2][L]: AccP, AccQ in permuted order
    float2* partial;           // [frame][2][gridDim.x][HT]: LS lag sums c, x (levinson_kernel's layout)
    int HT;
    const float2* tw;
};

// shared memory: [fft::SmemSeeded with tw2 rows | staging L float2 | AccP, AccQ 2 L float2 | window staging L float]
template <int R3> using FpSmem = fft::SmemSeeded<R3, fft::Tw2Rows<R3>>;
template <int R3> constexpr int framepass_smem_float2() {
    return FpSmem<R3>::SMEM_FLOAT2 + 3 * fft::Geo<R3>::L + fft::Geo<R3>::L / 2;
}

// a unit of a CTA's run: Doppler block u < F, else LS-only tail segment u - F
struct FpUnit {
    int lo, hi, ls_end;        // samples [lo, hi); X_ls takes [lo, ls_end)
    int nseg, Bs, nk;          // nk: items per segment (4 block, 3 tail)
};

__device__ __forceinline__ FpUnit fp_unit(const FramePassParams& p, int u) {
    FpUnit g;
    if (u < p.F) {
        const long long base = (long long)u * p.D + p.c0;
        g.lo = (int)max(base - (p.ntaps - 1), 0ll);
        g.hi = (int)min(base + 1, (long long)p.n);
        g.ls_end = u + 1 < p.F ? (int)min((long long)g.hi, max(base + p.D - (p.ntaps - 1), 0ll)) : g.hi;
        const int len = g.hi > g.lo ? g.hi - g.lo : 0;
        g.nseg = (len + p.Bmax - 1) / p.Bmax;
        g.Bs = g.nseg ? (len + g.nseg - 1) / g.nseg : 0;
        g.nk = 4;
    } else {
        g.lo = p.tail_lo + (u - p.F) * p.Bt;
        g.hi = min(g.lo + p.Bt, p.n);
        g.ls_end = g.hi;
        g.nseg = 1;
        g.Bs = p.Bt;
        g.nk = 3;
    }
    return g;
}

template <int R3> constexpr int framepass_min_ctas() { return R3 == 8 ? 2 : 1; }

// CTA c of a frame walks units [c U / gridDim.x, (c + 1) U / gridDim.x), U = F + ntail.  Items of a segment: 0 = Ys'
// (staged), 1 = Yr' (staged), 2 = X_ls and 3 = X_caf (both read Yr''s slots, M - 1 further on, written by other
// threads: the barriers of Yr''s transform order those copies before the reads).  Only the window is staged for X_caf
// (in X_ls's hook); the next segment's Ys' copies are issued after the first barrier of the segment's last transform,
// when every thread has read the slots.
template <int R3>
__global__ void __launch_bounds__(16 * R3, framepass_min_ctas<R3>()) frame_pass_kernel(const __grid_constant__ FramePassParams p) {
    using G = fft::Geo<R3>;
    extern __shared__ __align__(16) float2 sm[];
    const int t = threadIdx.x;
    const FpSmem<R3> S(sm, p.tw, t);
    float2* stg = sm + FpSmem<R3>::SMEM_FLOAT2;
    float2* accs = stg + G::L;                                   // AccP [r T + t], AccQ [L + r T + t]
    float* wst = reinterpret_cast<float*>(accs + 2 * G::L);
    const float2* ref = p.ref + (size_t)blockIdx.y * p.frame_stride;
    const float2* srv = p.srv + (size_t)blockIdx.y * p.frame_stride;
    const int U = p.F + p.ntail;
    const int u0 = (int)((long long)blockIdx.x * U / gridDim.x), u1 = (int)((long long)(blockIdx.x + 1) * U / gridDim.x);
    const int off = p.M - 1;                                     // X's samples in Yr''s window

    // (unit, segment, kind) of the item being transformed and of the next one
    int cu = u0, cq = 0, ck = 0;
    FpUnit cg = fp_unit(p, cu);
    while (cu < u1 && cg.nseg == 0) { ++cu; if (cu < u1) cg = fp_unit(p, cu); }
    auto issue = [&](int u, const FpUnit& g, int q, int kind) {
        const int i0 = g.lo + q * g.Bs;
        if (kind == 0) stage_sig<G::T, true>(stg, t, srv, i0 - p.peek, G::L, p.n, 0);
        else if (kind == 1) stage_sig<G::T, true>(stg, t, ref, i0 - off, G::L, p.n, 0);
        else if (kind == 3 && p.win) {
            const int ln = min(g.Bs, g.hi - i0);
            const float* w0 = p.win + i0 + t;
#pragma unroll
            for (int n1 = 0; n1 < 16; ++n1)
                if (n1 * G::T < ln) cp_async4(wst + t + n1 * G::T, w0 + n1 * G::T, n1 * G::T + t < ln);
        }
        cp_async_commit();
    };
    if (cu < u1) issue(cu, cg, 0, 0);
    fft::stage_tw2<R3, fft::Tw2Rows<R3>>(sm, p.tw, t);
    __syncthreads();

    float2 accC[16], accX[16], ys[16], yr[16], v[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) accC[r] = accX[r] = ys[r] = yr[r] = make_float2(0.f, 0.f);
#pragma unroll 1
    while (cu < u1) {
        const int i0 = cg.lo + cq * cg.Bs;
        // the item after this one
        int nu = cu, nq = cq, nk = ck + 1;
        FpUnit ng = cg;
        if (nk == cg.nk) {
            nk = 0;
            if (++nq == cg.nseg) {
                nq = 0;
                do { ++nu; if (nu < u1) ng = fp_unit(p, nu); } while (nu < u1 && ng.nseg == 0);
            }
        }
        if (ck >= 2) {
            const int ln = min(cg.Bs, cg.hi - i0);
            const int lx = ck == 2 ? max(0, min(ln, cg.ls_end - i0)) : ln;
            if (ck == 3) cp_async_wait_all();                            // the window
#pragma unroll
            for (int n1 = 0; n1 < 16; ++n1) {
                const int i = n1 * G::T + t;
                v[n1] = i < lx ? stg[i + off] : make_float2(0.f, 0.f);
            }
            if (ck == 3 && p.win) {
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
        fft::fft_n2p<R3>(v, t, S, [&] { if (nu < u1 && !(nk == 2)) issue(nu, ng, nq, nk); });
        // Ys', Yr', accC and accX are updated in place, not by assignments on separate branches: with branches ptxas
        // kept each array in two register sets and copied it back and forth on every item (~100 MOV per item; without
        // them the frame pass at C2 takes 8 % less time)
        if (ck < 2) {
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                ys[r] = ck == 0 ? v[r] : ys[r];
                yr[r] = ck == 1 ? v[r] : yr[r];
            }
        } else if (ck == 2) {
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                cmacc(accC[r], v[r], yr[r]);                             // accC += X_ls conj(Yr')
                cmacc(accX[r], v[r], ys[r]);                             // accX += X_ls conj(Ys')
            }
        } else {
            // AccP += X_caf conj(Ys'), AccQ += X_caf conj(Yr'), from zero on the block's first segment; its last
            // segment writes the sums out
            const bool first = cq == 0, last = cq + 1 == cg.nseg;
            float2* dst = p.acc + ((size_t)blockIdx.y * p.F + cu) * 2 * G::L;
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                float2 a = make_float2(0.f, 0.f), b = make_float2(0.f, 0.f);
                if (!first) {
                    a = accs[r * G::T + t];
                    b = accs[G::L + r * G::T + t];
                }
                cmacc(b, v[r], yr[r]);
                cmacc(a, v[r], ys[r]);
                if (last) {
                    dst[r * G::T + t] = a;
                    dst[G::L + r * G::T + t] = b;
                } else {
                    accs[r * G::T + t] = a;
                    accs[G::L + r * G::T + t] = b;
                }
            }
        }
        if (nu != cu) cg = ng;
        cu = nu; cq = nq; ck = nk;
    }
    // LS lag sums: c[m] is lag m + M - 1 of accC (Yr' starts M - 1 before the segment), x[m] lag m of accX
    const float inv = 1.0f / (float)G::L;
#pragma unroll 1
    for (int w = 0; w < 2; ++w) {
#pragma unroll
        for (int r = 0; r < 16; ++r) v[r] = w ? accX[r] : accC[r];
        fft::fft_p2n<R3>(v, t, S);
        float2* row = p.partial + ((size_t)(blockIdx.y * 2 + w) * gridDim.x + blockIdx.x) * p.HT;
        const int sh = w ? 0 : off;
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int m = n1 * G::T + t - sh;
            if (m >= 0 && m < p.M) row[m] = make_float2(v[n1].x * inv, v[n1].y * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------ combine
struct CafCombineParams {
    const float2* acc;         // [frame][F][2][L] from frame_pass_kernel
    const float2* wp;          // [frame][L] taps spectrum, permuted order
    int F, R, peek;
    float2* P;                 // [frame][F][HT]; P[j][d], d = 0..R
    int HT;
    const float2* tw;
};

// CTA c walks blocks c, c + gridDim.x, ... of frame blockIdx.y
template <int R3>
__global__ void __launch_bounds__(16 * R3) caf_combine_kernel(const __grid_constant__ CafCombineParams p) {
    using G = fft::Geo<R3>;
    extern __shared__ __align__(16) float2 sm[];
    const int t = threadIdx.x;
    const fft::Smem<R3> S(sm);
    fft::stage_twiddles<R3>(sm, p.tw, t);
    __syncthreads();
    const float2* wp = p.wp + (size_t)blockIdx.y * G::L;
    float2 w[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) w[r] = __ldg(wp + r * G::T + t);
    const float inv = 1.0f / (float)G::L;
#pragma unroll 1
    for (int j = blockIdx.x; j < p.F; j += gridDim.x) {
        const float2* src = p.acc + ((size_t)blockIdx.y * p.F + j) * 2 * G::L;
        float2 v[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const float2 a = __ldg(src + r * G::T + t), q = cmulc(__ldg(src + G::L + r * G::T + t), w[r]);
            v[r] = make_float2(a.x - q.x, a.y - q.y);                   // AccP - AccQ conj(W')
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
// The one-pass frame runs at L = 2048 (R3 = 8) only: at R3 = 16 its shared memory (over 200 KB) does not fit.
constexpr int FP_R3 = 8;

inline cudaError_t framepass_set_attrs(int smem_limit) {
    cudaError_t e = cudaFuncSetAttribute(frame_pass_kernel<FP_R3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(caf_combine_kernel<FP_R3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_limit);
}

// CTAs per SM of each kernel at its launch configuration (0 if the runtime cannot answer)
inline int frame_pass_ctas_per_sm() {
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, frame_pass_kernel<FP_R3>, 16 * FP_R3,
                                                      framepass_smem_float2<FP_R3>() * sizeof(float2)) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return v;
}

inline int caf_combine_ctas_per_sm() {
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, caf_combine_kernel<FP_R3>, 16 * FP_R3,
                                                      fft::Geo<FP_R3>::SMEM_FLOAT2 * sizeof(float2)) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return v;
}

inline void launch_frame_pass(const FramePassParams& p, int ncta, int nf, cudaStream_t st) {
    frame_pass_kernel<FP_R3><<<dim3(ncta, nf), 16 * FP_R3, framepass_smem_float2<FP_R3>() * sizeof(float2), st>>>(p);
}

inline void launch_caf_combine(const CafCombineParams& p, int ncta, int nf, cudaStream_t st) {
    caf_combine_kernel<FP_R3><<<dim3(ncta, nf), 16 * FP_R3, fft::Geo<FP_R3>::SMEM_FLOAT2 * sizeof(float2), st>>>(p);
}

}  // namespace fftc
}  // namespace prc
