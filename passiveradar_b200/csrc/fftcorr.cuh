// fftcorr.cuh -- the frame's three heavy steps as block correlations / overlap-save filtering in the frequency
// domain (FP32, fftcore.cuh), reading the caller's complex64 channels directly: no intermediate planes in HBM.
//
//   lscorr_fft_kernel   c[m] = sum_i ref[i] conj(ref[i+m]),  x[m] = sum_i ref[i] conj(srv[i+m-peek]),  m < M
//                       (first column of A^H A and A^H srv of LS_Filter, reference clutter_removal.py:34-45, up to the
//                       conjugation levinson_kernel applies).  The channel is cut into segments of Bs <= L - M + 1
//                       samples; per segment X = spectrum of the zero-padded reference segment, Yr / Ys = spectra of
//                       the L reference / surveillance samples that start with it: X conj(Yr) and X conj(Ys) are the
//                       spectra of the segment's lag sums for 0 <= m < M (lags reach at most L - 1, no wrap).
//                       Three transforms per segment, spectra accumulated in registers over the CTA's segments, one
//                       permuted->natural transform per correlation and CTA at the end.
//   taps_spectrum_kernel  W'(f): spectrum of the solved taps placed at (k - (M-1)) mod L, in permuted order.
//   fir_fft_kernel      out = srv - circular FIR(ref, w)  (clutter_removal.py:51) by overlap-save: one forward
//                       transform of L reference samples, times W', one transform back, L - M + 1 outputs.
//   caf_fft_kernel      CAF block sums P[j][d] = sum_{i in Doppler block j} ref[i] win[i] conj(s[(i+d) mod n]),
//                       d = 0..R (range_doppler_processing.py:81-86), s = srv or -- FUSED -- the cleaned channel
//                       formed in the frequency domain as S - R_seg W' (valid because the circular-convolution
//                       wrap lands in the part of the segment no lag 0..R touches).  Segments of <= L - R - (M-1)
//                       samples; spectra X conj(S_clean) accumulated per Doppler block; one transform back.
//
// All kernels take a batch of frames in gridDim.y (frame_stride samples apart).  Every hot loop has ONE transform
// call site (a loop body with two or three inlined transforms is 37-43 KB of SASS and misses the 32 KB instruction
// cache on every iteration) and its input is
// staged one transform ahead with cp.async.  Algebra pinned on the CPU by scripts/fft/model.py (numpy) and
// scripts/fft/emul.cu (thread-by-thread run of fftcore.cuh).
#pragma once
#include <cuda_runtime.h>

#include "fftcore.cuh"

namespace prc {
namespace fftc {

using fft::cmul;
using fft::cmulc;

// ---- asynchronous, thread-private input staging --------------------------------------------------------------
// Thread t copies the 16 samples it will itself transform (elements n1 T + t) into its own shared-memory slots
// with cp.async (8-byte copies, zero fill through src-size 0), one transform ahead; cp.async.wait_group makes its
// own copies visible to it, so the staging needs no block-wide barrier and no branch.  The copies of the next
// transform are issued after the first barrier of the current one (fft_n2p's hook), when the slots have been read.
__device__ __forceinline__ void cp_async8(float2* dst, const float2* src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    const int sz = valid ? 8 : 0;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    const int sz = valid ? 4 : 0;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// stage sig[(base + i)], i = n1 T + t < len (zero beyond; circular mod n, or zero outside [0, n) when linear);
// base may be up to one period outside [0, n) and the L elements cross the end of the channel at most once.
// A copy that is switched off (src-size 0) reads nothing, so its source address is not sanitised.
// FULL: len == L is known at compile time.  The common case -- the L elements lie inside [0, n) -- is one LDGSTS per
// element with immediate offsets (the index arithmetic of the general case costs as many issue slots as the copies).
template <int T, bool FULL>
__device__ __forceinline__ void stage_sig(float2* stg, int t, const float2* __restrict__ sig, long long base, int len,
                                          int n, int linear) {
    if (base >= 0 && base + 16 * T <= n) {
        const float2* p0 = sig + base + t;
        float2* d0 = stg + t;
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1)
            if (FULL || n1 * T < len) cp_async8(d0 + n1 * T, p0 + n1 * T, FULL || n1 * T + t < len);   // rows beyond len: not staged
        return;
    }
    int lo = 0, hi = FULL ? 16 * T : len, wrap = 0x7fffffff;
    if (linear) {                                   // valid i: 0 <= base + i < n
        lo = base < 0 ? (int)(-base) : 0;
        const long long h = (long long)n - base;
        hi = h < (long long)hi ? (h < 0 ? 0 : (int)h) : hi;
    } else {
        if (base < 0) base += n;
        if (base >= n) base -= n;
        wrap = (int)(n - base);                     // first element that has wrapped around
    }
    const float2* p0 = sig + base;
#pragma unroll
    for (int n1 = 0; n1 < 16; ++n1) {
        const int i = n1 * T + t;
        const int off = i - (i >= wrap ? n : 0);
        if (FULL || n1 * T < len) cp_async8(stg + i, p0 + off, i >= lo && i < hi);
    }
}

// len: what the item was staged with (rows n1 T >= len were not staged: zero)
template <int T, bool FULL>
__device__ __forceinline__ void fetch_staged(float2 (&v)[16], const float2* stg, int t, int len) {
    cp_async_wait_all();
    const float2* s0 = stg + t;
#pragma unroll
    for (int n1 = 0; n1 < 16; ++n1) v[n1] = (FULL || n1 * T < len) ? s0[n1 * T] : make_float2(0.f, 0.f);
}

// acc += a conj(b)
__device__ __forceinline__ void cmacc(float2& acc, const float2 a, const float2 b) {
    acc.x = fmaf(a.x, b.x, fmaf(a.y, b.y, acc.x));
    acc.y = fmaf(a.y, b.x, fmaf(-a.x, b.y, acc.y));
}

// ------------------------------------------------------------------------------------------------ LS correlations
struct LsCorrParams {
    const float2* ref;
    const float2* srv;
    long long frame_stride;
    int n, M, peek, linear;
    int nseg, Bs;              // nseg segments of Bs samples (the last one shorter), Bs <= L - M + 1
    float2* partial;           // [frame][2][gridDim.x][HT]
    int HT;
    const float2* tw;
};

// shared memory: [fft::Smem (2 exchange buffers, twiddles) | staging L float2]
template <int R3> constexpr int lscorr_smem_float2() { return fft::Geo<R3>::SMEM_FLOAT2 + fft::Geo<R3>::L; }

// CTAs per SM the register allocation of lscorr_fft_kernel is held to.  R3 = 8: 68.6 KB of shared memory fits three
// times in an SM, and an allocation of 175 registers x 128 threads would let only two in -- at <= 168 registers,
// without spills, three fit.  R3 = 16 is held to one CTA per SM by its shared memory; 0 leaves the
// allocation of the other instantiations to ptxas as before.
template <int R3> constexpr int lscorr_min_ctas() { return R3 == 8 ? 3 : 0; }

// CTA c of a frame takes segments c, c + gridDim.x, ...; items per segment: 0 = zero-padded reference segment (X),
// 1 = L reference samples from the segment start (Yr), 2 = L surveillance samples from start - peek (Ys).
// X is the first len samples of Yr, and a thread stages the same elements for both: the L reference samples are
// staged once, for item 0, which zeroes the elements from len on in its registers, and item 1 reads the same slots
// again (a third fewer copies from L2 and shared-memory stores; the transforms see the same inputs).
template <int R3>
__global__ void __launch_bounds__(16 * R3, lscorr_min_ctas<R3>()) lscorr_fft_kernel(const __grid_constant__ LsCorrParams p) {
    using G = fft::Geo<R3>;
    extern __shared__ __align__(16) float2 sm[];
    const int t = threadIdx.x;
    const fft::Smem<R3> S(sm);
    float2* stg = sm + G::SMEM_FLOAT2;
    const float2* ref = p.ref + (size_t)blockIdx.y * p.frame_stride;
    const float2* srv = p.srv + (size_t)blockIdx.y * p.frame_stride;
    const int nmine = ((int)blockIdx.x < p.nseg) ? (p.nseg - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int nitems = 3 * nmine;

    auto issue = [&](int it) {
        const int q = it / 3, kind = it - 3 * q;
        if (kind == 1) return;                      // Yr: still in the slots item 0 read
        const int sgm = blockIdx.x + q * gridDim.x;
        const long long i0 = (long long)sgm * p.Bs;
        if (kind == 0) stage_sig<G::T, true>(stg, t, ref, i0, G::L, p.n, p.linear);
        else stage_sig<G::T, true>(stg, t, srv, i0 - p.peek, G::L, p.n, p.linear);
        cp_async_commit();
    };

    if (nitems) issue(0);
    fft::stage_twiddles<R3>(sm, p.tw, t);
    __syncthreads();

    float2 accC[16], accX[16], X[16], v[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) accC[r] = accX[r] = X[r] = make_float2(0.f, 0.f);
#pragma unroll 1
    for (int it = 0; it < nitems; ++it) {
        const int kind = it % 3;
        fetch_staged<G::T, true>(v, stg, t, G::L);
        if (kind == 0) {                            // X: the segment's len samples, zero padded
            const int len = min(p.Bs, p.n - ((int)blockIdx.x + (it / 3) * (int)gridDim.x) * p.Bs);
#pragma unroll
            for (int n1 = 0; n1 < 16; ++n1)
                if (n1 * G::T + t >= len) v[n1] = make_float2(0.f, 0.f);
        }
        fft::fft_n2p<R3>(v, t, S, [&] { if (it + 1 < nitems) issue(it + 1); });
        if (kind == 0) {
#pragma unroll
            for (int r = 0; r < 16; ++r) X[r] = v[r];
        } else if (kind == 1) {
#pragma unroll
            for (int r = 0; r < 16; ++r) cmacc(accC[r], X[r], v[r]);        // accC += X conj(Yr)
        } else {
#pragma unroll
            for (int r = 0; r < 16; ++r) cmacc(accX[r], X[r], v[r]);        // accX += X conj(Ys)
        }
    }
    const float inv = 1.0f / (float)G::L;
#pragma unroll 1
    for (int w = 0; w < 2; ++w) {
#pragma unroll
        for (int r = 0; r < 16; ++r) v[r] = w ? accX[r] : accC[r];
        fft::fft_p2n<R3>(v, t, S);
        float2* row = p.partial + ((size_t)(blockIdx.y * 2 + w) * gridDim.x + blockIdx.x) * p.HT;
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int m = n1 * G::T + t;
            if (m < p.M) row[m] = make_float2(v[n1].x * inv, v[n1].y * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------ taps spectrum
struct TapSpecParams {
    const float2* taps;        // [frame][M]
    int M;
    float2* wp;                // [frame][L], permuted order: wp[r * T + t]
    const float2* tw;
};

template <int R3>
__global__ void __launch_bounds__(16 * R3) taps_spectrum_kernel(const __grid_constant__ TapSpecParams p) {
    using G = fft::Geo<R3>;
    extern __shared__ __align__(16) float2 sm[];
    const int t = threadIdx.x;
    const fft::Smem<R3> S(sm);
    fft::stage_twiddles<R3>(sm, p.tw, t);
    __syncthreads();
    const float2* taps = p.taps + (size_t)blockIdx.x * p.M;
    float2 v[16];
#pragma unroll
    for (int n1 = 0; n1 < 16; ++n1) {
        const int k = (n1 * G::T + t + p.M - 1) & (G::L - 1);      // h[(k - (M-1)) mod L] = w[k]
        v[n1] = (k < p.M) ? taps[k] : make_float2(0.f, 0.f);
    }
    fft::fft_n2p<R3>(v, t, S);
    float2* wp = p.wp + (size_t)blockIdx.x * G::L;
#pragma unroll
    for (int r = 0; r < 16; ++r) wp[r * G::T + t] = v[r];
}

// ------------------------------------------------------------------------------------------------ overlap-save FIR
struct FirFftParams {
    const float2* ref;
    const float2* srv;
    float2* out;
    long long frame_stride;
    const float2* wp;          // [frame][L]
    int n, M, peek, linear;
    int nseg;                  // segments of L - M + 1 outputs; CTA walks segments blockIdx.x, + gridDim.x, ...
    const float2* tw;
};

template <int R3> constexpr int fir_smem_float2() { return fft::Geo<R3>::SMEM_FLOAT2 + fft::Geo<R3>::L; }

template <int R3>
__global__ void __launch_bounds__(16 * R3) fir_fft_kernel(const __grid_constant__ FirFftParams p) {
    using G = fft::Geo<R3>;
    extern __shared__ __align__(16) float2 sm[];
    const int t = threadIdx.x;
    const fft::Smem<R3> S(sm);
    float2* stg = sm + G::SMEM_FLOAT2;
    const float2* ref = p.ref + (size_t)blockIdx.y * p.frame_stride;
    const float2* srv = p.srv + (size_t)blockIdx.y * p.frame_stride;
    float2* out = p.out + (size_t)blockIdx.y * p.frame_stride;
    const float2* wp = p.wp + (size_t)blockIdx.y * G::L;
    const int Bf = G::L - p.M + 1;
    const float inv = 1.0f / (float)G::L;
    auto issue = [&](int sgm) {
        stage_sig<G::T, true>(stg, t, ref, (long long)sgm * Bf + p.peek - (p.M - 1), G::L, p.n, p.linear);
        cp_async_commit();
    };
    if ((int)blockIdx.x < p.nseg) issue(blockIdx.x);
    fft::stage_twiddles<R3>(sm, p.tw, t);
    __syncthreads();
#pragma unroll 1
    for (int sgm = blockIdx.x; sgm < p.nseg; sgm += gridDim.x) {
        const long long p0 = (long long)sgm * Bf;
        float2 v[16];
        fetch_staged<G::T, true>(v, stg, t, G::L);
        fft::fft_n2p<R3>(v, t, S, [&] { if (sgm + (int)gridDim.x < p.nseg) issue(sgm + gridDim.x); });
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const float2 y = cmul(v[r], __ldg(wp + r * G::T + t));
            v[r] = make_float2(y.x, -y.y);                   // transform of conj(Y) = L conj(y)
        }
        float2 sv[16];                                       // surveillance samples of this segment: in flight during the transform
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int i = n1 * G::T + t;
            const long long o = p0 + i;
            sv[n1] = (i < Bf && o < p.n) ? __ldg(srv + o) : make_float2(0.f, 0.f);
        }
        fft::fft_p2n<R3>(v, t, S);
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int i = n1 * G::T + t;
            const long long o = p0 + i;
            if (i < Bf && o < p.n) out[o] = make_float2(sv[n1].x - v[n1].x * inv, sv[n1].y + v[n1].y * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------ CAF block sums
struct CafFftParams {
    const float2* ref;
    const float2* srv;
    long long frame_stride;
    const float* win;          // n floats shared by all frames, or NULL
    const float2* wp;          // [frame][L] taps spectrum (FUSED) or NULL
    int n, R, F, M, peek;      // M, peek: the fused clutter filter
    long long D;               // Doppler block j sums samples i = j D + c0 - m, m = 0..ntaps-1, 0 <= i < n
    int c0, ntaps;
    int Bmax;                  // segment length limit: L - R - (M - 1)
    float2* P;                 // [frame][F][HT]; P[j][d], d = 0..R
    int HT;
    const float2* tw;
};

// shared memory: [fft::Smem | staging L float2 | window staging L float]
template <int R3> constexpr int caf_smem_float2() { return fft::Geo<R3>::SMEM_FLOAT2 + fft::Geo<R3>::L + fft::Geo<R3>::L / 2; }

// Items of a Doppler block: per segment the surveillance samples (kind 0), with FUSED the reference samples the
// clutter filter needs (kind 1), and the windowed reference (kind 2); one transform call site for all of them.
// With FUSED, kind 1 stages ref[i0 - off ..] with off = M - 1 - peek, and the ln <= Bmax reference samples of kind 2
// lie inside that window (off + Bmax <= L): kind 2 reads them from the slots kind 1 staged, shifted by off, and
// stages only the window.  The slots are written by other threads, so this relies on the barriers of kind 1's
// transform (every thread waited for its own copies before it); the next segment's copies are issued after the
// first barrier of kind 2's transform, when every thread has read them.
template <int R3, bool FUSED>
__global__ void __launch_bounds__(16 * R3) caf_fft_kernel(const __grid_constant__ CafFftParams p) {
    using G = fft::Geo<R3>;
    constexpr int NK = FUSED ? 3 : 2;
    extern __shared__ __align__(16) float2 sm[];
    const int t = threadIdx.x;
    const fft::Smem<R3> S(sm);
    float2* stg = sm + G::SMEM_FLOAT2;
    float* wst = reinterpret_cast<float*>(stg + G::L);
    const float2* ref = p.ref + (size_t)blockIdx.y * p.frame_stride;
    const float2* srv = p.srv + (size_t)blockIdx.y * p.frame_stride;
    const float2* wp = FUSED ? p.wp + (size_t)blockIdx.y * G::L : nullptr;
    const float inv = 1.0f / (float)G::L;
    const int off = p.M - 1 - p.peek;
    const bool reuse = FUSED && off >= 0 && off + p.Bmax <= G::L;      // kind 2 reads kind 1's slots
    bool tw_staged = false;
#pragma unroll 1
    for (int j = blockIdx.x; j < p.F; j += gridDim.x) {
        long long lo = (long long)j * p.D + p.c0 - (p.ntaps - 1);
        long long hi = (long long)j * p.D + p.c0 + 1;
        if (lo < 0) lo = 0;
        if (hi > p.n) hi = p.n;
        const int len = hi > lo ? (int)(hi - lo) : 0;
        const int nseg = (len + p.Bmax - 1) / p.Bmax;
        const int Bs = nseg ? (len + nseg - 1) / nseg : 0;
        const int nitems = nseg * NK;
        auto issue = [&](int it) {
            const int q = it / NK, kind = FUSED ? it - q * NK : 2 * (it - q * NK);
            const long long i0 = lo + (long long)q * Bs;
            const int ln = (int)min((long long)Bs, hi - i0);
            if (kind == 0) {
                // L samples from i0 (circular); positions >= ln + R are never reached by lags 0..R
                stage_sig<G::T, true>(stg, t, srv, i0, G::L, p.n, 0);
            } else if (kind == 1) {
                stage_sig<G::T, true>(stg, t, ref, i0 + p.peek - (p.M - 1), G::L, p.n, 0);
            } else {
                if (!reuse) stage_sig<G::T, false>(stg, t, ref, i0, ln, p.n, 0);
                if (p.win) {
                    const float* w0 = p.win + i0 + t;
#pragma unroll
                    for (int n1 = 0; n1 < 16; ++n1)
                        if (n1 * G::T < ln) cp_async4(wst + t + n1 * G::T, w0 + n1 * G::T, n1 * G::T + t < ln);
                }
            }
            cp_async_commit();
        };
        if (nitems) issue(0);
        if (!tw_staged) {
            fft::stage_twiddles<R3>(sm, p.tw, t);
            __syncthreads();
            tw_staged = true;
        }
        float2 acc[16], sg[16], v[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) acc[r] = sg[r] = make_float2(0.f, 0.f);
#pragma unroll 1
        for (int it = 0; it < nitems; ++it) {
            const int q = it / NK, kind = FUSED ? it - q * NK : 2 * (it - q * NK);
            if (kind == 2) {
                const int ln = (int)min((long long)Bs, hi - (lo + (long long)q * Bs));
                if (reuse) {
                    cp_async_wait_all();                            // the window
#pragma unroll
                    for (int n1 = 0; n1 < 16; ++n1) {
                        const int i = n1 * G::T + t;
                        v[n1] = i < ln ? stg[i + off] : make_float2(0.f, 0.f);
                    }
                } else {
                    fetch_staged<G::T, false>(v, stg, t, ln);
                }
                if (p.win) {
#pragma unroll
                    for (int n1 = 0; n1 < 16; ++n1) {
                        if (n1 * G::T < ln) {
                            const float w = wst[t + n1 * G::T];
                            v[n1].x *= w;
                            v[n1].y *= w;
                        }
                    }
                }
            } else {
                fetch_staged<G::T, true>(v, stg, t, G::L);
            }
            fft::fft_n2p<R3>(v, t, S, [&] { if (it + 1 < nitems) issue(it + 1); });
            if (kind == 0) {
#pragma unroll
                for (int r = 0; r < 16; ++r) sg[r] = v[r];
            } else if (kind == 1) {
#pragma unroll
                for (int r = 0; r < 16; ++r) {               // cleaned surveillance spectrum: S - R_seg W'
                    const float2 y = cmul(v[r], __ldg(wp + r * G::T + t));
                    sg[r].x -= y.x;
                    sg[r].y -= y.y;
                }
            } else {
#pragma unroll
                for (int r = 0; r < 16; ++r) cmacc(acc[r], v[r], sg[r]);         // acc += X conj(S_clean)
            }
        }
        if (nitems) fft::fft_p2n<R3>(acc, t, S);
        float2* row = p.P + ((size_t)blockIdx.y * p.F + j) * p.HT;
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int d = n1 * G::T + t;
            if (d <= p.R) row[d] = make_float2(acc[n1].x * inv, acc[n1].y * inv);
        }
    }
}

}  // namespace fftc
}  // namespace prc
