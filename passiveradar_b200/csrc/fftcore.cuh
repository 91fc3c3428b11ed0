// fftcore.cuh -- register/shared-memory complex FFT of length L = 256 * R3 (R3 = 4, 8, 16) for one group of
// T = L / 16 threads, 16 points per thread.  FP32, hand-written for the FFT-domain correlation kernels
// (fftcorr.cuh).  Replaces nothing in the reference by itself: the reference's lag loops
// (range_doppler_processing.py:81-86, clutter_removal.py:34-51) are evaluated as block correlations in the
// frequency domain (SURVEY.md section 7, hard part 2).
//
// Decomposition (L = 16 * 16 * R3):  n = n1 * (16 R3) + n2 * R3 + n3,   k = k1 + 16 k2 + 256 k3
//
//   W_L^{nk} = W_16^{n1 k1} * W_L^{(n2 R3 + n3) k1} * W_16^{n2 k2} * W_{16 R3}^{n3 k2} * W_R3^{n3 k3}
//
// fft_n2p ("natural to permuted", decimation in frequency):
//   pass 1   thread t = n2 R3 + n3 holds x[n1 T + t], n1 = 0..15 (coalesced loads): DFT16 over n1, times W_L^{t k1}
//   exch 1   E1[k1][n2][n3]  ->  thread (k1, n3) = k1 R3 + n3 reads n2 = 0..15
//   pass 2   DFT16 over n2, times W_{16 R3}^{n3 k2}
//   exch 2   E2[k1][n3][k2]  ->  thread (k1, j) = k1 R3 + j reads n3 = 0..R3-1 for k2 = j + R3 h, h < 16 / R3
//   pass 3   DFT_R3 over n3: register h R3 + k3 holds X[k1 + 16 (j + R3 h) + 256 k3]        ("permuted order")
//
// fft_p2n ("permuted to natural") is the TRANSPOSE of that factorisation: the DFT matrix is symmetric, so running
// the passes in reverse order with the same small DFTs and the same twiddles is again the forward DFT, now from
// permuted-order registers to natural order x[n1 T + t].  An inverse transform is never needed: the correlation
// kernels accumulate Zc = X conj(Y) in permuted order and fft_p2n(Zc)[m] = L * sum_i x[i] conj(y[i + m]).
//
// Shared memory: two exchange buffers of EX = 16 * 17 * R3 float2 (padded: every 64-bit access pattern below is
// bank-conflict free per half-warp), so one transform needs two block-wide barriers and consecutive transforms
// need none between them.  Twiddle tables (built in float64 by fft_twiddle_kernel, staged to shared memory):
//   tw1[k1 * T + t]   = W_L^{t k1}            (L entries)
//   tw2[k2 * R3 + n3] = W_{16 R3}^{n3 k2}     (16 R3 entries)
//
// Every per-thread phase is a __host__ __device__ function of (registers, t, buffers): the same code is run
// thread-by-thread on the CPU by scripts/fft/emul.cu and tests/test_fft_emulation.py to pin the index algebra
// against a float64 DFT without a GPU.
#pragma once
#include <cuda_runtime.h>

namespace prc {
namespace fft {

#define PRC_HD __host__ __device__ __forceinline__

template <int R3> struct Geo {
    static constexpr int L = 256 * R3;      // transform length
    static constexpr int T = 16 * R3;       // threads per transform
    static constexpr int S = 17 * R3;       // padded k1 stride of both exchange layouts (float2)
    static constexpr int EX = 16 * S;       // float2 per exchange buffer
    static constexpr int H = 16 / R3;       // DFT_R3's per thread in pass 3
    static constexpr int TW1 = L, TW2 = 16 * R3;
    static constexpr int SMEM_FLOAT2 = 2 * EX + TW1 + TW2;
};

// complex add / subtract: on the device one packed FP32x2 instruction each (FADD2 / FFMA2 with -1: the same two
// roundings as the scalar form, half the issue slots -- the transforms are issue-bound, not FP32-lane-bound)
#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ >= 1000) && !defined(PRC_SCALAR_FFT)
PRC_HD float2 cadd(float2 a, float2 b) { return __fadd2_rn(a, b); }
PRC_HD float2 csub(float2 a, float2 b) { return __ffma2_rn(b, make_float2(-1.f, -1.f), a); }
#else
PRC_HD float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
PRC_HD float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
#endif
PRC_HD float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
PRC_HD float2 cmulc(float2 a, float2 b) { return make_float2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y); }   // a conj(b)
PRC_HD float2 mul_mi(float2 a) { return make_float2(a.y, -a.x); }      // a * (-i)

// forward DFT4 (W4 = -i), in place, natural order
PRC_HD void dft4(float2& a, float2& b, float2& c, float2& d) {
    const float2 t0 = cadd(a, c), t1 = csub(a, c), t2 = cadd(b, d), t3 = mul_mi(csub(b, d));
    a = cadd(t0, t2);
    c = csub(t0, t2);
    b = cadd(t1, t3);
    d = csub(t1, t3);
}

template <int R> struct Dft;

template <> struct Dft<4> {
    static PRC_HD void run(float2* v) { dft4(v[0], v[1], v[2], v[3]); }
};

template <> struct Dft<8> {
    // n = 2a + b, k = c + 4d:  X[c + 4d] = sum_b W8^{bc} (-1)^{bd} sum_a x[2a + b] W4^{ac}
    static PRC_HD void run(float2* v) {
        const float r = 0.70710678118654752440f;
        dft4(v[0], v[2], v[4], v[6]);         // y0[c] at v[2c]
        dft4(v[1], v[3], v[5], v[7]);         // y1[c] at v[2c + 1]
        const float2 y1 = make_float2((v[3].x + v[3].y) * r, (v[3].y - v[3].x) * r);       // * W8^1 = (1 - i)/sqrt2
        const float2 y2 = mul_mi(v[5]);                                                  // * W8^2 = -i
        const float2 y3 = make_float2((v[7].y - v[7].x) * r, -(v[7].x + v[7].y) * r);      // * W8^3 = (-1 - i)/sqrt2
        const float2 a0 = v[0], a1 = v[2], a2 = v[4], a3 = v[6], b0 = v[1];
        v[0] = cadd(a0, b0); v[4] = csub(a0, b0);
        v[1] = cadd(a1, y1); v[5] = csub(a1, y1);
        v[2] = cadd(a2, y2); v[6] = csub(a2, y2);
        v[3] = cadd(a3, y3); v[7] = csub(a3, y3);
    }
};

template <> struct Dft<16> {
    // n = 4a + b, k = c + 4d:  X[c + 4d] = sum_b W16^{bc} W4^{bd} sum_a x[4a + b] W4^{ac}
    static PRC_HD void run(float2* v) {
        const float c1 = 0.92387953251128675613f, s1 = 0.38268343236508977173f, r = 0.70710678118654752440f;
        dft4(v[0], v[4], v[8], v[12]);        // y_b[c] lands at v[4c + b]
        dft4(v[1], v[5], v[9], v[13]);
        dft4(v[2], v[6], v[10], v[14]);
        dft4(v[3], v[7], v[11], v[15]);
        // twiddles W16^{bc}, b, c = 1..3   (W16^m = cos(pi m / 8) - i sin(pi m / 8))
        v[5] = cmul(v[5], make_float2(c1, -s1));                                        // b=1 c=1: W^1
        v[9] = make_float2((v[9].x + v[9].y) * r, (v[9].y - v[9].x) * r);               // b=1 c=2: W^2
        v[13] = cmul(v[13], make_float2(s1, -c1));                                      // b=1 c=3: W^3
        v[6] = make_float2((v[6].x + v[6].y) * r, (v[6].y - v[6].x) * r);               // b=2 c=1: W^2
        v[10] = mul_mi(v[10]);                                                          // b=2 c=2: W^4
        v[14] = make_float2((v[14].y - v[14].x) * r, -(v[14].x + v[14].y) * r);         // b=2 c=3: W^6
        v[7] = cmul(v[7], make_float2(s1, -c1));                                        // b=3 c=1: W^3
        v[11] = make_float2((v[11].y - v[11].x) * r, -(v[11].x + v[11].y) * r);         // b=3 c=2: W^6
        v[15] = cmul(v[15], make_float2(-c1, s1));                                      // b=3 c=3: W^9
        // X[c + 4d] = DFT4 over b of v[4c + b]; output index c + 4d
        float2 o[16];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float2 p = v[4 * c], q = v[4 * c + 1], s = v[4 * c + 2], u = v[4 * c + 3];
            dft4(p, q, s, u);
            o[c] = p; o[c + 4] = q; o[c + 8] = s; o[c + 12] = u;
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = o[i];
    }
};

// ---- natural -> permuted -------------------------------------------------------------------------------------
template <int R3>
PRC_HD void n2p_pass1(float2 (&v)[16], int t, float2* __restrict__ ea, const float2* __restrict__ tw1) {
    using G = Geo<R3>;
    float2 w[16];                      // twiddle loads in flight while the butterflies run
#pragma unroll
    for (int k1 = 1; k1 < 16; ++k1) w[k1] = tw1[k1 * G::T + t];
    Dft<16>::run(v);
    const int n2 = t / R3, n3 = t - n2 * R3;
    float2* dst = ea + n2 * R3 + n3;
    dst[0] = v[0];
#pragma unroll
    for (int k1 = 1; k1 < 16; ++k1) dst[k1 * G::S] = cmul(v[k1], w[k1]);
}

template <int R3>
PRC_HD void n2p_pass2(float2 (&v)[16], int t, const float2* __restrict__ ea, float2* __restrict__ eb,
                      const float2* __restrict__ tw2) {
    using G = Geo<R3>;
    const int k1 = t / R3, n3 = t - k1 * R3;
    const float2* src = ea + k1 * G::S + n3;
#pragma unroll
    for (int n2 = 0; n2 < 16; ++n2) v[n2] = src[n2 * R3];
    float2 w[16];
#pragma unroll
    for (int k2 = 1; k2 < 16; ++k2) w[k2] = tw2[k2 * R3 + n3];
    Dft<16>::run(v);
    float2* dst = eb + k1 * G::S + n3 * 17;
    dst[0] = v[0];
#pragma unroll
    for (int k2 = 1; k2 < 16; ++k2) dst[k2] = cmul(v[k2], w[k2]);
}

template <int R3>
PRC_HD void n2p_pass3(float2 (&v)[16], int t, const float2* __restrict__ eb) {
    using G = Geo<R3>;
    const int k1 = t / R3, j = t - k1 * R3;
    const float2* src = eb + k1 * G::S + j;
#pragma unroll
    for (int h = 0; h < G::H; ++h) {
#pragma unroll
        for (int n3 = 0; n3 < R3; ++n3) v[h * R3 + n3] = src[n3 * 17 + R3 * h];
        Dft<R3>::run(&v[h * R3]);
    }
}

// frequency held by register r of thread t after fft_n2p (and expected by fft_p2n)
template <int R3>
PRC_HD int perm_freq(int t, int r) {
    const int k1 = t / R3, j = t - k1 * R3;
    const int h = r / R3, k3 = r - h * R3;
    return k1 + 16 * (j + R3 * h) + 256 * k3;
}

// ---- permuted -> natural (transposed factorisation) ---------------------------------------------------------
template <int R3>
PRC_HD void p2n_pass1(float2 (&v)[16], int t, float2* __restrict__ eb) {
    using G = Geo<R3>;
    const int k1 = t / R3, j = t - k1 * R3;
    float2* dst = eb + k1 * G::S + j;
#pragma unroll
    for (int h = 0; h < G::H; ++h) {
        Dft<R3>::run(&v[h * R3]);
#pragma unroll
        for (int n3 = 0; n3 < R3; ++n3) dst[n3 * 17 + R3 * h] = v[h * R3 + n3];
    }
}

template <int R3>
PRC_HD void p2n_pass2(float2 (&v)[16], int t, const float2* __restrict__ eb, float2* __restrict__ ea,
                      const float2* __restrict__ tw2) {
    using G = Geo<R3>;
    const int k1 = t / R3, n3 = t - k1 * R3;
    const float2* src = eb + k1 * G::S + n3 * 17;
    float2 w[16];
#pragma unroll
    for (int k2 = 1; k2 < 16; ++k2) w[k2] = tw2[k2 * R3 + n3];
#pragma unroll
    for (int k2 = 0; k2 < 16; ++k2) v[k2] = src[k2];
#pragma unroll
    for (int k2 = 1; k2 < 16; ++k2) v[k2] = cmul(v[k2], w[k2]);
    Dft<16>::run(v);
    float2* dst = ea + k1 * G::S + n3;
#pragma unroll
    for (int n2 = 0; n2 < 16; ++n2) dst[n2 * R3] = v[n2];
}

template <int R3>
PRC_HD void p2n_pass3(float2 (&v)[16], int t, const float2* __restrict__ ea, const float2* __restrict__ tw1) {
    using G = Geo<R3>;
    const int n2 = t / R3, n3 = t - n2 * R3;
    const float2* src = ea + n2 * R3 + n3;
    float2 w[16];
#pragma unroll
    for (int k1 = 1; k1 < 16; ++k1) w[k1] = tw1[k1 * G::T + t];
#pragma unroll
    for (int k1 = 0; k1 < 16; ++k1) v[k1] = src[k1 * G::S];
#pragma unroll
    for (int k1 = 1; k1 < 16; ++k1) v[k1] = cmul(v[k1], w[k1]);
    Dft<16>::run(v);
}

#ifdef __CUDACC__
// Block-wide transforms: every thread of the group (blockDim.x == T) calls them; `sm` = [ea | eb | tw1 | tw2].
template <int R3> struct Smem {
    float2* ea; float2* eb; const float2* tw1; const float2* tw2;
    __device__ __forceinline__ explicit Smem(float2* base)
        : ea(base), eb(base + Geo<R3>::EX), tw1(base + 2 * Geo<R3>::EX), tw2(base + 2 * Geo<R3>::EX + Geo<R3>::TW1) {}
};

template <int R3>
__device__ __forceinline__ void fft_n2p(float2 (&v)[16], int t, const Smem<R3>& s) {
    n2p_pass1<R3>(v, t, s.ea, s.tw1);
    __syncthreads();
    n2p_pass2<R3>(v, t, s.ea, s.eb, s.tw2);
    __syncthreads();
    n2p_pass3<R3>(v, t, s.eb);
}

// same, with `after_pass1()` run once the group's first barrier has passed (every register of v has been consumed by
// then): the place to start asynchronous copies that overwrite the shared-memory slots v was fetched from
template <int R3, class Hook>
__device__ __forceinline__ void fft_n2p(float2 (&v)[16], int t, const Smem<R3>& s, Hook after_pass1) {
    n2p_pass1<R3>(v, t, s.ea, s.tw1);
    __syncthreads();
    after_pass1();
    n2p_pass2<R3>(v, t, s.ea, s.eb, s.tw2);
    __syncthreads();
    n2p_pass3<R3>(v, t, s.eb);
}

template <int R3>
__device__ __forceinline__ void fft_p2n(float2 (&v)[16], int t, const Smem<R3>& s) {
    p2n_pass1<R3>(v, t, s.eb);
    __syncthreads();
    p2n_pass2<R3>(v, t, s.eb, s.ea, s.tw2);
    __syncthreads();
    p2n_pass3<R3>(v, t, s.ea, s.tw1);
}

// stage the twiddle tables (global, [tw1 | tw2]) into shared memory; caller synchronises
template <int R3>
__device__ __forceinline__ void stage_twiddles(float2* base, const float2* __restrict__ tw_global, int t) {
    using G = Geo<R3>;
    float2* dst = base + 2 * G::EX;
    for (int i = t; i < G::TW1 + G::TW2; i += G::T) dst[i] = tw_global[i];
}

// tw[0 .. L) = tw1, tw[L .. L + 16 R3) = tw2, evaluated in float64
template <int R3>
__global__ void fft_twiddle_kernel(float2* tw) {
    using G = Geo<R3>;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < G::TW1) {
        const int k1 = i / G::T, t = i - k1 * G::T;
        double s, c;
        sincospi(-2.0 * (double)((long long)t * k1 % G::L) / (double)G::L, &s, &c);
        tw[i] = make_float2((float)c, (float)s);
    } else if (i < G::TW1 + G::TW2) {
        const int q = i - G::TW1;
        const int k2 = q / R3, n3 = q - k2 * R3;
        double s, c;
        sincospi(-2.0 * (double)(n3 * k2) / (double)(16 * R3), &s, &c);
        tw[i] = make_float2((float)c, (float)s);
    }
}
#endif

}  // namespace fft
}  // namespace prc
