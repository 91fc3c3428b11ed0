// frontend.cuh -- the arithmetic of the front end that feeds the hot path (SURVEY.md section 8(f).2):
//   deinterleave_IQ  (reference passiveRadar/signal_utils.py:19-22)
//   frequency_shift  (signal_utils.py:24-27, float32 phase ramp reproduced)
//   resample         (signal_utils.py:15-17: scipy resample_poly(x, up, dn, padtype='line'))
// Its one set of kernels, which run one chunk (prc_iq_mix_c64, prc_frontend_c64) or many (prc_frontend_chunks_c64),
// is in recording.cuh, and the CFAR detector behind it in detect.cuh.  All of it is bandwidth-bound element-wise /
// short-FIR work: one pass over the raw samples, shared-memory staging of the FIR window.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace prc {

enum IqKind { IQ_C64 = 0, IQ_I8 = 1, IQ_I16 = 2 };
enum MixMode { MIX_NONE = 0, MIX_C64 = 1, MIX_C128 = 2, MIX_F64 = 3, MIX_FS64 = 4 };

struct MixParams {
    const void* in;
    int kind;            // IqKind
    long long n;         // complex samples
    int mode;            // MixMode
    float B;             // float32(2 pi fc): imaginary part of complex64(1j*2*pi*fc)
    float rFs;           // fl32(1 / float32(Fs)): numpy divides a complex array by a real scalar as a
                         // multiplication by the reciprocal (loops.c.src: scl = 1.0/(in2r + in2i*rat))
    double po;           // phase offset (MIX_C64: rounded to float32 first, like numpy's weak scalar)
    double B64, rFs64;   // MIX_F64 / MIX_FS64: the same in float64 (fc or Fs was a NumPy float64 scalar)
};

// complex sample i of raw interleaved I/Q, read as scalars (the recording chain's chunks and decimate.cuh's slabs)
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

// x[i] * exp(1j * theta_i) with numpy's evaluation order:
//   theta32 = fl32(fl32(B * fl32(i)) * fl32(1/Fs))                                  (complex64 arange, weak python scalars)
//   MIX_C64 : theta = fl32(theta32 + fl32(po)), exp and product in float32     (phase_offset a python scalar)
//   MIX_C128: theta = double(theta32) + po, exp in float64                     (phase_offset a numpy float64, main.py:127-130)
//   MIX_F64 : theta = (2 pi fc) * double(fl32(i)) / Fs + po in float64          (fc a numpy float64 scalar)
//   MIX_FS64: theta = double(fl32(B * fl32(i))) / Fs + po in float64            (only Fs a numpy float64 scalar)
// The float64 angle (up to ~1e7 rad) is reduced to [-pi, pi] in double (two-constant Cody-Waite) and the
// sine/cosine taken in float32: absolute error ~1e-7, far inside the 1e-5 parity budget.
__device__ __forceinline__ float2 mix_sample(const MixParams& p, float2 v, long long i) {
    if (p.mode == MIX_NONE) return v;
    const float th32 = __fmul_rn(__fmul_rn(p.B, (float)i), p.rFs);
    double a;
    if (p.mode == MIX_C64) a = (double)__fadd_rn(th32, (float)p.po);
    else if (p.mode == MIX_C128) a = (double)th32 + p.po;
    else if (p.mode == MIX_F64) a = (p.B64 * (double)(float)i) * p.rFs64 + p.po;   // the ramp itself is still arange(dtype=complex64)
    else a = (double)__fmul_rn(p.B, (float)i) * p.rFs64 + p.po;
    const double k = rint(a * 0.15915494309189535);
    double r = fma(-k, 6.283185307179586, a);
    r = fma(-k, 2.4492935982947064e-16, r);
    float sn, cs;
    __sincosf((float)r, &sn, &cs);        // |r| <= pi: absolute error < 5e-7 (CUDA C Programming Guide, intrinsic functions)
    return make_float2(__fmaf_rn(v.x, cs, -__fmul_rn(v.y, sn)), __fmaf_rn(v.x, sn, __fmul_rn(v.y, cs)));
}

// ---------------------------------------------------------------------------------------------------
// resample_poly(x, up, down, padtype='line') as one polyphase pass.
//   y[m] = sum_k hpad[k] * xup[(m + n_pre_remove) * down - k],   xup[i * up] = xext[i]
// hpad = n_pre_pad zeros + h (already scaled by up), xext = x extended by a line through its end points
// (scipy _upfirdn_apply.pyx MODE_LINE: x[0] + idx * slope on the left, x[n-1] + (idx - n + 1) * slope on
// the right, slope = (x[n-1] - x[0]) / (n - 1)).  One thread per output sample; a CTA stages the
// polyphase taps [phase][j] and its window of mixed, deinterleaved input samples in shared memory, so the raw
// samples are read from HBM exactly once.
// ---------------------------------------------------------------------------------------------------
struct ResampleParams {
    MixParams mix;        // input description of chunk 0 (mode MIX_NONE for plain resample)
    int up, down;
    int n_pre_pad, n_pre_remove;
    int tpp;              // taps per phase = ceil((n_pre_pad + nh) / up), made odd (table row stride)
    long long n_out;
    const float* hp;      // polyphase table [up][tpp]: hp[ph][j] = hpad[ph + j * up]
    int span;             // input samples staged per CTA
};

constexpr int RS_THREADS = 256;

__device__ __forceinline__ size_t rs_table_bytes(const ResampleParams& p) {
    return ((size_t)p.up * p.tpp * 4 + 15) & ~(size_t)15;
}

// output m of the CTA whose window of xext starts at i_lo
__device__ __forceinline__ float2 rs_sum(const ResampleParams& p, const float* hp, const float2* xs, long long i_lo,
                                         long long m) {
    const long long T = (m + p.n_pre_remove) * (long long)p.down;
    const long long ih = T / p.up;
    const int ph = (int)(T - ih * p.up);                     // hpad index of the newest sample: k = ph + j * up
    const float* h = hp + (size_t)ph * p.tpp;
    const float2* x = xs + (ih - i_lo);                      // x[-j] = xext[ih - j]
    float ar = 0.f, ai = 0.f, br = 0.f, bi = 0.f;            // two chains: shorter dependency, pairwise-like sum
    int j = 0;
    for (; j + 1 < p.tpp; j += 2) {
        const float h0 = h[j], h1 = h[j + 1];
        const float2 v0 = x[-j], v1 = x[-j - 1];
        ar = fmaf(h0, v0.x, ar); ai = fmaf(h0, v0.y, ai);
        br = fmaf(h1, v1.x, br); bi = fmaf(h1, v1.y, bi);
    }
    if (j < p.tpp) {
        const float h0 = h[j];
        const float2 v0 = x[-j];
        ar = fmaf(h0, v0.x, ar); ai = fmaf(h0, v0.y, ai);
    }
    return make_float2(ar + br, ai + bi);
}

}  // namespace prc
