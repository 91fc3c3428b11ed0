// spectrum.cuh -- batched Welch power spectral density with matplotlib.mlab.psd's definition (DESIGN.md section 16).
// Everything is float64 / complex128 whatever the input dtype, as chanoff.cuh is: a preview is read in dB down to the
// noise floor, where single-precision transform noise would show.
//
//   spec_twiddle   tw[k] = exp(-2 pi i k / P), k < P / 2, built with sincospi (exact arguments)
//   spec_segments  one CTA per (chunk of consecutive segments, frame): each segment is widened, windowed, zero-padded
//                  to P = pad_to points and transformed in shared memory (radix-2 decimation in frequency: natural in,
//                  bit-reversed out); |X|^2 is summed over the chunk's segments in registers, in that bit-reversed
//                  order, and written once as the chunk's partial spectrum
//   spec_finish    per output bin: the frame's partials summed in chunk order, scaled, divided by the segment count,
//                  one-sided bins doubled, written in mlab's order
//
// The chunking of a frame's segments depends on (n, nfft, noverlap, pad_to) only (segments_per_cta), never on the batch
// size or the device, and the finishing sum runs in a fixed order: a frame of a batch is bit-identical to that frame
// computed alone.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace prc {
namespace spec {

// input dtypes (include/prcore.h PRC_DT_*): the four the estimator accepts
enum Dtype { DT_F32 = 3, DT_F64 = 4, DT_C64 = 5, DT_C128 = 6 };
inline bool dt_ok(int dt) { return dt == DT_F32 || dt == DT_F64 || dt == DT_C64 || dt == DT_C128; }

constexpr int THREADS = 256;
constexpr int MIN_LOG2 = 4;             // pad_to in [16, 8192]
constexpr int MAX_LOG2 = 13;            // 8192 complex128 = 128 KB of shared memory per CTA
constexpr int MAX_CHUNKS = 64;          // CTAs (partial spectra) per frame at most
constexpr int FIN_THREADS = 256;

// segments per CTA: at most MAX_CHUNKS chunks per frame, as few segments per chunk as that allows
inline long long segments_per_cta(long long nseg) { return (nseg + MAX_CHUNKS - 1) / MAX_CHUNKS; }

struct SegParams {
    const void* x;          // frame f starts at element f * stride
    int dt;
    long long n, stride;    // samples per frame, elements between frames
    int nfft, m;            // segment length, pad_to = 2^m
    long long step;         // nfft - noverlap
    long long nseg;         // segments per frame
    long long per_cta;      // segments per chunk
    int nchunk;             // chunks per frame
    const double* win;      // nfft window values
    const double2* tw;      // 2^(m-1) twiddles
    double* part;           // [frame of the launch][chunk][2^m], bit-reversed bin order
    long long f0;           // first frame of the launch
};

__device__ __forceinline__ double2 load_sample(const void* p, int dt, long long i) {
    if (dt == DT_C64) {
        const float2 v = static_cast<const float2*>(p)[i];
        return make_double2((double)v.x, (double)v.y);
    }
    if (dt == DT_C128) return static_cast<const double2*>(p)[i];
    if (dt == DT_F32) return make_double2((double)static_cast<const float*>(p)[i], 0.0);
    return make_double2(static_cast<const double*>(p)[i], 0.0);
}

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
    return make_double2(fma(a.x, b.x, -a.y * b.y), fma(a.x, b.y, a.y * b.x));
}

// ACC = accumulators per thread = max(1, P / THREADS)
template <int ACC>
__global__ void __launch_bounds__(THREADS, 1) spec_segments_kernel(const SegParams p) {
    extern __shared__ double2 sm[];
    const int P = 1 << p.m, H = P >> 1;
    const long long f = p.f0 + blockIdx.y;
    const long long s0 = (long long)blockIdx.x * p.per_cta;
    const long long s1 = min(s0 + p.per_cta, p.nseg);
    const long long base = f * p.stride;
    double acc[ACC];
#pragma unroll
    for (int k = 0; k < ACC; ++k) acc[k] = 0.0;
    for (long long s = s0; s < s1; ++s) {
        const long long start = s * p.step;
        for (int e = threadIdx.x; e < P; e += THREADS) {
            double2 v = make_double2(0.0, 0.0);
            if (e < p.nfft && start + e < p.n) {            // zero padding to pad_to, and of a frame shorter than nfft
                const double w = p.win[e];
                v = load_sample(p.x, p.dt, base + start + e);
                v.x *= w;
                v.y *= w;
            }
            sm[e] = v;
        }
        __syncthreads();
        for (int r = 0; r < p.m; ++r) {                    // stage r: span h = P / 2^(r+1), twiddle exp(-2 pi i j / 2h)
            const int lh = p.m - 1 - r, h = 1 << lh;
            for (int b = threadIdx.x; b < H; b += THREADS) {
                const int j = b & (h - 1);
                const int e1 = ((b >> lh) << (lh + 1)) | j, e2 = e1 + h;
                const double2 a = sm[e1], c = sm[e2];
                sm[e1] = make_double2(a.x + c.x, a.y + c.y);
                sm[e2] = cmul(make_double2(a.x - c.x, a.y - c.y), __ldg(&p.tw[j << r]));
            }
            __syncthreads();
        }
#pragma unroll
        for (int k = 0; k < ACC; ++k) {
            const int e = threadIdx.x + k * THREADS;
            if (e < P) {
                const double2 v = sm[e];
                acc[k] = fma(v.x, v.x, fma(v.y, v.y, acc[k]));
            }
        }
        __syncthreads();                                   // the next segment overwrites sm
    }
    double* out = p.part + ((long long)blockIdx.y * p.nchunk + blockIdx.x) * P;
#pragma unroll
    for (int k = 0; k < ACC; ++k) {
        const int e = threadIdx.x + k * THREADS;
        if (e < P) out[e] = acc[k];
    }
}

__global__ void spec_twiddle_kernel(double2* tw, int m) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (1 << (m - 1))) return;
    double s, c;
    sincospi(ldexp(-2.0, -m) * k, &s, &c);                 // -2 k / P: sincospi takes multiples of pi
    tw[k] = make_double2(c, s);
}

struct FinParams {
    const double* part;     // as SegParams::part
    int m, nchunk;
    long long nbins;        // output bins per frame
    int onesided;           // 0: two-sided, rotated so bin 0 is -Fs/2; 1: bins 0 .. P/2
    int nyq_double;         // one-sided: the P/2 bin is doubled too (mlab: when nfft is odd)
    double scale;           // caller's factor (1 / (Fs sum w^2) or 1 / (sum |w|)^2)
    double inv_nseg;        // 1 / segments per frame
    double* out;
    long long out_stride, f0;
};

__global__ void __launch_bounds__(FIN_THREADS) spec_finish_kernel(const FinParams p) {
    const long long j = (long long)blockIdx.x * FIN_THREADS + threadIdx.x;
    if (j >= p.nbins) return;
    const int P = 1 << p.m;
    const int k = p.onesided ? (int)j : (int)((j + (P >> 1)) & (P - 1));     // natural bin
    const int e = (int)(__brev((unsigned)k) >> (32 - p.m));                   // its place in the transform's output
    const double* src = p.part + (long long)blockIdx.y * p.nchunk * P + e;
    double s = 0.0;
    for (int c = 0; c < p.nchunk; ++c) s += src[(long long)c * P];
    double v = s * p.scale * p.inv_nseg;
    if (p.onesided && k > 0 && (k < (P >> 1) || p.nyq_double)) v *= 2.0;
    p.out[(p.f0 + blockIdx.y) * p.out_stride + j] = v;
}

// ---- launches (host side; prcore.cu brackets them with its profiling scopes and checks the launch) ----------------
inline size_t segments_smem(int m) { return ((size_t)1 << m) * sizeof(double2); }

template <int ACC>
inline cudaError_t set_attr_t(int lim) {
    return cudaFuncSetAttribute(spec_segments_kernel<ACC>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim);
}

inline cudaError_t set_attrs(int lim) {
    const cudaError_t e[6] = {set_attr_t<1>(lim), set_attr_t<2>(lim), set_attr_t<4>(lim), set_attr_t<8>(lim),
                              set_attr_t<16>(lim), set_attr_t<32>(lim)};
    for (cudaError_t x : e)
        if (x != cudaSuccess) return x;
    return cudaSuccess;
}

inline void launch_twiddle(double2* tw, int m, cudaStream_t st) {
    const int h = 1 << (m - 1);
    spec_twiddle_kernel<<<(h + 255) / 256, 256, 0, st>>>(tw, m);
}

// accumulators per thread of a transform of 2^m points: the instantiation launch_segments picks
inline int segments_acc(int m) { return m <= 8 ? 1 : 1 << (m - 8); }

inline void launch_segments(const SegParams& p, int nframes, cudaStream_t st) {
    const dim3 grid((unsigned)p.nchunk, (unsigned)nframes);
    const size_t smem = segments_smem(p.m);
    switch (segments_acc(p.m)) {
        case 1: spec_segments_kernel<1><<<grid, THREADS, smem, st>>>(p); break;
        case 2: spec_segments_kernel<2><<<grid, THREADS, smem, st>>>(p); break;
        case 4: spec_segments_kernel<4><<<grid, THREADS, smem, st>>>(p); break;
        case 8: spec_segments_kernel<8><<<grid, THREADS, smem, st>>>(p); break;
        case 16: spec_segments_kernel<16><<<grid, THREADS, smem, st>>>(p); break;
        default: spec_segments_kernel<32><<<grid, THREADS, smem, st>>>(p); break;
    }
}

inline void launch_finish(const FinParams& p, int nframes, cudaStream_t st) {
    spec_finish_kernel<<<dim3((unsigned)((p.nbins + FIN_THREADS - 1) / FIN_THREADS), (unsigned)nframes), FIN_THREADS, 0,
                         st>>>(p);
}

}  // namespace spec
}  // namespace prc
