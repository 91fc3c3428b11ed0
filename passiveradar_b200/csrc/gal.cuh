// gal.cuh -- GAL_JPE (reference clutter_removal.py:251-364): gradient-adaptive lattice + NLMS transversal stage,
// one frame per warp (delay lines up to GAL_WARP_MAX_D taps) or per CTA (up to GAL_MAX_D), state on chip.
//
// Per sample n (DESIGN.md section 10 gives the reference's rounding points and the mu1 type rules):
//   f[0] = b[0] = ref[n + peek],  f[m] = f[m-1] - conj(k[m]) bo[m-1],  b[m] = bo[m-1] - k[m] f[m-1]   (m < L)
//   k[m] += mu1 grad_m / (P[m-1] + 1e-10),  P, grad from f, bo, b of this sample                       (m < L)
//   b[m] = bo[m-1] (L <= m < D),  e = srv[n] - h^H b,  h += mu2 conj(e) b / (b^H b + 1e-10)
//   mu1 = min(0.999 mu1 + 1e-8 e^2, 5e-3)
// The forward errors are a prefix sum over the stages: f[m] = ref[n + peek] - sum_{j<=m} conj(k[j]) bo[j-1].  Each
// thread owns T consecutive stages/taps in registers and sums its own terms; a warp scan (plus, in the CTA variant, one
// exchange of warp totals through shared memory) gives the offsets.  Everything else is elementwise per tap except
// the two reductions h^H b and b^H b (butterfly, so every lane holds the bitwise same e).  The k update of sample n
// only feeds sample n + 1, so it overlaps the reductions.  Round-off of the reordered sums does not grow along the run
// (the reference's own output moves by ~2e-7 for a 1e-7 input perturbation over 6000 samples); the one accumulation
// that does drift, h's, is compensated (see the transversal stage).
#pragma once
#include <cuda_runtime.h>

namespace prc {

constexpr int GAL_MAX_D = 4096;         // largest delay line (the NLMS kernel's bound)
constexpr int GAL_CTA_T = 8;            // taps per thread, CTA-per-frame variant
constexpr int GAL_MAX_WARPS = GAL_MAX_D / (32 * GAL_CTA_T);
constexpr int GAL_WARP_MAX_D = 32 * 8;  // the warp-per-frame variant takes delay lines up to 256 taps
constexpr int GAL_WARP_FRAMES = 4;      // frames (one warp each) per CTA of the warp-per-frame variant

struct GalParams {
    const float2* ref;
    const float2* srv;
    float2* out;                // frame f at out + f * stride
    float2* k_out;              // nframes x D or null
    float2* h_out;              // nframes x D or null
    long long n, stride;        // samples per frame, distance between consecutive frames (samples)
    int nframes, L, D, peek;
    double mu1;                 // the caller's (Python float) step size
    float mu2;
};

__device__ __forceinline__ float2 gal_cmul(float2 a, float2 b) {
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

template <int T, bool CTA>
__global__ void __launch_bounds__(CTA ? 32 * GAL_MAX_WARPS : 32 * GAL_WARP_FRAMES)
gal_jpe_kernel(const __grid_constant__ GalParams p) {
    constexpr unsigned FULL = 0xffffffffu;
    __shared__ float2 s_tot[CTA ? GAL_MAX_WARPS : 1];     // per-warp totals of the stage prefix sum
    __shared__ float4 s_red[CTA ? GAL_MAX_WARPS : 1];     // per-warp partial h^H b (x, y) and b^H b (z)
    __shared__ float2 s_edge[CTA ? GAL_MAX_WARPS : 1];    // last b of each warp (bo[m-1] of the next warp's lane 0)
    // compensation terms of h (see below), one per tap: warp variant in static shared memory, CTA variant in the
    // dynamic shared memory (gal_smem(): nthr * T float2, then P as nthr * T floats)
    __shared__ float2 s_hcw[CTA ? 1 : GAL_WARP_FRAMES * 32 * T];
    extern __shared__ float2 gal_dyn[];
    const int lane = threadIdx.x & 31;
    const int warp = CTA ? (int)(threadIdx.x >> 5) : 0;
    const int nwarp = CTA ? (int)(blockDim.x >> 5) : 1;
    const int tid = CTA ? (int)threadIdx.x : lane;
    const int nthr = CTA ? (int)blockDim.x : 32;
    const int frame = CTA ? (int)blockIdx.x : (int)(blockIdx.x * GAL_WARP_FRAMES + (threadIdx.x >> 5));
    float2* hc = CTA ? gal_dyn : s_hcw + (threadIdx.x >> 5) * 32 * T;      // hc[j * nthr + tid]
    float* s_P = reinterpret_cast<float*>(gal_dyn + (CTA ? nthr * T : 0));  // CTA variant: s_P[j * nthr + tid]
    if (!CTA && frame >= p.nframes) return;                // whole warps only; this variant never synchronises the CTA
    const float2* ref = p.ref + (size_t)frame * p.stride;
    const float2* srv = p.srv + (size_t)frame * p.stride;
    float2* out = p.out + (size_t)frame * p.stride;
    const int L = p.L, D = p.D, m0 = tid * T;
    const long long nsteps = p.n - p.peek - 1 > 0 ? p.n - p.peek - 1 : 0;
    for (long long i = nsteps + tid; i < p.n; i += nthr) out[i] = make_float2(0.f, 0.f);     // the last peek + 1 samples

    float2 k[T], b[T], h[T];
    float P[CTA ? 1 : T];       // P[j] is the reference's P[m - 1] of stage m = m0 + j (the CTA variant keeps it in s_P
                                // to stay within the 128 registers of a 512-thread CTA)
#pragma unroll
    for (int j = 0; j < T; ++j) {
        k[j] = b[j] = h[j] = make_float2(0.f, 0.f);
        hc[j * nthr + tid] = make_float2(0.f, 0.f);
        if constexpr (CTA) s_P[j * nthr + tid] = 1e-8f;
        else P[j] = 1e-8f;
    }
    if (CTA) {
        if (tid < GAL_MAX_WARPS) s_edge[tid] = make_float2(0.f, 0.f);
        __syncthreads();
    }
    // mu1: a Python float (mu_d) until the first update, complex64 (mu_c) afterwards, a Python float again whenever
    // the clamp at 5e-3 wins -- identical in every thread
    bool mu_py = true;
    double mu_d = p.mu1;
    float2 mu_c = make_float2(0.f, 0.f);
    const float mu2 = p.mu2;
    const float omb2 = (float)(1.0 - 0.9 * 0.9);

    // inputs of the next 32 samples, one per lane (broadcast by shuffle), fetched one chunk ahead
    float2 nx = make_float2(0.f, 0.f), ns = make_float2(0.f, 0.f);
    if (lane < nsteps) { nx = ref[lane + p.peek]; ns = srv[lane]; }
    for (long long c0 = 0; c0 < nsteps; c0 += 32) {
        const float2 cx = nx, cs = ns;
        if (c0 + 32 + lane < nsteps) { nx = ref[c0 + 32 + lane + p.peek]; ns = srv[c0 + 32 + lane]; }
        const int cn = nsteps - c0 < 32 ? (int)(nsteps - c0) : 32;
        float2 keep = make_float2(0.f, 0.f);
        for (int t = 0; t < cn; ++t) {
            const float2 x0 = make_float2(__shfl_sync(FULL, cx.x, t), __shfl_sync(FULL, cx.y, t));
            const float2 sv = make_float2(__shfl_sync(FULL, cs.x, t), __shfl_sync(FULL, cs.y, t));
            // ---- bo[m0 - 1]: the previous thread's last backward error (b still holds last sample's values = bo)
            float2 bprev = make_float2(__shfl_up_sync(FULL, b[T - 1].x, 1), __shfl_up_sync(FULL, b[T - 1].y, 1));
            if (lane == 0) bprev = (CTA && warp > 0) ? s_edge[warp - 1] : make_float2(0.f, 0.f);
            // ---- stage terms c[m] = conj(k[m]) bo[m-1] (c[0] = -ref: f[m] = -(inclusive prefix)), local prefix
            float2 s[T];
            float2 acc = make_float2(0.f, 0.f);
#pragma unroll
            for (int j = 0; j < T; ++j) {
                const int m = m0 + j;
                const float2 bm1 = j ? b[j - 1] : bprev;
                float2 c = make_float2(0.f, 0.f);
                if (m == 0) c = make_float2(-x0.x, -x0.y);
                else if (m < L) c = make_float2(k[j].x * bm1.x + k[j].y * bm1.y, k[j].x * bm1.y - k[j].y * bm1.x);
                acc.x += c.x;
                acc.y += c.y;
                s[j] = acc;
            }
            float2 inc = acc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float tx = __shfl_up_sync(FULL, inc.x, o), ty = __shfl_up_sync(FULL, inc.y, o);
                if (lane >= o) { inc.x += tx; inc.y += ty; }
            }
            float2 ex = make_float2(__shfl_up_sync(FULL, inc.x, 1), __shfl_up_sync(FULL, inc.y, 1));
            if (lane == 0) ex = make_float2(0.f, 0.f);
            if (CTA) {
                if (lane == 31) s_tot[warp] = inc;
                __syncthreads();                                  // A: warp totals of the prefix sum
                float2 wx = make_float2(0.f, 0.f);
                for (int w = 0; w < warp; ++w) { wx.x += s_tot[w].x; wx.y += s_tot[w].y; }
                ex.x += wx.x;
                ex.y += wx.y;
            }
            // ---- new backward errors (b is overwritten in place: bm1 carries the old value one tap on), reflection-
            // coefficient update, partial reductions over the delay line
            float2 fm1 = make_float2(-ex.x, -ex.y);               // f[m0 - 1]
            float2 bm1 = bprev;                                   // bo[m - 1]
            float hr = 0.f, hi = 0.f, bb = 0.f;
#pragma unroll
            for (int j = 0; j < T; ++j) {
                const int m = m0 + j;
                const float2 bo = b[j];
                const float2 fm = make_float2(-(ex.x + s[j].x), -(ex.y + s[j].y));
                float2 nb;
                if (m == 0) {
                    nb = x0;
                } else if (m < L) {
                    const float2 kf = gal_cmul(k[j], fm1);
                    nb = make_float2(bm1.x - kf.x, bm1.y - kf.y);
                    const float Em = (fm1.x * fm1.x + fm1.y * fm1.y) + (bm1.x * bm1.x + bm1.y * bm1.y);
                    float pj;
                    if constexpr (CTA) pj = s_P[j * nthr + tid];
                    else pj = P[j];
                    pj = 0.9f * pj + omb2 * Em;
                    if constexpr (CTA) s_P[j * nthr + tid] = pj;
                    else P[j] = pj;
                    // grad = conj(f[m-1]) b[m] + bo[m-1] conj(f[m])
                    const float2 g = make_float2(fm1.x * nb.x + fm1.y * nb.y + bm1.x * fm.x + bm1.y * fm.y,
                                                 fm1.x * nb.y - fm1.y * nb.x + bm1.y * fm.x - bm1.x * fm.y);
                    float2 q;
                    if (mu_py) {
                        const float mf = (float)mu_d;
                        q = make_float2(mf * g.x, mf * g.y);
                    } else {
                        q = gal_cmul(mu_c, g);
                    }
                    const float r = __frcp_rn(pj + 1e-10f);     // complex64 / real complex64 = reciprocal multiply
                    k[j].x += q.x * r;
                    k[j].y += q.y * r;
                } else if (m < D) {
                    nb = bm1;                                     // delay line
                } else {
                    nb = make_float2(0.f, 0.f);
                }
                fm1 = fm;
                bm1 = bo;
                b[j] = nb;
                hr += h[j].x * nb.x + h[j].y * nb.y;              // conj(h) b
                hi += h[j].x * nb.y - h[j].y * nb.x;
                bb += nb.x * nb.x + nb.y * nb.y;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {                    // butterfly: every lane ends with the same bits
                hr += __shfl_xor_sync(FULL, hr, o);
                hi += __shfl_xor_sync(FULL, hi, o);
                bb += __shfl_xor_sync(FULL, bb, o);
            }
            if (CTA) {
                if (lane == 0) s_red[warp] = make_float4(hr, hi, bb, 0.f);
                if (lane == 31) s_edge[warp] = b[T - 1];
                __syncthreads();                                  // B: partial reductions, warp edges
                hr = hi = bb = 0.f;
                for (int w = 0; w < nwarp; ++w) {
                    const float4 v = s_red[w];
                    hr += v.x; hi += v.y; bb += v.z;
                }
            }
            // ---- transversal NLMS stage
            const float2 e = make_float2(sv.x - hr, sv.y - hi);
            const float r2 = __frcp_rn(bb + 1e-10f);
            // h is a compensated (Kahan) sum of its increments: added one by one in complex64, as the reference does,
            // they random-walk h away from the exact recurrence (2.4e-5 of max|srv| at the output over a 2^19-sample CPI,
            // against 9e-7 compensated); the increments themselves keep the reference's rounding points
            const float2 cc = make_float2(mu2 * e.x, -(mu2 * e.y));        // mu2 conj(e)
#pragma unroll
            for (int j = 0; j < T; ++j) {
                const float2 u = gal_cmul(cc, b[j]);
                float2 c = hc[j * nthr + tid];
                const float yx = u.x * r2 - c.x, yy = u.y * r2 - c.y;
                const float tx = h[j].x + yx, ty = h[j].y + yy;
                c.x = (tx - h[j].x) - yx;
                c.y = (ty - h[j].y) - yy;
                h[j] = make_float2(tx, ty);
                hc[j * nthr + tid] = c;
            }
            if (lane == t) keep = e;
            // ---- mu1 = min(0.999 mu1 + 1e-8 e**2, 5e-3): complex64 against 5e-3, real part first
            const float2 d = make_float2(1e-8f * (e.x * e.x - e.y * e.y), 1e-8f * (e.x * e.y + e.y * e.x));
            float xr, xi;
            if (mu_py) { xr = (float)(0.999 * mu_d) + d.x; xi = 0.f + d.y; }
            else { xr = 0.999f * mu_c.x + d.x; xi = 0.999f * mu_c.y + d.y; }
            if (xr > 5e-3f || (xr == 5e-3f && xi > 0.f)) { mu_py = true; mu_d = 5e-3; }
            else { mu_py = false; mu_c = make_float2(xr, xi); }
        }
        if (warp == 0 && lane < cn) out[c0 + lane] = keep;
    }
#pragma unroll
    for (int j = 0; j < T; ++j) {
        const int m = m0 + j;
        if (m < D) {
            if (p.k_out) p.k_out[(size_t)frame * D + m] = k[j];
            if (p.h_out) p.h_out[(size_t)frame * D + m] = h[j];
        }
    }
}

// dynamic shared memory of the CTA-per-frame variant with `threads` threads
inline size_t gal_smem(int threads) { return (size_t)threads * GAL_CTA_T * (sizeof(float2) + sizeof(float)); }

}  // namespace prc
