// prcore_corr.cu -- the correlation family of libprcore.so: LS_Filter (direct form and FFT-domain), LS_Filter_Toeplitz
// and LS_Filter_Multiple, fast_xambg, direct_xambg, and the frame (LS_Filter -> fast_xambg) with its one-pass FFT-domain
// path and its shared-reference form for several surveillance channels; their planners, launches and C entry points,
// and the options that select their paths.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdlib>
#include <mutex>
#include <string>
#include <vector>

#include "prcore_host.h"
#include "kernels.cuh"
#include "lagstream.cuh"
#include "fftcorr.cuh"
#include "framepass.cuh"
#include "framemulti.cuh"

namespace prcore {

using namespace prc;

// Register tile of the FP32 sliding-window kernels (lagcorr, lagstream, fir_apply; DESIGN.md section 3.8):
// TILE_I x TILE_D = 10 x 10 complex MACs per step (samples x lags, or taps x outputs), lane stride
// 10 complex = 80 B (odd multiple of 16 B => conflict-free 128-bit shared loads).
constexpr int TILE_I = 10, TILE_D = 10;
constexpr int FIR_THREADS = 128;

std::atomic<int> g_fft{1};            // FFT-domain correlation / overlap-save kernels (fftcorr.cuh); PRC_FFT=0: FP32 direct form
std::atomic<int> g_fft_min_n{8192};   // ... for channels of at least this many samples (PRC_FFT_MIN_N)
std::atomic<int> g_frame_onepass{1};  // FFT-domain frame: LS lag sums and CAF block spectra in one pass (framepass.cuh); 0: two passes
std::once_flag g_env_once;

// The options start from the environment: read once, before the first plan or the first prc_set_option / prc_get_option
void read_env() {
    if (const char* e = getenv("PRC_FFT")) g_fft.store(atoi(e));
    if (const char* e = getenv("PRC_FFT_MIN_N")) g_fft_min_n.store(atoi(e));
}

int corr_set_attrs(int lim) {
    CU(cudaFuncSetAttribute(lagcorr_kernel<TILE_I, TILE_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(lagstream_kernel<TILE_I, TILE_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(fir_apply_kernel<TILE_I, TILE_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(levinson_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(levinson_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(doppler_fft_pow2_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(doppler_fft_pow2_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(doppler_fft_pow2_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
#define PRC_FFT_ATTRS(R3)                                                                                              \
    CU(cudaFuncSetAttribute(fftc::lscorr_fft_kernel<R3>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));           \
    CU(cudaFuncSetAttribute(fftc::taps_spectrum_kernel<R3>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));        \
    CU(cudaFuncSetAttribute(fftc::fir_fft_kernel<R3>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));              \
    CU(cudaFuncSetAttribute(fftc::caf_fft_kernel<R3, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));       \
    CU(cudaFuncSetAttribute(fftc::caf_fft_kernel<R3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    PRC_FFT_ATTRS(4)
    PRC_FFT_ATTRS(8)
    PRC_FFT_ATTRS(16)
#undef PRC_FFT_ATTRS
    CU(fftc::framepass_set_attrs(lim));
    CU(fftc::framemulti_set_attrs(lim));
    return PRC_OK;
}

// --------------------------------------------------------------------------- geometry
struct Geo {
    int H, G, steps, nchunk, chunk_len, threads;
    size_t smem;
    int HT;
};

int choose_geo(int blk_len, long long outer, int nlag, int nsm, Geo* g) {
    const int TI = TILE_I, TD = TILE_D;
    g->H = ceil_div(nlag, TD);
    g->HT = g->H * TD;
    if (g->H > 512) return fail(PRC_E_INVALID, "%d lags exceed the supported maximum of %d", nlag, 512 * TD);
    int gmax = std::max(1, std::min(32, 256 / g->H));
    long long target = (long long)nsm * 8;
    long long nchunk = std::max<long long>(1, (target + outer - 1) / outer);
    const int min_chunk = TI * gmax * 2;
    nchunk = std::min<long long>(nchunk, std::max(1, blk_len / min_chunk));
    for (;;) {
        g->chunk_len = ceil_div(blk_len, nchunk);
        g->nchunk = ceil_div(blk_len, g->chunk_len);
        g->G = std::max(1, std::min(gmax, ceil_div(g->chunk_len, TI * 4)));
        g->steps = ceil_div(ceil_div(g->chunk_len, g->G), TI);
        const size_t Lpad = (size_t)g->G * g->steps * TI;
        g->smem = std::max(3 * Lpad + g->HT, (size_t)g->G * g->HT) * sizeof(float2);
        if (g->smem <= 100 * 1024 || g->chunk_len <= TI) break;
        nchunk = nchunk * 2;
    }
    if (g->smem > SMEM_LIMIT) return fail(PRC_E_INVALID, "lag-correlation tile needs %zu B of shared memory", g->smem);
    g->threads = ((g->H * g->G + 31) / 32) * 32;
    return PRC_OK;
}

struct StreamGeo {
    int HT, threads, ncta;
    size_t smem;
    LagStreamParams sp;   // the geometry's fields (blk_len, nblk, total .. maxpieces); operands, block starts and
                          // s_linear are the caller's
};

// CTAs per problem: fill every SM with two co-resident CTAs, but keep >= 2 full steps per CTA
int choose_stream(int blk_len, int nblk, int nprob, int nlag, int nsm, StreamGeo* g) {
    const int TI = TILE_I, TD = TILE_D;
    LagStreamParams& s = g->sp;
    s = LagStreamParams{};
    s.blk_len = blk_len;
    s.nblk = nblk;
    s.H = ceil_div(nlag, TD);
    g->HT = s.H * TD;
    if (s.H > 512) return fail(PRC_E_INVALID, "%d lags exceed the supported maximum of %d", nlag, 512 * TD);
    int G = std::max(1, std::min(32, 256 / s.H));
    s.total = (long long)nblk * blk_len;
    long long want = std::max(1, 2 * nsm / nprob);
    const long long min_per_cta = (long long)G * TI * 2;
    want = std::min<long long>(want, std::max<long long>(1, s.total / min_per_cta));
    s.per_cta = (s.total + want - 1) / want;
    g->ncta = (int)((s.total + s.per_cta - 1) / s.per_cta);
    s.G = (int)std::max<long long>(1, std::min<long long>(G, (s.per_cta + TI - 1) / TI));
    s.steps = std::max(2, 100 / TI);
    while (s.steps > 1 && (long long)s.G * s.steps * TI > s.per_cta + s.G * TI) --s.steps;
    for (;;) {
        const size_t Lmax = (size_t)s.G * s.steps * TI;
        g->smem = (2 * (2 * Lmax + g->HT) + 2 * (size_t)s.G * g->HT) * sizeof(float2);   // staging, sums, compensations
        if (g->smem <= 100 * 1024 || s.steps == 1) break;
        --s.steps;
    }
    if (g->smem > SMEM_LIMIT) return fail(PRC_E_INVALID, "lag-correlation tile needs %zu B of shared memory", g->smem);
    s.maxpieces = (int)std::min<long long>(g->ncta, (blk_len + s.per_cta - 2) / s.per_cta + 1);
    g->threads = ((s.H * s.G + 31) / 32) * 32;
    return PRC_OK;
}

void launch_lagstream(dim3 grid, int threads, size_t smem, cudaStream_t st, const LagStreamParams& sp) {
    lagstream_kernel<TILE_I, TILE_D><<<grid, threads, smem, st>>>(sp);
}

// --------------------------------------------------------------------------- FFT-domain path (fftcorr.cuh)
// A batch of frames: nf channels pairs `stride` samples apart (inputs), results laid out frame after frame.
inline int r3_index(int r3) { return r3 == 4 ? 0 : (r3 == 8 ? 1 : 2); }
inline size_t fft_smem(int r3) { return (size_t)(2 * 16 * 17 * r3 + 256 * r3 + 16 * r3) * sizeof(float2); }   // fft::Geo<R3>::SMEM_FLOAT2: exchange buffers + twiddles, no staging

// R3 = 4 / 8 / 16  <->  L = 1024 / 2048 / 4096
#define PRC_R3_SWITCH(r3, STMT)                        \
    switch (r3) {                                      \
        case 4: { constexpr int R3 = 4; STMT; } break; \
        case 8: { constexpr int R3 = 8; STMT; } break; \
        default: { constexpr int R3 = 16; STMT; } break; \
    }

int fft_twiddles(Ctx* c, int r3, const float2** tw) {
    const int k = r3_index(r3);
    const int cnt = 256 * r3 + 16 * r3;
    if (!c->fft_tw_ready[k]) {
        TRY(c->fft_tw[k].ensure((size_t)cnt * sizeof(float2)));
        PRC_R3_SWITCH(r3, (fft::fft_twiddle_kernel<R3><<<ceil_div(cnt, 256), 256, 0, c->stream>>>(c->fft_tw[k].as<float2>())));
        TRY(check_launch("fft_twiddle_kernel"));
        c->fft_tw_ready[k] = true;
    }
    *tw = c->fft_tw[k].as<float2>();
    return PRC_OK;
}

// FFT-domain kernels whose grids are sized to one wave of CTAs for the whole batch
enum FftKern { FK_LS = 0, FK_FIR = 1, FK_FRAME = 2, FK_COMBINE = 3 };   // FRAME, COMBINE: R3 = 8 only

// CTAs of one instantiation an SM holds at once, at the block size and dynamic shared memory it is launched with:
// registers (and the launch bounds that cap them) and shared memory decide it, so the grids follow the build rather
// than a number written next to them.  Asked once per context.  1 if the runtime cannot answer (the grid stays
// correct, only smaller; the launch itself then reports what is wrong).
int fft_ctas_per_sm(Ctx* c, FftKern k, int r3) {
    int& cached = c->fft_ctas[k][r3_index(r3)];
    if (cached > 0) return cached;
    int v = 0;
    cudaError_t e = cudaSuccess;
    if (k == FK_LS) {
        PRC_R3_SWITCH(r3, (e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, fftc::lscorr_fft_kernel<R3>, 16 * R3,
                                                                           fftc::lscorr_smem_float2<R3>() * sizeof(float2))));
    } else if (k == FK_FIR) {
        PRC_R3_SWITCH(r3, (e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, fftc::fir_fft_kernel<R3>, 16 * R3,
                                                                           fftc::fir_smem_float2<R3>() * sizeof(float2))));
    } else {
        v = k == FK_FRAME ? fftc::frame_pass_ctas_per_sm() : fftc::caf_combine_ctas_per_sm();
    }
    if (e != cudaSuccess || v < 1) {
        cudaGetLastError();
        return 1;
    }
    cached = v;
    return v;
}

// ---- LS correlations: segments of the channel
struct LsFftPlan {
    bool on = false;
    int r3 = 8, nseg = 0, Bs = 0, ncta = 0, HT = 0;
};

LsFftPlan ls_fft_plan(Ctx* c, long long n, int M, int nf) {
    LsFftPlan pl;
    std::call_once(g_env_once, read_env);
    if (!g_fft.load() || n < g_fft_min_n.load() || M < 1 || M > 2048) return pl;
    pl.r3 = M <= 1024 ? 8 : 16;
    const int L = 256 * pl.r3;
    if (n < 2 * L) return pl;
    const int bmax = L - M + 1;                        // lags 0..M-1 of a segment stay inside its L-sample window
    pl.nseg = (int)((n + bmax - 1) / bmax);
    pl.Bs = (int)((n + pl.nseg - 1) / pl.nseg);
    pl.nseg = (int)((n + pl.Bs - 1) / pl.Bs);
    // CTAs of one transform group (16 R3 threads), as many per SM as are resident at once (R3 = 8: 3, R3 = 16: 1): the
    // whole batch is ONE wave of CTAs, every CTA walks its share of a frame's segments (any split works: segments are
    // independent)
    const long long slots = (long long)fft_ctas_per_sm(c, FK_LS, pl.r3) * c->nsm;
    pl.ncta = (int)std::max<long long>(1, std::min<long long>(pl.nseg, slots / nf));
    pl.HT = (M + 1) & ~1;
    pl.on = true;
    return pl;
}

int ls_fft_corr(Ctx* c, const LsFftPlan& pl, const float2* ref, const float2* srv, long long n, Batch bt, int M, int peek,
                bool linear) {
    const float2* tw;
    TRY(fft_twiddles(c, pl.r3, &tw));
    TRY(c->partial.ensure((size_t)bt.nf * 2 * pl.ncta * pl.HT * sizeof(float2)));
    fftc::LsCorrParams p{};
    p.ref = ref; p.srv = srv; p.frame_stride = bt.stride;
    p.n = (int)n; p.M = M; p.peek = peek; p.linear = linear ? 1 : 0;
    p.nseg = pl.nseg; p.Bs = pl.Bs;
    p.partial = c->partial.as<float2>(); p.HT = pl.HT; p.tw = tw;
    {
        ProfScope ps(c, K_LAGCORR_LS);
        PRC_R3_SWITCH(pl.r3, (fftc::lscorr_fft_kernel<R3><<<dim3(pl.ncta, bt.nf), 16 * R3, fftc::lscorr_smem_float2<R3>() * sizeof(float2), c->stream>>>(p)));
    }
    return check_launch("lscorr_fft_kernel");
}

// (T + reg I) w = rhs for nf frames from the lag sums in c->partial: taps -> taps [nf][M], status -> status [nf].
// thr: threads of a levinson_kernel<1> CTA (M <= 1024); 0: one thread per unknown (a CTA of 1024 threads would own a
// whole SM's registers and could not share it with the other slots' transform CTAs; the recursion only ever uses
// ceil(M / 32) warps)
int levinson_launch(Ctx* c, int nchunk, int HT, int M, double reg, int nf, float2* taps, int* status, int thr = 0) {
    LevinsonParams lp{};
    lp.partial = c->partial.as<float2>();
    lp.nchunk = nchunk; lp.HT = HT; lp.M = M; lp.reg = reg;
    lp.taps = taps; lp.status = status;
    {
        ProfScope ps(c, K_LEVINSON);
        if (!thr) thr = std::max(64, (M + 31) & ~31);
        if (M <= 1024) levinson_kernel<1><<<nf, thr, levinson_smem(M, thr), c->stream>>>(lp);
        else levinson_kernel<4><<<nf, 512, levinson_smem(M, 512), c->stream>>>(lp);
    }
    return check_launch("levinson_kernel");
}

// W' of c->lstaps (from frame f0 on) for transform length 256 r3 -> wp [nf][L]
int taps_spectrum(Ctx* c, int r3, int M, int nf, DBuf* wp, int f0 = 0) {
    const float2* tw;
    TRY(fft_twiddles(c, r3, &tw));
    TRY(wp->ensure((size_t)nf * 256 * r3 * sizeof(float2)));
    fftc::TapSpecParams p{};
    p.taps = c->lstaps.as<float2>() + (size_t)f0 * M; p.M = M; p.wp = wp->as<float2>(); p.tw = tw;
    {
        ProfScope ps(c, K_MISC);
        PRC_R3_SWITCH(r3, (fftc::taps_spectrum_kernel<R3><<<nf, 16 * R3, fft_smem(R3), c->stream>>>(p)));
    }
    return check_launch("taps_spectrum_kernel");
}

// out = srv - FIR(ref, c->lstaps from frame f0 on) by overlap-save (circular, or zero-extended when linear)
int fir_fft(Ctx* c, int r3, const float2* ref, const float2* srv, float2* out, long long n, Batch bt, int M, int peek,
            bool linear, int f0 = 0) {
    const float2* tw;
    TRY(fft_twiddles(c, r3, &tw));
    TRY(taps_spectrum(c, r3, M, bt.nf, &c->wp_fir, f0));
    const int L = 256 * r3;
    fftc::FirFftParams p{};
    p.ref = ref; p.srv = srv; p.out = out; p.frame_stride = bt.stride;
    p.wp = c->wp_fir.as<float2>();
    p.n = (int)n; p.M = M; p.peek = peek; p.linear = linear ? 1 : 0;
    p.nseg = ceil_div(n, L - M + 1);
    p.tw = tw;
    // one wave of CTAs for the whole batch (R3 = 8: 3 resident per SM, 68 KB of shared memory each)
    const long long slots = (long long)fft_ctas_per_sm(c, FK_FIR, r3) * c->nsm;
    const int per_frame = (int)std::max<long long>(1, std::min<long long>(p.nseg, slots / bt.nf));
    {
        ProfScope ps(c, K_FIR);
        PRC_R3_SWITCH(r3, (fftc::fir_fft_kernel<R3><<<dim3(per_frame, bt.nf), 16 * R3, fftc::fir_smem_float2<R3>() * sizeof(float2), c->stream>>>(p)));
    }
    return check_launch("fir_fft_kernel");
}

// ---- CAF block sums
int decimator_offset(long long ntaps, long long D) {   // resample_poly alignment, up = 1
    const long long half = (ntaps - 1) / 2;
    const long long pre_pad = D - half % D;
    const long long pre_remove = (half + pre_pad) / D;
    return (int)(pre_remove * D - pre_pad);
}

// fast_xambg's decimator: factor D = int(n / F) and ntaps taps (taps: device float32; NULL: a boxcar of D + 1, or no
// filter at all when D = 1).  Doppler block j covers samples j D + c0 - (ntaps - 1) .. j D + c0.
struct Decimator {
    long long D, ntaps;
    int c0;
    const float* taps;
    bool boxcar() const { return taps == nullptr && ntaps == D + 1; }
};

// dtaps32: the tap-weighted decimator (ndtaps taps), or NULL.  No checks: D < 1 is the callers' to refuse.
Decimator decimator(long long n, int F, const float* dtaps32, long long ndtaps) {
    Decimator d{n / F, 1, 0, nullptr};
    if (d.D <= 1) return d;   // resample_poly(x, 1, 1) returns x (scipy _signaltools.py:4028)
    d.ntaps = dtaps32 ? ndtaps : d.D + 1;
    d.c0 = decimator_offset(d.ntaps, d.D);
    d.taps = dtaps32;
    return d;
}

struct CafFftPlan {
    bool on = false;
    int r3 = 8, Bmax = 0, HT = 0;
};

// mfuse: taps of the clutter filter fused into the surveillance operand (0: none)
CafFftPlan caf_fft_plan(long long n, int R, int F, const Decimator& dm, int mfuse) {
    CafFftPlan pl;
    const long long ntaps = dm.ntaps;
    std::call_once(g_env_once, read_env);
    if (!g_fft.load() || n < g_fft_min_n.load() || !dm.boxcar() || dm.D < 32 || F < 1) return pl;
    double best = 0.0;
    for (int r3 : {4, 8, 16}) {
        const int L = 256 * r3;
        const long long bmax = (long long)L - R - std::max(mfuse - 1, 0);
        if (bmax < L / 4 || n < L) continue;
        const long long nseg = (ntaps + bmax - 1) / bmax;
        const double cost = (double)(nseg * (mfuse ? 3 : 2) + 1) * L * ilog2(L);
        if (!pl.on || cost < best) {
            pl.on = true; pl.r3 = r3; pl.Bmax = (int)bmax; best = cost;
        }
    }
    pl.HT = (R + 2) & ~1;
    return pl;
}

// P[frame][j][d] -> c->fftP; wp == nullptr: plain CAF of (ref, srv); else srv is cleaned on the fly with the taps
// spectrum wp ([nf][L], same r3)
int caf_fft(Ctx* c, const CafFftPlan& pl, const float2* ref, const float2* srv, long long n, Batch bt, int R, int F,
            const float* win32, const Decimator& dm, const float2* wp, int M, int peek) {
    const float2* tw;
    TRY(fft_twiddles(c, pl.r3, &tw));
    TRY(c->fftP.ensure((size_t)bt.nf * F * pl.HT * sizeof(float2)));
    fftc::CafFftParams p{};
    p.ref = ref; p.srv = srv; p.frame_stride = bt.stride; p.win = win32; p.wp = wp;
    p.n = (int)n; p.R = R; p.F = F; p.M = M; p.peek = peek;
    p.D = dm.D; p.c0 = dm.c0; p.ntaps = (int)dm.ntaps; p.Bmax = pl.Bmax;
    p.P = c->fftP.as<float2>(); p.HT = pl.HT; p.tw = tw;
    const dim3 grid(F, bt.nf);
    {
        ProfScope ps(c, K_LAGCORR_CAF);
        if (wp) { PRC_R3_SWITCH(pl.r3, (fftc::caf_fft_kernel<R3, true><<<grid, 16 * R3, fftc::caf_smem_float2<R3>() * sizeof(float2), c->stream>>>(p))); }
        else { PRC_R3_SWITCH(pl.r3, (fftc::caf_fft_kernel<R3, false><<<grid, 16 * R3, fftc::caf_smem_float2<R3>() * sizeof(float2), c->stream>>>(p))); }
    }
    return check_launch("caf_fft_kernel");
}

// --------------------------------------------------------------------------- device pipelines
// All pointers are device pointers; everything is enqueued on c->stream.

// The CAF's block sums as the Doppler stage reads them: [nf][F][nchunk][HT] at src.  per_cta > 0: the lagstream
// layout, block j holds stream_pieces(j, blk_len, per_cta) of its nchunk rows; 0: all nchunk rows.
struct BlockSums {
    const float2* src;
    int nchunk, HT, blk_len;
    long long per_cta;
};

// Doppler stage: the block sums of nf frames -> out [nf][F][R + 1]
int doppler_stage(Ctx* c, const BlockSums& bs, int R, int F, int nf, float2* out) {
    if (c->tw_F != F) {
        TRY(c->tw.ensure((size_t)F * sizeof(float2)));
        twiddle_kernel<<<ceil_div(F, 256), 256, 0, c->stream>>>(c->tw.as<float2>(), F);
        TRY(check_launch("twiddle_kernel"));
        c->tw_F = F;
    }
    DopplerParams d{};
    d.partial = bs.src;
    d.tw = c->tw.as<float2>();
    d.out = out;
    d.F = F; d.R = R; d.nchunk = bs.nchunk; d.HT = bs.HT;
    d.partial_fstride = (long long)F * bs.nchunk * bs.HT;
    d.out_fstride = (long long)F * (R + 1);
    d.blk_len = bs.blk_len; d.per_cta = bs.per_cta;
    int logF = 0;
    while ((1 << logF) < F) ++logF;
    d.logF = logF;
    const bool pow2 = (1 << logF) == F && F >= 2;
    ProfScope ps_doppler(c, K_DOPPLER);
    if (pow2 && F <= 8192) {
        if (F <= 1024 && (long long)ceil_div(R + 1, 8) * nf >= c->nsm) {
            const size_t sm = (size_t)2 * F * 8 * sizeof(float2);
            doppler_fft_pow2_kernel<8><<<dim3(ceil_div(R + 1, 8), nf), 256, sm, c->stream>>>(d);
        } else if (F <= 4096) {     // also the small-grid case: 2 columns per CTA fill more SMs
            const size_t sm = (size_t)2 * F * 2 * sizeof(float2);
            doppler_fft_pow2_kernel<2><<<dim3(ceil_div(R + 1, 2), nf), 256, sm, c->stream>>>(d);
        } else {
            const size_t sm = (size_t)2 * F * sizeof(float2);
            doppler_fft_pow2_kernel<1><<<dim3(R + 1, nf), 256, sm, c->stream>>>(d);
        }
        TRY(check_launch("doppler_fft_pow2_kernel"));
    } else {
        TRY(c->pbuf.ensure((size_t)F * (R + 1) * sizeof(float2)));
        for (int fr = 0; fr < nf; ++fr) {      // any F: chunk sum + direct DFT, frame by frame
            chunk_sum_kernel<<<ceil_div((long long)F * (R + 1), 256), 256, 0, c->stream>>>(
                d.partial + (size_t)fr * d.partial_fstride, c->pbuf.as<float2>(), F, R, bs.nchunk, bs.HT, bs.blk_len, bs.per_cta, d);
            TRY(check_launch("chunk_sum_kernel"));
            doppler_dft_kernel<<<dim3(ceil_div(R + 1, 128), F), 128, 0, c->stream>>>(
                c->pbuf.as<float2>(), c->tw.as<float2>(), out + (size_t)fr * d.out_fstride, F, R);
            TRY(check_launch("doppler_dft_kernel"));
        }
    }
    return PRC_OK;
}

// bt.nf > 1 (a batch of frames) and fuse_wp != nullptr (clutter filter applied inside the CAF kernel, taps spectrum
// [nf][L] for the transform length of caf_fft_plan(..., fuse_M)) exist on the FFT-domain path only
int xambg_device(Ctx* c, const float2* ref, const float2* srv, long long n, int R, int F,
                 const float* win32, const float* dtaps32, long long ndtaps, float2* out, Batch bt = Batch{},
                 const float2* fuse_wp = nullptr, int fuse_M = 0, int fuse_peek = 0) {
    if (n <= 0 || n >= (1ll << 31) - 4096) return fail(PRC_E_INVALID, "n=%lld unsupported", n);
    if (F < 1 || R < 0) return fail(PRC_E_INVALID, "freq_bins=%d / range_bins=%d invalid", F, R);
    const Decimator dm = decimator(n, F, dtaps32, ndtaps);
    if (dm.D < 1) return fail(PRC_E_INVALID, "decimation factor int(n/freq_bins) is 0 (n=%lld, freq_bins=%d)", n, F);
    if (dm.ntaps > (1ll << 30)) return fail(PRC_E_INVALID, "decimator too long");
    const int ntaps = (int)dm.ntaps;
    const CafFftPlan fp = caf_fft_plan(n, R, F, dm, fuse_wp ? fuse_M : 0);
    if ((bt.nf > 1 || fuse_wp) && !fp.on)
        return fail(PRC_E_INVALID, "batched / fused CAF needs the FFT-domain path (n=%lld, F=%d, R=%d not eligible)", n, F, R);
    BlockSums bs;
    if (fp.on) {
        // ---- FFT-domain block correlations (fftcorr.cuh): one CTA per Doppler block, P[j][d] straight from the channels
        TRY(caf_fft(c, fp, ref, srv, n, bt, R, F, win32, dm, fuse_wp, fuse_M, fuse_peek));
        bs = {c->fftP.as<float2>(), 1, fp.HT, ntaps, 0};
    } else if (dm.taps == nullptr && ntaps >= 64) {   // tiny Doppler blocks: one flush per block would dominate
        StreamGeo sg;
        TRY(choose_stream(ntaps, F, 1, R + 1, c->nsm, &sg));
        TRY(c->partial.ensure((size_t)F * sg.sp.maxpieces * sg.HT * sizeof(float2)));
        const float2* xw = ref;
        if (win32) {
            TRY(c->refw.ensure((size_t)n * sizeof(float2)));
            {
                ProfScope ps(c, K_MISC);
                weight_kernel<<<ceil_div(n, 256), 256, 0, c->stream>>>(ref, win32, c->refw.as<float2>(), (int)n);
            }
            TRY(check_launch("weight_kernel"));
            xw = c->refw.as<float2>();
        }
        LagStreamParams sp = sg.sp;
        sp.x = xw;
        sp.s[0] = srv; sp.s[1] = srv;
        sp.n = (int)n;
        sp.blk_first_lo = (long long)dm.c0 - (ntaps - 1);
        sp.blk_stride = dm.D;
        sp.partial = c->partial.as<float2>();
        {
            ProfScope ps(c, K_LAGCORR_CAF);
            launch_lagstream(dim3(sg.ncta, 1), sg.threads, sg.smem, c->stream, sp);
        }
        TRY(check_launch("lagstream_kernel(caf)"));
        bs = {c->partial.as<float2>(), sp.maxpieces, sg.HT, ntaps, sp.per_cta};
    } else {
        Geo g{};
        TRY(choose_geo(ntaps, F, R + 1, c->nsm, &g));
        TRY(c->partial.ensure((size_t)F * g.nchunk * g.HT * sizeof(float2)));
        LagCorrParams p{};
        p.x = ref;
        p.s[0] = srv; p.s[1] = srv;
        p.dmin[0] = 0; p.dmin[1] = 0;
        p.win = win32;
        p.taps = dm.taps;
        p.n = (int)n;
        p.blk_first_lo = (long long)dm.c0 - (ntaps - 1);
        p.blk_stride = dm.D;
        p.blk_len = ntaps;
        p.nblk = F;
        p.nchunk = g.nchunk;
        p.chunk_len = g.chunk_len;
        p.H = g.H; p.G = g.G; p.steps = g.steps;
        p.partial = c->partial.as<float2>();
        {
            ProfScope ps(c, K_LAGCORR_CAF);
            const dim3 grid((unsigned)((long long)F * g.nchunk), 1);
            lagcorr_kernel<TILE_I, TILE_D><<<grid, g.threads, g.smem, c->stream>>>(p);
        }
        TRY(check_launch("lagcorr_kernel(caf)"));
        bs = {c->partial.as<float2>(), g.nchunk, g.HT, ntaps, 0};
    }
    return doppler_stage(c, bs, R, F, bt.nf, out);
}

// bt.nf > 1 (a batch of frames; taps_out then receives [nf][M]) and out == nullptr (only the taps are wanted: the
// caller applies them inside the CAF kernel) exist on the FFT-domain path only.  status_at: the int of c->status the
// direct-form solve reports to.
int ls_device(Ctx* c, const float2* ref, const float2* srv, long long n, int filter_len, int peek,
              double reg, float2* out, float2* taps_out, bool linear = false, Batch bt = Batch{}, int status_at = 0) {
    // linear: LS_Filter_Toeplitz semantics -- correlations and FIR treat ref/srv as zero outside [0, n)
    if (n <= 0 || n >= (1ll << 31) - 4096) return fail(PRC_E_INVALID, "n=%lld unsupported", n);
    if (filter_len < 0 || peek < 0 || filter_len + peek < 1)
        return fail(PRC_E_INVALID, "filter_len=%d peek=%d invalid", filter_len, peek);
    const int M = filter_len + peek;
    if (M > 2048) return fail(PRC_E_INVALID, "%d taps exceed the Toeplitz solver's maximum of 2048", M);
    const LsFftPlan lf = ls_fft_plan(c, n, M, bt.nf);
    if ((bt.nf > 1 || !out) && !lf.on)
        return fail(PRC_E_INVALID, "batched LS filter needs the FFT-domain path (n=%lld, %d taps not eligible)", n, M);
    if (lf.on) {
        // ---- FFT-domain path (fftcorr.cuh): block spectra -> lag sums -> float64 Toeplitz solve -> overlap-save FIR
        TRY(ls_fft_corr(c, lf, ref, srv, n, bt, M, peek, linear));
        TRY(c->lstaps.ensure((size_t)bt.nf * M * sizeof(float2)));
        TRY(c->status.ensure((size_t)bt.nf * sizeof(int)));
        TRY(levinson_launch(c, lf.ncta, lf.HT, M, reg, bt.nf, c->lstaps.as<float2>(), c->status.as<int>()));
        if (out) TRY(fir_fft(c, lf.r3, ref, srv, out, n, bt, M, peek, linear));
        if (taps_out)
            CU(cudaMemcpyAsync(taps_out, c->lstaps.p, (size_t)bt.nf * M * sizeof(float2), cudaMemcpyDeviceToDevice, c->stream));
        return PRC_OK;
    }
    TRY(c->lstaps.ensure((size_t)M * sizeof(float2)));
    TRY(c->status.ensure((size_t)(status_at + 1) * sizeof(int)));
    StreamGeo sg;
    TRY(choose_stream((int)n, 1, 2, M, c->nsm, &sg));
    TRY(c->partial.ensure((size_t)2 * sg.sp.maxpieces * sg.HT * sizeof(float2)));
    LagStreamParams sp = sg.sp;
    sp.x = ref;
    sp.s[0] = ref; sp.s[1] = srv;
    sp.dmin[1] = -peek;
    sp.n = (int)n;
    sp.s_linear = linear ? 1 : 0;
    sp.partial = c->partial.as<float2>();
    {
        ProfScope ps(c, K_LAGCORR_LS);
        launch_lagstream(dim3(sg.ncta, 2), sg.threads, sg.smem, c->stream, sp);
    }
    TRY(check_launch("lagstream_kernel(ls)"));
    // one CTA; its chunks are the pieces of the single block (== ncta)
    TRY(levinson_launch(c, sp.maxpieces, sg.HT, M, reg, 1, c->lstaps.as<float2>(), c->status.as<int>() + status_at, 1024));

    FirParams fp{};
    fp.ref = ref; fp.srv = srv; fp.taps = c->lstaps.as<float2>(); fp.out = out;
    fp.n = (int)n; fp.M = M; fp.peek = peek;
    fp.linear = linear ? 1 : 0;
    fp.Mpad = ceil_div(M, TILE_I) * TILE_I;
    if (fp.Mpad & 1) fp.Mpad += TILE_I;      // keep the ref window 16-byte aligned behind the taps
    const int LO = FIR_THREADS * TILE_D;
    const size_t sm = (size_t)(fp.Mpad + LO + fp.Mpad) * sizeof(float2);
    if (sm > SMEM_LIMIT) return fail(PRC_E_INVALID, "%d taps exceed the FIR kernel's shared memory", M);
    {
        ProfScope ps(c, K_FIR);
        fir_apply_kernel<TILE_I, TILE_D><<<ceil_div(n, LO), FIR_THREADS, sm, c->stream>>>(fp);
    }
    TRY(check_launch("fir_apply_kernel"));
    if (taps_out)
        CU(cudaMemcpyAsync(taps_out, c->lstaps.p, (size_t)M * sizeof(float2), cudaMemcpyDeviceToDevice, c->stream));
    return PRC_OK;
}

// LS_Filter_Toeplitz (reference clutter_removal.py:109-160) on the device: roll (and optionally
// frequency-shift) the reference, then the LS pipeline in linear mode with reg = 0 and all
// filterLen + peek taps causal on the rolled reference.
// bt.nf > 1: a batch of frames, every buffer (ref, srv, out, the rolled reference) bt.stride samples apart (FFT-domain path)
int ls_toeplitz_device(Ctx* c, const float2* ref, const float2* srv, long long n, int filter_len, int peek,
                       bool shift, double fc, double fs, float2* out, float2* taps_out, Batch bt = Batch{}) {
    if (n <= 0 || n >= (1ll << 31) - 4096) return fail(PRC_E_INVALID, "n=%lld unsupported", n);
    if (filter_len < 0 || peek < 0 || filter_len + peek < 1)
        return fail(PRC_E_INVALID, "filter_len=%d peek=%d invalid", filter_len, peek);
    const long long stride = bt.nf > 1 ? bt.stride : n;
    TRY(c->rs.ensure(((size_t)(bt.nf - 1) * stride + n) * sizeof(float2)));
    // complex64(1j*2*pi*fc) * complex64(n) / Fs, evaluated like numpy does (see shift_roll_kernel)
    const float B = (float)(2.0 * 3.14159265358979323846 * fc);
    {
        ProfScope ps(c, K_MISC);
        shift_roll_kernel<<<dim3(ceil_div(n, 256), bt.nf), 256, 0, c->stream>>>(ref, c->rs.as<float2>(), (int)n, peek, shift ? 1 : 0, B,
                                                                                 1.0f / (float)fs, stride);
    }
    TRY(check_launch("shift_roll_kernel"));
    return ls_device(c, c->rs.as<float2>(), srv, n, filter_len + peek, 0, 0.0, out, taps_out, true, bt);
}

// ---- direct_xambg (reference range_doppler_processing.py:93-124) ---------------------------------
// row f: xcorr(frequency_shift(ref, (f - F/2)/CPI, Fs), srv, R, 0): a LINEAR lag correlation of the
// frequency-shifted reference (float32 phase ramp, complex64 exp -- as the reference) with srv.
int direct_xambg_device(Ctx* c, const float2* ref, const float2* srv, long long n, int R, int F, double fs, float2* out) {
    if (n <= 0 || n >= (1ll << 31) - 4096) return fail(PRC_E_INVALID, "n=%lld unsupported", n);
    if (R < 0 || F < 1) return fail(PRC_E_INVALID, "range_bins=%d freq_bins=%d invalid", R, F);
    if (!(fs > 0)) return fail(PRC_E_INVALID, "sample_rate must be > 0");
    TRY(c->rs.ensure((size_t)n * sizeof(float2)));
    StreamGeo sg;
    TRY(choose_stream((int)n, 1, 1, R + 1, c->nsm, &sg));
    TRY(c->partial.ensure((size_t)sg.sp.maxpieces * sg.HT * sizeof(float2)));
    const double cpi = (double)n / fs;
    for (int f = 0; f < F; ++f) {
        const double df = ((double)f - 0.5 * (double)F) / cpi;
        TRY(frequency_shift_device(c, ref, n, df, fs, c->rs.as<float2>()));
        LagStreamParams sp = sg.sp;
        sp.x = c->rs.as<float2>();
        sp.s[0] = srv; sp.s[1] = srv;
        sp.n = (int)n;
        sp.s_linear = 1;
        sp.partial = c->partial.as<float2>();
        {
            ProfScope ps(c, K_LAGCORR_CAF);
            launch_lagstream(dim3(sg.ncta, 1), sg.threads, sg.smem, c->stream, sp);
            piece_sum_kernel<<<ceil_div(R + 1, 128), 128, 0, c->stream>>>(c->partial.as<float2>(), sp.maxpieces, sg.HT, R,
                                                                     out + (size_t)f * (R + 1));
        }
        TRY(check_launch("lagstream_kernel(direct_xambg)"));
    }
    return PRC_OK;
}

// window (host or device, double or float) -> device float
int stage_window(Ctx* c, const void* window, long long n, int mem_kind, unsigned flags, const float** win32) {
    *win32 = nullptr;
    if (!window) return PRC_OK;
    if (flags & PRC_FLAG_WINDOW_F32)
        return stage_in(c, window, mem_kind, 1, (size_t)n * sizeof(float), (size_t)n * sizeof(float), c->win32, flags, win32);
    const double* w64;
    TRY(stage_in(c, window, mem_kind, 1, (size_t)n * sizeof(double), (size_t)n * sizeof(double), c->win64, flags, &w64));
    TRY(c->win32.ensure((size_t)n * sizeof(float)));
    f64_to_f32_kernel<<<ceil_div(n, 256), 256, 0, c->stream>>>(w64, c->win32.as<float>(), n);
    TRY(check_launch("f64_to_f32_kernel"));
    *win32 = c->win32.as<float>();
    return PRC_OK;
}

int check_ls_status(Ctx* c, unsigned flags, int nf = 1) {
    if (flags & PRC_FLAG_ASYNC) return PRC_OK;   // caller owns the synchronisation; status stays on the device (prc_ls_status)
    std::vector<int> st((size_t)nf, 0);
    CU(cudaMemcpyAsync(st.data(), c->status.p, (size_t)nf * sizeof(int), cudaMemcpyDeviceToHost, /*status*/ c->stream));
    CU(cudaStreamSynchronize(c->stream));
    for (int i = 0; i < nf; ++i)
        if (st[i] != 0)
            return fail(PRC_E_SINGULAR, "LS normal equations are not positive definite (singular Gram matrix, frame %d)", i);
    return PRC_OK;
}

// ---- one-pass FFT-domain frame (framepass.cuh): LS lag sums and the CAF's per-block spectra AccP, AccQ from one set
// of window transforms, then the Toeplitz solve, W', and AccP - AccQ conj(W') per block
struct OnePassPlan {
    bool on = false;
    int Bmax = 0, ntail = 0, Bt = 0;
    long long tail_lo = 0;
    Decimator dm{};
};

// AccP / AccQ spectra of one chunk of frames: 2 L complex64 per Doppler block and frame (8 MiB per frame at 256 blocks
// of L = 2048); larger batches run in chunks of frames that fit
constexpr size_t FP_ACC_CAP = 256u << 20;

// Taken when both FFT-domain plans are on, the clutter filter has at least one tap before peek (so Yr' starts at or
// before Ys'), the segment limit of both the LS lags and the CAF lags at L = 2048 is at least L / 4, and the transform
// count x L log L is below that of the two passes (lscorr_fft_kernel + caf_fft_kernel<FUSED>).  Otherwise off, and the
// frame runs exactly as before.
OnePassPlan onepass_plan(const LsFftPlan& lf, const CafFftPlan& cf, long long n, int filter_len, int peek, int R, int F,
                         const Decimator& dm) {
    OnePassPlan op;
    if (!g_frame_onepass.load() || !lf.on || !cf.on || filter_len < 1) return op;
    const int M = filter_len + peek;
    const long long L = 256 * fftc::FP_R3;
    const long long bls = L - 2ll * M + 2;                       // lags M-1 .. 2M-2 of X_ls conj(Yr')
    const long long bmax = std::min(bls, L - M - R - peek + 1);  // CAF lags peek .. R + peek of the cleaned window
    if (bmax < L / 4 || n < L) return op;
    const long long D = dm.D, ntaps = dm.ntaps;
    const int c0 = dm.c0;
    if (c0 - (ntaps - 1) > 0) return op;                         // samples before the first block: not a layout we run
    op.tail_lo = std::min((long long)(F - 1) * D + c0 + 1, n);
    const long long tail = n - op.tail_lo;
    op.ntail = (int)((tail + bls - 1) / bls);
    op.Bt = op.ntail ? (int)((tail + op.ntail - 1) / op.ntail) : 0;
    double one = 3.0 * op.ntail, two_caf = 0.0;
    for (int j = 0; j < F; ++j) {
        const long long lo = std::max((long long)j * D + c0 - (ntaps - 1), 0ll), hi = std::min((long long)j * D + c0 + 1, n);
        const long long len = std::max(hi - lo, 0ll);
        one += 4.0 * ((len + bmax - 1) / bmax) + 1.0;            // + the combine's transform
        two_caf += 3.0 * ((len + cf.Bmax - 1) / cf.Bmax) + 1.0;
    }
    const double one_cost = one * L * ilog2((int)L);
    const double two_cost = 3.0 * lf.nseg * (256.0 * lf.r3) * ilog2(256 * lf.r3) + two_caf * (256.0 * cf.r3) * ilog2(256 * cf.r3);
    if (one_cost >= two_cost) return op;
    op.on = true;
    op.Bmax = (int)bmax;
    op.dm = dm;
    return op;
}

int frame_onepass(Ctx* c, const OnePassPlan& op, const float2* ref, const float2* srv, long long n, Batch bt, int filter_len,
                  int peek, double reg, int R, int F, const float* win32, float2* maps, float2* taps_out, float2* cleaned_out) {
    if (n >= (1ll << 31) - 4096) return fail(PRC_E_INVALID, "n=%lld unsupported", n);
    if (op.dm.ntaps > (1ll << 30)) return fail(PRC_E_INVALID, "decimator too long");   // as fast_xambg refuses it
    constexpr int R3 = fftc::FP_R3;
    constexpr int L = 256 * R3;
    const int M = filter_len + peek;
    const float2* tw;
    TRY(fft_twiddles(c, R3, &tw));
    const size_t per_frame = (size_t)F * 2 * L * sizeof(float2);
    const int chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)bt.nf, FP_ACC_CAP / per_frame));
    const int HT = (M + 1) & ~1, HTc = (R + 2) & ~1;
    TRY(c->fpacc.ensure(per_frame * chunk));
    TRY(c->lstaps.ensure((size_t)bt.nf * M * sizeof(float2)));
    TRY(c->status.ensure((size_t)bt.nf * sizeof(int)));
    TRY(c->fftP.ensure((size_t)chunk * F * HTc * sizeof(float2)));
    const int units = F + op.ntail;
    for (int f0 = 0; f0 < bt.nf; f0 += chunk) {
        const int nf = std::min(chunk, bt.nf - f0);
        const Batch b{nf, bt.stride};
        const float2* r = ref + (size_t)f0 * bt.stride;
        const float2* s = srv + (size_t)f0 * bt.stride;
        // one wave of CTAs (two per SM), each walking a run of Doppler blocks (and tail segments) of its frame
        const long long slots = (long long)fft_ctas_per_sm(c, FK_FRAME, R3) * c->nsm;
        const int ncta = (int)std::max<long long>(1, std::min<long long>(units, slots / nf));
        TRY(c->partial.ensure((size_t)nf * 2 * ncta * HT * sizeof(float2)));
        fftc::FramePassParams p{};
        p.ref = r; p.srv = s; p.frame_stride = bt.stride; p.win = win32;
        p.n = (int)n; p.M = M; p.peek = peek; p.F = F;
        p.D = op.dm.D; p.c0 = op.dm.c0; p.ntaps = (int)op.dm.ntaps; p.Bmax = op.Bmax;
        p.tail_lo = (int)op.tail_lo; p.ntail = op.ntail; p.Bt = op.Bt;
        p.acc = c->fpacc.as<float2>(); p.partial = c->partial.as<float2>(); p.HT = HT; p.tw = tw;
        {
            ProfScope ps(c, K_LAGCORR_CAF);
            fftc::launch_frame_pass(p, ncta, nf, c->stream);
        }
        TRY(check_launch("frame_pass_kernel"));
        TRY(levinson_launch(c, ncta, HT, M, reg, nf, c->lstaps.as<float2>() + (size_t)f0 * M, c->status.as<int>() + f0));
        TRY(taps_spectrum(c, R3, M, nf, &c->wp_caf, f0));
        if (cleaned_out) TRY(fir_fft(c, R3, r, s, cleaned_out + (size_t)f0 * bt.stride, n, b, M, peek, false, f0));
        fftc::CafCombineParams q{};
        q.acc = c->fpacc.as<float2>(); q.wp = c->wp_caf.as<float2>();
        q.F = F; q.R = R; q.peek = peek;
        q.P = c->fftP.as<float2>(); q.HT = HTc; q.tw = tw;
        const long long cslots = (long long)fft_ctas_per_sm(c, FK_COMBINE, R3) * c->nsm;
        const int gc = (int)std::max<long long>(1, std::min<long long>(F, cslots / nf));
        {
            ProfScope ps(c, K_CAF_COMBINE);
            fftc::launch_caf_combine(q, gc, nf, c->stream);
        }
        TRY(check_launch("caf_combine_kernel"));
        TRY(doppler_stage(c, BlockSums{c->fftP.as<float2>(), 1, HTc, (int)op.dm.ntaps, 0}, R, F, nf, maps + (size_t)f0 * F * (R + 1)));
    }
    if (taps_out)
        CU(cudaMemcpyAsync(taps_out, c->lstaps.p, (size_t)bt.nf * M * sizeof(float2), cudaMemcpyDeviceToDevice, c->stream));
    return PRC_OK;
}

// The paths of one call of the frame: FFT-domain LS and CAF (the latter with the clutter filter fused), and the one-pass
// frame that replaces the two.  fft(): the batched FFT-domain frame runs; otherwise the direct-form kernels, frame by
// frame.
struct FramePlan {
    LsFftPlan ls;
    CafFftPlan caf;
    OnePassPlan one;
    bool fft() const { return ls.on && caf.on; }
};

FramePlan frame_plan(Ctx* c, long long n, int nf, int filter_len, int peek, int R, int F) {
    const int M = filter_len + peek;
    const Decimator dm = decimator(n, F, nullptr, 0);
    FramePlan fp;
    fp.ls = ls_fft_plan(c, n, M, nf);
    fp.caf = caf_fft_plan(n, R, F, dm, M);
    fp.one = onepass_plan(fp.ls, fp.caf, n, filter_len, peek, R, F, dm);
    return fp;
}

// one frame (or, on the FFT-domain path, a batch of frames) of  LS_Filter -> fast_xambg  on device pointers
int frame_device(Ctx* c, const FramePlan& fp, const float2* ref, const float2* srv, long long n, Batch bt, int filter_len,
                 int peek, double reg, int R, int F, const float* win32, float2* maps, float2* taps_out, float2* cleaned_out) {
    const int M = filter_len + peek;
    if (fp.one.on)
        return frame_onepass(c, fp.one, ref, srv, n, bt, filter_len, peek, reg, R, F, win32, maps, taps_out, cleaned_out);
    if (fp.fft()) {
        // FFT-domain frame: lag sums -> Toeplitz solve -> taps spectrum -> CAF with the clutter filter applied to the
        // surveillance spectrum inside the kernel (the cleaned channel exists only if the caller asks for it)
        TRY(ls_device(c, ref, srv, n, filter_len, peek, reg, cleaned_out, taps_out, false, bt));
        TRY(taps_spectrum(c, fp.caf.r3, M, bt.nf, &c->wp_caf));
        return xambg_device(c, ref, srv, n, R, F, win32, nullptr, 0, maps, bt, c->wp_caf.as<float2>(), M, peek);
    }
    // FP32 direct-form kernels, frame by frame; frame fr reports its Toeplitz-solve status in status[fr]
    TRY(c->clean.ensure((size_t)n * sizeof(float2)));
    TRY(c->status.ensure((size_t)bt.nf * sizeof(int)));
    for (int fr = 0; fr < bt.nf; ++fr) {
        const float2* r = ref + (size_t)fr * bt.stride;
        const float2* sv = srv + (size_t)fr * bt.stride;
        float2* dclean = cleaned_out ? cleaned_out + (size_t)fr * bt.stride : c->clean.as<float2>();
        TRY(ls_device(c, r, sv, n, filter_len, peek, reg, dclean, taps_out ? taps_out + (size_t)fr * M : nullptr, false,
                      Batch{}, fr));
        TRY(xambg_device(c, r, dclean, n, R, F, win32, nullptr, 0, maps + (size_t)fr * F * (R + 1)));
    }
    return PRC_OK;
}

// ---- several surveillance channels against one reference (framemulti.cuh)
// The shared pass runs where the one-pass plan is on and at least this many channels share the reference: the
// smallest K at which scripts/multichannel_bench.py measured it faster than K one-pass frames (DESIGN.md section 20)
constexpr int FM_MIN_SHARED_K = 2;

// nchan = K shared-reference frames of one chunk after another: the one-pass plan's partition, one frame_multi_pass
// launch, then levinson_launch, taps_spectrum and caf_combine_multi on K nf problems ([k][f] within the chunk) and the
// Doppler stage channel by channel.  The CTAs of a frame walk its units exactly as frame_onepass's do for the same
// frames per launch, so each channel is bit for bit prc_frames_c64(ref, srv_k) when the batch fits one chunk of both.
int frames_shared(Ctx* c, const OnePassPlan& op, const float2* ref, const float2* srv, long long n, Batch bt, int K,
                  long long chan_stride, int filter_len, int peek, double reg, int R, int F, const float* win32,
                  float2* maps, float2* taps_out) {
    if (n >= (1ll << 31) - 4096) return fail(PRC_E_INVALID, "n=%lld unsupported", n);
    if (op.dm.ntaps > (1ll << 30)) return fail(PRC_E_INVALID, "decimator too long");
    constexpr int R3 = fftc::FP_R3;
    constexpr int L = 256 * R3;
    const int M = filter_len + peek;
    const float2* tw;
    TRY(fft_twiddles(c, R3, &tw));
    const size_t per_frame = (size_t)(1 + K) * F * L * sizeof(float2);
    const int chunk = (int)std::max<size_t>(1, std::min<size_t>((size_t)bt.nf, FP_ACC_CAP / per_frame));
    const int HT = (M + 1) & ~1, HTc = (R + 2) & ~1;
    const size_t map_elems = (size_t)F * (R + 1);
    TRY(c->fpacc.ensure(per_frame * chunk));
    TRY(c->lstaps.ensure((size_t)K * chunk * M * sizeof(float2)));
    TRY(c->status.ensure((size_t)K * chunk * sizeof(int)));
    TRY(c->mstatus.ensure((size_t)K * bt.nf * sizeof(int)));
    TRY(c->fftP.ensure((size_t)K * chunk * F * HTc * sizeof(float2)));
    const int units = F + op.ntail;
    for (int f0 = 0; f0 < bt.nf; f0 += chunk) {
        const int nf = std::min(chunk, bt.nf - f0);
        const int np = K * nf;
        // frame_onepass's grid for nf frames per launch (two of its CTAs per SM), so that the partitions agree
        const long long slots = (long long)fft_ctas_per_sm(c, FK_FRAME, R3) * c->nsm;
        const int ncta = (int)std::max<long long>(1, std::min<long long>(units, slots / nf));
        TRY(c->partial.ensure((size_t)np * 2 * ncta * HT * sizeof(float2)));
        fftc::FrameMultiParams p{};
        fftc::FramePassParams& b = p.fp;
        b.ref = ref + (size_t)f0 * bt.stride; b.srv = srv + (size_t)f0 * bt.stride; b.frame_stride = bt.stride;
        b.win = win32;
        b.n = (int)n; b.M = M; b.peek = peek; b.F = F;
        b.D = op.dm.D; b.c0 = op.dm.c0; b.ntaps = (int)op.dm.ntaps; b.Bmax = op.Bmax;
        b.tail_lo = (int)op.tail_lo; b.ntail = op.ntail; b.Bt = op.Bt;
        b.acc = c->fpacc.as<float2>(); b.partial = c->partial.as<float2>(); b.HT = HT; b.tw = tw;
        p.chan_stride = chan_stride;
        {
            ProfScope ps(c, K_FRAME_MULTI);
            fftc::launch_frame_multi(p, K, ncta, nf, c->stream);
        }
        TRY(check_launch("frame_multi_pass_kernel"));
        TRY(levinson_launch(c, ncta, HT, M, reg, np, c->lstaps.as<float2>(), c->status.as<int>()));
        TRY(taps_spectrum(c, R3, M, np, &c->wp_caf));
        fftc::CafCombineMultiParams q{};
        q.acc = c->fpacc.as<float2>(); q.wp = c->wp_caf.as<float2>();
        q.F = F; q.R = R; q.peek = peek; q.nf = nf; q.nchan = K;
        q.P = c->fftP.as<float2>(); q.HT = HTc; q.tw = tw;
        const long long cslots = (long long)fft_ctas_per_sm(c, FK_COMBINE, R3) * c->nsm;
        const int gc = (int)std::max<long long>(1, std::min<long long>(F, cslots / np));
        {
            ProfScope ps(c, K_CAF_COMBINE);
            fftc::launch_caf_combine_multi(q, gc, np, c->stream);
        }
        TRY(check_launch("caf_combine_multi_kernel"));
        // the Doppler stage as frame_onepass runs it on nf frames: its kernel choice depends on the frame count
        for (int k = 0; k < K; ++k)
            TRY(doppler_stage(c, BlockSums{c->fftP.as<float2>() + (size_t)k * nf * F * HTc, 1, HTc, (int)op.dm.ntaps, 0}, R, F,
                              nf, maps + ((size_t)k * bt.nf + f0) * map_elems));
        // taps and status of the chunk's [k][f] problems -> [k][frame]
        if (taps_out)
            CU(cudaMemcpy2DAsync(taps_out + (size_t)f0 * M, (size_t)bt.nf * M * sizeof(float2), c->lstaps.p,
                                 (size_t)nf * M * sizeof(float2), (size_t)nf * M * sizeof(float2), K, cudaMemcpyDeviceToDevice,
                                 c->stream));
        CU(cudaMemcpy2DAsync(c->mstatus.as<int>() + f0, (size_t)bt.nf * sizeof(int), c->status.p, (size_t)nf * sizeof(int),
                             (size_t)nf * sizeof(int), K, cudaMemcpyDeviceToDevice, c->stream));
    }
    TRY(c->status.ensure((size_t)K * bt.nf * sizeof(int)));
    CU(cudaMemcpyAsync(c->status.p, c->mstatus.p, (size_t)K * bt.nf * sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
    return PRC_OK;
}

// nchan channels of bt.nf frames each, channel k's frames chan_stride samples after channel 0's; maps [k][frame][F][R+1],
// taps_out [k][frame][M] or NULL, status words [k][frame] in c->status.  One channel is prc_frames_c64's frame_device
// call; several take the shared pass where it pays (FM_MIN_SHARED_K) and otherwise frame_device channel by channel.
int frames_multi_device(Ctx* c, const FramePlan& fp, const float2* ref, const float2* srv, long long n, Batch bt, int nchan,
                        long long chan_stride, int filter_len, int peek, double reg, int R, int F, const float* win32,
                        float2* maps, float2* taps_out) {
    if (nchan == 1)
        return frame_device(c, fp, ref, srv, n, bt, filter_len, peek, reg, R, F, win32, maps, taps_out, nullptr);
    if (fp.one.on && nchan >= FM_MIN_SHARED_K)
        return frames_shared(c, fp.one, ref, srv, n, bt, nchan, chan_stride, filter_len, peek, reg, R, F, win32, maps, taps_out);
    const int M = filter_len + peek;
    TRY(c->mstatus.ensure((size_t)nchan * bt.nf * sizeof(int)));
    for (int k = 0; k < nchan; ++k) {
        TRY(frame_device(c, fp, ref, srv + (long long)k * chan_stride, n, bt, filter_len, peek, reg, R, F, win32,
                         maps + (size_t)k * bt.nf * F * (R + 1), taps_out ? taps_out + (size_t)k * bt.nf * M : nullptr, nullptr));
        CU(cudaMemcpyAsync(c->mstatus.as<int>() + (size_t)k * bt.nf, c->status.p, (size_t)bt.nf * sizeof(int),
                           cudaMemcpyDeviceToDevice, c->stream));
    }
    TRY(c->status.ensure((size_t)nchan * bt.nf * sizeof(int)));
    CU(cudaMemcpyAsync(c->status.p, c->mstatus.p, (size_t)nchan * bt.nf * sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
    return PRC_OK;
}

// read-only names of the residency the one-wave grids are sized from (fft_ctas_per_sm, R3 = 8 -- the transform
// length of up to 1024 LS taps and of the CAF at config 2): the FftKern they report, -1 for any other name
int fft_ctas_option(const std::string& k) {
    if (k == "fft_ctas_ls") return FK_LS;
    if (k == "fft_ctas_fir") return FK_FIR;
    if (k == "fft_ctas_frame") return FK_FRAME;
    return -1;
}

// ---- bodies the single-frame entry points share with their batched twins
// prc_xambg_c64 / prc_xambg_frames_c64 after their checks, with c locked; bt: the caller's frames.  taps32 (device,
// float32) is the tap-weighted decimator, which only the single-frame entry takes, or NULL
int xambg_entry(Ctx* c, const prc_c64* ref, const prc_c64* srv, long long n, Batch bt, int range_bins, int freq_bins,
                const void* window, const float* taps32, long long ndtaps, prc_c64* out, int mem_kind, unsigned flags) {
    const size_t nb = (size_t)n * sizeof(float2), sb = (size_t)bt.stride * sizeof(float2);
    const size_t ob = (size_t)freq_bins * (range_bins + 1) * sizeof(float2) * bt.nf;
    const float2 *dref, *dsrv;
    float2* dout;
    TRY(stage_in(c, ref, mem_kind, bt.nf, nb, sb, c->ref, flags, &dref));
    TRY(stage_in(c, srv, mem_kind, bt.nf, nb, sb, c->srv, flags, &dsrv));
    TRY(stage_out(out, mem_kind, ob, c->out, &dout));
    if (mem_kind == PRC_MEM_HOST) bt.stride = n;      // staged frames are packed
    const float* win32;
    TRY(stage_window(c, window, n, mem_kind, flags, &win32));
    if (caf_fft_plan(n, range_bins, freq_bins, decimator(n, freq_bins, taps32, ndtaps), 0).on || bt.nf == 1) {
        TRY(xambg_device(c, dref, dsrv, n, range_bins, freq_bins, win32, taps32, ndtaps, dout, bt));
    } else {
        for (int fr = 0; fr < bt.nf; ++fr)       // direct-form kernels, frame by frame
            TRY(xambg_device(c, dref + (size_t)fr * bt.stride, dsrv + (size_t)fr * bt.stride, n, range_bins, freq_bins, win32,
                             nullptr, 0, dout + (size_t)fr * freq_bins * (range_bins + 1)));
    }
    TRY(unstage(c, out, dout, mem_kind, 1, ob, ob, flags));
    return finish(c, flags);
}

// LS_Filter_Multiple's bins (prc_ls_multiple_c64 / prc_ls_multiple_frames_c64) on bt.nf frames, every buffer bt.stride
// samples apart: the last bin writes out and, when taps is given, its taps
int ls_bins(Ctx* c, const float2* ref, const float2* srv, long long n, Batch bt, int filter_len, int peek,
            double sample_rate, const double* doppler_bins, int nbins, float2* out, float2* taps, unsigned flags) {
    const size_t span = ((size_t)(bt.nf - 1) * bt.stride + n) * sizeof(float2);
    if (nbins > 1) TRY(c->clean.ensure(span));
    if (nbins > 2) TRY(c->clean2.ensure(span));
    // bins are applied one after the other on the running residual (clutter_removal.py:178-187)
    const float2* cur = srv;
    for (int b = 0; b < nbins; ++b) {
        const double fc = doppler_bins ? doppler_bins[b] : 0.0;
        const bool last = (b == nbins - 1);
        float2* dst = last ? out : (((nbins - 1 - b) & 1) ? c->clean.as<float2>() : c->clean2.as<float2>());
        TRY(ls_toeplitz_device(c, ref, cur, n, filter_len, peek, fc != 0.0, fc, sample_rate, dst, last ? taps : nullptr, bt));
        if (!(flags & PRC_FLAG_ASYNC)) TRY(check_ls_status(c, 0, bt.nf));      // singular systems are reported per bin
        cur = dst;
    }
    return PRC_OK;
}

}  // namespace prcore

using namespace prcore;

// =========================================================================== C ABI
#pragma GCC visibility push(default)
extern "C" {

int prc_xambg_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int range_bins, int freq_bins,
                  const void* window, const double* dtaps, int64_t ndtaps, prc_c64* out, int mem_kind,
                  int device, void* stream, unsigned flags) {
    Batch bt;
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, 1, n, &bt, range_bins, freq_bins));
    if (dtaps && ndtaps < 1) return fail(PRC_E_INVALID, "ndtaps=%lld invalid", (long long)ndtaps);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const float* taps32 = nullptr;
    if (dtaps) {
        const double* t64;
        TRY(stage_in(c, dtaps, mem_kind, 1, (size_t)ndtaps * sizeof(double), (size_t)ndtaps * sizeof(double), c->dtaps64,
                     flags, &t64));
        TRY(c->dtaps32.ensure((size_t)ndtaps * sizeof(float)));
        f64_to_f32_kernel<<<ceil_div(ndtaps, 256), 256, 0, c->stream>>>(t64, c->dtaps32.as<float>(), ndtaps);
        TRY(check_launch("f64_to_f32_kernel"));
        taps32 = c->dtaps32.as<float>();
    }
    return xambg_entry(c, ref, srv, n, bt, range_bins, freq_bins, window, taps32, ndtaps, out, mem_kind, flags);
}

int prc_ls_filter_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int filter_len, int peek, float reg,
                      prc_c64* out, prc_c64* taps, int mem_kind, int device, void* stream, unsigned flags) {
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, 1, n, nullptr));
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t nb = (size_t)n * sizeof(float2), mb = (size_t)(filter_len + peek) * sizeof(float2);
    const float2 *dref, *dsrv;
    float2* dout;
    TRY(stage_in(c, ref, mem_kind, 1, nb, nb, c->ref, flags, &dref));
    TRY(stage_in(c, srv, mem_kind, 1, nb, nb, c->srv, flags, &dsrv));
    TRY(stage_out(out, mem_kind, nb, c->clean, &dout));
    float2* dtaps = mem_kind == PRC_MEM_DEVICE ? reinterpret_cast<float2*>(taps) : nullptr;   // host: from c->lstaps
    TRY(ls_device(c, dref, dsrv, n, filter_len, peek, (double)reg, dout, dtaps));
    TRY(unstage(c, out, dout, mem_kind, 1, nb, nb, flags));
    TRY(unstage(c, taps, c->lstaps.p, mem_kind, 1, mb, mb, flags));
    TRY(check_ls_status(c, flags));
    return finish(c, flags);
}

int prc_xambg_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                         int range_bins, int freq_bins, const void* window, prc_c64* out, int mem_kind, int device,
                         void* stream, unsigned flags) {
    Batch bt;
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, nframes, frame_stride, &bt, range_bins, freq_bins));
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    return xambg_entry(c, ref, srv, n, bt, range_bins, freq_bins, window, nullptr, 0, out, mem_kind, flags);
}

int prc_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                   int filter_len, int peek, float reg, int range_bins, int freq_bins, const void* window,
                   prc_c64* out_maps, prc_c64* taps_out, prc_c64* cleaned_out, int mem_kind, int device, void* stream,
                   unsigned flags) {
    Batch bt;
    TRY(stack_args(ref, srv, out_maps, "ref/srv/out_maps", mem_kind, n, nframes, frame_stride, &bt, range_bins, freq_bins));
    if (filter_len < 0 || peek < 0 || filter_len + peek < 1)
        return fail(PRC_E_INVALID, "filter_len=%d peek=%d invalid", filter_len, peek);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const int M = filter_len + peek;
    const FramePlan fp = frame_plan(c, n, nframes, filter_len, peek, range_bins, freq_bins);
    // host taps are read from c->lstaps after the call, which holds every frame's taps on the FFT-domain path only
    if (mem_kind == PRC_MEM_HOST && taps_out && nframes > 1 && !fp.fft())
        return fail(PRC_E_INVALID, "taps_out with host pointers and nframes > 1 needs the FFT-domain path");
    const size_t nb = (size_t)n * sizeof(float2), sb = (size_t)bt.stride * sizeof(float2);
    const size_t ob = (size_t)freq_bins * (range_bins + 1) * sizeof(float2);
    const size_t tb = (size_t)nframes * M * sizeof(float2);
    const float2 *dref, *dsrv;
    float2 *dmap, *dclean;
    TRY(stage_in(c, ref, mem_kind, nframes, nb, sb, c->ref, flags, &dref));
    TRY(stage_in(c, srv, mem_kind, nframes, nb, sb, c->srv, flags, &dsrv));
    TRY(stage_out(out_maps, mem_kind, ob * nframes, c->out, &dmap));
    TRY(stage_out(cleaned_out, mem_kind, nb * nframes, c->clean, &dclean));
    float2* dtaps = mem_kind == PRC_MEM_DEVICE ? reinterpret_cast<float2*>(taps_out) : nullptr;   // host: from c->lstaps
    if (mem_kind == PRC_MEM_HOST) bt.stride = n;      // staged frames are packed
    const float* win32;
    TRY(stage_window(c, window, n, mem_kind, flags, &win32));
    TRY(frame_device(c, fp, dref, dsrv, n, bt, filter_len, peek, (double)reg, range_bins, freq_bins, win32, dmap, dtaps, dclean));
    TRY(unstage(c, out_maps, dmap, mem_kind, 1, ob * nframes, ob * nframes, flags));
    TRY(unstage(c, taps_out, c->lstaps.p, mem_kind, 1, tb, tb, flags));
    TRY(unstage(c, cleaned_out, dclean, mem_kind, nframes, nb, sb, flags));
    TRY(check_ls_status(c, flags, nframes));
    return finish(c, flags);
}

int prc_frame_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int filter_len, int peek, float reg,
                  int range_bins, int freq_bins, const void* window, prc_c64* out_map, prc_c64* taps_out,
                  prc_c64* cleaned_out, int mem_kind, int device, void* stream, unsigned flags) {
    return prc_frames_c64(ref, srv, n, 1, n, filter_len, peek, reg, range_bins, freq_bins, window, out_map, taps_out,
                          cleaned_out, mem_kind, device, stream, flags);
}

int prc_frames_multi_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                         int nchan, int64_t chan_stride, int filter_len, int peek, float reg, int range_bins,
                         int freq_bins, const void* window, prc_c64* maps, prc_c64* taps_out,
                         int device, void* stream, unsigned flags) {
    if (nchan < 1 || nchan > fftc::FM_MAX_CHANNELS)
        return fail(PRC_E_INVALID, "nchan=%d invalid (1 <= nchan <= %d)", nchan, fftc::FM_MAX_CHANNELS);
    Batch bt;
    TRY(stack_args(ref, srv, maps, "ref/srv/maps", PRC_MEM_DEVICE, n, nframes, frame_stride, &bt, range_bins, freq_bins));
    if (filter_len < 0 || peek < 0 || filter_len + peek < 1)
        return fail(PRC_E_INVALID, "filter_len=%d peek=%d invalid", filter_len, peek);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const FramePlan fp = frame_plan(c, n, nframes, filter_len, peek, range_bins, freq_bins);
    const float* win32;
    TRY(stage_window(c, window, n, PRC_MEM_DEVICE, flags, &win32));
    TRY(frames_multi_device(c, fp, reinterpret_cast<const float2*>(ref), reinterpret_cast<const float2*>(srv), n, bt, nchan,
                            chan_stride, filter_len, peek, (double)reg, range_bins, freq_bins, win32,
                            reinterpret_cast<float2*>(maps), reinterpret_cast<float2*>(taps_out)));
    TRY(check_ls_status(c, flags, nchan * nframes));
    return finish(c, flags);
}

int prc_set_option(const char* name, int value) {
    if (!name) return fail(PRC_E_INVALID, "name is NULL");
    std::call_once(g_env_once, read_env);
    const std::string k(name);
    if (k == "fft") g_fft.store(value);
    else if (k == "fft_min_n") g_fft_min_n.store(value);
    else if (k == "frame_onepass") g_frame_onepass.store(value);
    else if (fft_ctas_option(k) >= 0)
        return fail(PRC_E_INVALID, "option '%s' is read-only (CTAs per SM of the build's kernels on this device)", name);
    else return fail(PRC_E_INVALID, "unknown option '%s'", name);
    return PRC_OK;
}

int prc_get_option(const char* name, int* value) {
    if (!name || !value) return fail(PRC_E_INVALID, "name/value is NULL");
    std::call_once(g_env_once, read_env);
    const std::string k(name);
    if (k == "fft") *value = g_fft.load();
    else if (k == "fft_min_n") *value = g_fft_min_n.load();
    else if (k == "frame_onepass") *value = g_frame_onepass.load();
    else if (fft_ctas_option(k) >= 0) {
        int dev = 0;
        CU(cudaGetDevice(&dev));
        Ctx* c;
        TRY(get_ctx(dev, nullptr, &c));
        std::lock_guard<std::mutex> lk(c->mu);
        *value = fft_ctas_per_sm(c, (FftKern)fft_ctas_option(k), 8);
    }
    else return fail(PRC_E_INVALID, "unknown option '%s'", name);
    return PRC_OK;
}

int prc_ls_toeplitz_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int filter_len, int peek,
                        prc_c64* out, prc_c64* taps, int mem_kind, int device, void* stream, unsigned flags) {
    return prc_ls_multiple_c64(ref, srv, n, filter_len, peek, 1.0, nullptr, 1, out, taps, mem_kind, device, stream, flags);
}

int prc_ls_multiple_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int filter_len, int peek,
                        double sample_rate, const double* doppler_bins, int nbins, prc_c64* out, prc_c64* taps_last,
                        int mem_kind, int device, void* stream, unsigned flags) {
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, 1, n, nullptr));
    if (nbins < 1) return fail(PRC_E_INVALID, "nbins=%d invalid", nbins);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t nb = (size_t)n * sizeof(float2), mb = (size_t)(filter_len + peek) * sizeof(float2);
    const float2 *dref, *dsrv;
    float2* dout;
    TRY(stage_in(c, ref, mem_kind, 1, nb, nb, c->ref, flags, &dref));
    TRY(stage_in(c, srv, mem_kind, 1, nb, nb, c->srv, flags, &dsrv));
    TRY(stage_out(out, mem_kind, nb, c->out, &dout));
    float2* dtaps = mem_kind == PRC_MEM_DEVICE ? reinterpret_cast<float2*>(taps_last) : nullptr;   // host: from c->lstaps
    TRY(ls_bins(c, dref, dsrv, n, Batch{}, filter_len, peek, sample_rate, doppler_bins, nbins, dout, dtaps, flags));
    TRY(unstage(c, out, dout, mem_kind, 1, nb, nb, flags));
    TRY(unstage(c, taps_last, c->lstaps.p, mem_kind, 1, mb, mb, flags));
    return finish(c, flags);
}

int prc_ls_multiple_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                               int filter_len, int peek, double sample_rate, const double* doppler_bins, int nbins,
                               prc_c64* out, int mem_kind, int device, void* stream, unsigned flags) {
    if (mem_kind != PRC_MEM_DEVICE) return fail(PRC_E_INVALID, "prc_ls_multiple_frames_c64 takes device pointers (mem_kind=%d)", mem_kind);
    if (nframes < 1 || nbins < 1) return fail(PRC_E_INVALID, "nframes=%d nbins=%d invalid", nframes, nbins);
    Batch bt;
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, nframes, frame_stride, &bt));
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    TRY(ls_bins(c, reinterpret_cast<const float2*>(ref), reinterpret_cast<const float2*>(srv), n, bt, filter_len, peek,
                sample_rate, doppler_bins, nbins, reinterpret_cast<float2*>(out), nullptr, flags));
    return finish(c, flags);
}

int prc_direct_xambg_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int range_bins, int freq_bins,
                         double sample_rate, prc_c64* out, int mem_kind, int device, void* stream, unsigned flags) {
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, 1, n, nullptr));
    if (range_bins < 0 || freq_bins < 1) return fail(PRC_E_INVALID, "range_bins=%d freq_bins=%d invalid", range_bins, freq_bins);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t nb = (size_t)n * sizeof(float2);
    const size_t ob = (size_t)freq_bins * (range_bins + 1) * sizeof(float2);
    const float2 *dref, *dsrv;
    float2* dout;
    TRY(stage_in(c, ref, mem_kind, 1, nb, nb, c->ref, flags, &dref));
    TRY(stage_in(c, srv, mem_kind, 1, nb, nb, c->srv, flags, &dsrv));
    TRY(stage_out(out, mem_kind, ob, c->out, &dout));
    TRY(direct_xambg_device(c, dref, dsrv, n, range_bins, freq_bins, sample_rate, dout));
    TRY(unstage(c, out, dout, mem_kind, 1, ob, ob, flags));
    return finish(c, flags);
}

}  // extern "C"
#pragma GCC visibility pop
