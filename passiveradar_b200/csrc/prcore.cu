// prcore.cu -- host side of libprcore.so: C ABI (include/prcore.h), workspaces, launches.
//
// Build (see passiveradar_b200/build.py):
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo \
//        -Xcompiler -fPIC -shared -Iinclude -o passiveradar_b200/libprcore.so prcore.cu
//
// Threading model: one workspace ("Ctx") per (device, caller stream), or per
// (device, calling thread) when the caller passes stream == NULL.  A Ctx owns grow-only
// device buffers; all work of one call is enqueued on the Ctx's stream, so buffer reuse
// is ordered by the stream.  Nothing here falls back to the CPU.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "prcore.h"
#include "kernels.cuh"
#include "lagstream.cuh"
#include "frontend.cuh"
#include "detect.cuh"
#include "nlms_block.cuh"
#include "gal.cuh"
#include "track.cuh"
#include "fftcorr.cuh"
#include "chanoff.cuh"
#include "lssvd.cuh"
#include "framepass.cuh"
#include "recording.cuh"
#include "render.cuh"
#include "spectrum.cuh"
#include "decimate.cuh"

namespace {

using namespace prc;

// Register tile of the FP32 sliding-window kernels (lagcorr, lagstream, fir_apply; DESIGN.md section 3.8):
// TILE_I x TILE_D = 10 x 10 complex MACs per step (samples x lags, or taps x outputs), lane stride
// 10 complex = 80 B (odd multiple of 16 B => conflict-free 128-bit shared loads).
constexpr int TILE_I = 10, TILE_D = 10;
constexpr int FIR_THREADS = 128;
constexpr size_t SMEM_LIMIT = 200 * 1024;

thread_local std::string g_err;
std::atomic<uint64_t> g_launches{0};

// optional per-kernel timing (prc_profile_*): CUDA events on the launching stream around each launch
enum KernelId { K_LAGCORR_LS = 0, K_LEVINSON, K_FIR, K_LAGCORR_CAF, K_DOPPLER, K_NLMS, K_MISC, K_GAL, K_TRK_MEAS, K_TRK_MULTI,
                K_TRK_SIMPLE, K_CHANOFF_LOAD, K_CHANOFF_IIR, K_CHANOFF_FFT, K_CHANOFF_ARGMAX, K_SVD_CORR, K_SVD_EIG, K_SVD_FIR,
                K_CAF_COMBINE, K_FRONTEND_CHUNKS, K_CFAR_FRAMES, K_PERSISTENCE,
                K_PERCENTILE, K_PSD_SEGMENTS, K_PSD_FINISH, K_DECIMATE, K_NORM_SUM, K_NORM_SCALE, K_COUNT };
const char* const kKernelNames[K_COUNT] = {"lagcorr_ls", "levinson", "fir_apply", "lagcorr_caf",
                                           "doppler_fft", "nlms", "misc", "gal_jpe", "track_meas",
                                           "track_multi", "track_simple", "chanoff_load", "chanoff_iir",
                                           "chanoff_fft", "chanoff_argmax", "svd_corr", "svd_eig", "svd_fir",
                                           "caf_combine", "frontend_chunks", "cfar_frames",
                                           "persistence", "percentile", "psd_segments", "psd_finish",
                                           "decimate", "norm_sum", "norm_scale"};
std::atomic<int> g_prof_on{0};
std::mutex g_prof_mu;
double g_prof_ms[K_COUNT] = {0};
uint64_t g_prof_n[K_COUNT] = {0};
struct ProfRec { int id; cudaEvent_t a, b; };

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CU(call)                                                                               \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess)                                                                 \
            return fail(PRC_E_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, \
                        __LINE__);                                                             \
    } while (0)

#define TRY(call)               \
    do {                        \
        int r_ = (call);        \
        if (r_ != PRC_OK) return r_; \
    } while (0)

struct DBuf {
    void* p = nullptr;
    size_t cap = 0;
    int ensure(size_t bytes) {
        if (bytes <= cap) return PRC_OK;
        if (p) {
            cudaError_t e = cudaFree(p);   // implicit device sync: nothing in flight still uses it
            p = nullptr;
            cap = 0;
            if (e != cudaSuccess) return fail(PRC_E_CUDA, "cudaFree: %s", cudaGetErrorString(e));
        }
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            p = nullptr;
            return fail(PRC_E_NOMEM, "cudaMalloc(%zu): %s", want, cudaGetErrorString(e));
        }
        cap = want;
        return PRC_OK;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <class T> T* as() const { return static_cast<T*>(p); }
};

struct Ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int nsm = 148;
    std::mutex mu;
    DBuf fe_in, fe_out, fe_hp;                     // front end: raw IQ, resampled, polyphase taps
    DBuf fe_po, fe_cends;                          // front end: phase offsets, end points of every chunk
    DBuf rd_in, rd_out, rd_det, rd_part, rd_w;     // CFAR_2D and the frame chain of range_doppler_plot.py: maps, results,
                                                   // detections, CFAR partial sums, weights
    uint64_t fe_hp_key = 0;                        // which taps fe_hp holds
    DBuf rs, clean2;          // LS_Filter_Toeplitz: rolled / frequency-shifted reference, ping-pong output
    DBuf refw, ref, srv, out, clean, partial, win32, win64, dtaps32, dtaps64, lstaps, tw, pbuf, status,
        nl_init, nl_taps, gal_k, gal_h;
    DBuf svd_part, svd_cr, svd_ws, svd_taps, svd_rank;   // LS_Filter_SVD: lag-sum partials, c / rhs, A and Z
                                                         // of frames that exceed shared memory, float64 taps, ranks
    DBuf trk_map, trk_plan, trk_stats, trk_slots, trk_out, trk_cnt;   // trackers: host maps, summation tree, per-frame
                                                                      // mean / thr / count, candidate slots, results
    int trk_plan_n = -1, trk_nnodes = 0, trk_nlevels = 0;             // map size trk_plan was built for, its shape
    int tw_F = 0;
    void* pin[2] = {nullptr, nullptr};      // page-locked bounce buffers for pageable host arrays (h2d / d2h below)
    cudaEvent_t pin_ev[2] = {nullptr, nullptr};
    bool pin_ready = false;
    DBuf fft_tw[3], wp_fir, wp_caf, fftP;     // FFT-domain path: twiddle tables (L = 1024 / 2048 / 4096), taps spectra, CAF block sums
    DBuf fpacc;                               // one-pass frame: AccP / AccQ spectra per Doppler block [nf][F][2][L]
    bool fft_tw_ready[3] = {false, false, false};
    int fft_ctas[4][3] = {};  // CTAs per SM of the one-wave FFT-domain kernels, [FftKern][r3_index] (0: not asked yet)
    std::vector<ProfRec> recs;
    void release() {
        cudaSetDevice(device);
        rs.release();
        clean2.release();
        for (DBuf& b : fft_tw) b.release();
        for (bool& r : fft_tw_ready) r = false;
        for (DBuf* b : {&wp_fir, &wp_caf, &fftP, &fpacc}) b->release();
        for (DBuf* b : {&fe_in, &fe_out, &fe_hp, &fe_po, &fe_cends, &rd_in, &rd_out, &rd_det, &rd_part, &rd_w})
            b->release();
        for (DBuf* b : {&refw, &ref, &srv, &out, &clean, &partial, &win32, &win64, &dtaps32, &dtaps64, &lstaps,
                        &tw, &pbuf, &status, &nl_init, &nl_taps, &gal_k, &gal_h, &trk_map, &trk_plan, &trk_stats,
                        &trk_slots, &trk_out, &trk_cnt, &svd_part, &svd_cr, &svd_ws, &svd_taps, &svd_rank})
            b->release();
        trk_plan_n = -1;
        if (pin_ready) {
            for (int k = 0; k < 2; ++k) { cudaFreeHost(pin[k]); cudaEventDestroy(pin_ev[k]); pin[k] = nullptr; pin_ev[k] = nullptr; }
            pin_ready = false;
        }
        if (own_stream && stream) cudaStreamDestroy(stream);
        stream = nullptr;
    }
};

std::mutex g_mu;
std::map<std::pair<int, void*>, Ctx*> g_stream_ctx;   // (device, caller stream)
std::vector<Ctx*> g_all_ctx;
std::atomic<bool> g_attrs_set[64];
std::atomic<uint64_t> g_epoch{1};                      // bumped by prc_shutdown
std::atomic<int> g_fft{1};            // FFT-domain correlation / overlap-save kernels (fftcorr.cuh); PRC_FFT=0: FP32 direct form
std::atomic<int> g_fft_min_n{8192};   // ... for channels of at least this many samples (PRC_FFT_MIN_N)
std::atomic<int> g_frame_onepass{1};  // FFT-domain frame: LS lag sums and CAF block spectra in one pass (framepass.cuh); 0: two passes
std::once_flag g_env_once;

// Workspaces of a thread that called with stream == NULL.  They are released when the thread exits (dask's thread pool
// retires worker threads): otherwise every short-lived caller would strand ~60 MB of device memory until prc_shutdown.
struct TlsCtx {
    Ctx* ctx[64] = {nullptr};
    uint64_t epoch = 0;
    ~TlsCtx() {
        if (epoch != g_epoch.load()) return;              // prc_shutdown already freed them
        std::lock_guard<std::mutex> lk(g_mu);
        if (epoch != g_epoch.load()) return;
        for (Ctx*& c : ctx) {
            if (!c) continue;
            for (size_t i = 0; i < g_all_ctx.size(); ++i)
                if (g_all_ctx[i] == c) {
                    g_all_ctx.erase(g_all_ctx.begin() + i);
                    break;
                }
            if (c->stream) cudaStreamSynchronize(c->stream);
            for (ProfRec& r : c->recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
            c->release();
            delete c;
            c = nullptr;
        }
    }
};
thread_local TlsCtx g_tls;

void read_env() {
    if (const char* e = getenv("PRC_FFT")) g_fft.store(atoi(e));
    if (const char* e = getenv("PRC_FFT_MIN_N")) g_fft_min_n.store(atoi(e));
}

int set_kernel_attrs(int device) {
    if (g_attrs_set[device].load()) return PRC_OK;
    const int lim = (int)SMEM_LIMIT;
    CU(cudaFuncSetAttribute(lagcorr_kernel<TILE_I, TILE_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(lagstream_kernel<TILE_I, TILE_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(fir_apply_kernel<TILE_I, TILE_D>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(levinson_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(levinson_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(doppler_fft_pow2_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(doppler_fft_pow2_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(doppler_fft_pow2_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<1, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<2, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<4, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(gal_jpe_kernel<GAL_CTA_T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(lssvd::svd_eig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<float, TRK_MODE_MEAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<float, TRK_MODE_SLOTS>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<float, TRK_MODE_MEAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<double, TRK_MODE_MEAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<double, TRK_MODE_SLOTS>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<double, TRK_MODE_MEAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
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
    CU(spec::set_attrs(lim));
    CU(dec::set_attrs(lim));
    g_attrs_set[device].store(true);
    return PRC_OK;
}

int get_ctx(int device, void* stream, Ctx** out) {
    std::call_once(g_env_once, read_env);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(PRC_E_CUDA, "no CUDA device available (%s); libprcore has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    if (device < 0 || device >= ndev || device >= 64) return fail(PRC_E_INVALID, "device %d out of range (0..%d)", device, ndev - 1);
    CU(cudaSetDevice(device));
    TRY(set_kernel_attrs(device));
    if (stream == nullptr) {
        if (g_tls.epoch != g_epoch.load()) {
            for (auto& c : g_tls.ctx) c = nullptr;
            g_tls.epoch = g_epoch.load();
        }
        Ctx*& c = g_tls.ctx[device];
        if (!c) {
            Ctx* n = new Ctx();
            n->device = device;
            n->own_stream = true;
            cudaError_t se = cudaStreamCreateWithFlags(&n->stream, cudaStreamNonBlocking);
            if (se != cudaSuccess) {
                delete n;
                return fail(PRC_E_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(se));
            }
            cudaDeviceGetAttribute(&n->nsm, cudaDevAttrMultiProcessorCount, device);
            std::lock_guard<std::mutex> lk(g_mu);
            g_all_ctx.push_back(n);
            c = n;
        }
        *out = c;
        return PRC_OK;
    }
    std::lock_guard<std::mutex> lk(g_mu);
    auto key = std::make_pair(device, stream);
    auto it = g_stream_ctx.find(key);
    if (it == g_stream_ctx.end()) {
        Ctx* n = new Ctx();
        n->device = device;
        n->stream = static_cast<cudaStream_t>(stream);
        n->own_stream = false;
        cudaDeviceGetAttribute(&n->nsm, cudaDevAttrMultiProcessorCount, device);
        g_all_ctx.push_back(n);
        it = g_stream_ctx.emplace(key, n).first;
    }
    *out = it->second;
    return PRC_OK;
}

int check_launch(const char* what) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(PRC_E_CUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
    return PRC_OK;
}

struct ProfScope {          // brackets one launch with events when profiling is enabled
    Ctx* c;
    int id;
    cudaEvent_t a = nullptr;
    ProfScope(Ctx* c_, int id_) : c(c_), id(id_) {
        if (g_prof_on.load(std::memory_order_relaxed)) {
            cudaEventCreate(&a);
            cudaEventRecord(a, c->stream);
        }
    }
    ~ProfScope() {
        if (a) {
            cudaEvent_t b;
            cudaEventCreate(&b);
            cudaEventRecord(b, c->stream);
            c->recs.push_back({id, a, b});
        }
    }
};

// --------------------------------------------------------------------------- geometry
struct Geo {
    int H, G, steps, nchunk, chunk_len, threads;
    size_t smem;
    int HT;
};

int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

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
struct Batch {
    int nf = 1;
    long long stride = 0;
};

inline int r3_index(int r3) { return r3 == 4 ? 0 : (r3 == 8 ? 1 : 2); }
inline size_t fft_smem(int r3) { return (size_t)(2 * 16 * 17 * r3 + 256 * r3 + 16 * r3) * sizeof(float2); }   // fft::Geo<R3>::SMEM_FLOAT2: exchange buffers + twiddles, no staging
inline int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

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

// ---- front end (frontend.cuh) -------------------------------------------------------------------
size_t iq_bytes(int kind, long long n) {
    return (size_t)n * (kind == IQ_I8 ? 2 : kind == IQ_I16 ? 4 : 8);
}

MixParams make_mix(const void* in, int kind, long long n, int mode, double fc, double fs, double po) {
    MixParams m{};
    m.in = in; m.kind = kind; m.n = n; m.mode = mode;
    m.B = (float)(2.0 * 3.14159265358979323846 * fc);
    m.rFs = 1.0f / (float)fs;
    m.po = po;
    m.B64 = 2.0 * 3.14159265358979323846 * fc;
    m.rFs64 = 1.0 / fs;
    return m;
}

// scipy.signal.resample_poly(x, up, down, padtype='line') geometry (scipy/signal/_signaltools.py, resample_poly)
struct ResampleGeo { int up, down, n_pre_pad, n_pre_remove, tpp; long long n_out; };

int resample_geo(long long n_in, int up, int down, int nh, ResampleGeo* g) {
    if (up < 1 || down < 1) return fail(PRC_E_INVALID, "up and down must be >= 1");
    if (nh < 1 || (nh & 1) == 0) return fail(PRC_E_INVALID, "nh=%d: the filter must have 2*half_len+1 taps", nh);
    long long a = up, b = down;
    while (b) { const long long t = a % b; a = b; b = t; }
    up /= (int)a; down /= (int)a;
    const int half_len = (nh - 1) / 2;
    g->up = up; g->down = down;
    g->n_pre_pad = down - half_len % down;
    g->n_pre_remove = (half_len + g->n_pre_pad) / down;
    g->n_out = (n_in * up + down - 1) / down;
    g->tpp = ceil_div(g->n_pre_pad + nh, up) | 1;     // odd row stride: the `up` phase rows of the table start in distinct shared-memory banks
    return PRC_OK;
}

// The geometry, shared-memory check and polyphase table of one resample CTA.  h: host doubles (already multiplied by
// `up`, as resample_poly does before upfirdn).
int resample_table(Ctx* c, const ResampleGeo& g, const double* h, int nh, ResampleParams* out, size_t* smem_out) {
    ResampleParams& rp = *out;
    rp.up = g.up; rp.down = g.down;
    rp.n_pre_pad = g.n_pre_pad; rp.n_pre_remove = g.n_pre_remove; rp.tpp = g.tpp;
    rp.n_out = g.n_out;
    rp.span = (int)(((long long)(RS_THREADS - 1) * g.down) / g.up) + 2 + g.tpp;
    const size_t hp_bytes = (((size_t)g.up * g.tpp * 4 + 15) & ~(size_t)15);
    const size_t smem = hp_bytes + (size_t)rp.span * sizeof(float2);
    if (smem > SMEM_LIMIT)
        return fail(PRC_E_INVALID, "resample %d/%d with %d taps needs %zu bytes of shared memory per CTA", g.up, g.down, nh, smem);
    // polyphase table built on the host (nh ~ 2.4k taps) and cached per context: re-uploaded only when
    // the taps change (FNV-1a over the doubles), so steady-state calls enqueue kernels only
    uint64_t key = 1469598103934665603ull;
    auto mixin = [&key](const void* ptr, size_t bytes) {
        const unsigned char* b = static_cast<const unsigned char*>(ptr);
        for (size_t q = 0; q < bytes; ++q) { key ^= b[q]; key *= 1099511628211ull; }
    };
    mixin(h, (size_t)nh * sizeof(double));
    mixin(&g.up, sizeof(int));
    mixin(&g.down, sizeof(int));
    if (key != c->fe_hp_key || !c->fe_hp.p) {
        std::vector<float> hp((size_t)g.up * g.tpp, 0.f);
        for (int k = g.n_pre_pad; k < g.n_pre_pad + nh; ++k) hp[(size_t)(k % g.up) * g.tpp + k / g.up] = (float)h[k - g.n_pre_pad];
        TRY(c->fe_hp.ensure(hp.size() * sizeof(float)));
        CU(cudaMemcpyAsync(c->fe_hp.p, hp.data(), hp.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));     // hp is a stack-lifetime host buffer
        c->fe_hp_key = key;
    }
    rp.hp = c->fe_hp.as<float>();
    *smem_out = smem;
    return PRC_OK;
}

// nchunks chunks of mix.n samples each, chunk b at raw sample b * chunk_stride of mix.in, mixed with phase offset po[b]
// (device doubles; NULL: mix.po, for a single chunk), its output at out + b * out_stride (recording.cuh)
rec::ChunkParams chunk_params(const MixParams& mix, int nchunks, long long chunk_stride, const double* po, long long out_stride) {
    rec::ChunkParams p{};
    p.rs.mix = mix;
    p.chunk_bytes = (long long)iq_bytes(mix.kind, chunk_stride);
    p.out_stride = out_stride;
    p.po = po;
    p.nchunks = nchunks;
    return p;
}

// deinterleave_IQ + frequency_shift of the chunks: all of the front end when up == down == 1 (resample_poly returns a
// copy), and all a mix alone needs (no taps)
int mix_chunks_device(Ctx* c, KernelId kid, const rec::ChunkParams& p, float2* out) {
    ProfScope ps(c, kid);
    rec::launch_mix(p, out, c->stream);
    return check_launch("rec_mix_kernel");
}

int frontend_device(Ctx* c, KernelId kid, rec::ChunkParams p, const ResampleGeo& g, const double* h, int nh, float2* out) {
    if (g.up == 1 && g.down == 1) return mix_chunks_device(c, kid, p, out);
    size_t smem = 0;
    TRY(resample_table(c, g, h, nh, &p.rs, &smem));
    TRY(c->fe_cends.ensure((size_t)p.nchunks * 2 * sizeof(float2)));
    p.ends = c->fe_cends.as<float2>();
    static std::atomic<bool> attr_set[64];
    if (!attr_set[c->device].exchange(true)) CU(rec::allow_smem((int)SMEM_LIMIT));
    {
        ProfScope ps(c, kid);
        rec::launch_resample(p, smem, out, c->stream);
    }
    return check_launch("rec_resample_kernel");
}

// ---- CFAR_2D (detect.cuh) -----------------------------------------------------------------------
// CFAR_2D's limits, messages and window geometry
int cfar_window(int rows, int cols, int fw, int gw, CfarParams* p) {
    if (rows < 1 || cols < 1) return fail(PRC_E_INVALID, "rows=%d cols=%d invalid", rows, cols);
    if (rows > CFAR_MAX_ROWS)          // one CTA row of tiles per gridDim.y index
        return fail(PRC_E_INVALID, "rows=%d exceed the CFAR maximum of %d rows", rows, CFAR_MAX_ROWS);
    if (fw < 1 || fw > CFAR_MAX_FW) return fail(PRC_E_INVALID, "fw=%d outside [1, %d]", fw, CFAR_MAX_FW);
    if (gw < 0 || fw * fw - gw * gw == 0) return fail(PRC_E_INVALID, "fw=%d gw=%d: fw^2 - gw^2 must not be 0", fw, gw);
    *p = CfarParams{};
    p->rows = rows; p->cols = cols; p->fw = fw;
    // python: e1 = (fw - gw) // 2 (floor), e2 = fw - e1 + 1; slices clip to [0, fw]
    int e1 = (fw - gw) >= 0 ? (fw - gw) / 2 : -((gw - fw + 1) / 2);
    int e2 = fw - e1 + 1;
    if (e1 < 0) e1 = std::max(0, e1 + fw);     // negative slice start counts from the end
    p->e1 = std::min(e1, fw); p->e2 = std::min(std::max(e2, 0), fw);
    p->c = (fw - 1) / 2;
    p->scale = 1.0 / ((double)fw * fw - (double)gw * gw);
    return PRC_OK;
}

int cfar_frames_device(Ctx* c, KernelId kid, CfarParams& p, int nframes) {
    TRY(c->rd_part.ensure((size_t)nframes * CFAR_MEAN_CTAS * sizeof(double)));
    p.partial = c->rd_part.as<double>();
    {   // under a lock: a concurrent first call must not launch before the attribute is set
        static std::mutex attr_mu;
        static bool attr_set[64];
        std::lock_guard<std::mutex> g(attr_mu);
        if (!attr_set[c->device]) {
            CU(allow_cfar_smem((int)SMEM_LIMIT));
            attr_set[c->device] = true;
        }
    }
    {
        ProfScope ps(c, kid);
        launch_cfar(p, nframes, c->stream);
    }
    return check_launch("cfar_frames_kernel");
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
        const MixParams m = make_mix(ref, IQ_C64, n, MIX_C64, df, fs, 0.0);
        TRY(mix_chunks_device(c, K_MISC, chunk_params(m, 1, 0, nullptr, 0), c->rs.as<float2>()));
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

// bt.nf independent frames run as one CTA each (the recurrence of a frame is serial, the frames are not)
int nlms_device(Ctx* c, const float2* ref, const float2* srv, long long n, int filter_len, int peek, float mu,
                int block_len, const float2* init, float2* out, float2* taps_out, Batch bt = Batch{}, bool init_shared = true) {
    if (n <= 0 || n >= (1ll << 31) - 4096) return fail(PRC_E_INVALID, "n=%lld unsupported", n);
    if (filter_len < 0 || peek < 0 || filter_len + peek < 1)
        return fail(PRC_E_INVALID, "filter_len=%d peek=%d invalid", filter_len, peek);
    if (block_len < 1) return fail(PRC_E_INVALID, "block_len=%d invalid", block_len);
    const int M = filter_len + peek;
    if (M > 1024 * NLMS_MAXT) return fail(PRC_E_INVALID, "%d taps exceed the NLMS kernel's maximum of %d", M, 1024 * NLMS_MAXT);
    NlmsParams p{};
    p.ref = ref; p.srv = srv; p.init = init; p.out = out; p.taps_out = taps_out;
    p.n = (int)n; p.filter_len = filter_len; p.peek = peek; p.mu = mu; p.block_len = block_len;
    p.frame_stride = bt.nf > 1 ? bt.stride : 0; p.init_shared = init_shared ? 1 : 0;
    // exact evaluation 32 samples at a time (nlms_block.cuh); block_len > 1 (block_NLMS) freezes the taps inside a
    // user block
    const size_t sb = nlms_block_smem(M);
    ProfScope ps(c, K_NLMS);
    if (bt.nf > c->nsm && M <= 2048) {
        // more frames than SMs: 512-thread CTAs, two resident per SM (a 1024-thread CTA owns the SM's registers)
        if (M <= 512) nlms_block_kernel<1, 512><<<bt.nf, 512, sb, c->stream>>>(p);
        else if (M <= 1024) nlms_block_kernel<2, 512><<<bt.nf, 512, sb, c->stream>>>(p);
        else nlms_block_kernel<4, 512><<<bt.nf, 512, sb, c->stream>>>(p);
        return check_launch("nlms_block_kernel");
    }
    if (M <= 1024) nlms_block_kernel<1><<<bt.nf, NB_THREADS, sb, c->stream>>>(p);
    else if (M <= 2048) nlms_block_kernel<2><<<bt.nf, NB_THREADS, sb, c->stream>>>(p);
    else nlms_block_kernel<4><<<bt.nf, NB_THREADS, sb, c->stream>>>(p);
    return check_launch("nlms_block_kernel");
}

// GAL_JPE on bt.nf independent frames (gal.cuh): delay lines up to GAL_WARP_MAX_D taps run one frame per warp
// (GAL_WARP_FRAMES frames per CTA, shuffles only), longer ones one frame per CTA of ceil(D / 256) warps
int gal_check(long long n, int L, int D, int peek) {
    if (n <= 0) return fail(PRC_E_INVALID, "n=%lld invalid", n);
    if (L < 1) return fail(PRC_E_INVALID, "lattice_len=%d invalid (must be >= 1)", L);
    if (D < L) return fail(PRC_E_INVALID, "delay_line_len=%d must be >= lattice_len=%d", D, L);
    if (D > GAL_MAX_D)
        return fail(PRC_E_INVALID, "delay_line_len=%d exceeds the GAL_JPE kernel's maximum of %d", D, GAL_MAX_D);
    if (peek < 0) return fail(PRC_E_INVALID, "peek=%d invalid", peek);
    return PRC_OK;
}

int gal_device(Ctx* c, const float2* ref, const float2* srv, long long n, Batch bt, int L, int D, double mu1, double mu2,
               int peek, float2* out, float2* k_out, float2* h_out) {
    TRY(gal_check(n, L, D, peek));
    GalParams p{};
    p.ref = ref; p.srv = srv; p.out = out; p.k_out = k_out; p.h_out = h_out;
    p.n = n; p.stride = bt.stride; p.nframes = bt.nf;
    p.L = L; p.D = D; p.peek = peek; p.mu1 = mu1; p.mu2 = (float)mu2;
    ProfScope ps(c, K_GAL);
    if (D <= GAL_WARP_MAX_D) {
        const int grid = ceil_div(bt.nf, GAL_WARP_FRAMES), threads = 32 * GAL_WARP_FRAMES;
        if (D <= 32) gal_jpe_kernel<1, false><<<grid, threads, 0, c->stream>>>(p);
        else if (D <= 64) gal_jpe_kernel<2, false><<<grid, threads, 0, c->stream>>>(p);
        else if (D <= 128) gal_jpe_kernel<4, false><<<grid, threads, 0, c->stream>>>(p);
        else gal_jpe_kernel<8, false><<<grid, threads, 0, c->stream>>>(p);
        return check_launch("gal_jpe_kernel(warp)");
    }
    const int threads = 32 * ceil_div(D, 32 * GAL_CTA_T);
    gal_jpe_kernel<GAL_CTA_T, true><<<bt.nf, threads, gal_smem(threads), c->stream>>>(p);
    return check_launch("gal_jpe_kernel(cta)");
}

// ---- host <-> device copies of caller arrays.  dask hands the operators ordinary (pageable) numpy arrays from several
// threads at once (main.py:169-194); cudaMemcpyAsync from pageable memory goes through the driver's own staging, one
// copy at a time for the whole process.  Each workspace therefore owns two page-locked bounce buffers: the calling
// thread copies a chunk into one while the DMA engine drains the other, so concurrent callers overlap their host-side
// copies and their transfers.  Page-locked arrays (FramePipeline, prc_host_alloc / prc_host_register) and asynchronous
// calls (PRC_FLAG_ASYNC: the caller owns the synchronisation) take the plain cudaMemcpyAsync path.
constexpr size_t PIN_CHUNK = 4u << 20;

bool host_is_pinned(const void* ptr) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

int ensure_pin(Ctx* c) {
    if (c->pin_ready) return PRC_OK;
    for (int k = 0; k < 2; ++k) {
        CU(cudaHostAlloc(&c->pin[k], PIN_CHUNK, cudaHostAllocPortable));
        CU(cudaEventCreateWithFlags(&c->pin_ev[k], cudaEventDisableTiming));
    }
    c->pin_ready = true;
    return PRC_OK;
}

int h2d(Ctx* c, void* dst, const void* src, size_t bytes, unsigned flags) {
    if ((flags & PRC_FLAG_ASYNC) || bytes < (256u << 10) || host_is_pinned(src)) {
        CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->stream));
        return PRC_OK;
    }
    TRY(ensure_pin(c));
    int k = 0;
    for (size_t off = 0; off < bytes; off += PIN_CHUNK, k ^= 1) {
        const size_t len = std::min(PIN_CHUNK, bytes - off);
        CU(cudaEventSynchronize(c->pin_ev[k]));           // the transfer that last used this buffer has finished
        memcpy(c->pin[k], static_cast<const char*>(src) + off, len);
        CU(cudaMemcpyAsync(static_cast<char*>(dst) + off, c->pin[k], len, cudaMemcpyHostToDevice, c->stream));
        CU(cudaEventRecord(c->pin_ev[k], c->stream));
    }
    return PRC_OK;
}

int d2h(Ctx* c, void* dst, const void* src, size_t bytes, unsigned flags) {
    if ((flags & PRC_FLAG_ASYNC) || bytes < (256u << 10) || host_is_pinned(dst)) {
        CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
        return PRC_OK;
    }
    TRY(ensure_pin(c));
    const size_t nchunk = (bytes + PIN_CHUNK - 1) / PIN_CHUNK;
    for (size_t i = 0; i <= nchunk; ++i) {                // transfer of chunk i overlaps the host copy of chunk i - 1
        if (i < nchunk) {
            const size_t off = i * PIN_CHUNK, len = std::min(PIN_CHUNK, bytes - off);
            CU(cudaMemcpyAsync(c->pin[i & 1], static_cast<const char*>(src) + off, len, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaEventRecord(c->pin_ev[i & 1], c->stream));
        }
        if (i >= 1) {
            const size_t j = i - 1, off = j * PIN_CHUNK, len = std::min(PIN_CHUNK, bytes - off);
            CU(cudaEventSynchronize(c->pin_ev[j & 1]));
            memcpy(static_cast<char*>(dst) + off, c->pin[j & 1], len);
        }
    }
    return PRC_OK;
}

// ---- arguments and operands of the C entry points
bool bad_mem_kind(int k) { return k != PRC_MEM_HOST && k != PRC_MEM_DEVICE; }

// The checks of an entry point that takes ref / srv stacks, made before any CUDA call.  `names` names the three
// operands in the message; range_bins / freq_bins are the CAF's (the defaults pass).  *bt (when given): the frames and
// the caller's stride between them.
int stack_args(const void* a, const void* b, const void* o, const char* names, int mem_kind, long long n, int nframes,
               long long frame_stride, Batch* bt, int range_bins = 0, int freq_bins = 1) {
    if (!a || !b || !o) return fail(PRC_E_INVALID, "%s must not be NULL", names);
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    if (n <= 0) return fail(PRC_E_INVALID, "n=%lld invalid", n);
    if (nframes < 1) return fail(PRC_E_INVALID, "nframes=%d invalid", nframes);
    if (nframes > 1 && frame_stride < n) return fail(PRC_E_INVALID, "frame_stride=%lld smaller than n=%lld", frame_stride, n);
    if (freq_bins < 1 || range_bins < 0) return fail(PRC_E_INVALID, "freq_bins=%d / range_bins=%d invalid", freq_bins, range_bins);
    if (bt) {
        bt->nf = nframes;
        bt->stride = nframes > 1 ? frame_stride : n;
    }
    return PRC_OK;
}

// The checks the front-end entry points share, made before any CUDA call
int frontend_args(int mem_kind, long long n, int in_kind, int mode, double fs) {
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    if (n <= 0) return fail(PRC_E_INVALID, "n=%lld invalid", n);
    if (in_kind < IQ_C64 || in_kind > IQ_I16) return fail(PRC_E_INVALID, "in_kind=%d invalid", in_kind);
    if (mode < MIX_NONE || mode > MIX_FS64) return fail(PRC_E_INVALID, "mode=%d invalid", mode);
    if (mode != MIX_NONE && !(fs != 0.0)) return fail(PRC_E_INVALID, "fs must not be 0");
    return PRC_OK;
}

// `rows` rows of `row_bytes`: the host side's rows are `stride` bytes apart, the device side's packed.  One copy when
// the host rows are contiguous, one per row otherwise.
int rows_h2d(Ctx* c, void* dst, const void* src, size_t rows, size_t row_bytes, size_t stride, unsigned flags) {
    if (rows == 1 || stride == row_bytes) return h2d(c, dst, src, rows * row_bytes, flags);
    for (size_t r = 0; r < rows; ++r)
        TRY(h2d(c, static_cast<char*>(dst) + r * row_bytes, static_cast<const char*>(src) + r * stride, row_bytes, flags));
    return PRC_OK;
}

int rows_d2h(Ctx* c, void* dst, const void* src, size_t rows, size_t row_bytes, size_t stride, unsigned flags) {
    if (rows == 1 || stride == row_bytes) return d2h(c, dst, src, rows * row_bytes, flags);
    for (size_t r = 0; r < rows; ++r)
        TRY(d2h(c, static_cast<char*>(dst) + r * stride, static_cast<const char*>(src) + r * row_bytes, row_bytes, flags));
    return PRC_OK;
}

// A caller's input as the kernels read it: a device array (or NULL) where it is, a host one copied into `buf` with its
// rows packed (row stride row_bytes)
template <class T>
int stage_in(Ctx* c, const void* src, int mem_kind, size_t rows, size_t row_bytes, size_t stride, DBuf& buf,
             unsigned flags, const T** dev) {
    *dev = static_cast<const T*>(src);
    if (mem_kind == PRC_MEM_DEVICE || !src) return PRC_OK;
    TRY(buf.ensure(rows * row_bytes));
    *dev = buf.as<T>();
    return rows_h2d(c, buf.p, src, rows, row_bytes, stride, flags);
}

// Where the kernels write a caller's output: a device array (or NULL) itself, `bytes` of `buf` for a host one
template <class T>
int stage_out(void* dst, int mem_kind, size_t bytes, DBuf& buf, T** dev) {
    *dev = static_cast<T*>(dst);
    if (mem_kind == PRC_MEM_DEVICE || !dst) return PRC_OK;
    TRY(buf.ensure(bytes));
    *dev = buf.as<T>();
    return PRC_OK;
}

// Results, rows packed at `src`, back to a caller's host output whose rows are `stride` bytes apart; nothing to do for
// a device output (the kernels wrote it) or a NULL one
int unstage(Ctx* c, void* dst, const void* src, int mem_kind, size_t rows, size_t row_bytes, size_t stride, unsigned flags) {
    if (mem_kind == PRC_MEM_DEVICE || !dst) return PRC_OK;
    return rows_d2h(c, dst, src, rows, row_bytes, stride, flags);
}

// A parameter array of the call -> `buf`.  It is copied out of the caller's memory before the call returns: the
// transfer below is from pageable memory this function owns, which the runtime stages before cudaMemcpyAsync returns,
// so it is safe under PRC_FLAG_ASYNC even when the caller's array is page-locked and goes away right after the call
int copy_params(Ctx* c, const double* src, int count, DBuf& buf) {
    const std::vector<double> v(src, src + count);
    TRY(buf.ensure((size_t)count * sizeof(double)));
    CU(cudaMemcpyAsync(buf.p, v.data(), (size_t)count * sizeof(double), cudaMemcpyHostToDevice, c->stream));
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

int finish(Ctx* c, unsigned flags) {
    if (flags & PRC_FLAG_ASYNC) return PRC_OK;
    CU(cudaStreamSynchronize(c->stream));
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

// ---- Kalman trackers (track.cuh) -----------------------------------------------------------------
constexpr size_t TRK_SLOT_BUDGET = 256u << 20;     // candidate slots of one multi-tracker launch (bytes)

// python slice [start:stop] of an axis of length len
void py_slice(long long start, long long stop, long long len, int* lo, int* hi) {
    if (start < 0) { start += len; if (start < 0) start = 0; } else if (start > len) start = len;
    if (stop < 0) { stop += len; if (stop < 0) stop = 0; } else if (stop > len) stop = len;
    *lo = (int)start;
    *hi = (int)std::max(start, stop);
}

int trk_check(const void* maps, int rows, int cols, int nseq, int nframes, int64_t seq_stride, int64_t frame_stride,
              int mem_kind) {
    if (!maps) return fail(PRC_E_INVALID, "maps must not be NULL");
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    if (rows < 1 || cols < 1) return fail(PRC_E_INVALID, "rows=%d cols=%d invalid", rows, cols);
    if ((long long)rows * cols > TRK_MAX_CELLS)
        return fail(PRC_E_INVALID, "a %d x %d map exceeds the tracker kernels' maximum of %lld cells", rows, cols,
                    TRK_MAX_CELLS);
    if (nseq < 1 || nseq > 65535) return fail(PRC_E_INVALID, "nseq=%d outside [1, 65535]", nseq);
    if (nframes < 1) return fail(PRC_E_INVALID, "nframes=%d invalid", nframes);
    if (seq_stride < 0 || frame_stride < 0)
        return fail(PRC_E_INVALID, "seq_stride=%lld frame_stride=%lld invalid", (long long)seq_stride, (long long)frame_stride);
    return PRC_OK;
}

// NumPy's pairwise summation tree of n elements (split at n/2 rounded down to a multiple of 8 until <= 128),
// breadth-first, followed by the first node of every depth; built once per map size and context
int trk_plan(Ctx* c, int n) {
    if (c->trk_plan_n == n) return PRC_OK;
    std::vector<PwNode> nodes{PwNode{0, n, -1, 0}};
    std::vector<int> level{0};
    size_t lo = 0;
    for (;;) {
        const size_t hi = nodes.size();
        for (size_t q = lo; q < hi; ++q) {
            const PwNode nd = nodes[q];
            if (nd.len <= 128) continue;
            const int n2 = nd.len / 2 - (nd.len / 2) % 8;
            nodes[q].left = (int)nodes.size();
            nodes.push_back(PwNode{nd.off, n2, -1, 0});
            nodes.push_back(PwNode{nd.off + n2, nd.len - n2, -1, 0});
        }
        if (nodes.size() == hi) break;
        level.push_back((int)hi);
        lo = hi;
    }
    level.push_back((int)nodes.size());
    const size_t nb = nodes.size() * sizeof(PwNode), lb = level.size() * sizeof(int);
    TRY(c->trk_plan.ensure(nb + lb));
    CU(cudaMemcpyAsync(c->trk_plan.p, nodes.data(), nb, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(static_cast<char*>(c->trk_plan.p) + nb, level.data(), lb, cudaMemcpyHostToDevice, c->stream));
    c->trk_plan_n = n;
    c->trk_nnodes = (int)nodes.size();
    c->trk_nlevels = (int)level.size() - 1;
    return PRC_OK;
}

// maps -> device (frame-major, compact) when they are host arrays; fills the map part of mp
int trk_stage(Ctx* c, const void* maps, int rows, int cols, int nseq, int nframes, int64_t seq_stride,
              int64_t frame_stride, int mem_kind, unsigned flags, TrkMapParams* mp) {
    const size_t esz = (flags & PRC_FLAG_MAP_F64) ? 8 : 4;
    const long long n = (long long)rows * cols;
    *mp = TrkMapParams{};
    mp->maps = maps;
    mp->seq_stride = seq_stride;
    mp->frame_stride = frame_stride;
    if (mem_kind == PRC_MEM_HOST) {
        TRY(c->trk_map.ensure((size_t)nseq * nframes * n * esz));
        char* d = c->trk_map.as<char>();
        const char* h = static_cast<const char*>(maps);
        for (int s = 0; s < nseq; ++s)
            TRY(rows_h2d(c, d + (size_t)s * nframes * n * esz, h + (size_t)s * seq_stride * esz, nframes, n * esz,
                         (size_t)frame_stride * esz, flags));
        mp->maps = d;
        mp->seq_stride = (long long)nframes * n;
        mp->frame_stride = n;
    }
    TRY(trk_plan(c, (int)n));
    mp->rows = rows;
    mp->cols = cols;
    mp->n = (int)n;
    mp->nframes = nframes;
    mp->plan = c->trk_plan.as<PwNode>();
    mp->level = reinterpret_cast<const int*>(c->trk_plan.as<PwNode>() + c->trk_nnodes);
    mp->nnodes = c->trk_nnodes;
    mp->nlevels = c->trk_nlevels;
    // np.percentile(frame, 99.8), linear method: v = (n - 1) * 0.998, order statistics floor(v) and floor(v) + 1
    const double v = (double)(n - 1) * (99.8 / 100.0);
    mp->k = (int)std::floor(v);
    mp->g = v - (double)mp->k;
    py_slice(rows / 2 - 4, rows / 2 + 4, rows, &mp->dlo, &mp->dhi);
    mp->n_unbanded = std::max(0, cols - 16) * (rows - (mp->dhi - mp->dlo));
    // candidates sorted in shared memory: room for twice the usual count (n - 1 - k)
    const int want = std::max(256, 2 * ((int)n - 1 - mp->k) + 64);
    int cap = 256;
    while (cap < want && cap < TRK_MAX_CAP) cap <<= 1;
    mp->cap = cap;
    return PRC_OK;
}

// bin centres: rpts = linspace(range_extent, 0, cols), dpts = linspace(-1 * doppler_extent, doppler_extent, rows)
void trk_extent(TrkMapParams* mp, double doppler_extent, double range_extent) {
    mp->rng_start = range_extent;
    mp->dop_start = -1.0 * doppler_extent;
    mp->dop_stop = doppler_extent;
}

size_t trk_smem(const TrkMapParams& mp, int mode) {
    const size_t nv = ((size_t)mp.nnodes * 8 + 15) & ~(size_t)15;
    return mode == TRK_MODE_MEAN ? nv : nv + (size_t)mp.cap * (sizeof(unsigned long long) + sizeof(int));
}

// PRC_FLAG_TRACK_RESUME from host memory: the frame-0 records of every sequence (rec bytes, seq bytes apart) -> the
// staged history the kernels continue from
int trk_resume_h2d(Ctx* c, void* dev, const void* host, int nseq, size_t seq, size_t rec, unsigned flags) {
    for (int s = 0; s < nseq; ++s)
        TRY(h2d(c, static_cast<char*>(dev) + s * seq, static_cast<const char*>(host) + s * seq, rec, flags));
    return PRC_OK;
}

int trk_meas_launch(Ctx* c, const TrkMapParams& mp, bool f64, int mode, int nf, int nseq) {
    const size_t smem = trk_smem(mp, mode);
    if (smem > SMEM_LIMIT) return fail(PRC_E_INVALID, "tracker measurement kernel needs %zu B of shared memory", smem);
    const dim3 grid(nf, nseq);
    ProfScope ps(c, K_TRK_MEAS);
#define PRC_TRK_MEAS(T)                                                                                            \
    if (mode == TRK_MODE_MEAN) track_meas_kernel<T, TRK_MODE_MEAN><<<grid, TRK_THREADS, smem, c->stream>>>(mp);   \
    else if (mode == TRK_MODE_SLOTS) track_meas_kernel<T, TRK_MODE_SLOTS><<<grid, TRK_THREADS, smem, c->stream>>>(mp); \
    else track_meas_kernel<T, TRK_MODE_MEAS><<<grid, TRK_THREADS, smem, c->stream>>>(mp);
    if (f64) { PRC_TRK_MEAS(double) } else { PRC_TRK_MEAS(float) }
#undef PRC_TRK_MEAS
    return check_launch("track_meas_kernel");
}

// read-only names of the residency the one-wave grids are sized from (fft_ctas_per_sm, R3 = 8 -- the transform
// length of up to 1024 LS taps and of the CAF at config 2): the FftKern they report, -1 for any other name
int fft_ctas_option(const std::string& k) {
    if (k == "fft_ctas_ls") return FK_LS;
    if (k == "fft_ctas_fir") return FK_FIR;
    if (k == "fft_ctas_frame") return FK_FRAME;
    return -1;
}

// ---- channel offset / xcorr (chanoff.cuh) ---------------------------------------------------------------------------
constexpr int CHANOFF_MAX_ND = 64;          // largest decimation factor (its pole radius 0.9971 sets W ~ 14k samples)
constexpr int CHANOFF_MAX_LOG2 = 26;        // largest transform: 2^26 complex128 = 1 GiB per buffer

// Stream-ordered scratch of one call: once per run, and ~0.5 GB at main.py's shapes, so it is not kept in the Ctx
struct AsyncScratch {
    cudaStream_t st;
    std::vector<void*> ptrs;
    explicit AsyncScratch(cudaStream_t s) : st(s) {}
    ~AsyncScratch() { for (void* p : ptrs) cudaFreeAsync(p, st); }
    template <class T> int get(T** out, size_t bytes) {
        void* p = nullptr;
        cudaError_t e = cudaMallocAsync(&p, bytes ? bytes : 16, st);
        if (e != cudaSuccess) { cudaGetLastError(); return fail(PRC_E_NOMEM, "cudaMallocAsync(%zu): %s", bytes, cudaGetErrorString(e)); }
        ptrs.push_back(p);
        *out = static_cast<T*>(p);
        return PRC_OK;
    }
};

bool chanoff_bad_dtype(int dt) { return dt < chanoff::DT_I8 || dt > chanoff::DT_C128; }

// W: samples after which a zero-state start of the cascade agrees with the exact state below float64 round-off
// (DESIGN.md section 11): the transient decays as r^k for the largest pole radius r, times a polynomial in k for the
// four nearly repeated pole pairs, which the 256-sample margin covers
int chanoff_warmup(const chanoff::Sos& f, long long* warm) {
    double r = 0.0;
    for (int s = 0; s < chanoff::NSEC; ++s) {
        if (f.s[s][3] != 1.0) return fail(PRC_E_INVALID, "sos section %d: a0 = %g, must be 1", s, f.s[s][3]);
        const double a1 = f.s[s][4], a2 = f.s[s][5], disc = a1 * a1 - 4.0 * a2;
        const double rs = disc < 0.0 ? std::sqrt(a2) : std::max(std::fabs(-a1 + std::sqrt(disc)), std::fabs(-a1 - std::sqrt(disc))) / 2.0;
        r = std::max(r, rs);
    }
    if (!(r < 1.0)) return fail(PRC_E_INVALID, "the decimation filter is not stable (pole radius %g)", r);
    *warm = (long long)std::ceil(std::log(1e-18) / std::log(r)) + 256;
    return PRC_OK;
}

// xc[k] = sum_i a[i + k + p0] conj(b[i]) over the nvalid valid lags of correlate(A, pad(B, (pad_l, pad_r)), 'valid'),
// A, B = the inputs, decimated (f != nullptr: sosfiltfilt + [::nd]) or as they are.  mode ARG_ABS: |xc| -> out
// (optional) and res[0..1] = argmax, (argmax - nl) * nd; ARG_COMPLEX / ARG_REAL: the lags -> out.
int chanoff_device(Ctx* c, AsyncScratch& ws, const void* s1, int dt1, long long n1, const void* s2, int dt2, long long n2,
                   const chanoff::Sos* f, int nd, long long pad_l, long long pad_r, int mode, void* out, long long* res) {
    using namespace chanoff;
    const long long n1d = f ? (n1 + nd - 1) / nd : n1, n2d = f ? (n2 + nd - 1) / nd : n2;
    const long long lenb = n2d + pad_l + pad_r;
    const long long nvalid = (n1d >= lenb ? n1d - lenb : lenb - n1d) + 1;
    const long long p0 = (n1d >= lenb ? 0 : n1d - lenb) + pad_l;
    // circular length with no valid lag aliased: p + L beyond the support's top n1d - 1, p - L below -(n2d - 1)
    const long long need = std::max(std::max(std::max(n1d, n2d), std::max(p0 + nvalid - 1 + n2d, n1d - p0)), 2ll);
    int m = 1;
    while (m <= CHANOFF_MAX_LOG2 && (1ll << m) < need) ++m;
    if (m > CHANOFF_MAX_LOG2)
        return fail(PRC_E_INVALID, "the correlation needs a transform of %lld points; the maximum is 2^%d = %lld", need,
                    CHANOFF_MAX_LOG2, 1ll << CHANOFF_MAX_LOG2);
    const long long L = 1ll << m;
    double2 *X, *Y, *tlo, *thi;
    const int nhi = (int)std::max(1ll, (L / 2) >> TW_LO_BITS);
    TRY(ws.get(&X, (size_t)L * sizeof(double2)));
    TRY(ws.get(&Y, (size_t)L * sizeof(double2)));
    TRY(ws.get(&tlo, ((size_t)1 << TW_LO_BITS) * sizeof(double2)));
    TRY(ws.get(&thi, (size_t)nhi * sizeof(double2)));
    CU(cudaMemsetAsync(X + n1d, 0, (size_t)(L - n1d) * sizeof(double2), c->stream));
    CU(cudaMemsetAsync(Y + n2d, 0, (size_t)(L - n2d) * sizeof(double2), c->stream));
    if (f) {
        const long long nmax = std::max(n1, n2) + 2 * PADLEN;
        double* F;
        TRY(ws.get(&F, (size_t)nmax * sizeof(double2)));
        const void* src[2] = {s1, s2};
        const int dts[2] = {dt1, dt2};
        const long long ns[2] = {n1, n2};
        double2* dst[2] = {X, Y};
        for (int q = 0; q < 2; ++q) {
            IirParams ip{};
            ip.f = f[q];
            TRY(chanoff_warmup(f[q], &ip.warm));
            ip.dt = dts[q];
            ip.n = ns[q];
            ip.next = ns[q] + 2 * PADLEN;
            ip.chunk = std::max(256ll, (ip.next + 16383) / 16384);
            ip.nd = nd;
            const bool cplx = dt_complex(dts[q]);
            ProfScope ps(c, K_CHANOFF_IIR);
            ip.x = src[q];
            ip.y = F;
            launch_iir(ip, cplx, false, c->stream);
            TRY(check_launch("chanoff_iir_kernel(forward)"));
            ip.x = F;
            ip.y = dst[q];
            launch_iir(ip, cplx, true, c->stream);
            TRY(check_launch("chanoff_iir_kernel(backward)"));
        }
    } else {
        ProfScope ps(c, K_CHANOFF_LOAD);
        launch_load(s1, dt1, n1, X, c->nsm, c->stream);
        launch_load(s2, dt2, n2, Y, c->nsm, c->stream);
        TRY(check_launch("chanoff_load_kernel"));
    }
    // passes from the top index bits down: 8 bits (x 8 consecutive columns) while more than 11 remain, then the rest
    struct Pass { int lo, nb, c, s0; };
    std::vector<Pass> passes;
    for (int top = m; top > 0;) {
        const int nb = top <= FFT_TILE_BITS ? top : 8, lo = top - nb;
        passes.push_back(Pass{lo, nb, std::min(3, lo), m - top});
        top = lo;
    }
    {
        ProfScope ps(c, K_CHANOFF_FFT);
        launch_twiddle(tlo, thi, nhi, m, c->stream);
        TRY(check_launch("chanoff_twiddle_kernel"));
        FftParams fp{};
        fp.buf[0] = X; fp.buf[1] = Y;
        fp.tw_lo = tlo; fp.tw_hi = thi;
        fp.m = m;
        for (int k = 0; k < 2 * (int)passes.size(); ++k) {      // forward passes of X and Y, then the inverse of X conj(Y)
            const bool inverse = k >= (int)passes.size();
            const Pass& ps_ = inverse ? passes[2 * passes.size() - 1 - k] : passes[k];
            fp.lo = ps_.lo; fp.nb = ps_.nb; fp.c = ps_.c; fp.s0 = ps_.s0;
            fp.product = k == (int)passes.size();
            launch_fft_pass(fp, inverse, c->stream);
            TRY(check_launch("chanoff_fft_kernel"));
        }
    }
    ArgParams ap{};
    ap.cc = X; ap.L = L; ap.nvalid = nvalid; ap.p0 = p0;
    ap.scale = 1.0 / (double)L;
    ap.mode = mode;
    ap.out = out;
    const int nb = argmax_blocks(nvalid);
    ProfScope ps(c, K_CHANOFF_ARGMAX);
    if (mode == ARG_ABS) {
        TRY(ws.get(&ap.part_v, (size_t)nb * sizeof(double)));
        TRY(ws.get(&ap.part_k, (size_t)nb * sizeof(long long)));
    }
    launch_argmax(ap, nb, c->stream);
    TRY(check_launch("chanoff_argmax_kernel"));
    if (mode == ARG_ABS) {
        launch_argmax_final(ap.part_v, ap.part_k, nb, pad_l, nd, res, c->stream);
        TRY(check_launch("chanoff_argmax_final_kernel"));
    }
    return PRC_OK;
}

int chanoff_inputs(const void* s1, int dt1, int64_t n1, const void* s2, int dt2, int64_t n2, int mem_kind) {
    if (!s1 || !s2) return fail(PRC_E_INVALID, "s1/s2 must not be NULL");
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    if (chanoff_bad_dtype(dt1) || chanoff_bad_dtype(dt2)) return fail(PRC_E_INVALID, "dtype %d / %d invalid", dt1, dt2);
    if (n1 < 1 || n2 < 1) return fail(PRC_E_INVALID, "n1=%lld n2=%lld invalid", (long long)n1, (long long)n2);
    return PRC_OK;
}

// host inputs -> stream-ordered device copies of their raw bytes (int8 stays one byte per sample over PCIe)
int chanoff_stage(Ctx* c, AsyncScratch& ws, const void** s, int dt, int64_t n, int mem_kind, unsigned flags) {
    if (mem_kind == PRC_MEM_DEVICE) return PRC_OK;
    const size_t b = (size_t)n * chanoff::dt_size(dt);
    void* d;
    TRY(ws.get(&d, b));
    TRY(rows_h2d(c, d, *s, 1, b, b, flags));
    *s = d;
    return PRC_OK;
}

// ---- LS_Filter_SVD (lssvd.cuh) ----------------------------------------------------------------------------------------
constexpr size_t SVD_WS_BUDGET = 4ull << 30;     // A and Z of frames whose matrices exceed shared memory, per launch

int ls_svd_check(long long n, int filter_len, int peek) {
    if (n <= 0 || n >= (1ll << 31) - 4096) return fail(PRC_E_INVALID, "n=%lld unsupported", n);
    if (filter_len < 0 || peek < 0) return fail(PRC_E_INVALID, "filter_len=%d peek=%d invalid", filter_len, peek);
    const long long M = (long long)filter_len + peek;
    if (M < 1) return fail(PRC_E_INVALID, "filter_len + peek = 0: no taps");
    if (M > lssvd::MAX_M)
        return fail(PRC_E_INVALID, "%lld taps exceed the SVD filter's maximum of %d", M, lssvd::MAX_M);
    return PRC_OK;
}

// bt.nf frames: lag sums -> eigendecomposition and pseudo-inverse per frame -> residual; ranks to rank (device)
int ls_svd_device(Ctx* c, const float2* ref, const float2* srv, long long n, Batch bt, int filter_len, int peek,
                  float2* out, float2* taps_out, int* rank) {
    const int M = filter_len + peek;
    const lssvd::CorrGeo cg = lssvd::corr_geo(n, M);
    TRY(c->svd_part.ensure((size_t)bt.nf * 2 * M * cg.nparts * sizeof(double2)));
    TRY(c->svd_cr.ensure((size_t)bt.nf * 2 * M * sizeof(double2)));
    TRY(c->svd_taps.ensure((size_t)bt.nf * M * sizeof(double2)));
    {
        ProfScope ps(c, K_SVD_CORR);
        lssvd::CorrParams p{};
        p.ref = ref; p.srv = srv; p.n = n; p.stride = bt.stride; p.M = M; p.peek = peek;
        p.span = cg.span; p.nparts = cg.nparts; p.ntiles = cg.ntiles;
        p.part = c->svd_part.as<double2>();
        lssvd::launch_corr(p, bt.nf, c->stream);
        TRY(check_launch("svd_corr_kernel"));
        lssvd::launch_reduce(p.part, cg.nparts, (long long)bt.nf * 2 * M, c->svd_cr.as<double2>(), c->stream);
        TRY(check_launch("svd_reduce_kernel"));
    }
    {
        ProfScope ps(c, K_SVD_EIG);
        const lssvd::EigGeo eg = lssvd::eig_geo(M, SMEM_LIMIT - 2 * lssvd::MAX_M * sizeof(double) - 64);      // s_rot and flags are static
        const size_t per = (eg.a_smem ? 0 : (size_t)M * M * sizeof(double2)) + (eg.z_smem ? 0 : (size_t)M * M * sizeof(double));
        const int group = per ? (int)std::max<size_t>(1, std::min<size_t>(bt.nf, SVD_WS_BUDGET / per)) : bt.nf;
        if (per) TRY(c->svd_ws.ensure((size_t)group * per));
        for (int f0 = 0; f0 < bt.nf; f0 += group) {
            lssvd::EigParams p{};
            p.cr = c->svd_cr.as<double2>() + (size_t)f0 * 2 * M;
            p.M = M;
            p.nframes = std::min(group, bt.nf - f0);
            p.a_smem = eg.a_smem; p.z_smem = eg.z_smem;
            p.gA = eg.a_smem ? nullptr : c->svd_ws.as<double2>();
            p.gZ = eg.z_smem ? nullptr : reinterpret_cast<double*>(c->svd_ws.as<char>() + (eg.a_smem ? 0 : (size_t)group * M * M * sizeof(double2)));
            p.taps = c->svd_taps.as<double2>() + (size_t)f0 * M;
            p.taps_out = taps_out ? taps_out + (size_t)f0 * M : nullptr;
            p.rank = rank + f0;
            lssvd::launch_eig(p, eg, c->stream);
            TRY(check_launch("svd_eig_kernel"));
        }
    }
    ProfScope ps(c, K_SVD_FIR);
    lssvd::FirParams p{};
    p.ref = ref; p.srv = srv; p.out = out; p.n = n; p.stride = bt.stride; p.M = M; p.peek = peek;
    p.taps = c->svd_taps.as<double2>();
    lssvd::launch_fir(p, bt.nf, c->stream);
    return check_launch("svd_fir_kernel");
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

// ---- Welch PSD (spectrum.cuh) -----------------------------------------------------------------------------------
constexpr size_t PSD_PART_BUDGET = 256u << 20;     // partial spectra of one launch; larger batches run in groups

// nframes frames -> their spectra: twiddles once, then per group of frames the segment transforms and the finishing
// sums.  The groups only bound the scratch: a frame's chunks and its finishing sum do not depend on them.
int psd_device(Ctx* c, const void* x, int dt, long long n, int nframes, long long stride, int nfft, int noverlap, int m,
               const double* win, double scale, int onesided, double* out, long long out_stride) {
    using namespace spec;
    const long long P = 1ll << m, step = nfft - noverlap;
    const long long nseg = n < nfft ? 1 : (n - noverlap) / step;      // mlab zero-pads a short frame to one segment
    const long long per_cta = segments_per_cta(nseg);
    const int nchunk = (int)((nseg + per_cta - 1) / per_cta);
    const size_t frame_part = (size_t)nchunk * P * sizeof(double);
    const size_t fit = std::max<size_t>(1, PSD_PART_BUDGET / frame_part);
    const int group = (int)std::min<size_t>(std::min<size_t>((size_t)nframes, 65535), fit);
    AsyncScratch ws(c->stream);
    double2* tw;
    double* part;
    TRY(ws.get(&tw, (size_t)(P / 2) * sizeof(double2)));
    TRY(ws.get(&part, frame_part * group));
    SegParams sp{};
    sp.x = x; sp.dt = dt; sp.n = n; sp.stride = stride;
    sp.nfft = nfft; sp.m = m; sp.step = step; sp.nseg = nseg; sp.per_cta = per_cta; sp.nchunk = nchunk;
    sp.win = win; sp.tw = tw; sp.part = part;
    FinParams fp{};
    fp.part = part; fp.m = m; fp.nchunk = nchunk;
    fp.nbins = onesided ? P / 2 + 1 : P;
    fp.onesided = onesided;
    fp.nyq_double = nfft & 1;
    fp.scale = scale;
    fp.inv_nseg = 1.0 / (double)nseg;
    fp.out = out; fp.out_stride = out_stride;
    {
        ProfScope ps(c, K_PSD_SEGMENTS);
        launch_twiddle(tw, m, c->stream);
    }
    TRY(check_launch("spec_twiddle_kernel"));
    for (int f0 = 0; f0 < nframes; f0 += group) {
        const int nf = std::min(group, nframes - f0);
        sp.f0 = fp.f0 = f0;
        {
            ProfScope ps(c, K_PSD_SEGMENTS);
            launch_segments(sp, nf, c->stream);
        }
        TRY(check_launch("spec_segments_kernel"));
        {
            ProfScope ps(c, K_PSD_FINISH);
            launch_finish(fp, nf, c->stream);
        }
        TRY(check_launch("spec_finish_kernel"));
    }
    return PRC_OK;
}

// ---- FIR decimator and normalize (decimate.cuh) ------------------------------------------------------------------
// nrows rows of n samples -> ceil(n / q) outputs each: the taps to the device in the accumulator's precision, then one
// launch per 65535 rows (grid.y); a row's result does not depend on which launch it is in.
int decimate_device(Ctx* c, dec::DecParams p, int acc, int nrows, const double* taps) {
    using namespace dec;
    const size_t nt = (size_t)20 * p.q + 1;
    AsyncScratch ws(c->stream);
    if (acc == 0 || acc == 1) {
        std::vector<float> t32(nt);
        for (size_t j = 0; j < nt; ++j) t32[j] = (float)taps[j];
        float* d;
        TRY(ws.get(&d, nt * sizeof(float)));
        CU(cudaMemcpyAsync(d, t32.data(), nt * sizeof(float), cudaMemcpyHostToDevice, c->stream));
        p.taps = d;
    } else {
        double* d;
        TRY(ws.get(&d, nt * sizeof(double)));
        CU(cudaMemcpyAsync(d, taps, nt * sizeof(double), cudaMemcpyHostToDevice, c->stream));
        p.taps = d;
    }
    for (int r0 = 0; r0 < nrows; r0 += 65535) {
        {
            ProfScope ps(c, K_DECIMATE);
            launch_decimate(p, acc, r0, std::min(65535, nrows - r0), c->stream);
        }
        TRY(check_launch("dec_kernel"));
    }
    return PRC_OK;
}

int normalize_device(Ctx* c, const void* x, int dt, long long n, void* y) {
    using namespace dec;
    NormParams p{};
    p.x = x; p.dt = dt; p.n = n; p.y = y;
    p.nctas = norm_ctas(n);
    p.per_cta = (n + p.nctas - 1) / p.nctas;
    AsyncScratch ws(c->stream);
    TRY(ws.get(&p.part, (size_t)p.nctas * sizeof(double)));
    {
        ProfScope ps(c, K_NORM_SUM);
        launch_norm_sum(p, c->stream);
    }
    TRY(check_launch("norm_sum_kernel"));
    {
        ProfScope ps(c, K_NORM_SCALE);
        launch_norm_scale(p, c->nsm, c->stream);
    }
    return check_launch("norm_scale_kernel");
}

}  // namespace

// =========================================================================== C ABI
extern "C" {

int prc_version(void) { return PRC_VERSION; }

const char* prc_last_error(void) { return g_err.c_str(); }

int prc_device_count(int* count) {
    if (!count) return fail(PRC_E_INVALID, "count is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        *count = 0;
        return fail(PRC_E_CUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    }
    *count = n;
    return PRC_OK;
}

int prc_init(int device) {
    Ctx* c;
    return get_ctx(device, nullptr, &c);
}

void prc_shutdown(void) {
    std::lock_guard<std::mutex> lk(g_mu);
    for (Ctx* c : g_all_ctx) {
        c->release();
        delete c;
    }
    g_all_ctx.clear();
    g_stream_ctx.clear();
    g_epoch.fetch_add(1);
}

int prc_sync(int device, void* stream) {
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    CU(cudaStreamSynchronize(c->stream));
    return PRC_OK;
}

uint64_t prc_launch_count(void) { return g_launches.load(); }

int prc_profile_enable(int on) {
    g_prof_on.store(on ? 1 : 0);
    return PRC_OK;
}

// Drains every workspace's pending event pairs (synchronising their streams) into the totals.
int prc_profile_collect(void) {
    std::lock_guard<std::mutex> lk(g_mu);
    std::lock_guard<std::mutex> lp(g_prof_mu);
    for (Ctx* c : g_all_ctx) {
        std::lock_guard<std::mutex> lc(c->mu);
        if (c->recs.empty()) continue;
        cudaSetDevice(c->device);
        for (ProfRec& r : c->recs) {
            cudaEventSynchronize(r.b);
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
                g_prof_ms[r.id] += ms;
                g_prof_n[r.id] += 1;
            }
            cudaEventDestroy(r.a);
            cudaEventDestroy(r.b);
        }
        c->recs.clear();
    }
    return PRC_OK;
}

int prc_profile_kernels(void) { return K_COUNT; }

int prc_profile_read(int idx, const char** name, double* total_ms, uint64_t* launches) {
    if (idx < 0 || idx >= K_COUNT) return fail(PRC_E_INVALID, "kernel index %d out of range", idx);
    std::lock_guard<std::mutex> lp(g_prof_mu);
    if (name) *name = kKernelNames[idx];
    if (total_ms) *total_ms = g_prof_ms[idx];
    if (launches) *launches = g_prof_n[idx];
    return PRC_OK;
}

int prc_profile_reset(void) {
    std::lock_guard<std::mutex> lp(g_prof_mu);
    for (int i = 0; i < K_COUNT; ++i) { g_prof_ms[i] = 0; g_prof_n[i] = 0; }
    return PRC_OK;
}

int prc_host_alloc(void** ptr, uint64_t bytes) {
    if (!ptr) return fail(PRC_E_INVALID, "ptr is NULL");
    CU(cudaHostAlloc(ptr, bytes ? bytes : 1, cudaHostAllocPortable));
    return PRC_OK;
}
int prc_host_free(void* ptr) {
    CU(cudaFreeHost(ptr));
    return PRC_OK;
}
int prc_host_register(void* ptr, uint64_t bytes) {
    CU(cudaHostRegister(ptr, bytes, cudaHostRegisterPortable));
    return PRC_OK;
}
int prc_host_unregister(void* ptr) {
    CU(cudaHostUnregister(ptr));
    return PRC_OK;
}

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

int prc_nlms_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int filter_len, int peek, float mu,
                 int block_len, const prc_c64* init_taps, prc_c64* out, prc_c64* taps_out, int mem_kind,
                 int device, void* stream, unsigned flags) {
    return prc_nlms_frames_c64(ref, srv, n, 1, n, filter_len, peek, mu, block_len, init_taps, out, taps_out, mem_kind,
                               device, stream, flags);
}

int prc_nlms_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                        int filter_len, int peek, float mu, int block_len, const prc_c64* init_taps, prc_c64* out,
                        prc_c64* taps_out, int mem_kind, int device, void* stream, unsigned flags) {
    Batch bt;
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, nframes, frame_stride, &bt));
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t nb = (size_t)n * sizeof(float2), sb = (size_t)bt.stride * sizeof(float2);
    const int M = filter_len + peek;
    const size_t mb = (size_t)(M > 0 ? M : 1) * sizeof(float2);
    const float2 *dref, *dsrv, *dinit;
    float2 *dout, *dtaps;
    TRY(stage_in(c, ref, mem_kind, nframes, nb, sb, c->ref, flags, &dref));
    TRY(stage_in(c, srv, mem_kind, nframes, nb, sb, c->srv, flags, &dsrv));
    TRY(stage_in(c, init_taps, mem_kind, 1, mb, mb, c->nl_init, flags, &dinit));
    TRY(stage_out(out, mem_kind, nb * nframes, c->clean, &dout));
    TRY(stage_out(taps_out, mem_kind, mb * nframes, c->nl_taps, &dtaps));
    if (mem_kind == PRC_MEM_HOST) bt.stride = n;      // staged frames are packed
    TRY(nlms_device(c, dref, dsrv, n, filter_len, peek, mu, block_len, dinit, dout, dtaps, bt, true));
    TRY(unstage(c, out, dout, mem_kind, nframes, nb, sb, flags));
    TRY(unstage(c, taps_out, dtaps, mem_kind, 1, mb * nframes, mb * nframes, flags));
    return finish(c, flags);
}

int prc_gal_jpe_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                           int lattice_len, int delay_line_len, double mu1, double mu2, int peek,
                           prc_c64* out, prc_c64* k_out, prc_c64* h_out,
                           int mem_kind, int device, void* stream, unsigned flags) {
    Batch bt;
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, nframes, frame_stride, &bt));
    TRY(gal_check(n, lattice_len, delay_line_len, peek));      // before any CUDA call
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t nb = (size_t)n * sizeof(float2), sb = (size_t)bt.stride * sizeof(float2);
    const size_t db = (size_t)delay_line_len * sizeof(float2);
    const float2 *dref, *dsrv;
    float2 *dout, *dk, *dh;
    TRY(stage_in(c, ref, mem_kind, nframes, nb, sb, c->ref, flags, &dref));
    TRY(stage_in(c, srv, mem_kind, nframes, nb, sb, c->srv, flags, &dsrv));
    TRY(stage_out(out, mem_kind, nb * nframes, c->clean, &dout));
    TRY(stage_out(k_out, mem_kind, db * nframes, c->gal_k, &dk));
    TRY(stage_out(h_out, mem_kind, db * nframes, c->gal_h, &dh));
    if (mem_kind == PRC_MEM_HOST) bt.stride = n;      // staged frames are packed
    TRY(gal_device(c, dref, dsrv, n, bt, lattice_len, delay_line_len, mu1, mu2, peek, dout, dk, dh));
    TRY(unstage(c, out, dout, mem_kind, nframes, nb, sb, flags));
    TRY(unstage(c, k_out, dk, mem_kind, 1, db * nframes, db * nframes, flags));
    TRY(unstage(c, h_out, dh, mem_kind, 1, db * nframes, db * nframes, flags));
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

int prc_ls_status(int device, void* stream, int* status, int nframes) {
    if (!status || nframes < 1) return fail(PRC_E_INVALID, "status must not be NULL, nframes >= 1");
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->status.cap < (size_t)nframes * sizeof(int)) return fail(PRC_E_INVALID, "no LS solve of %d frames has run on this stream", nframes);
    CU(cudaMemcpyAsync(status, c->status.p, (size_t)nframes * sizeof(int), cudaMemcpyDeviceToHost, /*status*/ c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return PRC_OK;
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

int prc_iq_mix_c64(const void* in, int in_kind, int64_t n, int mode, double fc, double fs, double phase_offset,
                   prc_c64* out, int mem_kind, int device, void* stream, unsigned flags) {
    if (!in || !out) return fail(PRC_E_INVALID, "in/out must not be NULL");
    TRY(frontend_args(mem_kind, n, in_kind, mode, fs));
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t ib = iq_bytes(in_kind, n), ob = (size_t)n * sizeof(float2);
    const void* din;
    float2* dout;
    TRY(stage_in(c, in, mem_kind, 1, ib, ib, c->fe_in, flags, &din));
    TRY(stage_out(out, mem_kind, ob, c->fe_out, &dout));
    TRY(mix_chunks_device(c, K_MISC, chunk_params(make_mix(din, in_kind, n, mode, fc, fs, phase_offset), 1, 0, nullptr, 0),
                          dout));
    TRY(unstage(c, out, dout, mem_kind, 1, ob, ob, flags));
    return finish(c, flags);
}

int prc_resample_out_len(int64_t n_in, int up, int down, int nh, int64_t* n_out) {
    if (!n_out) return fail(PRC_E_INVALID, "n_out must not be NULL");
    ResampleGeo g;
    TRY(resample_geo(n_in, up, down, nh, &g));
    *n_out = g.n_out;
    return PRC_OK;
}

int prc_frontend_c64(const void* in, int in_kind, int64_t n, int mode, double fc, double fs, double phase_offset,
                     int up, int down, const double* h, int nh, prc_c64* out, int64_t out_capacity,
                     int mem_kind, int device, void* stream, unsigned flags) {
    if (!in || !out || !h) return fail(PRC_E_INVALID, "in/out/h must not be NULL");
    TRY(frontend_args(mem_kind, n, in_kind, mode, fs));
    ResampleGeo g;
    TRY(resample_geo(n, up, down, nh, &g));
    if (out_capacity < g.n_out) return fail(PRC_E_INVALID, "out holds %lld samples, %lld needed", (long long)out_capacity, g.n_out);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t ib = iq_bytes(in_kind, n);
    const void* din;
    float2* dout;
    TRY(stage_in(c, in, mem_kind, 1, ib, ib, c->fe_in, flags, &din));
    TRY(stage_out(out, mem_kind, (size_t)g.n_out * sizeof(float2), c->fe_out, &dout));
    TRY(frontend_device(c, K_MISC, chunk_params(make_mix(din, in_kind, n, mode, fc, fs, phase_offset), 1, 0, nullptr, 0), g,
                        h, nh, dout));
    TRY(unstage(c, out, dout, mem_kind, 1, (size_t)g.n_out * sizeof(float2), (size_t)g.n_out * sizeof(float2), flags));
    return finish(c, flags);
}

int prc_frontend_chunks_c64(const void* in, int in_kind, int64_t n, int nchunks, int64_t chunk_stride, int mode,
                            double fc, double fs, const double* phase_offsets, int up, int down, const double* h, int nh,
                            prc_c64* out, int64_t out_stride, int64_t out_capacity, int mem_kind, int device,
                            void* stream, unsigned flags) {
    if (!in || !out || !h || !phase_offsets) return fail(PRC_E_INVALID, "in/out/h/phase_offsets must not be NULL");
    TRY(frontend_args(mem_kind, n, in_kind, mode, fs));
    if (nchunks < 1 || nchunks > 65535) return fail(PRC_E_INVALID, "nchunks=%d outside [1, 65535]", nchunks);
    if (nchunks > 1 && chunk_stride < 0) return fail(PRC_E_INVALID, "chunk_stride=%lld invalid", (long long)chunk_stride);
    ResampleGeo g;
    TRY(resample_geo(n, up, down, nh, &g));
    if (nchunks > 1 && out_stride < g.n_out)
        return fail(PRC_E_INVALID, "out_stride=%lld smaller than the %lld samples of one chunk", (long long)out_stride, g.n_out);
    const long long ostride = nchunks > 1 ? out_stride : g.n_out;
    const long long cstride = nchunks > 1 ? chunk_stride : n;
    const long long need = (long long)(nchunks - 1) * ostride + g.n_out;
    if (out_capacity < need) return fail(PRC_E_INVALID, "out holds %lld samples, %lld needed", (long long)out_capacity, need);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t ib = iq_bytes(in_kind, (long long)(nchunks - 1) * cstride + n), cb = (size_t)g.n_out * sizeof(float2);
    const void* din;
    float2* dout;
    TRY(stage_in(c, in, mem_kind, 1, ib, ib, c->fe_in, flags, &din));
    TRY(stage_out(out, mem_kind, nchunks * cb, c->fe_out, &dout));
    const long long dstride = mem_kind == PRC_MEM_HOST ? g.n_out : ostride;      // staged chunks are packed
    TRY(copy_params(c, phase_offsets, nchunks, c->fe_po));
    TRY(frontend_device(c, K_FRONTEND_CHUNKS,
                        chunk_params(make_mix(din, in_kind, n, mode, fc, fs, 0.0), nchunks, cstride, c->fe_po.as<double>(),
                                     dstride),
                        g, h, nh, dout));
    TRY(unstage(c, out, dout, mem_kind, nchunks, cb, (size_t)ostride * sizeof(float2), flags));
    return finish(c, flags);
}

int prc_cfar2d_f32(const void* x, int rows, int cols, int fw, int gw, const float* thresh, float* cr_out,
                   uint8_t* det_out, int mem_kind, int device, void* stream, unsigned flags) {
    if (!x || (!cr_out && !det_out)) return fail(PRC_E_INVALID, "x and one of cr_out/det_out must not be NULL");
    if (det_out && !thresh) return fail(PRC_E_INVALID, "det_out needs a threshold");
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    CfarParams p;
    TRY(cfar_window(rows, cols, fw, gw, &p));
    const bool cplx = (flags & PRC_FLAG_ABS_C64) != 0;
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t cells = (size_t)rows * cols, inb = cells * (cplx ? sizeof(float2) : sizeof(float));
    TRY(stage_in(c, x, mem_kind, 1, inb, inb, c->rd_in, flags, &p.x));
    TRY(stage_out(cr_out, mem_kind, cells * sizeof(float), c->rd_out, &p.cr));
    TRY(stage_out(det_out, mem_kind, cells, c->rd_det, &p.det));
    p.is_complex = cplx ? 1 : 0;
    p.thresh = thresh ? *thresh : 0.f;
    TRY(cfar_frames_device(c, K_MISC, p, 1));
    TRY(unstage(c, cr_out, p.cr, mem_kind, 1, cells * sizeof(float), cells * sizeof(float), flags));
    TRY(unstage(c, det_out, p.det, mem_kind, 1, cells, cells, flags));
    return finish(c, flags);
}

int prc_cfar2d_frames(const void* x, int rows, int cols, int nframes, int64_t frame_stride, int fw, int gw,
                      void* cr_out, int64_t cr_stride, int mem_kind, int device, void* stream, unsigned flags) {
    if (!x || !cr_out) return fail(PRC_E_INVALID, "x and cr_out must not be NULL");
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    CfarParams p;
    TRY(cfar_window(rows, cols, fw, gw, &p));
    if (nframes < 0 || nframes > 65535) return fail(PRC_E_INVALID, "nframes=%d outside [0, 65535]", nframes);
    const long long cells = (long long)rows * cols;
    if (nframes > 1 && (frame_stride < cells || cr_stride < cells))
        return fail(PRC_E_INVALID, "frame_stride=%lld / cr_stride=%lld smaller than the %lld cells of a map",
                    (long long)frame_stride, (long long)cr_stride, cells);
    const bool cplx = (flags & PRC_FLAG_ABS_C64) != 0, f64 = (flags & PRC_FLAG_CR_F64) != 0;
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    if (nframes == 0) return finish(c, flags);
    const size_t ine = cplx ? sizeof(float2) : sizeof(float), oute = f64 ? sizeof(double) : sizeof(float);
    const long long xs = nframes > 1 ? frame_stride : cells, os = nframes > 1 ? cr_stride : cells;
    TRY(stage_in(c, x, mem_kind, nframes, cells * ine, xs * ine, c->rd_in, flags, &p.x));
    TRY(stage_out(cr_out, mem_kind, (size_t)nframes * cells * oute, c->rd_out, &p.cr));
    p.is_complex = cplx ? 1 : 0;
    p.frame_stride = mem_kind == PRC_MEM_HOST ? cells : xs;      // staged frames are packed
    p.out_stride = mem_kind == PRC_MEM_HOST ? cells : os;
    p.cr_f64 = f64 ? 1 : 0;
    TRY(cfar_frames_device(c, K_CFAR_FRAMES, p, nframes));
    TRY(unstage(c, cr_out, p.cr, mem_kind, nframes, cells * oute, os * oute, flags));
    return finish(c, flags);
}

int prc_persistence_frames(const void* x, int rows, int cols, int nframes, int64_t frame_stride, int n_carry, int hold,
                           const double* weights, double* out, int mem_kind, int device, void* stream, unsigned flags) {
    if (!x || !out || !weights) return fail(PRC_E_INVALID, "x/weights/out must not be NULL");
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    if (rows < 1 || cols < 1) return fail(PRC_E_INVALID, "rows=%d cols=%d invalid", rows, cols);
    if ((rows + rdr::PST_TY - 1) / rdr::PST_TY > 65535)
        return fail(PRC_E_INVALID, "rows=%d exceed the persistence maximum of %d rows", rows, 65535 * rdr::PST_TY);
    if (hold < 1) return fail(PRC_E_INVALID, "hold=%d must be >= 1", hold);
    if (nframes < 0) return fail(PRC_E_INVALID, "nframes=%d invalid", nframes);
    if (n_carry < 0 || n_carry > hold - 1)
        return fail(PRC_E_INVALID, "n_carry=%d outside [0, hold - 1 = %d]", n_carry, hold - 1);
    const long long cells = (long long)rows * cols;
    const int total = n_carry + nframes;
    if (total > 1 && frame_stride < cells)
        return fail(PRC_E_INVALID, "frame_stride=%lld smaller than the %lld cells of a map", (long long)frame_stride, cells);
    const bool f64 = (flags & PRC_FLAG_MAP_F64) != 0, prod32 = (flags & PRC_FLAG_PROD_F32) != 0;
    if (f64 && prod32) return fail(PRC_E_INVALID, "float32 products need a float32 stack (PRC_FLAG_MAP_F64 is set)");
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    if (nframes == 0) return finish(c, flags);
    TRY(copy_params(c, weights, std::min(hold, total), c->rd_w));      // the weights the call uses
    rdr::PersistParams p{};
    const size_t ine = f64 ? sizeof(double) : sizeof(float);
    const long long xs = total > 1 ? frame_stride : cells;
    const size_t ob = (size_t)nframes * cells * sizeof(double);
    TRY(stage_in(c, x, mem_kind, total, cells * ine, xs * ine, c->rd_in, flags, &p.x));
    TRY(stage_out(out, mem_kind, ob, c->rd_out, &p.out));
    p.frame_stride = mem_kind == PRC_MEM_HOST ? cells : xs;      // staged frames are packed
    p.f64 = f64 ? 1 : 0;
    p.f32prod = prod32 ? 1 : 0;
    p.oriented = (flags & PRC_FLAG_ORIENT) ? 1 : 0;
    p.rows = rows; p.cols = cols;
    p.n_carry = n_carry; p.nframes = nframes; p.hold = hold;
    p.w = c->rd_w.as<double>();
    {
        ProfScope ps(c, K_PERSISTENCE);
        rdr::launch_persistence(p, c->stream);
    }
    TRY(check_launch("pst_kernel"));
    TRY(unstage(c, out, p.out, mem_kind, 1, ob, ob, flags));
    return finish(c, flags);
}

int prc_percentiles_frames(const double* x, int64_t n, int nframes, int64_t frame_stride, const double* q,
                           const double* scale, int nq, double* out, int mem_kind, int device, void* stream,
                           unsigned flags) {
    if (!x || !out || !q) return fail(PRC_E_INVALID, "x/q/out must not be NULL");
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    if (n < 1 || n > rdr::PCT_MAX_N) return fail(PRC_E_INVALID, "n=%lld outside [1, %d]", (long long)n, rdr::PCT_MAX_N);
    if (nq < 1 || nq > rdr::PCT_MAX_Q) return fail(PRC_E_INVALID, "nq=%d outside [1, %d]", nq, rdr::PCT_MAX_Q);
    if (nframes < 0) return fail(PRC_E_INVALID, "nframes=%d invalid", nframes);
    if (nframes > 1 && frame_stride < n)
        return fail(PRC_E_INVALID, "frame_stride=%lld smaller than n=%lld", (long long)frame_stride, (long long)n);
    rdr::PctParams p{};
    p.n = (int)n;
    p.nq = nq;
    for (int j = 0; j < nq; ++j) {
        if (!(q[j] >= 0.0 && q[j] <= 100.0)) return fail(PRC_E_INVALID, "q[%d]=%g outside [0, 100]", j, q[j]);
        // np.percentile on float64 data, linear method: v = (n - 1) * (q / 100.0); order statistics floor(v) and
        // floor(v) + 1, gamma = v - floor(v).  From v >= n - 1 on both are the maximum and NumPy's gamma is v + 1.
        const double v = (double)(n - 1) * (q[j] / 100.0);
        if (v >= (double)(n - 1)) {
            p.k[j] = (int)(n - 1);
            p.g[j] = v + 1.0;
        } else {
            p.k[j] = (int)std::floor(v);
            p.g[j] = v - std::floor(v);
        }
        p.scale[j] = scale ? scale[j] : 1.0;
    }
    p.has_scale = scale ? 1 : 0;
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    if (nframes == 0) return finish(c, flags);
    const long long xs = nframes > 1 ? frame_stride : n;
    const size_t ob = (size_t)nframes * nq * sizeof(double);
    TRY(stage_in(c, x, mem_kind, nframes, (size_t)n * sizeof(double), xs * sizeof(double), c->rd_in, flags, &p.x));
    TRY(stage_out(out, mem_kind, ob, c->rd_out, &p.out));
    p.frame_stride = mem_kind == PRC_MEM_HOST ? n : xs;      // staged frames are packed
    {
        ProfScope ps(c, K_PERCENTILE);
        rdr::launch_percentiles(p, nframes, c->stream);
    }
    TRY(check_launch("pct_kernel"));
    TRY(unstage(c, out, p.out, mem_kind, 1, ob, ob, flags));
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

int prc_get_measurements_frames(const void* maps, int rows, int cols, int nseq, int nframes, int64_t seq_stride,
                                int64_t frame_stride, double doppler_extent, double range_extent,
                                int64_t meas_capacity, int32_t* counts, double* meas,
                                int mem_kind, int device, void* stream, unsigned flags) {
    TRY(trk_check(maps, rows, cols, nseq, nframes, seq_stride, frame_stride, mem_kind));
    if (!counts) return fail(PRC_E_INVALID, "counts must not be NULL");
    if (meas_capacity < 0 || (meas_capacity > 0 && !meas))
        return fail(PRC_E_INVALID, "meas_capacity=%lld needs a meas buffer", (long long)meas_capacity);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    TrkMapParams mp;
    TRY(trk_stage(c, maps, rows, cols, nseq, nframes, seq_stride, frame_stride, mem_kind, flags, &mp));
    trk_extent(&mp, doppler_extent, range_extent);
    const size_t nfr = (size_t)nseq * nframes;
    const size_t ob = nfr * 3 * (size_t)meas_capacity * sizeof(double);
    TRY(c->trk_stats.ensure(nfr * 2 * sizeof(double)));
    mp.mean = c->trk_stats.as<double>();
    mp.thr = mp.mean + nfr;
    TRY(stage_out(counts, mem_kind, nfr * sizeof(int), c->trk_cnt, &mp.count));
    TRY(stage_out(meas, mem_kind, ob, c->trk_out, &mp.out));
    mp.f0 = 0;
    mp.out_cap = meas_capacity;
    mp.out_nf = nframes;
    TRY(trk_meas_launch(c, mp, (flags & PRC_FLAG_MAP_F64) != 0, TRK_MODE_MEAS, nframes, nseq));
    TRY(unstage(c, counts, mp.count, mem_kind, 1, nfr * sizeof(int), nfr * sizeof(int), flags));
    TRY(unstage(c, ob ? meas : nullptr, mp.out, mem_kind, 1, ob, ob, flags));
    return finish(c, flags);
}

int prc_multitarget_track_frames(const void* maps, int rows, int cols, int nseq, int nframes, int64_t seq_stride,
                                 int64_t frame_stride, double doppler_extent, double range_extent, int n_tracks,
                                 prc_track* history, int mem_kind, int device, void* stream, unsigned flags) {
    TRY(trk_check(maps, rows, cols, nseq, nframes, seq_stride, frame_stride, mem_kind));
    if (n_tracks < 0 || n_tracks > TRK_MAX_TRACKS)
        return fail(PRC_E_INVALID, "n_tracks=%d outside [0, %d], the multi-target tracker's maximum", n_tracks,
                    TRK_MAX_TRACKS);
    if (n_tracks > 0 && !history) return fail(PRC_E_INVALID, "history must not be NULL");
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    if (n_tracks == 0) return finish(c, flags);
    TrkMapParams mp;
    TRY(trk_stage(c, maps, rows, cols, nseq, nframes, seq_stride, frame_stride, mem_kind, flags, &mp));
    trk_extent(&mp, doppler_extent, range_extent);
    const bool f64 = (flags & PRC_FLAG_MAP_F64) != 0;
    const size_t nfr = (size_t)nseq * nframes;
    const size_t slot = 3 * (size_t)mp.cap * sizeof(double);
    const int fc = (int)std::max<size_t>(1, std::min<size_t>(nframes, TRK_SLOT_BUDGET / (slot * nseq)));
    TRY(c->trk_stats.ensure(nfr * (2 * sizeof(double) + sizeof(int))));
    TRY(c->trk_slots.ensure((size_t)nseq * fc * slot));
    mp.mean = c->trk_stats.as<double>();
    mp.thr = mp.mean + nfr;
    mp.count = reinterpret_cast<int*>(mp.thr + nfr);
    mp.out = c->trk_slots.as<double>();
    mp.out_cap = mp.cap;
    mp.out_nf = fc;
    const size_t hb = nfr * n_tracks * sizeof(prc_track);
    prc_track* dh;
    TRY(stage_out(history, mem_kind, hb, c->trk_out, &dh));
    const bool resume = (flags & PRC_FLAG_TRACK_RESUME) != 0;
    if (resume && mem_kind == PRC_MEM_HOST)
        TRY(trk_resume_h2d(c, dh, history, nseq, (size_t)nframes * n_tracks * sizeof(prc_track),
                           (size_t)n_tracks * sizeof(prc_track), flags));
    for (int f0 = 0; f0 < nframes; f0 += fc) {
        const int nf = std::min(fc, nframes - f0);
        mp.f0 = f0;
        TRY(trk_meas_launch(c, mp, f64, TRK_MODE_SLOTS, nf, nseq));
        TrkMultiParams tp{};
        tp.m = mp;
        tp.f64 = f64 ? 1 : 0;
        tp.hist = dh;
        tp.n_tracks = n_tracks;
        tp.f0 = f0;
        tp.f1 = f0 + nf;
        tp.slots = mp.out;
        tp.fc = fc;
        tp.resume = resume ? 1 : 0;
        {
            ProfScope ps(c, K_TRK_MULTI);
            track_multi_kernel<<<nseq, 32, 0, c->stream>>>(tp);
        }
        TRY(check_launch("track_multi_kernel"));
    }
    TRY(unstage(c, history, dh, mem_kind, 1, hb, hb, flags));
    return finish(c, flags);
}

int prc_simple_track_frames(const void* maps, int rows, int cols, int nseq, int nframes, int64_t seq_stride,
                            int64_t frame_stride, double range_extent, double doppler_extent,
                            prc_track_simple* history, int mem_kind, int device, void* stream, unsigned flags) {
    TRY(trk_check(maps, rows, cols, nseq, nframes, seq_stride, frame_stride, mem_kind));
    if (!history) return fail(PRC_E_INVALID, "history must not be NULL");
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    TrkMapParams mp;
    TRY(trk_stage(c, maps, rows, cols, nseq, nframes, seq_stride, frame_stride, mem_kind, flags, &mp));
    const bool f64 = (flags & PRC_FLAG_MAP_F64) != 0;
    const size_t nfr = (size_t)nseq * nframes;
    TRY(c->trk_stats.ensure(nfr * sizeof(double)));
    mp.mean = c->trk_stats.as<double>();
    TRY(trk_meas_launch(c, mp, f64, TRK_MODE_MEAN, nframes, nseq));
    const size_t hb = nfr * sizeof(prc_track_simple);
    prc_track_simple* dh;
    TRY(stage_out(history, mem_kind, hb, c->trk_out, &dh));
    const bool resume = (flags & PRC_FLAG_TRACK_RESUME) != 0;
    if (resume && mem_kind == PRC_MEM_HOST)
        TRY(trk_resume_h2d(c, dh, history, nseq, (size_t)nframes * sizeof(prc_track_simple), sizeof(prc_track_simple),
                           flags));
    TrkSimpleParams sp{};
    sp.m = mp;
    sp.hist = dh;
    sp.range_extent = range_extent;
    sp.doppler_extent = doppler_extent;
    py_slice(250, 260, rows, &sp.zlo, &sp.zhi);
    sp.resume = resume ? 1 : 0;
    {
        ProfScope ps(c, K_TRK_SIMPLE);
        if (f64) track_simple_kernel<double><<<nseq, TRK_SIMPLE_THREADS, 0, c->stream>>>(sp);
        else track_simple_kernel<float><<<nseq, TRK_SIMPLE_THREADS, 0, c->stream>>>(sp);
    }
    TRY(check_launch("track_simple_kernel"));
    TRY(unstage(c, history, dh, mem_kind, 1, hb, hb, flags));
    return finish(c, flags);
}

int prc_channel_offset(const void* s1, int dtype1, int64_t n1, const void* s2, int dtype2, int64_t n2, int nd, int64_t nl,
                       const double* sos, const double* zi, int64_t* offset, double* xc_abs,
                       int mem_kind, int device, void* stream, unsigned flags) {
    TRY(chanoff_inputs(s1, dtype1, n1, s2, dtype2, n2, mem_kind));
    if (!sos || !zi || !offset) return fail(PRC_E_INVALID, "sos/zi/offset must not be NULL");
    if (nd < 1 || nd > CHANOFF_MAX_ND) return fail(PRC_E_INVALID, "nd=%d outside [1, %d]", nd, CHANOFF_MAX_ND);
    if (nl < 0) return fail(PRC_E_INVALID, "nl=%lld invalid", (long long)nl);
    if (n1 <= chanoff::PADLEN || n2 <= chanoff::PADLEN)
        return fail(PRC_E_INVALID, "The length of the input vector x must be greater than padlen, which is %d.", chanoff::PADLEN);
    chanoff::Sos f[2];
    for (int q = 0; q < 2; ++q) {
        memcpy(f[q].s, sos + 24 * q, sizeof f[q].s);
        memcpy(f[q].zi, zi + 8 * q, sizeof f[q].zi);
        long long w;
        TRY(chanoff_warmup(f[q], &w));               // before any CUDA call
    }
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    AsyncScratch ws(c->stream);
    TRY(chanoff_stage(c, ws, &s1, dtype1, n1, mem_kind, flags));
    TRY(chanoff_stage(c, ws, &s2, dtype2, n2, mem_kind, flags));
    long long* res;
    TRY(ws.get(&res, 2 * sizeof(long long)));
    const long long n1d = (n1 + nd - 1) / nd, n2d = (n2 + nd - 1) / nd, lenb = n2d + 2 * nl;
    const long long nvalid = (n1d >= lenb ? n1d - lenb : lenb - n1d) + 1;
    double* xc = xc_abs;
    if (xc_abs && mem_kind == PRC_MEM_HOST) TRY(ws.get(&xc, (size_t)nvalid * sizeof(double)));
    TRY(chanoff_device(c, ws, s1, dtype1, n1, s2, dtype2, n2, f, nd, nl, nl, chanoff::ARG_ABS, xc, res));
    if (mem_kind == PRC_MEM_DEVICE) CU(cudaMemcpyAsync(offset, res + 1, sizeof(long long), cudaMemcpyDeviceToDevice, c->stream));
    TRY(unstage(c, offset, res + 1, mem_kind, 1, sizeof(long long), sizeof(long long), flags));
    TRY(unstage(c, xc_abs, xc, mem_kind, 1, (size_t)nvalid * sizeof(double), (size_t)nvalid * sizeof(double), flags));
    return finish(c, flags);
}

int prc_xcorr(const void* s1, int dtype1, int64_t n1, const void* s2, int dtype2, int64_t n2, int64_t nlead, int64_t nlag,
              void* out, int mem_kind, int device, void* stream, unsigned flags) {
    TRY(chanoff_inputs(s1, dtype1, n1, s2, dtype2, n2, mem_kind));
    if (!out) return fail(PRC_E_INVALID, "out must not be NULL");
    if (nlead < 0 || nlag < 0) return fail(PRC_E_INVALID, "nlead=%lld nlag=%lld invalid", (long long)nlead, (long long)nlag);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    AsyncScratch ws(c->stream);
    TRY(chanoff_stage(c, ws, &s1, dtype1, n1, mem_kind, flags));
    TRY(chanoff_stage(c, ws, &s2, dtype2, n2, mem_kind, flags));
    const bool cplx = chanoff::dt_complex(dtype1) || chanoff::dt_complex(dtype2);
    const long long lenb = n2 + nlag + nlead;
    const size_t ob = (size_t)((n1 >= lenb ? n1 - lenb : lenb - n1) + 1) * (cplx ? sizeof(double2) : sizeof(double));
    void* dout = out;
    if (mem_kind == PRC_MEM_HOST) TRY(ws.get(&dout, ob));
    TRY(chanoff_device(c, ws, s1, dtype1, n1, s2, dtype2, n2, nullptr, 1, nlag, nlead,
                       cplx ? chanoff::ARG_COMPLEX : chanoff::ARG_REAL, dout, nullptr));
    TRY(unstage(c, out, dout, mem_kind, 1, ob, ob, flags));
    return finish(c, flags);
}

int prc_ls_svd_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                          int filter_len, int peek, prc_c64* out, prc_c64* taps_out, int* rank_out,
                          int mem_kind, int device, void* stream, unsigned flags) {
    TRY(ls_svd_check(n, filter_len, peek));             // before any CUDA call
    Batch bt;
    TRY(stack_args(ref, srv, out, "ref/srv/out", mem_kind, n, nframes, frame_stride, &bt));
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const int M = filter_len + peek;
    const size_t nb = (size_t)n * sizeof(float2), sb = (size_t)bt.stride * sizeof(float2);
    const size_t mb = (size_t)M * sizeof(float2) * nframes, rb = (size_t)nframes * sizeof(int);
    const float2 *dref, *dsrv;
    float2 *dout, *dtaps;
    TRY(stage_in(c, ref, mem_kind, nframes, nb, sb, c->ref, flags, &dref));
    TRY(stage_in(c, srv, mem_kind, nframes, nb, sb, c->srv, flags, &dsrv));
    TRY(stage_out(out, mem_kind, nb * nframes, c->clean, &dout));
    TRY(stage_out(taps_out, mem_kind, mb, c->lstaps, &dtaps));
    int* drank;
    TRY(stage_out(rank_out, mem_kind, rb, c->svd_rank, &drank));
    if (!rank_out) {
        TRY(c->svd_rank.ensure(rb));
        drank = c->svd_rank.as<int>();
    }
    if (mem_kind == PRC_MEM_HOST) bt.stride = n;      // staged frames are packed
    TRY(ls_svd_device(c, dref, dsrv, n, bt, filter_len, peek, dout, dtaps, drank));
    TRY(unstage(c, out, dout, mem_kind, nframes, nb, sb, flags));
    TRY(unstage(c, taps_out, dtaps, mem_kind, 1, mb, mb, flags));
    TRY(unstage(c, rank_out, drank, mem_kind, 1, rb, rb, flags));
    return finish(c, flags);
}

int prc_psd_frames(const void* x, int dtype, int64_t n, int nframes, int64_t frame_stride, int nfft, int noverlap,
                   int pad_to, const double* window, double scale, int onesided, double* out, int64_t out_stride,
                   int device, void* stream, unsigned flags) {
    if (!x || !window || !out) return fail(PRC_E_INVALID, "x/window/out must not be NULL");
    if (!spec::dt_ok(dtype))
        return fail(PRC_E_INVALID, "dtype=%d invalid: PRC_DT_F32, PRC_DT_F64, PRC_DT_C64 or PRC_DT_C128", dtype);
    if (pad_to < (1 << spec::MIN_LOG2) || pad_to > (1 << spec::MAX_LOG2) || (pad_to & (pad_to - 1)))
        return fail(PRC_E_INVALID, "pad_to=%d must be a power of two in [%d, %d]", pad_to, 1 << spec::MIN_LOG2,
                    1 << spec::MAX_LOG2);
    if (nfft < 1 || nfft > pad_to) return fail(PRC_E_INVALID, "nfft=%d outside [1, pad_to=%d]", nfft, pad_to);
    if (noverlap < 0 || noverlap >= nfft) return fail(PRC_E_INVALID, "noverlap=%d outside [0, nfft=%d)", noverlap, nfft);
    if (n < 1) return fail(PRC_E_INVALID, "n=%lld invalid", (long long)n);
    if (nframes < 1) return fail(PRC_E_INVALID, "nframes=%d invalid", nframes);
    if (frame_stride < n)
        return fail(PRC_E_INVALID, "frame_stride=%lld smaller than n=%lld", (long long)frame_stride, (long long)n);
    if (onesided != 0 && onesided != 1) return fail(PRC_E_INVALID, "onesided=%d must be 0 or 1", onesided);
    const long long nbins = onesided ? pad_to / 2 + 1 : pad_to;
    if (out_stride < nbins)
        return fail(PRC_E_INVALID, "out_stride=%lld smaller than the %lld output bins", (long long)out_stride, nbins);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    TRY(psd_device(c, x, dtype, n, nframes, frame_stride, nfft, noverlap, ilog2(pad_to), window, scale, onesided, out,
                   out_stride));
    return finish(c, flags);
}

int prc_decimate_rows(const void* x, int src, int64_t n, int nrows, int64_t row_stride, int mode, double fc, double fs,
                      double phase_offset, const double* taps, int q, void* out, int64_t out_stride, int device,
                      void* stream, unsigned flags) {
    if (!x || !taps || !out) return fail(PRC_E_INVALID, "x/taps/out must not be NULL");
    const bool raw = src >= PRC_DEC_RAW;
    if (raw ? (src - PRC_DEC_RAW < PRC_IQ_C64 || src - PRC_DEC_RAW > PRC_IQ_I16) : (src < PRC_DT_I8 || src > PRC_DT_C128))
        return fail(PRC_E_INVALID, "src=%d invalid: a PRC_DT_* code, or PRC_DEC_RAW + PRC_IQ_C64 / PRC_IQ_I8 / PRC_IQ_I16",
                    src);
    if (raw && (mode < PRC_MIX_NONE || mode > PRC_MIX_FS64)) return fail(PRC_E_INVALID, "mode=%d invalid", mode);
    if (q < dec::MIN_Q || q > dec::MAX_Q)
        return fail(PRC_E_INVALID, "q=%d outside [%d, %d]: the decimation factor's limits", q, dec::MIN_Q, dec::MAX_Q);
    if (n < 1) return fail(PRC_E_INVALID, "n=%lld invalid", (long long)n);
    if (nrows < 1) return fail(PRC_E_INVALID, "nrows=%d invalid", nrows);
    if (nrows > 1 && row_stride < n)
        return fail(PRC_E_INVALID, "row_stride=%lld smaller than n=%lld", (long long)row_stride, (long long)n);
    const long long nout = (n + q - 1) / q;
    if (nrows > 1 && out_stride < nout)
        return fail(PRC_E_INVALID, "out_stride=%lld smaller than the %lld outputs per row", (long long)out_stride, nout);
    dec::DecParams p{};
    p.x = x; p.src = src; p.n = n; p.row_stride = row_stride; p.q = q; p.nout = nout;
    p.y = out; p.out_stride = out_stride;
    if (raw) p.mix = make_mix(x, src - PRC_DEC_RAW, n, mode, fc, fs, phase_offset);
    p.G = dec::group_lanes(q);
    dec::slab_geometry(q, p.G, &p.ks, &p.ksp, &p.nslab);
    const int acc = dec::acc_kind(src, raw ? mode : PRC_MIX_NONE);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    TRY(decimate_device(c, p, acc, nrows, taps));
    return finish(c, flags);
}

int prc_normalize(const void* x, int dtype, int64_t n, void* out, int device, void* stream, unsigned flags) {
    if (!x || !out) return fail(PRC_E_INVALID, "x/out must not be NULL");
    if (dtype < PRC_DT_I8 || dtype > PRC_DT_C128) return fail(PRC_E_INVALID, "dtype=%d invalid: a PRC_DT_* code", dtype);
    if (n < 1) return fail(PRC_E_INVALID, "n=%lld invalid", (long long)n);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    TRY(normalize_device(c, x, dtype, n, out));
    return finish(c, flags);
}

}  // extern "C"
