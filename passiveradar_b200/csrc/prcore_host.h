// prcore_host.h -- what the host modules of libprcore.so share: errors, workspaces, profiling scopes, launch checks,
// host staging and argument checks.  Internal; the C ABI is include/prcore.h.
//
// Threading model: one workspace ("Ctx") per (device, caller stream), or per (device, calling thread) when the caller
// passes stream == NULL.  A Ctx owns grow-only device buffers; all work of one call is enqueued on the Ctx's stream, so
// buffer reuse is ordered by the stream.  Nothing here falls back to the CPU.
//
// Modules (DESIGN.md section 3): prcore.cu (runtime), prcore_corr.cu, prcore_clutter.cu, prcore_signal.cu,
// prcore_detect.cu.  Each kernel header is included by exactly one of them; this header includes none.
#pragma once

#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <mutex>
#include <vector>

#include "prcore.h"

namespace prcore {

constexpr size_t SMEM_LIMIT = 200 * 1024;

// optional per-kernel timing (prc_profile_*): CUDA events on the launching stream around each launch
enum KernelId { K_LAGCORR_LS = 0, K_LEVINSON, K_FIR, K_LAGCORR_CAF, K_DOPPLER, K_NLMS, K_MISC, K_GAL, K_TRK_MEAS, K_TRK_MULTI,
                K_TRK_SIMPLE, K_CHANOFF_LOAD, K_CHANOFF_IIR, K_CHANOFF_FFT, K_CHANOFF_ARGMAX, K_SVD_CORR, K_SVD_EIG, K_SVD_FIR,
                K_CAF_COMBINE, K_FRONTEND_CHUNKS, K_CFAR_FRAMES, K_PERSISTENCE,
                K_PERCENTILE, K_PSD_SEGMENTS, K_PSD_FINISH, K_DECIMATE, K_NORM_SUM, K_NORM_SCALE, K_OS_CFAR, K_FRAME_MULTI, K_COUNT };
struct ProfRec { int id; cudaEvent_t a, b; };

int fail(int code, const char* fmt, ...);      // sets prc_last_error(); returns code

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
    DBuf() = default;
    DBuf(const DBuf&) = delete;
    DBuf& operator=(const DBuf&) = delete;
    ~DBuf() {
        if (p) cudaFree(p);
    }
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
    void* pin[2] = {nullptr, nullptr};      // page-locked bounce buffers for pageable host arrays (h2d / d2h)
    cudaEvent_t pin_ev[2] = {nullptr, nullptr};
    bool pin_ready = false;
    DBuf fft_tw[3], wp_fir, wp_caf, fftP;     // FFT-domain path: twiddle tables (L = 1024 / 2048 / 4096), taps spectra, CAF block sums
    DBuf fpacc;                               // one-pass frame: AccP / AccQ spectra per Doppler block [nf][F][2][L]
    DBuf mstatus;                             // frames of several channels: Toeplitz-solve status [nchan][nframes]
    bool fft_tw_ready[3] = {false, false, false};
    int fft_ctas[4][3] = {};  // CTAs per SM of the one-wave FFT-domain kernels, [FftKern][r3_index] (0: not asked yet)
    std::vector<ProfRec> recs;
    ~Ctx();       // prcore.cu
};

int get_ctx(int device, void* stream, Ctx** out);
int check_launch(const char* what);      // counts one launch (prc_launch_count) and reports a failed one

extern std::atomic<int> g_prof_on;
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

// A batch of frames: nf channels pairs `stride` samples apart (inputs), results laid out frame after frame.
struct Batch {
    int nf = 1;
    long long stride = 0;
};

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }
inline int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

// ---- host <-> device copies of caller arrays (prcore.cu)
int h2d(Ctx* c, void* dst, const void* src, size_t bytes, unsigned flags);
int d2h(Ctx* c, void* dst, const void* src, size_t bytes, unsigned flags);
int rows_h2d(Ctx* c, void* dst, const void* src, size_t rows, size_t row_bytes, size_t stride, unsigned flags);
int rows_d2h(Ctx* c, void* dst, const void* src, size_t rows, size_t row_bytes, size_t stride, unsigned flags);
int unstage(Ctx* c, void* dst, const void* src, int mem_kind, size_t rows, size_t row_bytes, size_t stride, unsigned flags);
int copy_params(Ctx* c, const double* src, int count, DBuf& buf);
int finish(Ctx* c, unsigned flags);

// ---- arguments and operands of the C entry points
int stack_args(const void* a, const void* b, const void* o, const char* names, int mem_kind, long long n, int nframes,
               long long frame_stride, Batch* bt, int range_bins = 0, int freq_bins = 1);
inline bool bad_mem_kind(int k) { return k != PRC_MEM_HOST && k != PRC_MEM_DEVICE; }

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

// ---- what the modules export to one another
// The shared-memory limits of each module's kernels (set_kernel_attrs, once per device)
int corr_set_attrs(int lim);
int clutter_set_attrs(int lim);
int signal_set_attrs(int lim);
int detect_set_attrs(int lim);

// frequency_shift of one complex64 channel through the front end's mix kernel (prcore_signal.cu), profiled as K_MISC:
// the rows of direct_xambg_device
int frequency_shift_device(Ctx* c, const float2* x, long long n, double fc, double fs, float2* out);

}  // namespace prcore
