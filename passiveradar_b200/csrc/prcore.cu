// prcore.cu -- runtime of libprcore.so: errors, workspaces and their teardown, kernel attributes, profiling, pinned
// host staging and argument checks, and the C entry points that belong to no operator family.  The operator families'
// host code lives in prcore_corr.cu, prcore_clutter.cu, prcore_signal.cu and prcore_detect.cu (prcore_host.h).
//
// Build (see passiveradar_b200/build.py):
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden \
//        -shared -Iinclude -o passiveradar_b200/libprcore.so prcore*.cu
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

#include "prcore_host.h"

namespace prcore {

thread_local std::string g_err;
std::atomic<uint64_t> g_launches{0};

const char* const kKernelNames[K_COUNT] = {"lagcorr_ls", "levinson", "fir_apply", "lagcorr_caf",
                                           "doppler_fft", "nlms", "misc", "gal_jpe", "track_meas",
                                           "track_multi", "track_simple", "chanoff_load", "chanoff_iir",
                                           "chanoff_fft", "chanoff_argmax", "svd_corr", "svd_eig", "svd_fir",
                                           "caf_combine", "frontend_chunks", "cfar_frames",
                                           "persistence", "percentile", "psd_segments", "psd_finish",
                                           "decimate", "norm_sum", "norm_scale", "os_cfar",
                                           "frame_multi"};
std::atomic<int> g_prof_on{0};
std::mutex g_prof_mu;
double g_prof_ms[K_COUNT] = {0};
uint64_t g_prof_n[K_COUNT] = {0};

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

// Waits for the work on the workspace's stream, then frees what it holds: pending profiling events, the page-locked
// bounce buffers, an owned stream and, through the members' destructors, every device buffer
Ctx::~Ctx() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    for (ProfRec& r : recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    if (pin_ready)
        for (int k = 0; k < 2; ++k) { cudaFreeHost(pin[k]); cudaEventDestroy(pin_ev[k]); }
    if (own_stream && stream) cudaStreamDestroy(stream);
}

std::mutex g_mu;
std::map<std::pair<int, void*>, Ctx*> g_stream_ctx;   // (device, caller stream)
std::vector<Ctx*> g_all_ctx;
std::atomic<bool> g_attrs_set[64];
std::atomic<uint64_t> g_epoch{1};                      // bumped by prc_shutdown

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
            delete c;
            c = nullptr;
        }
    }
};
thread_local TlsCtx g_tls;

int set_kernel_attrs(int device) {
    if (g_attrs_set[device].load()) return PRC_OK;
    const int lim = (int)SMEM_LIMIT;
    TRY(corr_set_attrs(lim));
    TRY(clutter_set_attrs(lim));
    TRY(signal_set_attrs(lim));
    TRY(detect_set_attrs(lim));
    g_attrs_set[device].store(true);
    return PRC_OK;
}

int get_ctx(int device, void* stream, Ctx** out) {
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

// ---- arguments of the C entry points
// The checks of an entry point that takes ref / srv stacks, made before any CUDA call.  `names` names the three
// operands in the message; range_bins / freq_bins are the CAF's (the defaults pass).  *bt (when given): the frames and
// the caller's stride between them.
int stack_args(const void* a, const void* b, const void* o, const char* names, int mem_kind, long long n, int nframes,
               long long frame_stride, Batch* bt, int range_bins, int freq_bins) {
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

int finish(Ctx* c, unsigned flags) {
    if (flags & PRC_FLAG_ASYNC) return PRC_OK;
    CU(cudaStreamSynchronize(c->stream));
    return PRC_OK;
}

}  // namespace prcore

using namespace prcore;

// =========================================================================== C ABI
#pragma GCC visibility push(default)
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
    for (Ctx* c : g_all_ctx) delete c;
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

}  // extern "C"
#pragma GCC visibility pop
