// prcore_detect.cu -- detection and tracking in libprcore.so: CFAR_2D (single map and frames), the ordered-statistic
// CFAR, the frame chain's persistence and percentiles, and the Kalman trackers; their launches and C entry points.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <mutex>
#include <vector>

#include "prcore_host.h"
#include "detect.cuh"
#include "oscfar.cuh"
#include "render.cuh"

namespace prcore {

using namespace prc;

int detect_set_attrs(int lim) {
    CU(cudaFuncSetAttribute(track_meas_kernel<float, TRK_MODE_MEAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<float, TRK_MODE_SLOTS>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<float, TRK_MODE_MEAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<double, TRK_MODE_MEAN>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<double, TRK_MODE_SLOTS>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(track_meas_kernel<double, TRK_MODE_MEAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    return PRC_OK;
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

// ---- ordered-statistic CFAR (oscfar.cuh) ---------------------------------------------------------------
// the cells of CFAR_2D's window: fw^2 minus the guard hole [e1, e2)^2 (empty when e2 <= e1)
int os_cells(const CfarParams& p) {
    const int hole = std::max(0, p.e2 - p.e1);
    return p.fw * p.fw - hole * hole;
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

}  // namespace prcore

using namespace prcore;

// =========================================================================== C ABI
#pragma GCC visibility push(default)
extern "C" {

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

int prc_os_cfar2d_frames(const void* x, int rows, int cols, int nframes, int64_t frame_stride, int fw, int gw, int k,
                         void* cr_out, int64_t cr_stride, int device, void* stream, unsigned flags) {
    if (!x || !cr_out) return fail(PRC_E_INVALID, "x and cr_out must not be NULL");
    oscfar::OsParams p;
    TRY(cfar_window(rows, cols, fw, gw, &p.c));
    if (nframes < 0 || nframes > 65535) return fail(PRC_E_INVALID, "nframes=%d outside [0, 65535]", nframes);
    const long long cells = (long long)rows * cols;
    if (nframes > 1 && (frame_stride < cells || cr_stride < cells))
        return fail(PRC_E_INVALID, "frame_stride=%lld / cr_stride=%lld smaller than the %lld cells of a map",
                    (long long)frame_stride, (long long)cr_stride, cells);
    const int n = os_cells(p.c);
    if (n < 1) return fail(PRC_E_INVALID, "fw=%d gw=%d: the guard hole covers the whole window (N = 0 cells)", fw, gw);
    if (k < 1 || k > n) return fail(PRC_E_INVALID, "k=%d outside [1, N = %d], the cells of the fw=%d gw=%d window", k, n,
                                    fw, gw);
    p.k = k;
    p.h0 = p.c.e1;
    p.h1 = std::max(p.c.e1, p.c.e2);
    p.c.x = x;
    p.c.is_complex = (flags & PRC_FLAG_ABS_C64) ? 1 : 0;
    p.c.cr = cr_out;
    p.c.cr_f64 = (flags & PRC_FLAG_CR_F64) ? 1 : 0;
    p.c.frame_stride = nframes > 1 ? frame_stride : cells;
    p.c.out_stride = nframes > 1 ? cr_stride : cells;
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    if (nframes == 0) return finish(c, flags);
    TRY(c->rd_part.ensure((size_t)nframes * CFAR_MEAN_CTAS * sizeof(double)));
    p.c.partial = c->rd_part.as<double>();
    {
        ProfScope ps(c, K_OS_CFAR);
        oscfar::launch_os_cfar(p, nframes, c->stream);
    }
    TRY(check_launch("os_select_kernel"));
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

}  // extern "C"
#pragma GCC visibility pop
