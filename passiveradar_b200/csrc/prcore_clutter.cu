// prcore_clutter.cu -- the adaptive and SVD clutter filters of libprcore.so: NLMS_filter / block_NLMS, GAL_JPE and
// LS_Filter_SVD; their launches and C entry points.
#include <cuda_runtime.h>

#include <algorithm>

#include "prcore_host.h"
#include "nlms_block.cuh"
#include "gal.cuh"
#include "lssvd.cuh"

namespace prcore {

using namespace prc;

int clutter_set_attrs(int lim) {
    CU(cudaFuncSetAttribute(nlms_block_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<1, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<2, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(nlms_block_kernel<4, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(gal_jpe_kernel<GAL_CTA_T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    CU(cudaFuncSetAttribute(lssvd::svd_eig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
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

}  // namespace prcore

using namespace prcore;

// =========================================================================== C ABI
#pragma GCC visibility push(default)
extern "C" {

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

}  // extern "C"
#pragma GCC visibility pop
