// prcore_signal.cu -- the signal front end of libprcore.so: deinterleave / mix / resample of raw IQ in chunks, decimate,
// normalize, the channel-offset estimator and xcorr, and the Welch PSD; their launches and C entry points.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <vector>

#include "prcore_host.h"
#include "recording.cuh"
#include "decimate.cuh"
#include "chanoff.cuh"
#include "spectrum.cuh"

namespace prcore {

using namespace prc;

int signal_set_attrs(int lim) {
    CU(spec::set_attrs(lim));
    CU(dec::set_attrs(lim));
    return PRC_OK;
}

// ---- front end (frontend.cuh) -------------------------------------------------------------------
size_t iq_bytes(int kind, long long n) {
    return (size_t)n * (kind == IQ_I8 ? 2 : kind == IQ_I16 ? 4 : 8);
}

// raw bytes from the first I to the last Q of n >= 1 complex samples `pitch` raw elements apart: with pitch 4 (one
// channel of a PRC_FLAG_CHANNEL_PAIR stream) the other channel's last sample, which may lie past the caller's buffer,
// is not part of it
size_t iq_span_bytes(int kind, long long n, int pitch) {
    return iq_bytes(kind, 1) / 2 * ((size_t)pitch * (size_t)(n - 1) + 2);
}

// raw elements from one complex sample to the next: 4 for one channel of a PRC_FLAG_CHANNEL_PAIR stream, 2 otherwise
int iq_pitch(unsigned flags) {
    return (flags & PRC_FLAG_CHANNEL_PAIR) ? 4 : 2;
}

// flags: the front-end entry points' own (PRC_FLAG_CHANNEL_PAIR); every other caller reads plain I/Q
MixParams make_mix(const void* in, int kind, long long n, int mode, double fc, double fs, double po, unsigned flags = 0) {
    MixParams m{};
    m.in = in; m.kind = kind; m.n = n; m.mode = mode;
    m.pitch = iq_pitch(flags);
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

// nchunks chunks of mix.n samples each, chunk b at complex sample b * chunk_stride of mix.in (samples mix.pitch raw
// elements apart), mixed with phase offset po[b] (device doubles; NULL: mix.po, for a single chunk), its output at
// out + b * out_stride (recording.cuh)
rec::ChunkParams chunk_params(const MixParams& mix, int nchunks, long long chunk_stride, const double* po, long long out_stride) {
    rec::ChunkParams p{};
    p.rs.mix = mix;
    p.chunk_bytes = (long long)(iq_bytes(mix.kind, 1) / 2 * mix.pitch) * chunk_stride;     // raw element size x pitch
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

int frequency_shift_device(Ctx* c, const float2* x, long long n, double fc, double fs, float2* out) {
    const MixParams m = make_mix(x, IQ_C64, n, MIX_C64, fc, fs, 0.0);
    return mix_chunks_device(c, K_MISC, chunk_params(m, 1, 0, nullptr, 0), out);
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

// The checks the front-end entry points share, made before any CUDA call
int frontend_args(int mem_kind, long long n, int in_kind, int mode, double fs) {
    if (bad_mem_kind(mem_kind)) return fail(PRC_E_INVALID, "mem_kind=%d invalid", mem_kind);
    if (n <= 0) return fail(PRC_E_INVALID, "n=%lld invalid", n);
    if (in_kind < IQ_C64 || in_kind > IQ_I16) return fail(PRC_E_INVALID, "in_kind=%d invalid", in_kind);
    if (mode < MIX_NONE || mode > MIX_FS64) return fail(PRC_E_INVALID, "mode=%d invalid", mode);
    if (mode != MIX_NONE && !(fs != 0.0)) return fail(PRC_E_INVALID, "fs must not be 0");
    return PRC_OK;
}

// ---- channel offset / xcorr (chanoff.cuh) ---------------------------------------------------------------------------
constexpr int CHANOFF_MAX_ND = 64;          // largest decimation factor (its pole radius 0.9971 sets W ~ 14k samples)
constexpr int CHANOFF_MAX_LOG2 = 26;        // largest transform: 2^26 complex128 = 1 GiB per buffer

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

}  // namespace prcore

using namespace prcore;

// =========================================================================== C ABI
#pragma GCC visibility push(default)
extern "C" {

int prc_iq_mix_c64(const void* in, int in_kind, int64_t n, int mode, double fc, double fs, double phase_offset,
                   prc_c64* out, int mem_kind, int device, void* stream, unsigned flags) {
    if (!in || !out) return fail(PRC_E_INVALID, "in/out must not be NULL");
    TRY(frontend_args(mem_kind, n, in_kind, mode, fs));
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    const size_t ib = iq_span_bytes(in_kind, n, iq_pitch(flags)), ob = (size_t)n * sizeof(float2);
    const void* din;
    float2* dout;
    TRY(stage_in(c, in, mem_kind, 1, ib, ib, c->fe_in, flags, &din));
    TRY(stage_out(out, mem_kind, ob, c->fe_out, &dout));
    TRY(mix_chunks_device(c, K_MISC, chunk_params(make_mix(din, in_kind, n, mode, fc, fs, phase_offset, flags), 1, 0,
                                                  nullptr, 0),
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
    const size_t ib = iq_span_bytes(in_kind, n, iq_pitch(flags));
    const void* din;
    float2* dout;
    TRY(stage_in(c, in, mem_kind, 1, ib, ib, c->fe_in, flags, &din));
    TRY(stage_out(out, mem_kind, (size_t)g.n_out * sizeof(float2), c->fe_out, &dout));
    TRY(frontend_device(c, K_MISC,
                        chunk_params(make_mix(din, in_kind, n, mode, fc, fs, phase_offset, flags), 1, 0, nullptr, 0), g,
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
    const size_t ib = iq_span_bytes(in_kind, (long long)(nchunks - 1) * cstride + n, iq_pitch(flags));
    const size_t cb = (size_t)g.n_out * sizeof(float2);
    const void* din;
    float2* dout;
    TRY(stage_in(c, in, mem_kind, 1, ib, ib, c->fe_in, flags, &din));
    TRY(stage_out(out, mem_kind, nchunks * cb, c->fe_out, &dout));
    const long long dstride = mem_kind == PRC_MEM_HOST ? g.n_out : ostride;      // staged chunks are packed
    TRY(copy_params(c, phase_offsets, nchunks, c->fe_po));
    TRY(frontend_device(c, K_FRONTEND_CHUNKS,
                        chunk_params(make_mix(din, in_kind, n, mode, fc, fs, 0.0, flags), nchunks, cstride,
                                     c->fe_po.as<double>(),
                                     dstride),
                        g, h, nh, dout));
    TRY(unstage(c, out, dout, mem_kind, nchunks, cb, (size_t)ostride * sizeof(float2), flags));
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
#pragma GCC visibility pop
