// prcore_array.cu -- array processing in libprcore.so: the beamscan of several surveillance channels' range-Doppler maps
// into one amplitude map and a bearing per cell (beamscan.cuh); its launch and C entry point.
#include <cuda_runtime.h>

#include <mutex>

#include "prcore_host.h"
#include "beamscan.cuh"

using namespace prcore;

// =========================================================================== C ABI
#pragma GCC visibility push(default)
extern "C" {

int prc_beamscan_frames(const prc_c64* maps, int rows, int cols, int nframes, int64_t frame_stride, int nchan,
                        int64_t chan_stride, const prc_c64* steering, int nangles, int wrap, float* amp_out,
                        float* pos_out, int64_t out_stride, int device, void* stream, unsigned flags) {
    using namespace prc::beam;
    if (!maps || !steering) return fail(PRC_E_INVALID, "maps and steering must not be NULL");
    if (!amp_out && !pos_out) return fail(PRC_E_INVALID, "amp_out and pos_out must not both be NULL");
    if (rows < 1 || cols < 1) return fail(PRC_E_INVALID, "rows=%d cols=%d invalid", rows, cols);
    const long long cells = (long long)rows * cols;
    if (cells > (long long)0x7fffffff * (BS_THREADS * BS_CPT))
        return fail(PRC_E_INVALID, "a %d x %d map exceeds the beamscan's maximum of %lld cells", rows, cols,
                    (long long)0x7fffffff * (BS_THREADS * BS_CPT));
    if (nframes < 0 || nframes > 65535) return fail(PRC_E_INVALID, "nframes=%d outside [0, 65535]", nframes);
    if (nchan < 1 || nchan > BS_MAX_CHAN) return fail(PRC_E_INVALID, "nchan=%d outside [1, %d]", nchan, BS_MAX_CHAN);
    if (nangles < 1 || nangles > BS_MAX_ANGLES)
        return fail(PRC_E_INVALID, "nangles=%d outside [1, %d]", nangles, BS_MAX_ANGLES);
    if (wrap != 0 && wrap != 1) return fail(PRC_E_INVALID, "wrap=%d must be 0 or 1", wrap);
    if (chan_stride < 0) return fail(PRC_E_INVALID, "chan_stride=%lld must be >= 0", (long long)chan_stride);
    if (nframes > 1 && (frame_stride < cells || out_stride < cells))
        return fail(PRC_E_INVALID, "frame_stride=%lld / out_stride=%lld smaller than the %lld cells of a map",
                    (long long)frame_stride, (long long)out_stride, cells);
    Ctx* c;
    TRY(get_ctx(device, stream, &c));
    std::lock_guard<std::mutex> lk(c->mu);
    if (nframes == 0) return finish(c, flags);
    TRY(copy_param_bytes(c, steering, (size_t)nangles * nchan * sizeof(prc_c64), c->bf_steer));
    BeamParams p{};
    p.maps = reinterpret_cast<const float2*>(maps);
    p.steer = c->bf_steer.as<float2>();
    p.amp = amp_out;
    p.pos = pos_out;
    p.cells = cells;
    p.frame_stride = nframes > 1 ? frame_stride : cells;
    p.chan_stride = chan_stride;
    p.out_stride = nframes > 1 ? out_stride : cells;
    p.nangles = nangles;
    p.wrap = wrap;
    {
        ProfScope ps(c, K_BEAMSCAN);
        launch_beamscan(p, nchan, nframes, c->stream);
    }
    TRY(check_launch("beamscan_kernel"));
    return finish(c, flags);
}

}  // extern "C"
#pragma GCC visibility pop
