/*
 * prcore.h -- C ABI of libprcore.so, the H100 (sm_90a) passive-radar DSP core.
 *
 * This is the drop-in boundary for the hot path of Max-Manning/passiveRadar.
 * The reference has no FFI of its own (it is pure Python), so each entry point
 * below names the *Python function* whose arithmetic it replaces; the Python
 * wrappers in passiveradar_b200/ keep those functions' signatures and bind these
 * symbols through ctypes (see INTEGRATION.md for the stub a maintainer of the
 * reference would add).
 *
 * Conventions
 *   - complex64 data are interleaved (re, im) float pairs: `prc_c64`.
 *   - every function returns PRC_OK (0) or a negative PRC_E_* code; the message
 *     for the calling thread is available from prc_last_error().
 *   - `mem_kind` says where the data pointers live:
 *         PRC_MEM_HOST   (0)  host memory; the library copies H2D / D2H itself
 *         PRC_MEM_DEVICE (1)  device memory on `device`; no copies are made
 *   - `stream` is a cudaStream_t (as void*).  NULL: the library uses a private
 *     stream owned by the calling thread and the call is synchronous.  Non-NULL:
 *     all work is enqueued on that stream; unless PRC_FLAG_ASYNC is set the call
 *     waits for it to finish before returning.
 *   - the library is re-entrant: dask's threaded scheduler calls the Python
 *     wrappers concurrently (main.py:169-194); ctypes drops the GIL, every
 *     (thread | stream) owns its workspace, errors are thread-local.
 *   - inputs are never modified; outputs are caller-allocated.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point
 *     fails with PRC_E_CUDA.
 */
#ifndef PRCORE_H
#define PRCORE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct prc_c64 { float re, im; } prc_c64;

#define PRC_VERSION 200          /* 0.2.0 */

/* status codes */
#define PRC_OK            0
#define PRC_E_INVALID    -1      /* bad argument (message says which) */
#define PRC_E_CUDA       -2      /* CUDA runtime error / no device */
#define PRC_E_SINGULAR   -3      /* LS normal equations not positive definite */
#define PRC_E_NOMEM      -4

/* mem_kind */
#define PRC_MEM_HOST      0
#define PRC_MEM_DEVICE    1

/* flags */
#define PRC_FLAG_ASYNC        1u   /* do not synchronise `stream` before returning */
#define PRC_FLAG_WINDOW_F32   2u   /* `window` points at float, not double */
#define PRC_FLAG_ABS_C64      4u   /* prc_cfar2d_f32, prc_cfar2d_frames, prc_os_cfar2d_frames: `x` is a complex64 map,
                                    * |x| is used */
#define PRC_FLAG_MAP_F64      8u   /* tracker entry points, prc_persistence_frames: maps are float64, not float32 */
#define PRC_FLAG_CR_F64      16u   /* prc_cfar2d_frames, prc_os_cfar2d_frames: cr_out receives the float64 CR, not its
                                    * float32 rounding */
#define PRC_FLAG_PROD_F32    32u   /* prc_persistence_frames: float32 products float32(x) * float32(w) */
#define PRC_FLAG_ORIENT      64u   /* prc_persistence_frames: frames are written as fliplr(P.T) */
#define PRC_FLAG_TRACK_RESUME 128u /* tracker entry points: continue from the frame-0 records of `history` */
#define PRC_FLAG_CHANNEL_PAIR 256u /* prc_iq_mix_c64, prc_frontend_c64, prc_frontend_chunks_c64: `in` is one channel of a
                                    * two-channel stream whose complex samples alternate between the channels */
/* Every entry point ignores the flags that are not its own. */

/* ---- lifecycle / diagnostics ------------------------------------------------ */
int         prc_version(void);
const char* prc_last_error(void);                /* thread-local, never NULL */
int         prc_device_count(int* count);
int         prc_init(int device);                /* optional: create the context early */
void        prc_shutdown(void);                  /* free every workspace and private stream */
int         prc_sync(int device, void* stream);  /* cudaStreamSynchronize on `stream` (or the thread's) */
uint64_t    prc_launch_count(void);              /* kernels launched by this library so far */

/* per-kernel device timing (CUDA events on the launching stream around every launch).
 * enable -> run -> collect (synchronises) -> read(idx) for idx < prc_profile_kernels() */
int prc_profile_enable(int on);
int prc_profile_collect(void);
int prc_profile_kernels(void);
int prc_profile_read(int idx, const char** name, double* total_ms, uint64_t* launches);
int prc_profile_reset(void);

/* pinned host memory helpers (so numpy buffers can take the async copy path) */
int prc_host_alloc(void** ptr, uint64_t bytes);
int prc_host_free(void* ptr);
int prc_host_register(void* ptr, uint64_t bytes);
int prc_host_unregister(void* ptr);

/* ---- cross-ambiguity function ---------------------------------------------------
 * Replaces fast_xambg(), reference passiveRadar/range_doppler_processing.py:12-90,
 * for inputs already padded to their final length `n` (the zero-padding of :52-55,
 * named windows of :57-58 and the (F, R+1, 1) reshape stay in the Python wrapper).
 *
 *   out[f*(range_bins+1) + k],  f = 0..freq_bins-1 (fftshift-ed Doppler),
 *                               k = 0..range_bins   (delay range_bins - k)
 *
 * window : n doubles (or floats with PRC_FLAG_WINDOW_F32) or NULL      (:83-84)
 * dtaps  : decimator taps (doubles) or NULL for the reference's default boxcar of
 *          int(n/freq_bins)+1 ones (:69-72); ndtaps = their count         (:73-78)
 */
int prc_xambg_c64(const prc_c64* ref, const prc_c64* srv, int64_t n,
                  int range_bins, int freq_bins,
                  const void* window, const double* dtaps, int64_t ndtaps,
                  prc_c64* out, int mem_kind, int device, void* stream, unsigned flags);

/* ---- block least-squares clutter filter ---------------------------------------------
 * Replaces LS_Filter(), reference passiveRadar/clutter_removal.py:6-56.
 *   out  : n cleaned surveillance samples
 *   taps : filter_len + peek taps, or NULL                                    (:53-56)
 * The Gram matrix of :39 is Hermitian Toeplitz (circular autocorrelation of ref);
 * the library computes its first column and the right-hand side of :45 as lag
 * correlations, solves (T + reg I) w = rhs in float64 and applies the circular FIR
 * of :51.
 */
int prc_ls_filter_c64(const prc_c64* ref, const prc_c64* srv, int64_t n,
                      int filter_len, int peek, float reg,
                      prc_c64* out, prc_c64* taps,
                      int mem_kind, int device, void* stream, unsigned flags);

/* ---- Toeplitz least-squares clutter filter (what main.py actually calls) ---------------------------
 * prc_ls_toeplitz_c64 replaces LS_Filter_Toeplitz(), reference passiveRadar/clutter_removal.py:109-160:
 * reference rolled by -peek (:139), LINEAR (zero-padded) auto/cross correlations (:142-147), Levinson
 * solve without regularisation (:150, float64 here as in SciPy), linear convolution + subtraction
 * (:153-155).  prc_ls_multiple_c64 replaces LS_Filter_Multiple() (:162-187): the filter is applied once
 * per Doppler bin on the running residual, the reference being frequency-shifted by bin Hz first
 * (signal_utils.py:24-27, float32 phase ramp as in the reference).  doppler_bins == NULL means [0].
 * Results are complex64; the Python wrappers widen them to complex128 like the reference returns.
 */
int prc_ls_toeplitz_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int filter_len, int peek,
                        prc_c64* out, prc_c64* taps, int mem_kind, int device, void* stream, unsigned flags);
int prc_ls_multiple_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int filter_len, int peek,
                        double sample_rate, const double* doppler_bins, int nbins,
                        prc_c64* out, prc_c64* taps_last,
                        int mem_kind, int device, void* stream, unsigned flags);

/* prc_ls_multiple_frames_c64: LS_Filter_Multiple on nframes independent chunks per call (device pointers; frame i at
 * ref/srv/out + i*frame_stride): what main.py:169-176 does per dask chunk, several chunks at a time.  One launch of each
 * kernel per Doppler bin covers the batch.
 */
int prc_ls_multiple_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                               int filter_len, int peek, double sample_rate, const double* doppler_bins, int nbins,
                               prc_c64* out, int mem_kind, int device, void* stream, unsigned flags);

/* ---- NLMS / block-NLMS clutter filter ---------------------------------------------------
 * Replaces NLMS_filter(), reference passiveRadar/clutter_removal.py:189-249
 * (block_len == 1) and provides block_NLMS (block_len > 1; not in the reference,
 * defined in DESIGN.md).
 *   init_taps : filter_len + peek initial taps or NULL (zeros)              (:218-225)
 *   out       : n samples; out[0:filter_len] and out[n-peek:] are zero        (:231,:244)
 *   taps_out  : final taps or NULL                                            (:246-249)
 */
int prc_nlms_c64(const prc_c64* ref, const prc_c64* srv, int64_t n,
                 int filter_len, int peek, float mu, int block_len,
                 const prc_c64* init_taps, prc_c64* out, prc_c64* taps_out,
                 int mem_kind, int device, void* stream, unsigned flags);

/* ---- one CPI frame: LS_Filter -> fast_xambg with filterLen = range_bins-like chaining ----
 * The composition main.py performs per chunk (main.py:169-194 with LS_Filter in place
 * of LS_Filter_Multiple): cleaned = LS_Filter(ref, srv, filter_len, reg, peek);
 * map = fast_xambg(ref, cleaned, range_bins, freq_bins, n, window).
 * The cleaned surveillance channel stays in device memory.
 *   taps_out, cleaned_out : optional (NULL to skip)
 */
int prc_frame_c64(const prc_c64* ref, const prc_c64* srv, int64_t n,
                  int filter_len, int peek, float reg,
                  int range_bins, int freq_bins, const void* window,
                  prc_c64* out_map, prc_c64* taps_out, prc_c64* cleaned_out,
                  int mem_kind, int device, void* stream, unsigned flags);

/* prc_frames_c64: the same composition for `nframes` frames in one call -- frame i reads ref + i*frame_stride and
 * srv + i*frame_stride (strides in samples; device or host pointers as mem_kind says) and writes
 * out_maps + i*freq_bins*(range_bins+1), taps_out + i*(filter_len+peek), cleaned_out + i*frame_stride.  This is the unit
 * of work of the dask graph (one chunk = one frame, main.py:169-194) handed over several chunks at a time, so that one
 * launch of each kernel covers the whole batch (gridDim.y = frame).  prc_frame_c64 is nframes = 1.
 * With PRC_FLAG_ASYNC the Toeplitz-solve status of every frame stays on the device: prc_ls_status() reads it back
 * (0 = ok, 1 = normal equations not positive definite) after synchronising `stream`.
 */
int prc_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                   int filter_len, int peek, float reg, int range_bins, int freq_bins, const void* window,
                   prc_c64* out_maps, prc_c64* taps_out, prc_c64* cleaned_out,
                   int mem_kind, int device, void* stream, unsigned flags);
int prc_ls_status(int device, void* stream, int* status, int nframes);

/* prc_frames_multi_c64: prc_frames_c64 for nchan surveillance channels that share one reference channel (one reference
 * antenna and up to four surveillance antennas of one coherent receiver).  Frame f of the reference is at
 * ref + f*frame_stride; frame f of surveillance channel k at srv + k*chan_stride + f*frame_stride (strides in samples,
 * any chan_stride, 0 included: the inputs are only read).  maps receives [nchan][nframes][freq_bins][range_bins+1],
 * taps_out (or NULL) [nchan][nframes][filter_len+peek]; the status words are [nchan][nframes] (prc_ls_status with
 * nchan*nframes).  Channel k's taps and map are those of prc_frames_c64(ref, srv_k) on the same frames; where the
 * one-pass frame runs and nchan >= 2 the reference's transforms, its lag sums and its part of the CAF block spectra are
 * formed once for all channels (csrc/framemulti.cuh).  All pointers are DEVICE pointers (no mem_kind).  Flags:
 * PRC_FLAG_ASYNC, PRC_FLAG_WINDOW_F32 as in prc_frames_c64.  Limits (PRC_E_INVALID before any CUDA call):
 * 1 <= nchan <= 4, plus prc_frames_c64's.  nchan = 1 is exactly prc_frames_c64 on device pointers.
 */
int prc_frames_multi_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                         int nchan, int64_t chan_stride, int filter_len, int peek, float reg, int range_bins,
                         int freq_bins, const void* window, prc_c64* maps, prc_c64* taps_out,
                         int device, void* stream, unsigned flags);

/* The other two operators of the path on nframes independent frames per call (same layout rules as prc_frames_c64):
 * prc_nlms_frames_c64 -- NLMS_filter / block_NLMS (clutter_removal.py:189-249): the recurrence of one frame is serial,
 *   so every frame gets its own CTA (one SM) and the batch fills the GPU; init_taps (filter_len + peek taps or NULL)
 *   is shared by all frames, taps_out receives nframes * (filter_len + peek) taps.
 * prc_xambg_frames_c64 -- fast_xambg (range_doppler_processing.py:12-90, default boxcar decimator) with one window for
 *   all frames; out receives nframes maps of freq_bins x (range_bins + 1).
 */
int prc_nlms_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                        int filter_len, int peek, float mu, int block_len, const prc_c64* init_taps,
                        prc_c64* out, prc_c64* taps_out, int mem_kind, int device, void* stream, unsigned flags);
int prc_xambg_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                         int range_bins, int freq_bins, const void* window, prc_c64* out,
                         int mem_kind, int device, void* stream, unsigned flags);

/* ---- gradient-adaptive lattice joint process estimator ------------------------------------------------
 * prc_gal_jpe_frames_c64 replaces GAL_JPE(), reference passiveRadar/clutter_removal.py:251-364, on nframes
 * independent frames (frame i at ref/srv/out + i*frame_stride; a single frame is nframes = 1): a lattice of
 * lattice_len stages (gradient-adaptive reflection coefficients, step mu1, which the recurrence itself adapts
 * and clamps at 5e-3) feeds an NLMS transversal filter of delay_line_len taps (step mu2).  peek = number of
 * non-causal taps: sample n uses ref[n + peek].
 *   out   : n samples per frame; the last peek + 1 are zero                              (:317-359)
 *   k_out : nframes * delay_line_len final reflection coefficients, or NULL              (:361-362)
 *   h_out : nframes * delay_line_len final transversal taps, or NULL                     (:361-362)
 * Requires 1 <= lattice_len <= delay_line_len <= 4096 and peek >= 0 (PRC_E_INVALID otherwise).  The sample
 * recurrence of a frame is serial: a frame runs on one warp (delay_line_len <= 256) or one CTA, and a batch
 * of frames fills the GPU.  Arithmetic is complex64 with the reference's rounding points (DESIGN.md).
 */
int prc_gal_jpe_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                           int lattice_len, int delay_line_len, double mu1, double mu2, int peek,
                           prc_c64* out, prc_c64* k_out, prc_c64* h_out,
                           int mem_kind, int device, void* stream, unsigned flags);

/* ---- SVD least-squares clutter filter ------------------------------------------------------------------
 * prc_ls_svd_frames_c64 replaces LS_Filter_SVD(), reference passiveRadar/clutter_removal.py:58-107, on nframes
 * independent frames (frame i at ref/srv/out + i*frame_stride; a single frame is nframes = 1).  With the data
 * matrix A[:, k] = roll(ref, k - peek), M = filter_len + peek columns, the taps are the minimum-norm least-squares
 * solution of A taps = srv, computed from the Hermitian Toeplitz Gram matrix A^H A (A itself is never formed):
 * its eigenvalues below max(1e-20, 1e-10 * largest) -- singular values of A below max(1e-10, 1e-5 * largest) --
 * are dropped (DESIGN.md section 13).  All arithmetic is float64; out is rounded to complex64 once.
 *   out      : n samples per frame, srv - A taps                                           (:102)
 *   taps_out : nframes * M taps rounded to complex64, or NULL                              (:99)
 *   rank_out : nframes ints, or NULL: the number of kept singular values; -1 when the input is not finite or the
 *              eigensolver does not converge, and that frame's out and taps are NaN
 * Requires n >= 1, filter_len >= 0, peek >= 0 and 1 <= M <= 1024 (PRC_E_INVALID naming the limit otherwise).
 * One CTA per frame runs the eigensolver, so a batch of frames is what fills the GPU.
 */
int prc_ls_svd_frames_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int nframes, int64_t frame_stride,
                          int filter_len, int peek, prc_c64* out, prc_c64* taps_out, int* rank_out,
                          int mem_kind, int device, void* stream, unsigned flags);

/* ---- run-time switches (also read once from the environment: PRC_FFT, PRC_FFT_MIN_N) ----------------
 *   "fft"        1 (default): LS correlations, clutter FIR and CAF block sums as FFT-domain block correlations
 *                (csrc/fftcorr.cuh);  0: FP32 direct form (csrc/lagstream.cuh, kernels.cuh)
 *   "fft_min_n"  smallest channel length the FFT-domain path takes (default 8192)
 *   "frame_onepass"  1 (default): prc_frames_c64 / prc_frame_c64 on the FFT-domain path form the LS lag sums and the
 *                CAF's per-block spectra in one pass over the channels (csrc/framepass.cuh) where the plan allows it
 *                (L = 2048, filter_len >= 1, fewer transforms than two passes);  0: lscorr_fft_kernel, then the fused
 *                caf_fft_kernel.  Acceptance and results within float32 round-off are the same either way.
 * Read-only (prc_get_option only; prc_set_option returns PRC_E_INVALID):
 *   "fft_ctas_ls", "fft_ctas_fir"  CTAs per SM of lscorr_fft_kernel and fir_fft_kernel at L = 2048 on the calling
 *                 thread's current device, as the runtime's occupancy calculator gives it for the launch
 *                 configuration: the number their one-wave grids are sized from
 *   "fft_ctas_frame"  the same for frame_pass_kernel (the one-pass frame; 2 on an H100)
 */
int prc_set_option(const char* name, int value);
int prc_get_option(const char* name, int* value);

/* ---- direct (time-domain) cross-ambiguity function ------------------------------------------------
 * Replaces direct_xambg(), reference passiveRadar/range_doppler_processing.py:93-124: for Doppler bin f
 * the reference channel is frequency-shifted by (f - freq_bins/2) / CPI Hz (signal_utils.py:24-27,
 * float32 phase ramp and complex64 exponential as in the reference) and LINEARLY cross-correlated
 * with srv (xcorr(ref_shifted, srv, range_bins, 0), signal_utils.py:29-32).  out: freq_bins x
 * (range_bins + 1) complex64, column k <-> delay range_bins - k (same orientation as prc_xambg_c64).
 */
int prc_direct_xambg_c64(const prc_c64* ref, const prc_c64* srv, int64_t n, int range_bins, int freq_bins,
                         double sample_rate, prc_c64* out, int mem_kind, int device, void* stream, unsigned flags);

/* ---- front end: the chain main.py:105-166 runs on every input chunk before the clutter filter -------
 * in_kind : PRC_IQ_C64 (n complex64 samples), PRC_IQ_I8 / PRC_IQ_I16 (2n interleaved I,Q integers:
 *           deinterleave_IQ(), reference passiveRadar/signal_utils.py:19-22)
 * mode    : PRC_MIX_NONE, or frequency_shift(x, fc, fs, phase_offset) (signal_utils.py:24-27) with the
 *           reference's float32 phase ramp; PRC_MIX_C64 = phase_offset is a Python scalar (complex64
 *           arithmetic throughout), PRC_MIX_C128 = phase_offset is a NumPy float64 (main.py:127-130;
 *           the exponential is then evaluated in float64).  Results are complex64 either way.
 * in      : I and Q are read as scalars, so `in` may sit at any raw element, odd ones included (a raw array
 *           sliced by a channel offset, main.py:87-92).
 * PRC_FLAG_CHANNEL_PAIR: `in` is one channel of a stream that holds two channels' I/Q as
 *           [ref_I[0], ref_Q[0], srv_I[0], srv_Q[0], ref_I[1], ...] (PRconfig.yaml's interleaved_input_channels):
 *           complex sample i is read from raw elements 4i and 4i+1 of `in`.  Pass the stream's element 0 for the
 *           reference channel and element 2 for the surveillance channel, plus 4 * start for a channel trimmed to
 *           start at sample `start`.  n and chunk_stride count the channel's complex samples; every other argument
 *           and check is unchanged.  From host memory exactly the raw span the channel's samples occupy is copied,
 *           its first I to its last Q (2 * (2 * N - 1) elements for N samples), so the surveillance channel's buffer
 *           may end at its last Q.
 * prc_frontend_c64 additionally applies resample() = scipy.signal.resample_poly(x, up, down,
 * padtype='line') (signal_utils.py:15-17) in the same pass: h = the nh = 2*half_len+1 low-pass taps
 * ALREADY multiplied by up (what resample_poly hands to upfirdn; host doubles, designed by the caller
 * with scipy.signal.firwin exactly as resample_poly does).  out receives prc_resample_out_len() samples.
 * With n = 1 the line extension's slope is 0/0 and every output is NaN, as resample_poly gives.  One CTA
 * stages its taps and input window in at most 200 KB of shared memory: at up = 1 the largest down is 89, at
 * up = 2 it is 171; a ratio beyond returns PRC_E_INVALID with the bytes it needs.
 */
#define PRC_IQ_C64   0
#define PRC_IQ_I8    1
#define PRC_IQ_I16   2
#define PRC_MIX_NONE 0
#define PRC_MIX_C64  1
#define PRC_MIX_C128 2
#define PRC_MIX_F64  3   /* fc was a NumPy float64 scalar: the phase ramp is evaluated in float64 */
#define PRC_MIX_FS64 4   /* only fs was a NumPy float64 scalar: float32 product, float64 division */
int prc_iq_mix_c64(const void* in, int in_kind, int64_t n, int mode, double fc, double fs, double phase_offset,
                   prc_c64* out, int mem_kind, int device, void* stream, unsigned flags);
int prc_resample_out_len(int64_t n_in, int up, int down, int nh, int64_t* n_out);
int prc_frontend_c64(const void* in, int in_kind, int64_t n, int mode, double fc, double fs, double phase_offset,
                     int up, int down, const double* h, int nh, prc_c64* out, int64_t out_capacity,
                     int mem_kind, int device, void* stream, unsigned flags);
/* prc_frontend_chunks_c64: prc_frontend_c64 on nchunks chunks of n complex samples in one launch, what main.py:105-166
 * does to every chunk of a recording.  Chunk b starts at complex sample b * chunk_stride of `in` (which may sit at
 * any raw element, as above), is mixed with phase_offsets[b] and resampled
 * with the line extension of its own end points.  phase_offsets is nchunks doubles in host memory whatever mem_kind
 * is; they are copied before the call returns, also with PRC_FLAG_ASYNC.  Its prc_resample_out_len() samples go to
 * out + b * out_stride (out_stride >= that length when nchunks > 1).  out_capacity counts complex samples from `out`.
 * Every chunk's output is bit-identical to a prc_frontend_c64 call on that chunk; the errors are the same.
 */
int prc_frontend_chunks_c64(const void* in, int in_kind, int64_t n, int nchunks, int64_t chunk_stride, int mode,
                            double fc, double fs, const double* phase_offsets, int up, int down, const double* h, int nh,
                            prc_c64* out, int64_t out_stride, int64_t out_capacity, int mem_kind, int device,
                            void* stream, unsigned flags);

/* ---- CFAR detector ---------------------------------------------------------------------------------
 * Replaces CFAR_2D(X, fw, gw, thresh), reference passiveRadar/target_detection.py:683-703: X / mean|X|
 * divided by the wrapped 2-D box average (fw x fw window minus the guard hole) + 1e-10.
 * x: rows x cols float32 (or complex64 with PRC_FLAG_ABS_C64: the magnitude is taken on the device, so
 * a map can go from prc_xambg_c64 to the detector without leaving HBM).  cr_out (float32) and/or
 * det_out (uint8, cr > *thresh) are written; thresh may be NULL when det_out is NULL.  The window sum and
 * the division are evaluated in float64, as the reference's float64 Tfilt makes convolve2d do, so signed
 * real maps are held to the reference too.  Limits: 1 <= fw <= 64, rows <= 524 280 (65 535 CTA rows of 8);
 * beyond either the call returns PRC_E_INVALID naming the limit.
 */
int prc_cfar2d_f32(const void* x, int rows, int cols, int fw, int gw, const float* thresh, float* cr_out,
                   uint8_t* det_out, int mem_kind, int device, void* stream, unsigned flags);

/* ---- the frame chain of range_doppler_plot.py:45-85 -------------------------------------------------------------
 * prc_cfar2d_frames: CFAR_2D(x[b], fw, gw) for b < nframes in one launch; map b at x + b*frame_stride elements (float32,
 *   or complex64 with PRC_FLAG_ABS_C64), its CR at cr_out + b*cr_stride elements: float32, bit-identical to a
 *   prc_cfar2d_f32 call on that map, or with PRC_FLAG_CR_F64 the float64 value that call rounds.  Limits and
 *   messages are prc_cfar2d_f32's; nframes <= 65535, strides >= rows*cols when nframes > 1.
 * prc_persistence_frames: persistence() of reference passiveRadar/plotting_tools.py:9-30 along the frame axis.  x holds
 *   n_carry carried frames followed by nframes new ones (frame f at x + f*frame_stride, rows x cols, float32 or float64
 *   with PRC_FLAG_MAP_F64); out receives, for every new frame k, P[k] = sum_{i < min(k+1, hold)} X[k-i] * weights[i]
 *   with k counted from the first carried frame, summed from +0.0 in the order i = 0, 1, ...  A stream continues across
 *   calls when the last min(k, hold-1) input frames are carried.  weights: min(hold, n_carry+nframes) host doubles
 *   (decay**i as the caller's Python computes it), copied before the call returns.  PRC_FLAG_PROD_F32 forms the
 *   products in float32 (a float32 stack and a float32 or Python-float decay under NumPy 2 promotion), else float64.
 *   out: nframes frames of rows*cols doubles, each P[k] (rows x cols) or, with PRC_FLAG_ORIENT, fliplr(P[k].T)
 *   (cols x rows).  Requires hold >= 1 and 0 <= n_carry <= hold-1.
 * prc_percentiles_frames: np.percentile(frame, q[j]) (linear method) of nframes float64 frames of n values (frame b
 *   at x + b*frame_stride), times scale[j] when scale is not NULL: out[b*nq + j].  1 <= n <= 2 147 483 135,
 *   1 <= nq <= 4, 0 <= q[j] <= 100;
 *   q and scale are host doubles.  Bit-identical to NumPy; a frame holding NaN gives NaN.  -0.0 and +0.0 rank as
 *   equal, and a statistic that falls on either is returned as +0.0.
 */
int prc_cfar2d_frames(const void* x, int rows, int cols, int nframes, int64_t frame_stride, int fw, int gw,
                      void* cr_out, int64_t cr_stride, int mem_kind, int device, void* stream, unsigned flags);
int prc_persistence_frames(const void* x, int rows, int cols, int nframes, int64_t frame_stride, int n_carry, int hold,
                           const double* weights, double* out, int mem_kind, int device, void* stream, unsigned flags);
int prc_percentiles_frames(const double* x, int64_t n, int nframes, int64_t frame_stride, const double* q,
                           const double* scale, int nq, double* out, int mem_kind, int device, void* stream,
                           unsigned flags);

/* ---- ordered-statistic CFAR (Rohling) ----------------------------------------------------------------------------
 * prc_os_cfar2d_frames: CFAR_2D's detector with the window's k-th smallest cell as the noise estimate, for nframes maps
 *   in one launch (not in the reference).  The window is exactly the cells CFAR_2D sums (its Tfilt, guard hole and
 *   'same' / wrap placement, quirks included); N = their count (299 at fw = 18, gw = 4).  For cell (i, j):
 *     T  = the k-th smallest of the N window values, 1 <= k <= N (signed values of a real map; hypotf(re, im) of a
 *          complex64 map with PRC_FLAG_ABS_C64)
 *     CR = (x[i, j] * inv_mean) / (T + 1e-10) in float64, with x[i, j] (its sign kept; |x| of a complex map) and
 *          inv_mean = rows*cols / sum|x| formed exactly as prc_cfar2d_frames forms them: the two differ only in the
 *          denominator.
 *   Map b at x + b*frame_stride elements (float32, or complex64 with PRC_FLAG_ABS_C64), its CR at cr_out + b*cr_stride
 *   elements: the float32 rounding of the float64 CR, or with PRC_FLAG_CR_F64 the float64 CR.  A frame's CR does not
 *   depend on nframes.  Maps must be finite.
 *   x and cr_out are DEVICE pointers (no mem_kind; callers stage host arrays themselves).
 *   Limits (PRC_E_INVALID, naming the limit, before any CUDA call): prc_cfar2d_frames's (1 <= fw <= 64, fw^2 != gw^2,
 *   rows <= 524 280, nframes <= 65535, strides >= rows*cols when nframes > 1), N >= 1 and 1 <= k <= N.
 */
int prc_os_cfar2d_frames(const void* x, int rows, int cols, int nframes, int64_t frame_stride, int fw, int gw, int k,
                         void* cr_out, int64_t cr_stride, int device, void* stream, unsigned flags);

/* ---- beamscan of several surveillance channels (not in the reference) -------------------------------------------
 * prc_beamscan_frames: for nframes frames of nchan complex64 rows x cols maps (channel k of frame f at
 *   maps + k*chan_stride + f*frame_stride elements, the layout prc_frames_multi_c64 writes, so its output is read in
 *   place) and a steering table S of nangles x nchan complex64 values (row a: the array response of grid angle a),
 *   per cell, in float32:
 *     P[a]  = | sum_k S[a, k] * m_k |^2, a = 0 .. nangles-1
 *     a*    = the first a with the largest P[a]
 *     amp   = sqrt(P[a*])
 *     den   = P[a*-1] - 2 P[a*] + P[a*+1]
 *     delta = clamp(0.5 (P[a*-1] - P[a*+1]) / den, -0.5, 0.5) if den < 0, else 0
 *     pos   = a* + delta  (a fractional grid index)
 *   wrap = 0: a sector grid, delta = 0 at a* = 0 and a* = nangles-1.  wrap = 1: a full-circle grid, neighbours taken
 *   mod nangles; pos lies in [-0.5, nangles - 0.5).  The CAF conjugates the surveillance channel, so an echo from
 *   theta gives m_k = conj(a_k(theta)) * c: S is the array response itself, not its conjugate.  Per-channel complex
 *   gains g_k are folded in by the caller as S[a, k] / conj(g_k).  A zero cell gives amp = 0, pos = 0; maps must be
 *   finite.  Frame f's amp and pos go to amp_out / pos_out + f*out_stride (either may be NULL, not both); a frame's
 *   results do not depend on nframes.
 *   maps, amp_out and pos_out are DEVICE pointers (no mem_kind); steering is a HOST array, copied before the call
 *   returns (PRC_FLAG_ASYNC included).  Limits (PRC_E_INVALID, naming the limit, before any CUDA call): rows, cols >= 1,
 *   0 <= nframes <= 65535, 1 <= nchan <= 4, 1 <= nangles <= 4096, wrap 0 or 1, chan_stride >= 0, frame_stride and
 *   out_stride >= rows*cols when nframes > 1, maps and steering not NULL.
 */
int prc_beamscan_frames(const prc_c64* maps, int rows, int cols, int nframes, int64_t frame_stride, int nchan,
                        int64_t chan_stride, const prc_c64* steering, int nangles, int wrap, float* amp_out,
                        float* pos_out, int64_t out_stride, int device, void* stream, unsigned flags);

/* ---- Kalman target trackers ------------------------------------------------------------------------
 * Replace get_measurements(), multitarget_tracker() and simple_target_tracker(), reference
 * passiveRadar/target_detection.py:164-681.  The records below are byte for byte the reference's NumPy
 * dtypes (packed, every field 8 bytes): prc_kalman = kalman_filter_dtype, prc_track = target_track_dtype,
 * prc_track_simple = target_track_dtype_simple.
 *
 * Maps: nseq sequences of nframes frames; frame i of sequence s is at maps + s*seq_stride + i*frame_stride
 * (elements), row-major rows x cols like the reference's data[:, :, i] (rows = Doppler bins, cols = range
 * bins).  float32, or float64 with PRC_FLAG_MAP_F64; arithmetic is float64 either way.  Maps must be finite.
 * Candidates are ordered by strength, descending; equal strengths in descending position of the transformed
 * frame (np.flip(np.argsort(s, kind="stable")); the reference's unstable sort leaves that order open).
 *
 * prc_get_measurements_frames: counts[s*nframes + i] = the frame's exact candidate count (up to rows*cols);
 *   its candidates go to meas + (s*nframes + i) * 3 * meas_capacity as three rows of meas_capacity doubles:
 *   range, Doppler, strength.  Only the first meas_capacity are written; meas_capacity = rows*cols never cuts.
 * prc_multitarget_track_frames: history[(s*nframes + i)*n_tracks + t] = track t after frame i of sequence s.
 *   0 <= n_tracks <= 64.
 * prc_simple_track_frames: history[s*nframes + i] = the tracker state after frame i of sequence s.
 * rows * cols <= 524288.
 *
 * PRC_FLAG_TRACK_RESUME (both trackers) continues sequences instead of starting them fresh.  On entry the
 * frame-0 records of every sequence -- history[s*nframes*n_tracks + t] (multi-target) or history[s*nframes]
 * (simple) -- hold the state to continue from, normally the last frame's records of an earlier call on the
 * same sequence; they are uploaded first with PRC_MEM_HOST.  On return they hold the state after frame 0, as
 * without the flag.  The simple tracker keeps the record's own range_extent / doppler_extent.  A sequence cut
 * anywhere and continued this way gives the same bytes as one call.
 */
typedef struct prc_kalman {
    double x[4], P[16], F1[16], F2[16], Q[16], H[8], R[4], S[4];
} prc_kalman;
typedef struct prc_track {
    int64_t status, lifetime;
    double measurement[2], estimate[2], measurement_history[20];
    prc_kalman kalman_state;
} prc_track;
typedef struct prc_track_simple {
    double lock_mode[4], measurement[2];
    int64_t measurement_idx[2];
    double estimate[2], range_extent, doppler_extent;
    prc_kalman kalman_state;
} prc_track_simple;
#ifdef __cplusplus
static_assert(sizeof(prc_kalman) == 672, "prc_kalman must match kalman_filter_dtype");
static_assert(sizeof(prc_track) == 880, "prc_track must match target_track_dtype");
static_assert(sizeof(prc_track_simple) == 768, "prc_track_simple must match target_track_dtype_simple");
#else
_Static_assert(sizeof(prc_kalman) == 672, "prc_kalman must match kalman_filter_dtype");
_Static_assert(sizeof(prc_track) == 880, "prc_track must match target_track_dtype");
_Static_assert(sizeof(prc_track_simple) == 768, "prc_track_simple must match target_track_dtype_simple");
#endif

int prc_get_measurements_frames(const void* maps, int rows, int cols, int nseq, int nframes, int64_t seq_stride,
                                int64_t frame_stride, double doppler_extent, double range_extent,
                                int64_t meas_capacity, int32_t* counts, double* meas,
                                int mem_kind, int device, void* stream, unsigned flags);
int prc_multitarget_track_frames(const void* maps, int rows, int cols, int nseq, int nframes, int64_t seq_stride,
                                 int64_t frame_stride, double doppler_extent, double range_extent, int n_tracks,
                                 prc_track* history, int mem_kind, int device, void* stream, unsigned flags);
int prc_simple_track_frames(const void* maps, int rows, int cols, int nseq, int nframes, int64_t seq_stride,
                            int64_t frame_stride, double range_extent, double doppler_extent,
                            prc_track_simple* history, int mem_kind, int device, void* stream, unsigned flags);

/* ---- channel offset estimator ---------------------------------------------------------------------
 * prc_channel_offset replaces find_channel_offset(s1, s2, nd, nl), reference passiveRadar/signal_utils.py:73-78:
 *   B1 = decimate(s1, nd), B2 = pad(decimate(s2, nd), (nl, nl)), xc = |correlate(B1, B2, 'valid')|,
 *   *offset = (argmax(xc) - nl) * nd   (the first maximum on ties).
 * decimate is scipy.signal.decimate's default: sosfiltfilt with the order-8 Chebyshev sections
 * cheby1(8, 0.05, 0.8 / nd, output='sos') (odd extension of 27 samples, computed in the input's own dtype as NumPy
 * does, so integer inputs wrap), then every nd-th sample.  sos: 2 x 4 x 6 doubles and zi: 2 x 4 x 2 doubles
 * (= sosfilt_zi(sos)), one block per signal, designed by the caller as decimate does for that signal's dtype (float32-
 * rounded for float32 / complex64 inputs).  All arithmetic is float64 / complex128 whatever the dtypes.
 *   offset : one int64 (host or device, as mem_kind says)
 *   xc_abs : NULL, or the |n1d - (n2d + 2 nl)| + 1 values of |xc| as doubles, n_d = ceil(n / nd)
 * Limits (PRC_E_INVALID): n1, n2 > 27; 1 <= nd <= 64; nl >= 0; a circular transform of at most 2^26 points.
 *
 * prc_xcorr replaces xcorr(s1, s2, nlead, nlag) = correlate(s1, pad(s2, (nlag, nlead)), 'valid') (:29-32): out
 * receives the |n1 - (n2 + nlag + nlead)| + 1 valid lags, complex128 when either input is complex, else float64.
 *
 * Scratch memory is allocated stream-ordered on the call's stream and released before the call returns it.
 */
#define PRC_DT_I8    0
#define PRC_DT_U8    1
#define PRC_DT_I16   2
#define PRC_DT_F32   3
#define PRC_DT_F64   4
#define PRC_DT_C64   5
#define PRC_DT_C128  6
int prc_channel_offset(const void* s1, int dtype1, int64_t n1, const void* s2, int dtype2, int64_t n2, int nd, int64_t nl,
                       const double* sos, const double* zi, int64_t* offset, double* xc_abs,
                       int mem_kind, int device, void* stream, unsigned flags);
int prc_xcorr(const void* s1, int dtype1, int64_t n1, const void* s2, int dtype2, int64_t n2, int64_t nlead, int64_t nlag,
              void* out, int mem_kind, int device, void* stream, unsigned flags);

/* ---- Welch power spectral density -----------------------------------------------------------------
 * prc_psd_frames computes matplotlib.mlab.psd (what plt.psd plots, signal_preview.py:52-72) of nframes frames of n
 * samples, frame f at element f * frame_stride of x (dtype PRC_DT_F32, PRC_DT_F64, PRC_DT_C64 or PRC_DT_C128, widened
 * on load).  Per frame: segments of nfft samples at a step of nfft - noverlap, (n - noverlap) / (nfft - noverlap) of
 * them (a ragged tail is dropped; a frame shorter than nfft is zero-padded to one segment); each segment times
 * window[0 .. nfft), zero-padded to pad_to points and transformed; |X|^2 summed over the segments, times scale, divided
 * by the segment count.  onesided = 0: pad_to bins rotated so that bin 0 is -Fs/2 (mlab's freqcenter = pad_to / 2);
 * onesided = 1: bins 0 .. pad_to/2, every bin but DC doubled, the pad_to/2 bin only when nfft is odd (mlab's rule).
 * Frame f's bins go to out + f * out_stride.  All arithmetic is float64 / complex128.  A frame's result does not
 * depend on nframes or on the device: a frame of a batch is bit-identical to the same frame computed alone.
 *
 * x, window and out are DEVICE pointers (the call has no mem_kind; callers stage host arrays themselves).
 * Limits (PRC_E_INVALID): pad_to a power of two in [16, 8192]; 1 <= nfft <= pad_to; 0 <= noverlap < nfft; n >= 1;
 * nframes >= 1; frame_stride >= n; out_stride >= the output bins; onesided 0 or 1; x, window, out not NULL.
 * Scratch memory is allocated stream-ordered on the call's stream and released before the call returns it.
 */
int prc_psd_frames(const void* x, int dtype, int64_t n, int nframes, int64_t frame_stride, int nfft, int noverlap,
                   int pad_to, const double* window, double scale, int onesided, double* out, int64_t out_stride,
                   int device, void* stream, unsigned flags);

/* ---- FIR decimation and normalisation ---------------------------------------------------------------
 * prc_decimate_rows replaces decimate(x, q) = scipy.signal.decimate(x, q, 20*q, ftype='fir', axis=0) (reference
 * passiveRadar/signal_utils.py:11-13) on nrows rows of n samples, row b at x + b * row_stride elements:
 *   y[m] = sum_{j=0}^{20q} taps[j] * x[m*q + 10q - j],  x = 0 outside [0, n),  m = 0 .. ceil(n/q) - 1,
 * written to out + b * out_stride elements.  taps: 20q + 1 host doubles (firwin(20q+1, 1/q, window='hamming'), rounded
 * to float32 by the caller for float32 / complex64 data, as decimate does); they are copied before the call returns.
 * src is a PRC_DT_* code, or PRC_DEC_RAW + PRC_IQ_C64 / PRC_IQ_I8 / PRC_IQ_I16 for raw interleaved I/Q (float32, int8,
 * int16; I and Q read as scalars) that is deinterleaved and mixed on load with mode, fc, fs and phase_offset exactly as
 * prc_iq_mix_c64 does (channel_preprocessing, signal_utils.py:80-85: the tuned signal is never stored).  For raw I/Q,
 * n and row_stride count complex samples.  Arithmetic and out's dtype:
 *   PRC_DT_F32                              float32 taps and sums, float32 out
 *   PRC_DT_C64, raw with PRC_MIX_NONE/C64   float32 taps and sums, complex64 out
 *   PRC_DT_I8, U8, I16, F64                 float64, float64 out
 *   PRC_DT_C128, raw with the other modes   float64 (raw: the complex64 mixed sample widened), complex128 out
 * A row's result does not depend on nrows or on its place in the batch: row b is bit-identical to a one-row call on it.
 * Limits (PRC_E_INVALID, naming the limit): 2 <= q <= 65536; n >= 1; nrows >= 1; row_stride >= n and out_stride >=
 * ceil(n/q) when nrows > 1; x, taps, out not NULL.
 *
 * prc_normalize replaces normalize(x) = x / mean(|x|) (signal_utils.py:7-9) on n contiguous elements of dtype: the
 * mean of |x| is summed in float64 in a fixed order (no atomics), and out receives NumPy's result dtype: float32 for
 * PRC_DT_F32, complex64 for PRC_DT_C64 (x times float32(1 / float32(mean))), complex128 for PRC_DT_C128, float64 for
 * the rest.  |x| of int8 and int16 wraps at -128 and -32768 as NumPy's abs does.  An all-zero x gives NaN.
 * Limits (PRC_E_INVALID): n >= 1; x, out not NULL.
 *
 * x and out of both are DEVICE pointers (no mem_kind; callers stage host arrays themselves).  Scratch memory is
 * allocated stream-ordered on the call's stream and released before the call returns it.
 */
#define PRC_DEC_RAW 16
int prc_decimate_rows(const void* x, int src, int64_t n, int nrows, int64_t row_stride, int mode, double fc, double fs,
                      double phase_offset, const double* taps, int q, void* out, int64_t out_stride, int device,
                      void* stream, unsigned flags);
int prc_normalize(const void* x, int dtype, int64_t n, void* out, int device, void* stream, unsigned flags);

#ifdef __cplusplus
}
#endif
#endif /* PRCORE_H */
