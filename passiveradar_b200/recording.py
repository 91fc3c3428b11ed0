"""Recording chain on one H100: raw two-channel IQ in, overlapped-CPI range-Doppler maps out (main.py:44-194).

``main.py`` turns a recording into a stack of range-Doppler maps with dask: it cuts each raw channel into chunks of
``input_chunk_length`` raw elements (half a CPI once resampled), runs the front end (``deinterleave_IQ`` ->
``frequency_shift`` -> ``resample``) and ``LS_Filter_Multiple`` on every chunk on its own, and then builds every CPI
with ``da.overlap.overlap(depth=window_overlap, boundary=0)``: frame ``k`` is ``[last window_overlap samples of chunk
k-1 | chunk k | first window_overlap samples of chunk k+1]``, zeros beyond the ends of the recording, and the two
halves of a frame were cleaned by different filters.  ``fast_xambg`` with a float64 Kaiser(5.0) window of
``cpi_samples`` then gives one map per chunk.

``RecordingPipeline`` does the same on the device, a batch of chunks at a time:

    pipe = RecordingPipeline.from_config(config)      # the dict the reference's getConfiguration returns
    xambg = pipe.run(ref_raw, srv_raw)                # (F, R+1, nframes) complex64, main.py's layout
    meta = pipe.metadata()                            # frame_timestamps, range_bins, doppler_bins (main.py:200-206)

* the front end of all chunks of a batch is one launch per channel (``prc_frontend_chunks_c64``), the clutter filter
  one call (``prc_ls_multiple_frames_c64``), the overlapped frames are gathered into a contiguous ``(frames, cpi)``
  buffer by a device copy and the maps are one call (``prc_xambg_frames_c64``);
* raw batches are staged in a pinned ring of two slots and copied on a side stream while the previous batch computes;
* the last chunk of a batch and the tail of the one before it are carried into the next batch, so every frame sees
  exactly the neighbours ``overlap`` gives it and the maps do not depend on the batch size.

Only a batch is ever held in host or device memory, so recordings of any length stream through.

Decisions where main.py cannot be followed literally:

* Negative channel offsets: main.py's non-interleaved branch slices ``ref[:-offset]`` and ``srv[offset:]``
  (main.py:93-97), which keeps only ``|offset|`` samples of each channel.  The interleaved branch's trim is applied
  instead (main.py:70-72): ``ref[:offset]``, ``srv[-offset:]``.
* ``overlap_cpi: False`` is refused: the reference's own ``getConfiguration`` raises ``KeyError`` there
  (config.py:77 reads ``config['cpi']``), so no reference run has that geometry.
* ``interleaved_input_channels: True`` (one raw source, ``[ref_I[0], ref_Q[0], srv_I[0], srv_Q[0], ref_I[1], ...]``)
  runs only with ``interleaved_chunking="separate"``, and is refused with ``NotImplementedError`` without it.  That
  branch of main.py (main.py:46-75) rechunks each channel to ``input_chunk_length`` complex samples, while its phase
  offsets, its declared resampled chunks and its overlap depth assume ``input_chunk_length // 2``: taken literally, every
  frame is longer than ``cpi_samples`` and ``fast_xambg``'s padding raises, so it makes no map.  ``"separate"`` cuts
  each channel into chunks of ``input_chunk_length // 2`` complex samples, as the separate-channel branch does; only
  where the samples come from changes.  The offset is then in complex samples: it is estimated as main.py:50-54 does,
  on ``[0::2]`` and ``[1::2]`` of ``deinterleave_IQ(stream[0:20 cpi])``, and trims as main.py:67-72 does.  With
  ``nb = ceil(len(stream) / (2 icl))`` raw blocks dask declares ``nb * (icl // 2)`` samples per channel, so
  ``N_chunks = min((nb * (icl // 2) - |offset|) // (icl // 2), num_frames) - 1``.  An interleaved recording and the
  same channels stored separately, at offset ``c`` against ``2 c`` raw elements, give bit-identical maps when both count
  the same chunks.
* A resampling ratio whose CTA needs more than the front end's 200 KB of shared memory is refused at construction with
  the library's message (``PrcoreError``).
* ``N_chunks = min(N_ref, N_srv, num_frames) - 1`` where ``N_x`` counts the ``input_chunk_length`` blocks dask cuts the
  trimmed raw channel into, a partial last block included (``map_blocks(..., chunks=(icl // 2,))`` declares every
  block ``icl // 2`` long, main.py:105-118).
"""
from __future__ import annotations

import math

import numpy as np
import scipy.signal as signal

from . import _lib
from .signal_utils import (_mix_mode, _offset_sections, _PADLEN, _raw_iq_kind, _raw_sources, _resample_taps,
                           find_channel_offset)

DOPPLER_BINS = (0, 1, -1, 2, -2)         # main.py:174: clutter at 0 Hz, +/-1 Hz, +/-2 Hz
LS_PEEK = 10                             # LS_Filter_Multiple's default (clutter_removal.py:162)
RS_THREADS = 256                         # outputs per resample CTA (frontend.cuh)
SMEM_LIMIT = 200 * 1024                  # shared memory a front-end CTA may use (prcore_host.h)


def resample_smem_refusal(up, dn):
    """The library's refusal of resample_poly(up, dn)'s CTA (prcore_signal.cu: resample_table), or None if it fits."""
    g = math.gcd(up, dn)
    up, dn = up // g, dn // g
    half_len = 10 * max(up, dn)
    nh = 2 * half_len + 1
    n_pre_pad = dn - half_len % dn
    tpp = -(-(n_pre_pad + nh) // up) | 1
    span = ((RS_THREADS - 1) * dn) // up + 2 + tpp
    smem = ((up * tpp * 4 + 15) & ~15) + span * 8
    if smem > SMEM_LIMIT:
        return f"resample {up}/{dn} with {nh} taps needs {smem} bytes of shared memory per CTA"
    return None


def trim(n_ref, n_srv, offset):
    """(ref_start, ref_stop, srv_start, srv_stop): the raw-element slices main.py:87-102 takes for a channel offset
    (negative offsets as main.py:70-72 does, see the module docstring)."""
    offset = int(offset)
    if offset > 0:
        r, s = slice(offset, None), slice(None, -offset)
    elif offset < 0:
        r, s = slice(None, offset), slice(-offset, None)
    else:
        r, s = slice(None), slice(None)
    r0, r1, _ = r.indices(n_ref)
    s0, s1, _ = s.indices(n_srv)
    return r0, max(r0, r1), s0, max(s0, s1)


class RecordingPipeline:
    """main.py's recording chain on one device; see the module docstring.  ``batch`` chunks are processed per step."""

    def __init__(self, config, *, batch=8, device=None, interleaved_chunking=None):
        self.interleaved = bool(config.get("interleaved_input_channels"))
        if interleaved_chunking is not None and not self.interleaved:
            raise ValueError("interleaved_chunking applies to interleaved_input_channels: True only")
        if self.interleaved and interleaved_chunking is None:
            raise NotImplementedError(
                "interleaved_input_channels: True needs interleaved_chunking='separate': main.py's interleaved branch "
                "rechunks to input_chunk_length complex samples while its phase offsets, resampled chunks and overlap "
                "assume input_chunk_length // 2, so taken literally its frames exceed cpi_samples and it makes no map; "
                "'separate' cuts each channel into input_chunk_length // 2 samples as the separate-channel branch does")
        if self.interleaved and interleaved_chunking != "separate":
            raise ValueError(f"interleaved_chunking={interleaved_chunking!r}: the one chunking offered is 'separate'")
        if self.interleaved and int(config["input_chunk_length"]) % 2:
            raise ValueError("interleaved_input_channels: True needs an even input_chunk_length (config.py makes it so)")
        if not config.get("overlap_cpi"):
            raise ValueError("overlap_cpi: False is not supported: the reference's getConfiguration raises KeyError "
                             "for it (config.py:77), so main.py never runs that geometry")
        self.cpi = int(config["cpi_samples"])
        self.up, self.dn = int(config["resamp_up"]), int(config["resamp_dn"])
        self.fs, self.fo = config["input_sample_rate"], config["offset_freq"]
        self.if_rate = float(config["IF_sample_rate"])
        self.icl = int(config["input_chunk_length"])
        self.depth = int(config["window_overlap"])
        self.R, self.F = int(config["num_range_cells"]), int(config["num_doppler_cells"])
        self.num_frames = int(config["num_frames"])
        self.frame_interval = config["frame_interval"]
        self.range_cell_width = config["range_cell_width"]
        self.doppler_cell_width = config["doppler_cell_width"]
        self.batch = max(1, int(batch))
        self.device = device
        self.n_in = self.icl // 2                                      # complex samples per chunk
        g = math.gcd(self.up, self.dn)
        self.Lc = -(-self.n_in * (self.up // g) // (self.dn // g))      # resampled samples per chunk
        self.frame_len = self.Lc + 2 * self.depth
        if self.frame_len > self.cpi:
            raise ValueError("index can't contain negative values")    # np.pad in fast_xambg (inputLen padding)
        if not 0 <= self.depth <= self.Lc:
            # a frame takes its overlap from the two neighbouring chunks only (config.py sets depth = cpi/4 <= Lc)
            raise ValueError(f"window_overlap={self.depth} must lie in [0, {self.Lc}], the resampled chunk length")
        if self.up // g != 1 or self.dn // g != 1:
            msg = resample_smem_refusal(self.up, self.dn)
            if msg:
                raise _lib.PrcoreError(_lib.PRC_E_INVALID, msg)
        # phase offsets are a float64 dask array in main.py:127-130, so frequency_shift sees a NumPy array
        self.mix_mode = _mix_mode(self.fo, self.fs, np.zeros(1))[0]
        self.taps = (_resample_taps(self.up // g, self.dn // g, self.mix_mode == _lib.MIX_C64) if g != self.up or
                     g != self.dn else np.ones(1))              # 1/1: resample_poly returns its input, no taps
        self.window = signal.get_window(("kaiser", 5.0), self.cpi)
        self.nframes = None
        self.offset = None

    @classmethod
    def from_config(cls, config, **kw):
        """From the dict ``passiveRadar.config.getConfiguration`` returns (main.py:231).  An interleaved config needs
        ``interleaved_chunking="separate"`` (see the module docstring)."""
        return cls(config, **kw)

    # ------------------------------------------------------------------ geometry (no device)
    def phase_offsets(self, nchunks):
        """main.py:125-130: 2 pi b ((icl // 2) % (fs // fo)) (fo / fs) for chunk b, float64."""
        mod_period = self.fs // self.fo
        per_block = (self.icl // 2) % mod_period
        return 2 * np.pi * np.arange(nchunks) * per_block * (self.fo / self.fs)

    def plan(self, n_ref, n_srv, offset):
        """Raw slices and chunk count main.py:86-120 gives raw channels of n_ref / n_srv elements.  Interleaved: n_ref
        is the stream's raw length, n_srv is None and the offset is in complex samples; the channel starts are in
        complex samples, and sample j of channel q (0 = ref, 1 = srv) is raw elements 4j + 2q and 4j + 2q + 1."""
        if self.interleaved:
            h, offset = self.n_in, int(offset)
            nb = -(-int(n_ref) // (2 * self.icl))                 # da.from_array(chunks=(2 icl,)) blocks
            nchunks = max(0, min((nb * h - abs(offset)) // h, self.num_frames) - 1)
            r0, s0 = max(offset, 0), max(-offset, 0)
            return {"ref_start": r0, "srv_start": s0, "ref_raw_start": 4 * r0, "srv_raw_start": 4 * s0 + 2,
                    "nchunks": nchunks, "phase_offsets": self.phase_offsets(nchunks)}
        r0, r1, s0, s1 = trim(n_ref, n_srv, offset)
        blocks = lambda n: -(-n // self.icl)
        nchunks = max(0, min(blocks(r1 - r0), blocks(s1 - s0), self.num_frames) - 1)
        return {"ref_start": r0, "srv_start": s0, "ref_len": r1 - r0, "srv_len": s1 - s0, "nchunks": nchunks,
                "phase_offsets": self.phase_offsets(nchunks)}

    def frame_window(self, k):
        """[start, stop) of frame k in the concatenated resampled stream (zeros outside [0, nchunks * Lc))."""
        return k * self.Lc - self.depth, (k + 1) * self.Lc + self.depth

    def metadata(self, nframes=None):
        """main.py:200-206, from the shape of the (F, R+1, nframes) result."""
        nframes = self.nframes if nframes is None else int(nframes)
        if nframes is None:
            raise ValueError("metadata() needs nframes before the first run")
        return {"frame_timestamps": np.arange(nframes) * self.frame_interval,
                "range_bins": np.arange(self.R + 1) * self.range_cell_width,
                "doppler_bins": np.arange(-1 * self.F, self.F) * self.doppler_cell_width}

    # ------------------------------------------------------------------ the batch loop
    def _stream(self, nchunks, torch_device, compute, emit):
        """Run the chunks in batches.  ``compute(c0, nb, ref_rows, srv_rows)`` writes the resampled reference and the
        cleaned surveillance channel of chunks c0 .. c0+nb-1 into the given (nb, Lc) rows; ``emit(j0, ref_frames,
        srv_frames)`` receives frames j0 .. j0+m-1 as (m, cpi) tensors, zero-padded past Lc + 2 depth.

        Row r of the channel buffers holds chunk c0 - 2 + r: rows 0 and 1 are carried from the previous batch (zeros
        before the first), and the row after the batch is zero for the last one, as overlap(boundary=0) pads."""
        import torch
        B, Lc, d = self.batch, self.Lc, self.depth
        bufs = [torch.zeros((B + 3) * Lc, dtype=torch.complex64, device=torch_device) for _ in range(2)]
        frames = [torch.zeros(B + 1, self.cpi, dtype=torch.complex64, device=torch_device) for _ in range(2)]
        for c0 in range(0, nchunks, B):
            nb = min(B, nchunks - c0)
            last = c0 + nb == nchunks
            compute(c0, nb, *(b[2 * Lc:(nb + 2) * Lc].view(nb, Lc) for b in bufs))
            if last:
                for b in bufs:
                    b[(nb + 2) * Lc:(nb + 3) * Lc].zero_()
            j0 = max(c0 - 1, 0)
            j1 = c0 + nb if last else c0 + nb - 1                 # frames j0 .. j1-1 have both neighbours now
            m = j1 - j0
            if m > 0:
                start = (j0 - c0 + 2) * Lc - d
                for b, f in zip(bufs, frames):
                    f[:m, :self.frame_len].copy_(b[start:start + (m - 1) * Lc + self.frame_len].unfold(0, self.frame_len, Lc))
                emit(j0, frames[0][:m], frames[1][:m])
            if not last:                                          # chunk c0+nb-1 and the tail of c0+nb-2
                for b in bufs:
                    b[Lc - d:2 * Lc].copy_(b[(nb + 1) * Lc - d:(nb + 2) * Lc].clone())

    # ------------------------------------------------------------------ device work of one batch
    def _setup(self):
        import torch
        if not torch.cuda.is_available():
            raise _lib.PrcoreError(_lib.PRC_E_CUDA, "RecordingPipeline needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.dev = _lib.current_device(self.device)
        self.tdev = torch.device("cuda", self.dev)
        with torch.cuda.device(self.tdev):
            self.stream = torch.cuda.Stream(device=self.tdev)
            self.copy_stream = torch.cuda.Stream(device=self.tdev)
        self.win_d = torch.from_numpy(np.ascontiguousarray(self.window, dtype=np.float64)).to(self.tdev)
        self.bins = np.ascontiguousarray(DOPPLER_BINS, dtype=np.float64)
        self.srv_rs = torch.empty(self.batch, self.Lc, dtype=torch.complex64, device=self.tdev)

    def _frontend(self, raw_ptr, kind, nb, phase_offsets, out_ptr):
        po = np.ascontiguousarray(phase_offsets, dtype=np.float64)
        _lib.check(self.lib.prc_frontend_chunks_c64(
            raw_ptr, kind, self.n_in, nb, self.n_in, self.mix_mode, float(self.fo), float(self.fs), po.ctypes.data,
            self.up, self.dn, self.taps.ctypes.data, self.taps.shape[0], out_ptr, self.Lc, nb * self.Lc,
            _lib.MEM_DEVICE, self.dev, self.stream.cuda_stream,
            _lib.FLAG_ASYNC | (_lib.FLAG_CHANNEL_PAIR if self.interleaved else 0)))

    def _clean(self, ref_rows, srv_rs, out_rows, nb):
        _lib.check(self.lib.prc_ls_multiple_frames_c64(
            ref_rows.data_ptr(), srv_rs.data_ptr(), self.Lc, nb, self.Lc, self.R, LS_PEEK, self.if_rate,
            self.bins.ctypes.data, self.bins.shape[0], out_rows.data_ptr(), _lib.MEM_DEVICE, self.dev,
            self.stream.cuda_stream, _lib.FLAG_ASYNC))

    def _maps(self, ref_frames, srv_frames, out):
        m = ref_frames.shape[0]
        _lib.check(self.lib.prc_xambg_frames_c64(
            ref_frames.data_ptr(), srv_frames.data_ptr(), self.cpi, m, self.cpi, self.R, self.F, self.win_d.data_ptr(),
            out.data_ptr(), _lib.MEM_DEVICE, self.dev, self.stream.cuda_stream, _lib.FLAG_ASYNC))

    def _offset_device(self, ref_d, srv_d):
        """find_channel_offset(ref[:10 cpi], srv[:10 cpi], 1, 5_000_000) (main.py:81-83) on device-resident raw data."""
        import torch
        a, b = ref_d[:10 * self.cpi], srv_d[:10 * self.cpi]
        dt = [_lib.DT_CODES[_lib.np_dtype(t.dtype)] for t in (a, b)]
        sos, zi = _offset_sections(1, a.dtype == torch.float32, b.dtype == torch.float32)
        off = torch.zeros(1, dtype=torch.int64, device=self.tdev)
        _lib.check(self.lib.prc_channel_offset(a.data_ptr(), dt[0], a.shape[0], b.data_ptr(), dt[1], b.shape[0], 1,
                                               5_000_000, sos.ctypes.data, zi.ctypes.data, off.data_ptr(), None,
                                               _lib.MEM_DEVICE, self.dev, self.stream.cuda_stream, 0))
        return int(off.item())

    def _offset_interleaved(self, head, kind):
        """find_channel_offset(refc1, srvc1, 1, 5_000_000) (main.py:50-54) for device-resident raw data head =
        stream[0:20 cpi]: refc1 and srvc1 are [0::2] and [1::2] of deinterleave_IQ(head), complex64, so the offset is
        in complex samples.  Both channels are read out of the stream in place."""
        import torch
        m = head.shape[0] // 2                                    # deinterleave_IQ's complex samples
        lens = ((m + 1) // 2, m // 2)
        if min(lens) <= _PADLEN:
            raise ValueError(f"The length of the input vector x must be greater than padlen, which is {_PADLEN}.")
        chans = [torch.empty(n, dtype=torch.complex64, device=self.tdev) for n in lens]
        for q in range(2):
            _lib.check(self.lib.prc_iq_mix_c64(head.data_ptr() + 2 * q * head.element_size(), kind, lens[q],
                                               _lib.MIX_NONE, 0.0, 1.0, 0.0, chans[q].data_ptr(), _lib.MEM_DEVICE,
                                               self.dev, self.stream.cuda_stream,
                                               _lib.FLAG_ASYNC | _lib.FLAG_CHANNEL_PAIR))
        sos, zi = _offset_sections(1, True, True)
        off = torch.zeros(1, dtype=torch.int64, device=self.tdev)
        _lib.check(self.lib.prc_channel_offset(chans[0].data_ptr(), _lib.DT_C64, lens[0], chans[1].data_ptr(),
                                               _lib.DT_C64, lens[1], 1, 5_000_000, sos.ctypes.data, zi.ctypes.data,
                                               off.data_ptr(), None, _lib.MEM_DEVICE, self.dev,
                                               self.stream.cuda_stream, 0))
        return int(off.item())

    def _reads(self, p):
        """Where the front end reads a plan's chunks: for each channel the raw element of its source where its chunk 0
        starts and the source it is in (0 or 1), and the raw elements from one chunk to the next."""
        if self.interleaved:
            return (p["ref_raw_start"], p["srv_raw_start"]), (0, 0), 4 * self.n_in
        return (p["ref_start"], p["srv_start"]), (0, 1), self.icl

    # ------------------------------------------------------------------ public entry points
    def run_device(self, ref_raw, srv_raw=None, maps=None, offset=None):
        """ref_raw, srv_raw: 1-D contiguous raw interleaved IQ CUDA tensors (int8, int16 or float32) on the pipeline's
        device; for an interleaved pipeline ref_raw is the one two-channel stream and srv_raw is None, and ``offset``
        is in complex samples.  Writes the maps as (nframes, F, R+1) complex64 into ``maps`` (allocated when None) on
        the device and returns it.  Work is forked from, and joined back into, the current torch stream: the raw tensors
        may still be being written by work queued there, and the maps are ready for work queued there after the call."""
        import torch
        srcs = _raw_sources(self.interleaved, ref_raw, srv_raw)
        self._setup()
        kinds = [_raw_iq_kind(name, t, self.tdev) for name, t in zip(("ref_raw", "srv_raw"), srcs)]
        cur = torch.cuda.current_stream(self.tdev)
        self.stream.wait_stream(cur)
        if offset is None:
            with torch.cuda.stream(self.stream):
                offset = (self._offset_interleaved(ref_raw[:20 * self.cpi], kinds[0]) if self.interleaved else
                          self._offset_device(ref_raw, srv_raw))
        p = self.plan(ref_raw.shape[0], None if self.interleaved else srv_raw.shape[0], offset)
        N = p["nchunks"]
        if maps is None:                  # allocated on the caller's stream, which it is returned to
            maps = torch.empty(N, self.F, self.R + 1, dtype=torch.complex64, device=self.tdev)
        elif (maps.device != self.tdev or maps.dtype != torch.complex64 or not maps.is_contiguous()
              or maps.dim() != 3 or maps.shape[0] < N or tuple(maps.shape[1:]) != (self.F, self.R + 1)):
            raise ValueError(f"maps must be a contiguous complex64 tensor of shape (>= {N}, {self.F}, {self.R + 1}) "
                             f"on {self.tdev}")
        with torch.cuda.stream(self.stream):
            starts, src, step = self._reads(p)
            size = [t.element_size() for t in srcs]
            base = [t.data_ptr() for t in srcs]

            def compute(c0, nb, ref_rows, srv_rows):
                po = p["phase_offsets"][c0:c0 + nb]
                raw = [base[src[q]] + (starts[q] + c0 * step) * size[src[q]] for q in range(2)]
                self._frontend(raw[0], kinds[src[0]], nb, po, ref_rows.data_ptr())
                self._frontend(raw[1], kinds[src[1]], nb, po, self.srv_rs.data_ptr())
                self._clean(ref_rows, self.srv_rs[:nb], srv_rows, nb)

            self._stream(N, self.tdev, compute, lambda j0, rf, sf: self._maps(rf, sf, maps[j0:j0 + rf.shape[0]]))
        cur.wait_stream(self.stream)
        self.nframes, self.offset = N, int(offset)
        return maps

    def run(self, ref_raw, srv_raw=None, offset=None):
        """ref_raw, srv_raw: 1-D raw interleaved IQ sources (ndarray, np.memmap, h5py dataset: anything sliceable),
        int8, int16 or float32; for an interleaved pipeline ref_raw is the one two-channel stream and srv_raw is None,
        and ``offset`` is in complex samples.  Returns main.py's ``xambg``: (F, R+1, nframes) complex64 on the host."""
        import torch
        from .frames import pinned_empty
        srcs = _raw_sources(self.interleaved, ref_raw, srv_raw)
        self._setup()
        dtypes = [np.dtype(x.dtype) for x in srcs]
        kinds = [_lib.IQ_KINDS[dt] for dt in dtypes]
        if offset is None and self.interleaved:
            with torch.cuda.stream(self.stream):             # the head's copy is ordered before its reads
                head = torch.from_numpy(np.ascontiguousarray(ref_raw[0:20 * self.cpi])).to(self.tdev)
                offset = self._offset_interleaved(head, kinds[0])
        elif offset is None:
            offset = find_channel_offset(ref_raw[0:10 * self.cpi], srv_raw[0:10 * self.cpi], 1, 5_000_000, device=self.dev)
        p = self.plan(ref_raw.shape[0], None if self.interleaved else srv_raw.shape[0], offset)
        N, B = p["nchunks"], self.batch
        starts, src, step = self._reads(p)
        # a batch of nb chunks from chunk c0 stages raw elements [win[j] + c0 step, + nb step + extra) of source j: the
        # stream's window holds both channels' chunks, the trimmed channel's |offset| samples later than the other's
        win, extra = ((0,), 4 * abs(int(offset))) if self.interleaved else (starts, 0)
        at = [starts[q] - win[src[q]] for q in range(2)]        # channel q's first chunk in its staged window
        out = np.empty((self.F, self.R + 1, N), dtype=np.complex64)
        # two slots of raw batches (pinned host, device), of maps (device, pinned host); kept for the next run, since
        # page-locking them costs more than a short recording takes
        tdt = [_lib.torch_dtype(dt) for dt in dtypes]
        slot = B * step + extra
        if getattr(self, "_ring_key", None) != (tuple(dtypes), slot, self.dev):
            self._ring = ([[torch.empty(slot, dtype=t, pin_memory=True) for t in tdt] for _ in range(2)],
                          [[torch.empty(slot, dtype=t, device=self.tdev) for t in tdt] for _ in range(2)],
                          [torch.empty(B + 1, self.F, self.R + 1, dtype=torch.complex64, device=self.tdev)
                           for _ in range(2)],
                          [pinned_empty((B + 1, self.F, self.R + 1)) for _ in range(2)])
            self._ring_key = (tuple(dtypes), slot, self.dev)
        host_raw, dev_raw, dev_maps, host_maps = self._ring
        copied = [torch.cuda.Event() for _ in range(2)]         # raw slot's host-to-device copy done
        read = [torch.cuda.Event() for _ in range(2)]           # raw slot's front end done
        landed = [torch.cuda.Event() for _ in range(2)]         # maps slot's device-to-host copy done
        pending = [None, None]                                  # (j0, m) of the maps in host_maps[s]
        state = {"batch": 0, "emitted": 0}

        def drain(s):
            if pending[s] is not None:
                landed[s].synchronize()
                j0, m = pending[s]
                out[:, :, j0:j0 + m] = host_maps[s][:m].transpose(1, 2, 0)
                pending[s] = None

        def compute(c0, nb, ref_rows, srv_rows):
            s = state["batch"] % 2
            state["batch"] += 1
            if state["batch"] > 2:
                copied[s].synchronize()                         # the slot's previous copy has left host memory
            L = nb * step + extra
            for j, x in enumerate(srcs):
                a = win[j] + c0 * step
                host_raw[s][j][:L].numpy()[:] = np.asarray(x[a:a + L])
            with torch.cuda.stream(self.copy_stream):
                self.copy_stream.wait_event(read[s])            # the batch two back has finished reading the slot
                for j in range(len(srcs)):
                    dev_raw[s][j][:L].copy_(host_raw[s][j][:L], non_blocking=True)
                copied[s].record(self.copy_stream)
            self.stream.wait_event(copied[s])
            po = p["phase_offsets"][c0:c0 + nb]
            raw = [dev_raw[s][src[q]].data_ptr() + at[q] * dev_raw[s][src[q]].element_size() for q in range(2)]
            self._frontend(raw[0], kinds[src[0]], nb, po, ref_rows.data_ptr())
            self._frontend(raw[1], kinds[src[1]], nb, po, self.srv_rs.data_ptr())
            read[s].record(self.stream)
            self._clean(ref_rows, self.srv_rs[:nb], srv_rows, nb)

        def emit(j0, rf, sf):
            s = state["emitted"] % 2
            state["emitted"] += 1
            drain(s)                                            # the slot's maps from two emits back are in `out`
            m = rf.shape[0]
            self._maps(rf, sf, dev_maps[s][:m])
            torch.from_numpy(host_maps[s])[:m].copy_(dev_maps[s][:m], non_blocking=True)
            landed[s].record(self.stream)
            pending[s] = (j0, m)

        with torch.cuda.stream(self.stream):
            self._stream(N, self.tdev, compute, emit)
        for s in range(2):
            drain(s)
        self.stream.synchronize()
        self.nframes, self.offset = N, int(offset)
        return out
