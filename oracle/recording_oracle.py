"""main.py:86-194 restated without dask -- TEST INFRASTRUCTURE ONLY.

A plain loop over chunks that calls, per chunk, the reference's own modules when ``build()`` placed them under
``oracle/_ref`` and the oracle ports otherwise (``frontend_oracle``, ``ls_filter_multiple_oracle``,
``fast_xambg_oracle``).  Dask is not part of this project's environment, so the dask calls of main.py are read from
dask's documented semantics:

* ``da.from_array(x, chunks=(icl,))`` cuts the raw channel into blocks of ``icl`` elements, the last one partial;
  ``map_blocks(deinterleave_IQ, ..., chunks=(icl // 2,))`` declares every output block ``icl // 2`` long, so
  ``ref_data.shape[0] // (icl // 2)`` is the number of raw blocks, a partial last block included (main.py:116-118).
* ``map_blocks(f, a, b, ...)`` with arrays of the same number of blocks calls ``f`` on block ``k`` of each: chunk ``k``
  of both channels, and block ``k`` (one element) of ``block_phase_offsets`` as a float64 array (main.py:133-149);
  the clutter filter gets chunk ``k`` of the resampled reference and surveillance channels (main.py:169-176).
* ``da.overlap.overlap(x, depth=d, boundary=0)`` extends block ``k`` by the last ``d`` samples of block ``k-1`` and
  the first ``d`` of block ``k+1``, with ``d`` zeros beyond either end of the array (main.py:180-181).
* ``map_blocks(fast_xambg, ..., chunks=(F, R+1, 1))`` stacks the per-frame maps along a new last axis (main.py:186-194).
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import scipy.signal as signal

HERE = os.path.dirname(os.path.abspath(__file__))
DOPPLER_BINS = [0, 1, -1, 2, -2]


def _ops():
    """(frontend, LS_Filter_Multiple, fast_xambg, kind): the reference's functions if oracle/_ref has them."""
    ref = os.path.join(HERE, "_ref")
    if os.path.isdir(os.path.join(ref, "passiveRadar")):
        if ref not in sys.path:
            sys.path.insert(0, ref)
        from passiveRadar import signal_utils as su, clutter_removal as cr, range_doppler_processing as rd
        front = lambda raw, fo, fs, po, up, dn: su.resample(su.frequency_shift(su.deinterleave_IQ(raw), fo, fs, po), up, dn)
        return front, cr.LS_Filter_Multiple, rd.fast_xambg, "reference"
    from .frontend_oracle import frontend_oracle
    from .clutter_oracle import ls_filter_multiple_oracle
    from .xambg_oracle import fast_xambg_oracle
    return frontend_oracle, ls_filter_multiple_oracle, fast_xambg_oracle, "port"


def raw_slices(config, n_ref, n_srv, offset):
    """main.py:87-120: the trimmed raw channels as (start, stop) pairs and N_chunks.  Negative offsets are trimmed as
    main.py:70-72 does (ref[:offset], srv[-offset:])."""
    icl = config["input_chunk_length"]
    idx = np.arange(n_ref), np.arange(n_srv)
    if offset > 0:
        r, s = idx[0][offset:], idx[1][:-offset]
    elif offset < 0:
        r, s = idx[0][:offset], idx[1][-offset:]
    else:
        r, s = idx
    n_blocks_ref = math.ceil(len(r) / icl) if len(r) else 0
    n_blocks_srv = math.ceil(len(s) / icl) if len(s) else 0
    n_chunks = min(n_blocks_ref * (icl // 2) // (icl // 2), n_blocks_srv * (icl // 2) // (icl // 2),
                   config["num_frames"]) - 1
    n_chunks = max(n_chunks, 0)
    r0 = int(r[0]) if len(r) else 0
    s0 = int(s[0]) if len(s) else 0
    return (r0, r0 + n_chunks * icl), (s0, s0 + n_chunks * icl), n_chunks


def block_phase_offsets(config, n_chunks):
    """main.py:125-130."""
    mod_period = config['input_sample_rate'] // config['offset_freq']
    offset_samples_per_block = (config['input_chunk_length'] // 2) % mod_period
    block_numbers = np.arange(n_chunks)
    return 2 * np.pi * block_numbers * offset_samples_per_block * (config['offset_freq'] / config['input_sample_rate'])


def overlap_frames(chunks, depth):
    """da.overlap.overlap(depth=depth, boundary=0) of equal-length blocks: one extended block per input block."""
    chunks = [np.asarray(c) for c in chunks]
    z = np.zeros(depth, dtype=chunks[0].dtype)
    out = []
    for k, c in enumerate(chunks):
        left = chunks[k - 1][len(chunks[k - 1]) - depth:] if k > 0 else z
        right = chunks[k + 1][:depth] if k + 1 < len(chunks) else z
        out.append(np.concatenate([left, c, right]))
    return out


def recording_oracle(config, ref_raw, srv_raw, offset, stages=False):
    """main.py's xambg, (F, R+1, N_chunks), for raw channels and a given channel offset.  ``stages=True`` also returns
    the per-chunk resampled reference, resampled surveillance and cleaned surveillance channels and the frames."""
    front, ls_multiple, xambg, _ = _ops()
    icl = config["input_chunk_length"]
    (r0, _), (s0, _), n_chunks = raw_slices(config, len(ref_raw), len(srv_raw), offset)
    po = block_phase_offsets(config, n_chunks)
    fo, fs = config["offset_freq"], config["input_sample_rate"]
    up, dn = config["resamp_up"], config["resamp_dn"]
    ref_rs, srv_rs, cleaned = [], [], []
    for k in range(n_chunks):
        a = np.asarray(ref_raw[r0 + k * icl:r0 + (k + 1) * icl])
        b = np.asarray(srv_raw[s0 + k * icl:s0 + (k + 1) * icl])
        ref_rs.append(front(a, fo, fs, po[k:k + 1], up, dn))
        srv_rs.append(front(b, fo, fs, po[k:k + 1], up, dn))
        cleaned.append(ls_multiple(ref_rs[-1], srv_rs[-1], config["num_range_cells"], config["IF_sample_rate"],
                                   DOPPLER_BINS))
    d = config["window_overlap"]
    ref_frames, srv_frames = overlap_frames(ref_rs, d), overlap_frames(cleaned, d)
    window = signal.get_window(('kaiser', 5.0), config['cpi_samples'])
    R, F = config["num_range_cells"], config["num_doppler_cells"]
    maps = [xambg(rf, sf, R, F, config["cpi_samples"], window) for rf, sf in zip(ref_frames, srv_frames)]
    out = np.concatenate(maps, axis=2).astype(np.complex64) if maps else np.zeros((F, R + 1, 0), np.complex64)
    if stages:
        return out, {"ref_rs": ref_rs, "srv_rs": srv_rs, "cleaned": cleaned, "ref_frames": ref_frames,
                     "srv_frames": srv_frames}
    return out


def dropin_composition(config, ref_raw, srv_raw, offset):
    """main.py's per-chunk calls made with the GPU drop-ins, as ``passiveradar_b200.install()`` gives them to main.py,
    in one thread without dask: every stage of every chunk is a host -> device -> host call.  Returns (F, R+1, N) and
    the per-chunk (resampled reference, resampled surveillance, cleaned surveillance)."""
    import passiveradar_b200 as prb
    icl = config["input_chunk_length"]
    (r0, _), (s0, _), n_chunks = raw_slices(config, len(ref_raw), len(srv_raw), offset)
    po = block_phase_offsets(config, n_chunks)
    fo, fs, up, dn = config["offset_freq"], config["input_sample_rate"], config["resamp_up"], config["resamp_dn"]
    front = lambda raw, k: prb.resample(prb.frequency_shift(prb.deinterleave_IQ(raw), fo, fs, po[k:k + 1]), up, dn)
    chunks = []
    for k in range(n_chunks):
        a = front(np.asarray(ref_raw[r0 + k * icl:r0 + (k + 1) * icl]), k)
        b = front(np.asarray(srv_raw[s0 + k * icl:s0 + (k + 1) * icl]), k)
        chunks.append((a, b, prb.LS_Filter_Multiple(a, b, config["num_range_cells"], config["IF_sample_rate"],
                                                    DOPPLER_BINS)))
    window = signal.get_window(('kaiser', 5.0), config['cpi_samples'])
    d = config["window_overlap"]
    frames = zip(overlap_frames([c[0] for c in chunks], d), overlap_frames([c[2] for c in chunks], d))
    maps = [prb.fast_xambg(a, b, config["num_range_cells"], config["num_doppler_cells"], config["cpi_samples"], window)
            for a, b in frames]
    return np.concatenate(maps, axis=2), chunks


def stage_truths(config, ref_rs, srv_rs):
    """float64 truths of the chain's later stages on given resampled chunks: ``ls_filter_multiple_truth`` per chunk,
    the overlapped frames of those cleaned chunks, and ``fast_xambg_truth`` per frame.  Returns (F, R+1, N) complex128."""
    from .clutter_oracle import ls_filter_multiple_truth
    from .xambg_oracle import fast_xambg_truth
    R, F, cpi, d = config["num_range_cells"], config["num_doppler_cells"], config["cpi_samples"], config["window_overlap"]
    cleaned = [ls_filter_multiple_truth(r, s, R, config["IF_sample_rate"], DOPPLER_BINS) for r, s in zip(ref_rs, srv_rs)]
    ref_f = overlap_frames([np.asarray(r, dtype=np.complex128) for r in ref_rs], d)
    window = signal.get_window(('kaiser', 5.0), cpi)
    maps = [fast_xambg_truth(a, b, R, F, cpi, window, fast=True) for a, b in zip(ref_f, overlap_frames(cleaned, d))]
    return np.concatenate(maps, axis=2)
