"""main.py's interleaved-channel branch (main.py:46-75) restated without dask -- TEST INFRASTRUCTURE ONLY.

One raw source holds both channels, ``[ref_I[0], ref_Q[0], srv_I[0], srv_Q[0], ref_I[1], ...]``.  main.py reads it with
``da.from_array(chunks=(2 icl,))``, ``map_blocks(deinterleave_IQ, chunks=(icl,))`` and takes ``[0::2]`` / ``[1::2]``
for the two channels, then trims them by the channel offset in complex samples.  Its ``rechunk((icl,))`` would make
every chunk ``icl`` complex samples, which no later line of main.py expects (``literal_geometry`` shows why it makes
no map), so each channel is cut into chunks of ``h = icl // 2`` samples as the separate-channel branch does, and the
per-chunk chain is ``recording_oracle``'s.  dask's semantics, as ``recording_oracle`` reads them:

* ``nb = ceil(n_raw / (2 icl))`` raw blocks, each declared ``icl`` complex samples long, a partial last block included,
  so ``[0::2]`` declares ``ceil(nb icl / 2)`` samples and ``[1::2]`` ``floor(nb icl / 2)``;
* ``N_chunks = min(N_ref, N_srv, num_frames) - 1`` with ``N_x`` the trimmed declared length over ``h`` (main.py:116-118).
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import scipy.signal as signal

from . import recording_oracle as ro

HERE = os.path.dirname(os.path.abspath(__file__))


def _chunk_ops():
    """(deinterleave_IQ, frequency_shift, resample): the reference's own if oracle/_ref has them, the ports otherwise."""
    ref = os.path.join(HERE, "_ref")
    if os.path.isdir(os.path.join(ref, "passiveRadar")):
        if ref not in sys.path:
            sys.path.insert(0, ref)
        from passiveRadar import signal_utils as su
        return su.deinterleave_IQ, su.frequency_shift, su.resample
    from .clutter_oracle import frequency_shift_oracle
    from .frontend_oracle import deinterleave_iq_oracle, resample_oracle
    return deinterleave_iq_oracle, frequency_shift_oracle, resample_oracle


def raw_slices_interleaved(config, n_raw, offset):
    """main.py:46-75 and 116-118 on a stream of n_raw raw elements: the trimmed channels as (start, stop) pairs in
    complex samples of each channel, and N_chunks.  Sample j of channel q is raw elements 4j + 2q, 4j + 2q + 1."""
    icl = config["input_chunk_length"]
    h = icl // 2
    nb = math.ceil(n_raw / (2 * icl))                   # da.from_array blocks
    declared = nb * icl                                 # map_blocks(deinterleave_IQ, chunks=(icl,))
    idx = np.arange(-(-declared // 2)), np.arange(declared // 2)      # [0::2], [1::2]
    if offset > 0:
        r, s = idx[0][offset:], idx[1][:-offset]
    elif offset < 0:
        r, s = idx[0][:offset], idx[1][-offset:]
    else:
        r, s = idx
    n_chunks = max(min(len(r) // h, len(s) // h, config["num_frames"]) - 1, 0)
    r0 = int(r[0]) if len(r) else max(offset, 0)
    s0 = int(s[0]) if len(s) else max(-offset, 0)
    return (r0, r0 + n_chunks * h), (s0, s0 + n_chunks * h), n_chunks


def literal_geometry(config):
    """The chunk, resampled-chunk and frame lengths of main.py's interleaved branch taken literally (chunks of icl
    complex samples), next to cpi_samples, the inputLen fast_xambg pads every frame to."""
    icl, up, dn = config["input_chunk_length"], config["resamp_up"], config["resamp_dn"]
    g = math.gcd(up, dn)
    resampled = -(-icl * (up // g) // (dn // g))        # resample_poly's output length
    return {"chunk": icl, "resampled": resampled, "frame": resampled + 2 * config["window_overlap"],
            "cpi": config["cpi_samples"]}


def recording_oracle_interleaved(config, stream, offset, stages=False):
    """main.py's xambg, (F, R+1, N_chunks), for one interleaved stream and a channel offset in complex samples.
    ``stages=True`` also returns the per-chunk stages as ``recording_oracle`` does."""
    deinterleave, shift, resample = _chunk_ops()
    _, ls_multiple, xambg, _ = ro._ops()
    h = config["input_chunk_length"] // 2
    (r0, _), (s0, _), n_chunks = raw_slices_interleaved(config, len(stream), offset)
    iq = deinterleave(np.asarray(stream))
    ref, srv = iq[0::2], iq[1::2]
    po = ro.block_phase_offsets(config, n_chunks)
    fo, fs = config["offset_freq"], config["input_sample_rate"]
    up, dn = config["resamp_up"], config["resamp_dn"]
    ref_rs, srv_rs, cleaned = [], [], []
    for k in range(n_chunks):
        ref_rs.append(resample(shift(ref[r0 + k * h:r0 + (k + 1) * h], fo, fs, po[k:k + 1]), up, dn))
        srv_rs.append(resample(shift(srv[s0 + k * h:s0 + (k + 1) * h], fo, fs, po[k:k + 1]), up, dn))
        cleaned.append(ls_multiple(ref_rs[-1], srv_rs[-1], config["num_range_cells"], config["IF_sample_rate"],
                                   ro.DOPPLER_BINS))
    d = config["window_overlap"]
    ref_frames, srv_frames = ro.overlap_frames(ref_rs, d), ro.overlap_frames(cleaned, d)
    window = signal.get_window(('kaiser', 5.0), config['cpi_samples'])
    R, F = config["num_range_cells"], config["num_doppler_cells"]
    maps = [xambg(rf, sf, R, F, config["cpi_samples"], window) for rf, sf in zip(ref_frames, srv_frames)]
    out = np.concatenate(maps, axis=2).astype(np.complex64) if maps else np.zeros((F, R + 1, 0), np.complex64)
    if stages:
        return out, {"ref_rs": ref_rs, "srv_rs": srv_rs, "cleaned": cleaned, "ref_frames": ref_frames,
                     "srv_frames": srv_frames}
    return out
