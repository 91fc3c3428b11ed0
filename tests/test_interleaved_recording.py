"""Recording chain on one interleaved two-channel source (PRconfig.yaml's interleaved_input_channels: True,
passiveradar_b200.recording with interleaved_chunking="separate"): the plan against main.py's interleaved branch under
dask's semantics, why the literal reading makes no map, the refusals and the flag's constant (no GPU needed); the
front end with PRC_FLAG_CHANNEL_PAIR against the same calls on the channel sliced out, the maps against the
separate-channel pipeline and the oracle chain, the offset estimate and the target position (GPU)."""
import os
import re

import numpy as np
import pytest
import scipy.signal as signal

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200.recording import RecordingPipeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIPPED, FAST = synth.RECORDING_CONFIGS["shipped"], synth.RECORDING_CONFIGS["fast"]
CONFIGS = {"shipped": SHIPPED, "fast": FAST}


def _inter(config, **kw):
    return dict(config, interleaved_input_channels=True, **kw)


def _pipe(config, **kw):
    return RecordingPipeline.from_config(_inter(config), interleaved_chunking="separate", **kw)


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", ["shipped", "fast"])
def test_plan_matches_main_py_interleaved_branch(name):
    from oracle import interleaved_oracle as io
    from oracle import recording_oracle as ro
    config = CONFIGS[name]
    icl = config["input_chunk_length"]
    h = icl // 2
    for num_frames in (config["num_frames"], 3):
        cfg = _inter(config, num_frames=num_frames)
        pipe = RecordingPipeline.from_config(cfg, interleaved_chunking="separate")
        assert pipe.n_in == h
        for k in (1, 2, 5):
            for extra in (0, 1, 2, 3, 4 * h - 1):
                n_raw = k * 2 * icl + extra
                for offset in (0, 3, -5, h - 1, h, -(h + 1)):
                    p = pipe.plan(n_raw, None, offset)
                    (r0, r1), (s0, s1), N = io.raw_slices_interleaved(cfg, n_raw, offset)
                    assert (p["nchunks"], p["ref_start"], p["srv_start"]) == (N, r0, s0), (n_raw, offset)
                    assert (p["ref_raw_start"], p["srv_raw_start"]) == (4 * r0, 4 * s0 + 2)
                    assert N <= num_frames - 1 or N == 0
                    # every chunk of both channels lies inside the stream's whole quads
                    assert N == 0 or N * h + abs(offset) <= n_raw // 4, (n_raw, offset, N)
                    np.testing.assert_array_equal(p["phase_offsets"], ro.block_phase_offsets(cfg, N))
    # the count is the floor of dask's declared length, not the separate branch's count of raw blocks
    assert _pipe(config).plan(3 * 2 * icl, None, 1)["nchunks"] == 1
    assert RecordingPipeline.from_config(config).plan(3 * icl, 3 * icl, 2)["nchunks"] == 2


@pytest.mark.parametrize("name,frame", [("shipped", 786432), ("fast", 98304)])
def test_literal_reading_makes_no_map(name, frame):
    """main.py's rechunk((input_chunk_length,)) taken literally: every frame is longer than cpi_samples, and
    fast_xambg's zero padding to inputLen = cpi_samples raises on it."""
    from oracle import interleaved_oracle as io
    from oracle import recording_oracle as ro
    config = CONFIGS[name]
    g = io.literal_geometry(config)
    assert g["frame"] == frame and g["resampled"] == config["cpi_samples"] and g["frame"] > g["cpi"]
    assert _pipe(config).frame_len == config["cpi_samples"]          # the chunking offered fills one CPI exactly
    xambg = ro._ops()[2]
    x = np.zeros(frame, np.complex64)
    with pytest.raises(ValueError, match="negative"):
        xambg(x, x, 4, 8, config["cpi_samples"], signal.get_window(("kaiser", 5.0), config["cpi_samples"]))


def test_interleaved_refusals_before_any_launch():
    before = _lib.launch_count() if os.path.exists(_lib.LIB_PATH) else None
    with pytest.raises(NotImplementedError, match="interleaved_chunking='separate'"):
        RecordingPipeline.from_config(_inter(FAST))
    with pytest.raises(ValueError, match="interleaved_chunking='literal'"):
        RecordingPipeline.from_config(_inter(FAST), interleaved_chunking="literal")
    with pytest.raises(ValueError, match="interleaved_input_channels: True only"):
        RecordingPipeline.from_config(FAST, interleaved_chunking="separate")
    with pytest.raises(ValueError, match="even input_chunk_length"):
        RecordingPipeline.from_config(_inter(FAST, input_chunk_length=2400257), interleaved_chunking="separate")
    raw = np.zeros(64, np.int8)
    inter, sep = _pipe(FAST), RecordingPipeline.from_config(FAST)
    with pytest.raises(ValueError, match="pass the one interleaved source only"):
        inter.run(raw, raw, offset=0)
    with pytest.raises(ValueError, match="pass the one interleaved source only"):
        inter.run_device(raw, raw, offset=0)
    with pytest.raises(ValueError, match="pass ref_raw and srv_raw"):
        sep.run(raw, offset=0)
    with pytest.raises(ValueError, match="pass ref_raw and srv_raw"):
        sep.run_device(raw, offset=0)
    if before is not None:
        assert _lib.launch_count() == before


def test_channel_pair_flag_matches_header():
    src = open(os.path.join(ROOT, "include", "prcore.h")).read()
    m = re.search(r"#define\s+PRC_FLAG_CHANNEL_PAIR\s+(\d+)u", src)
    assert m and int(m.group(1)) == _lib.FLAG_CHANNEL_PAIR == 256
    flags = [int(v) for v in re.findall(r"#define\s+PRC_FLAG_\w+\s+(\d+)u", src)]
    assert len(flags) == len(set(flags)), "every flag is its own bit"


# ------------------------------------------------------------------ GPU
_KINDS = ((np.int8, _lib.IQ_I8, "int8"), (np.int16, _lib.IQ_I16, "int16"), (np.float32, _lib.IQ_C64, "float32"))


def _channel(stream, q):
    """channel q's raw I/Q sliced out of a two-channel stream with NumPy"""
    return np.ascontiguousarray(stream.reshape(-1, 4)[:, 2 * q:2 * q + 2]).ravel()


@pytest.mark.gpu
def test_channel_pair_front_end_bit_identical_to_sliced_channel():
    """prc_iq_mix_c64, prc_frontend_c64 and prc_frontend_chunks_c64 with PRC_FLAG_CHANNEL_PAIR on channel q of a stream
    give the bits of the same calls on that channel's raw samples, from host and device memory; no chunk writes past
    its n_out samples.  A host input ends at the channel's last Q (the staged span is exactly the channel's)."""
    import torch
    from passiveradar_b200.signal_utils import _resample_taps
    lib = _lib.load()
    n, start, PAIR = 5003, 11, _lib.FLAG_CHANNEL_PAIR
    for dtype, kind, kname in _KINDS:
        for up, dn in ((13, 119), (3, 2), (1, 1)):
            for mode in (_lib.MIX_C64, _lib.MIX_C128):
                h = _resample_taps(up, dn, mode == _lib.MIX_C64) if up != dn else np.ones(1)
                n_out = -(-n * up // dn)
                for nchunks in (1, 2, 33):
                    total = start + nchunks * n
                    stream = synth.raw_iq(2 * total, kname, seed=nchunks + up + mode)
                    stream_d = torch.from_numpy(stream).cuda()
                    po = np.ascontiguousarray(2 * np.pi * np.arange(nchunks) * 9 * (100000 / 2400000) + 0.1)
                    for q in range(2):
                        chan = _channel(stream, q)[2 * start:]
                        a = 4 * start + 2 * q
                        host = stream[a:a + 2 * (2 * nchunks * n - 1)]      # first I to last Q of the channel
                        want = np.full((nchunks, n_out + 3), np.nan + 0j, dtype=np.complex64)
                        _lib.check(lib.prc_frontend_chunks_c64(chan.ctypes.data, kind, n, nchunks, n, mode, 100000.0,
                                                               2400000.0, po.ctypes.data, up, dn, h.ctypes.data,
                                                               h.shape[0], want.ctypes.data, n_out + 3, want.size,
                                                               _lib.MEM_HOST, 0, None, 0))
                        got = np.full_like(want, np.nan)
                        _lib.check(lib.prc_frontend_chunks_c64(host.ctypes.data, kind, n, nchunks, n, mode, 100000.0,
                                                               2400000.0, po.ctypes.data, up, dn, h.ctypes.data,
                                                               h.shape[0], got.ctypes.data, n_out + 3, got.size,
                                                               _lib.MEM_HOST, 0, None, PAIR))
                        got_d = torch.full((nchunks, n_out + 3), float("nan"), dtype=torch.complex64, device="cuda")
                        _lib.check(lib.prc_frontend_chunks_c64(stream_d.data_ptr() + a * stream.itemsize, kind, n,
                                                               nchunks, n, mode, 100000.0, 2400000.0, po.ctypes.data,
                                                               up, dn, h.ctypes.data, h.shape[0], got_d.data_ptr(),
                                                               n_out + 3, got_d.numel(), _lib.MEM_DEVICE, 0, None, PAIR))
                        torch.cuda.synchronize()
                        msg = f"{kname} {up}/{dn} mode {mode} nchunks {nchunks} channel {q}"
                        for g in (got, got_d.cpu().numpy()):
                            np.testing.assert_array_equal(g[:, :n_out].view(np.uint64), want[:, :n_out].view(np.uint64),
                                                          err_msg=msg)
                            assert np.isnan(g[:, n_out:]).all(), "a chunk's output spilled past its n_out samples"
                        # the single-chunk entry points on chunk 0
                        one = [np.empty(n, np.complex64), np.empty(n_out, np.complex64)]
                        one_d = [torch.empty(n, dtype=torch.complex64, device="cuda"),
                                 torch.empty(n_out, dtype=torch.complex64, device="cuda")]
                        ref = [np.empty(n, np.complex64), np.empty(n_out, np.complex64)]
                        host1 = stream[a:a + 2 * (2 * n - 1)]
                        for src, out, mem, flags in ((chan.ctypes.data, [x.ctypes.data for x in ref], _lib.MEM_HOST, 0),
                                                     (host1.ctypes.data, [x.ctypes.data for x in one], _lib.MEM_HOST,
                                                      PAIR),
                                                     (stream_d.data_ptr() + a * stream.itemsize,
                                                      [x.data_ptr() for x in one_d], _lib.MEM_DEVICE, PAIR)):
                            _lib.check(lib.prc_iq_mix_c64(src, kind, n, mode, 100000.0, 2400000.0, 0.3, out[0], mem, 0,
                                                          None, flags))
                            _lib.check(lib.prc_frontend_c64(src, kind, n, mode, 100000.0, 2400000.0, 0.3, up, dn,
                                                            h.ctypes.data, h.shape[0], out[1], n_out, mem, 0, None,
                                                            flags))
                        torch.cuda.synchronize()
                        for i in range(2):
                            for g in (one[i], one_d[i].cpu().numpy()):
                                np.testing.assert_array_equal(g.view(np.uint64), ref[i].view(np.uint64), err_msg=msg)


def _equal_count_recordings(config, nchunks, seed):
    """A recording both layouts cut into exactly nchunks chunks at any of the tests' offsets: one chunk more than
    nchunks of data, and num_frames capping both counts at nchunks."""
    ref, srv, _, _ = synth.recording_for(config, nchunks + 1, seed=seed)
    return dict(config, num_frames=nchunks + 1), ref, srv


@pytest.mark.gpu
@pytest.mark.parametrize("name,nchunks", [("fast", 8), ("shipped", 5)])
def test_interleaved_maps_bit_identical_to_separate_channels(name, nchunks):
    """The stream synth.interleave_channels(ref, srv) at offset c gives the separate-channel pipeline's maps on
    (ref, srv) at offset 2c raw elements, bit for bit, at the same batch size (the number of maps per call picks the
    CAF's path, so maps of different batch sizes may differ in the last bits): through run at batch 1 and 3,
    run_device and an np.memmap."""
    import tempfile
    import torch
    cfg, ref, srv = _equal_count_recordings(synth.RECORDING_CONFIGS[name], nchunks, seed=41)
    stream = synth.interleave_channels(ref, srv)
    stream_d = torch.from_numpy(stream).cuda()
    seps = {b: RecordingPipeline.from_config(cfg, batch=b) for b in (1, 3)}
    pipes = {b: RecordingPipeline.from_config(_inter(cfg), batch=b, interleaved_chunking="separate") for b in (1, 3)}
    with tempfile.TemporaryDirectory() as d:
        mm = np.memmap(os.path.join(d, "stream"), dtype=stream.dtype, mode="w+", shape=stream.shape)
        mm[:] = stream
        for c in (0, 7, -6):
            want = {b: p.run(ref, srv, offset=2 * c) for b, p in seps.items()}
            for b, pipe in pipes.items():
                assert want[b].shape[2] == nchunks
                np.testing.assert_array_equal(pipe.run(stream, offset=c), want[b], err_msg=f"offset {c} batch {b}")
                assert (pipe.nframes, pipe.offset) == (nchunks, c)
            got_d = pipes[3].run_device(stream_d, offset=c)
            np.testing.assert_array_equal(got_d.cpu().numpy().transpose(1, 2, 0), want[3], err_msg=f"offset {c} device")
            np.testing.assert_array_equal(pipes[1].run(mm, offset=c), want[1], err_msg=f"offset {c} memmap")
        del mm
    with pytest.raises(ValueError, match="contiguous"):
        pipes[3].run_device(stream_d[::2], offset=0)
    with pytest.raises(ValueError, match="must be a tensor on"):
        pipes[3].run_device(torch.from_numpy(stream), offset=0)
    with pytest.raises(TypeError):
        pipes[3].run_device(stream_d.to(torch.int32), offset=0)


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.gpu
def test_interleaved_pipeline_matches_oracle_chain():
    """Every map within 1e-5 + 1.2 x the oracle chain's own distance to the float64 stage truths of
    recording_oracle_interleaved (test_recording.py's end-to-end rule)."""
    from oracle import interleaved_oracle as io
    from oracle import recording_oracle as ro
    nchunks, c = 8, 7
    cfg, ref, srv = _equal_count_recordings(FAST, nchunks, seed=38)
    stream = synth.interleave_channels(ref, srv)
    got = RecordingPipeline.from_config(_inter(cfg), batch=3, interleaved_chunking="separate").run(stream, offset=c)
    want, st = io.recording_oracle_interleaved(_inter(cfg), stream, c, stages=True)
    assert got.shape == want.shape == (FAST["num_doppler_cells"], FAST["num_range_cells"] + 1, nchunks)
    truth = ro.stage_truths(cfg, st["ref_rs"], st["srv_rs"])
    errs = [_rel(got[:, :, k], want[:, :, k]) for k in range(nchunks)]
    own = [_rel(want[:, :, k], truth[:, :, k]) for k in range(nchunks)]
    print(f"[interleaved] maps vs oracle chain {max(errs):.2e}, oracle chain vs truths {max(own):.2e}")
    for k, e in enumerate(errs):
        assert e <= 1e-5 + 1.2 * own[k], (k, e, own[k])


@pytest.mark.gpu
@pytest.mark.parametrize("name,channel_delay", [("fast", 5), ("shipped", -5)])
def test_interleaved_offset_estimate_and_target_position(name, channel_delay):
    """srv lagging ref by c complex samples comes back as offset -c complex samples from host and device sources,
    find_channel_offset's value on [0::2] / [1::2] of deinterleave_IQ(stream[:20 cpi]); with it applied, the target
    peaks at column R - delay and Doppler row F/2 - fd T in every interior frame."""
    import torch
    from oracle.frontend_oracle import deinterleave_iq_oracle
    config = synth.RECORDING_CONFIGS[name]
    ref, srv, delay, kd = synth.recording_for(config, 5, channel_delay=channel_delay, seed=9)
    stream = synth.interleave_channels(ref, srv)
    cpi = config["cpi_samples"]
    iq = deinterleave_iq_oracle(stream[:20 * cpi])
    assert int(prb.find_channel_offset(iq[0::2], iq[1::2], 1, 5_000_000)) == -channel_delay
    pipe = _pipe(config)
    maps = pipe.run_device(torch.from_numpy(stream).cuda()).cpu().numpy()
    assert pipe.offset == -channel_delay
    N = pipe.plan(stream.shape[0], None, -channel_delay)["nchunks"]
    assert pipe.nframes == N >= 3
    hp = _pipe(config)
    np.testing.assert_array_equal(hp.run(stream), maps.transpose(1, 2, 0))
    assert hp.offset == -channel_delay
    R, F = config["num_range_cells"], config["num_doppler_cells"]
    for k in range(1, N - 1):
        m = np.abs(maps[k][:, :R - 4])                    # columns R-4 .. R hold the direct path's residue
        assert np.unravel_index(np.argmax(m), m.shape) == (F // 2 - kd, R - delay), k
