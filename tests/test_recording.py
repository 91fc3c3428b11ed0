"""Recording chain (main.py:44-194, passiveradar_b200.recording): the plan, the frame assembly, the refusals and the
metadata (no GPU needed); prc_frontend_chunks_c64 against per-chunk front-end calls, and RecordingPipeline against the
oracle chain and the per-chunk composition of the GPU drop-ins (GPU)."""
import os
import re

import numpy as np
import pytest
import scipy.signal as signal

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth
from passiveradar_b200.recording import RecordingPipeline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECORDING = os.path.join(ROOT, "passiveradar_b200", "csrc", "recording.cuh")

SHIPPED, FAST = synth.RECORDING_CONFIGS["shipped"], synth.RECORDING_CONFIGS["fast"]
# derived with the reference's getConfiguration from PRconfig.yaml with channel_bandwidth 25 kHz, cpi_seconds_nominal 2,
# max_doppler_nominal 32 and max_range_nominal 400: a ratio beyond the resampler
WIDE = {'cpi_samples': 65536, 'resamp_up': 17, 'resamp_dn': 1245, 'input_sample_rate': 2400000, 'offset_freq': 100000,
        'IF_sample_rate': 32771.0843373494, 'input_chunk_length': 4799548, 'window_overlap': 16384,
        'num_range_cells': 44, 'num_doppler_cells': 128, 'num_frames': 1200, 'overlap_cpi': True,
        'interleaved_input_channels': False, 'frame_interval': 0.9999058823529412,
        'range_cell_width': 9.148308823529412, 'doppler_cell_width': 0.5000470632530121}


# ------------------------------------------------------------------ CPU: plan, assembly, refusals, metadata
@pytest.mark.parametrize("config,Lc,depth,per_block", [(SHIPPED, 262144, 131072, 9), (FAST, 32768, 16384, 8)])
@pytest.mark.parametrize("offset", [0, 2, 7, -6])
def test_plan_matches_main_py_geometry(config, Lc, depth, per_block, offset):
    from oracle import recording_oracle as ro
    pipe = RecordingPipeline.from_config(config)
    icl = config["input_chunk_length"]
    assert (pipe.n_in, pipe.Lc, pipe.depth, pipe.frame_len) == (icl // 2, Lc, depth, config["cpi_samples"])
    for n_chunks_raw in (3.0, 5.5, 8.0):
        n = int(n_chunks_raw * icl) + 11
        p = pipe.plan(n, n + 5, offset)
        (r0, r1), (s0, s1), N = ro.raw_slices(config, n, n + 5, offset)
        assert (p["nchunks"], p["ref_start"], p["srv_start"]) == (N, r0, s0)
        assert p["ref_start"] + N * icl <= p["ref_start"] + p["ref_len"]
        assert p["srv_start"] + N * icl <= p["srv_start"] + p["srv_len"]
        want_r0 = max(offset, 0)
        want_s0 = max(-offset, 0)
        assert (p["ref_start"], p["srv_start"]) == (want_r0, want_s0)
        assert (p["ref_len"], p["srv_len"]) == (n - abs(offset), n + 5 - abs(offset))
        assert N == -(-(n - abs(offset)) // icl) - 1          # dask's block count of the shorter channel, minus one
    po = pipe.phase_offsets(5)
    assert po.dtype == np.float64
    np.testing.assert_array_equal(po, ro.block_phase_offsets(config, 5))
    np.testing.assert_array_equal(po, 2 * np.pi * np.arange(5) * per_block * (100000 / 2400000))
    assert pipe.mix_mode == _lib.MIX_C128
    for k in range(4):
        assert pipe.frame_window(k) == (k * Lc - depth, (k + 1) * Lc + depth)


@pytest.mark.parametrize("batch", [1, 2, 3, 7])
@pytest.mark.parametrize("nchunks", [1, 2, 5, 7])
def test_toy_chain_frames_equal_the_oracle_overlap(batch, nchunks):
    """Chunk k holds the value k (reference) and -k (cleaned surveillance): the batch loop's frames are exactly the
    ones overlap(depth, boundary=0) gives, whatever the batch size."""
    import torch
    from oracle import recording_oracle as ro
    pipe = RecordingPipeline.from_config(FAST, batch=batch)
    pipe.Lc, pipe.depth, pipe.cpi = 8, 3, 16              # a small geometry: frame_len 14 < cpi, zero-padded
    pipe.frame_len = pipe.Lc + 2 * pipe.depth
    ramp = np.arange(pipe.Lc) * 1j

    def compute(c0, nb, ref_rows, srv_rows):
        for i in range(nb):
            ref_rows[i] = torch.from_numpy((c0 + i + 1 + ramp).astype(np.complex64))
            srv_rows[i] = torch.from_numpy((-(c0 + i + 1) + ramp).astype(np.complex64))

    got = {}

    def emit(j0, rf, sf):
        for i in range(rf.shape[0]):
            assert j0 + i not in got
            got[j0 + i] = (rf[i].numpy().copy(), sf[i].numpy().copy())

    pipe._stream(nchunks, "cpu", compute, emit)
    assert sorted(got) == list(range(nchunks))
    want_r = ro.overlap_frames([(k + 1 + ramp).astype(np.complex64) for k in range(nchunks)], 3)
    want_s = ro.overlap_frames([(-(k + 1) + ramp).astype(np.complex64) for k in range(nchunks)], 3)
    for k in range(nchunks):
        np.testing.assert_array_equal(got[k][0], np.pad(want_r[k], (0, 2)))
        np.testing.assert_array_equal(got[k][1], np.pad(want_s[k], (0, 2)))


def test_refusals_before_any_launch():
    before = _lib.launch_count() if os.path.exists(_lib.LIB_PATH) else None
    with pytest.raises(NotImplementedError):
        RecordingPipeline.from_config(dict(FAST, interleaved_input_channels=True))
    with pytest.raises(ValueError, match="overlap_cpi"):
        RecordingPipeline.from_config(dict(FAST, overlap_cpi=False))
    with pytest.raises(_lib.PrcoreError, match=r"resample 17/1245 with 24901 taps needs 266384 bytes of shared memory"):
        RecordingPipeline.from_config(WIDE)
    with pytest.raises(ValueError, match="index can't contain negative values"):
        RecordingPipeline.from_config(dict(FAST, window_overlap=16385))
    with pytest.raises(ValueError, match="window_overlap=32769 must lie in"):
        RecordingPipeline.from_config(dict(FAST, window_overlap=32769, cpi_samples=1 << 18))
    with pytest.raises(ValueError, match="index can't contain negative values"):
        np.pad(np.zeros(4), (0, -1))                     # the message fast_xambg's inputLen padding gives
    if before is not None:
        assert _lib.launch_count() == before


def test_metadata_matches_main_py():
    pipe = RecordingPipeline.from_config(SHIPPED)
    m = pipe.metadata(7)
    F, R = SHIPPED["num_doppler_cells"], SHIPPED["num_range_cells"]
    xambg_shape = (F, R + 1, 7)
    np.testing.assert_array_equal(m["frame_timestamps"], np.arange(xambg_shape[2]) * SHIPPED['frame_interval'])
    np.testing.assert_array_equal(m["range_bins"], np.arange(xambg_shape[1]) * SHIPPED['range_cell_width'])
    np.testing.assert_array_equal(m["doppler_bins"],
                                  np.arange(-1 * xambg_shape[0], xambg_shape[0]) * SHIPPED['doppler_cell_width'])
    assert m["doppler_bins"].shape == (2 * F,)


def test_abi_entry_is_declared():
    assert "prc_frontend_chunks_c64" in _lib.SIGNATURES
    assert "prc_frontend_chunks_c64" in open(os.path.join(ROOT, "include", "prcore.h")).read()
    assert prb.RecordingPipeline is RecordingPipeline


def test_recording_kernels_build_for_sm90a_without_spills():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    blocks = [blk for blk in open(log).read().split("Compiling entry function")[1:]
              if "3prc3rec" in blk.split("\n")[0]]
    assert len(blocks) == 3, "ends, resample, mix"
    for blk in blocks:
        assert "'sm_90a'" in blk.split("\n")[0]
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in blk


# every launch in recording.cuh -> the GPU tests that reach it (a test of this file, or "tests/<file>::<test>")
FE, RS = "tests/test_gpu_frontend.py::", "tests/test_rows_sweep.py::"
COVERAGE = {
    "rec_ends_kernel": ["test_frontend_chunks_bit_identical_to_per_chunk_calls", "test_pipeline_matches_oracle_chain",
                        FE + "test_resample_matches_reference_golden",
                        RS + "test_resample_short_inputs"],                      # n = 1 (NaN as SciPy), 2, 3, 27
    "rec_resample_kernel": ["test_frontend_chunks_bit_identical_to_per_chunk_calls",
                            "test_pipeline_matches_oracle_chain",
                            FE + "test_resample_matches_reference_golden",
                            RS + "test_resample_ratio_grid",                   # 42 ratios; complex64, complex128, float64
                            RS + "test_resample_cta_boundaries",               # n_out = 255 .. 513 at 13/119 and 3/2
                            RS + "test_resample_shared_memory_limit",          # 1/89 and 2/171 fit, 1/90 and 2/173 not
                            RS + "test_frontend_mix_modes"],                   # int8 / int16 / float32 IQ, every mode
    "rec_mix_kernel": ["test_frontend_chunks_bit_identical_to_per_chunk_calls",
                       FE + "test_frequency_shift_follows_numpy_promotion",
                       RS + "test_frequency_shift_and_frontend_past_2_24_samples",   # 2^25 + 12345 samples
                       RS + "test_direct_xambg_shapes"],                       # one mix per Doppler bin, F = 1 .. 32
}


def _is_gpu_test(test_id):
    path, _, name = test_id.rpartition("::")
    src = open(os.path.join(ROOT, path) if path else os.path.abspath(__file__)).read()
    i = src.index(f"\ndef {name}(")
    decorators = src[src.rindex("\n\n", 0, i):i]
    return "@pytest.mark.gpu" in decorators or re.search(r"^pytestmark = pytest\.mark\.gpu$", src, re.M) is not None


def test_every_recording_launch_has_a_covering_gpu_test():
    src = open(RECORDING).read()
    sites = {m.group(1) + (m.group(2) or "") for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", src)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    for tests in COVERAGE.values():
        for t in tests:
            assert _is_gpu_test(t), f"{t} is not a GPU test"


# ------------------------------------------------------------------ GPU
def _chunks_call(ptr, kind, n, nchunks, stride, mode, po, up, dn, h, out_ptr, out_stride, cap, mem, stream=None):
    po = np.ascontiguousarray(po, dtype=np.float64)
    return _lib.load().prc_frontend_chunks_c64(ptr, kind, n, nchunks, stride, mode, 100000.0, 2400000.0,
                                               po.ctypes.data, up, dn, h.ctypes.data, h.shape[0], out_ptr,
                                               out_stride, cap, mem, 0, stream, 0)


@pytest.mark.gpu
def test_frontend_chunks_bit_identical_to_per_chunk_calls():
    import torch
    from passiveradar_b200.signal_utils import _resample_taps
    n = 5003
    for dtype, kind in ((np.int8, _lib.IQ_I8), (np.int16, _lib.IQ_I16), (np.float32, _lib.IQ_C64)):
        for up, dn in ((13, 119), (3, 2), (1, 1)):
            for mode in (_lib.MIX_C64, _lib.MIX_C128):
                for nchunks in (1, 2, 33):
                    raw = synth.raw_iq(nchunks * n + 8, {np.int8: "int8", np.int16: "int16", np.float32: "float32"}[dtype],
                                       seed=nchunks + up)
                    po = 2 * np.pi * np.arange(nchunks) * 9 * (100000 / 2400000) + 0.1
                    h = _resample_taps(up, dn, mode == _lib.MIX_C64) if up != dn else np.ones(1)
                    n_out = -(-n * up // dn)
                    out = np.full((nchunks, n_out + 3), np.nan + 0j, dtype=np.complex64)
                    _lib.check(_chunks_call(raw.ctypes.data, kind, n, nchunks, n, mode, po, up, dn, h,
                                            out.ctypes.data, n_out + 3, out.size, _lib.MEM_HOST))
                    for b in range(nchunks):
                        p = float(po[b]) if mode == _lib.MIX_C64 else np.array([po[b]])
                        want = prb.frontend(raw[2 * b * n:2 * (b + 1) * n], 100000, 2400000, p, up, dn)
                        assert want.shape == (n_out,)
                        np.testing.assert_array_equal(out[b, :n_out].view(np.uint64), want.view(np.uint64),
                                                      err_msg=f"{dtype.__name__} {up}/{dn} mode {mode} chunk {b}")
                    assert np.isnan(out[:, n_out:]).all(), "a chunk's output spilled past its n_out samples"
    # device pointers at an odd raw element (main.py slices by the channel offset in raw elements)
    raw = synth.raw_iq(4 * n + 8, "int8", seed=3)
    off, nchunks = 7, 3
    raw_d = torch.from_numpy(raw).cuda()
    po = np.array([0.0, 0.3, 0.6])
    h = _resample_taps(13, 119, False)
    n_out = -(-n * 13 // 119)
    out_d = torch.empty(nchunks, n_out, dtype=torch.complex64, device="cuda")
    _lib.check(_chunks_call(raw_d.data_ptr() + off, _lib.IQ_I8, n, nchunks, n, _lib.MIX_C128, po, 13, 119, h,
                            out_d.data_ptr(), n_out, out_d.numel(), _lib.MEM_DEVICE))
    torch.cuda.synchronize()
    got = out_d.cpu().numpy()
    for b in range(nchunks):
        want = prb.frontend(raw[off + 2 * b * n:off + 2 * (b + 1) * n], 100000, 2400000, np.array([po[b]]), 13, 119)
        np.testing.assert_array_equal(got[b].view(np.uint64), want.view(np.uint64))
    # so do prc_iq_mix_c64 and prc_frontend_c64: a device pointer at an odd raw element gives the host call's bits
    lib = _lib.load()
    for dtype, kind in ((np.int8, _lib.IQ_I8), (np.int16, _lib.IQ_I16)):
        iq = synth.raw_iq(n + 8, dtype.__name__, seed=4)
        host, iq_d = np.ascontiguousarray(iq[off:off + 2 * n]), torch.from_numpy(iq).cuda()
        mix, fe = np.empty(n, np.complex64), np.empty(n_out, np.complex64)
        mix_d = torch.empty(n, dtype=torch.complex64, device="cuda")
        fe_d = torch.empty(n_out, dtype=torch.complex64, device="cuda")
        for src, m, f, mem in ((host.ctypes.data, mix.ctypes.data, fe.ctypes.data, _lib.MEM_HOST),
                               (iq_d.data_ptr() + off * iq.itemsize, mix_d.data_ptr(), fe_d.data_ptr(), _lib.MEM_DEVICE)):
            _lib.check(lib.prc_iq_mix_c64(src, kind, n, _lib.MIX_C128, 100000.0, 2400000.0, 0.3, m, mem, 0, None, 0))
            _lib.check(lib.prc_frontend_c64(src, kind, n, _lib.MIX_C128, 100000.0, 2400000.0, 0.3, 13, 119, h.ctypes.data,
                                            h.shape[0], f, n_out, mem, 0, None, 0))
        torch.cuda.synchronize()
        np.testing.assert_array_equal(mix_d.cpu().numpy().view(np.uint64), mix.view(np.uint64), err_msg=dtype.__name__)
        np.testing.assert_array_equal(fe_d.cpu().numpy().view(np.uint64), fe.view(np.uint64), err_msg=dtype.__name__)
    # the resampler's shared-memory refusal and message are prc_frontend_c64's
    h = _resample_taps(17, 1245, False)
    o = np.empty(64, np.complex64)
    st = _chunks_call(raw.ctypes.data, _lib.IQ_I8, 100, 1, 100, _lib.MIX_C128, [0.0], 17, 1245, h, o.ctypes.data, 2, 64,
                      _lib.MEM_HOST)
    msg = _lib.load().prc_last_error().decode()
    st1 = _lib.load().prc_frontend_c64(raw.ctypes.data, _lib.IQ_I8, 100, _lib.MIX_C128, 100000.0, 2400000.0, 0.0, 17,
                                       1245, h.ctypes.data, h.shape[0], o.ctypes.data, 64, _lib.MEM_HOST, 0, None, 0)
    assert st == st1 == _lib.PRC_E_INVALID
    assert msg == _lib.load().prc_last_error().decode()
    from passiveradar_b200.recording import resample_smem_refusal
    assert msg == resample_smem_refusal(17, 1245)


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


class _Spy(RecordingPipeline):
    """The pipeline with every chunk's stage outputs (resampled reference, resampled surveillance, cleaned
    surveillance) copied out right after its batch computed them."""

    def _stream(self, nchunks, dev, compute, emit):
        self.stages = {}

        def spy(c0, nb, ref_rows, srv_rows):
            compute(c0, nb, ref_rows, srv_rows)
            for i in range(nb):
                self.stages[c0 + i] = tuple(t.cpu().numpy().copy() for t in (ref_rows[i], self.srv_rs[i], srv_rows[i]))

        super()._stream(nchunks, dev, spy, emit)


@pytest.mark.gpu
@pytest.mark.parametrize("name,nchunks", [("fast", 8), ("shipped", 5)])
def test_pipeline_matches_oracle_chain(name, nchunks):
    """Each stage on identical inputs within 1e-5 of its oracle (the cleaned chunks: of their float64 truth, and of
    the complex64 oracle up to 1.2 x that oracle's own distance to the truth); every map within 1e-5 of the oracle chain, or (all
    these frames carry clutter) within 1e-5 + 1.2 x the oracle chain's own distance to the float64 stage truths."""
    from oracle import recording_oracle as ro
    config = synth.RECORDING_CONFIGS[name]
    _, ls_oracle, xambg_oracle, _ = ro._ops()
    R, F, cpi, d = config["num_range_cells"], config["num_doppler_cells"], config["cpi_samples"], config["window_overlap"]
    window = signal.get_window(('kaiser', 5.0), cpi)
    from oracle import clutter_oracle as co
    fig = {"clean_vs_oracle": 0.0, "clean_vs_truth": 0.0, "clean_oracle_vs_truth": 0.0, "map_vs_oracle_same_frames": 0.0, "map_vs_chain": 0.0, "chain_vs_truth": 0.0}
    for offset in (0, 7, -6):
        ref, srv, _, _ = synth.recording_for(config, nchunks, seed=31 + offset)
        pipe = _Spy.from_config(config, batch=3)
        got = pipe.run(ref, srv, offset=offset)
        assert got.shape == (F, R + 1, nchunks)
        want, st = ro.recording_oracle(config, ref, srv, offset, stages=True)
        assert want.shape == got.shape
        # the clutter filter on the pipeline's own resampled chunks: within 1e-5 of |srv| of the float64 truth, and of
        # the complex64 oracle once that oracle's own round-off against the truth is allowed for (test_path_sweep's rule)
        for k in range(nchunks):
            r_rs, s_rs, clean = pipe.stages[k]
            den = np.abs(s_rs).max()
            o = ls_oracle(r_rs, s_rs, R, config["IF_sample_rate"], ro.DOPPLER_BINS)
            t = co.ls_filter_multiple_truth(r_rs, s_rs, R, config["IF_sample_rate"], ro.DOPPLER_BINS)
            e, g, own_c = (float(np.abs(x - y).max() / den) for x, y in ((clean, o), (clean, t), (o, t)))
            fig["clean_vs_oracle"] = max(fig["clean_vs_oracle"], e)
            fig["clean_vs_truth"] = max(fig["clean_vs_truth"], g)
            fig["clean_oracle_vs_truth"] = max(fig["clean_oracle_vs_truth"], own_c)
            assert g <= 1e-5 and e <= 1e-5 + 1.2 * own_c, (offset, k, e, g, own_c)
        # the CAF on the pipeline's own overlapped frames
        ref_f = ro.overlap_frames([pipe.stages[k][0] for k in range(nchunks)], d)
        srv_f = ro.overlap_frames([pipe.stages[k][2] for k in range(nchunks)], d)
        for k in range(nchunks):
            e = _rel(got[:, :, k], xambg_oracle(ref_f[k], srv_f[k], R, F, cpi, window)[:, :, 0])
            fig["map_vs_oracle_same_frames"] = max(fig["map_vs_oracle_same_frames"], e)
            assert e <= 1e-5, (offset, k, e)
        # end to end, against the oracle chain and its own distance to the float64 stage truths
        errs = [_rel(got[:, :, k], want[:, :, k]) for k in range(nchunks)]
        truth = ro.stage_truths(config, st["ref_rs"], st["srv_rs"])
        own = [_rel(want[:, :, k], truth[:, :, k]) for k in range(nchunks)]
        fig["map_vs_chain"] = max(fig["map_vs_chain"], max(errs))
        fig["chain_vs_truth"] = max(fig["chain_vs_truth"], max(own))
        for k, e in enumerate(errs):
            assert e <= 1e-5 + 1.2 * own[k], (offset, k, e, own[k])
    print(f"[recording] {name}: {fig}")


@pytest.mark.gpu
def test_clutter_free_frames_match_oracle_chain():
    from oracle import recording_oracle as ro
    ref, srv, _, _ = synth.recording_for(FAST, 6, clutter=False, seed=4)
    got = RecordingPipeline.from_config(FAST, batch=4).run(ref, srv, offset=0)
    want = ro.recording_oracle(FAST, ref, srv, 0)
    errs = [_rel(got[:, :, k], want[:, :, k]) for k in range(6)]
    print(f"[recording] clutter-free frames vs oracle chain: {max(errs):.2e}")
    assert max(errs) <= 1e-5


@pytest.mark.gpu
def test_pipeline_batch_sizes_sources_and_device_entry():
    import torch
    from oracle import recording_oracle as ro
    nchunks = 6
    ref, srv, _, _ = synth.recording_for(FAST, nchunks, seed=5)
    pipes = {b: _Spy.from_config(FAST, batch=b) for b in (1, 3, nchunks)}
    maps = {b: p.run(ref, srv, offset=7) for b, p in pipes.items()}
    # every chunk runs the same kernels over the same partition whatever the batch: bit-identical maps
    for b in (1, 3):
        np.testing.assert_array_equal(maps[b], maps[nchunks])
    # the per-chunk composition of the existing drop-ins (main.py under install(), one thread, no dask)
    comp, chunks = ro.dropin_composition(FAST, ref, srv, 7)
    worst = 0.0
    for k, (a, b, c) in enumerate(chunks):
        r_rs, s_rs, clean = pipes[nchunks].stages[k]
        np.testing.assert_array_equal(r_rs, a.astype(np.complex64))      # the front end: bit-identical
        np.testing.assert_array_equal(s_rs, b.astype(np.complex64))
        e = float(np.abs(clean - c).max() / np.abs(s_rs).max())
        worst = max(worst, e)
        assert e <= 3e-6                                  # DESIGN.md section 6: batch-versus-single
    print(f"[recording] cleaned chunks vs single-chunk LS_Filter_Multiple: {worst:.2e}")
    np.testing.assert_array_equal(maps[nchunks], comp)
    # np.memmap sources
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        mr = np.memmap(os.path.join(d, "r"), dtype=np.int8, mode="w+", shape=ref.shape)
        ms = np.memmap(os.path.join(d, "s"), dtype=np.int8, mode="w+", shape=srv.shape)
        mr[:], ms[:] = ref, srv
        got = RecordingPipeline.from_config(FAST, batch=4).run(mr, ms, offset=7)
        del mr, ms
    np.testing.assert_array_equal(got, maps[nchunks])
    # device-resident raw data written asynchronously on the caller's own stream: run_device orders after it
    pipe = RecordingPipeline.from_config(FAST, batch=4)
    user = torch.cuda.Stream()
    pr, ps = torch.from_numpy(ref).pin_memory(), torch.from_numpy(srv).pin_memory()
    with torch.cuda.stream(user):
        rd, sd = pr.to("cuda", non_blocking=True), ps.to("cuda", non_blocking=True)
        md = pipe.run_device(rd, sd, offset=7)
        host = md.to("cpu", non_blocking=False)
    np.testing.assert_array_equal(host.numpy().transpose(1, 2, 0), maps[nchunks])
    assert pipe.metadata()["frame_timestamps"].shape == (nchunks,)
    with pytest.raises(ValueError, match="contiguous"):
        pipe.run_device(rd[::2], sd[::2], offset=7)
    with pytest.raises(ValueError, match="must be a tensor on"):
        pipe.run_device(torch.from_numpy(ref), torch.from_numpy(srv), offset=7)
    with pytest.raises(TypeError):
        pipe.run_device(rd.to(torch.int32), sd.to(torch.int32), offset=7)


@pytest.mark.gpu
@pytest.mark.parametrize("name,channel_delay", [("fast", 5), ("shipped", -5)])
def test_offset_estimate_and_target_position(name, channel_delay):
    """srv lagging ref by c complex samples comes back as offset -2c raw elements (main.py estimates it on the raw
    interleaved arrays); with it applied, the target peaks at column R - delay and Doppler row F/2 - fd T in every
    interior frame."""
    import torch
    config = synth.RECORDING_CONFIGS[name]
    nchunks = 4
    ref, srv, delay, kd = synth.recording_for(config, nchunks, channel_delay=channel_delay, seed=9)
    cpi = config["cpi_samples"]
    assert int(prb.find_channel_offset(ref[:10 * cpi], srv[:10 * cpi], 1, 5_000_000)) == -2 * channel_delay
    pipe = RecordingPipeline.from_config(config)
    maps = pipe.run_device(torch.from_numpy(ref).cuda(), torch.from_numpy(srv).cuda()).cpu().numpy()
    assert pipe.offset == -2 * channel_delay
    assert pipe.nframes == nchunks
    R, F = config["num_range_cells"], config["num_doppler_cells"]
    for k in range(1, nchunks - 1):
        m = np.abs(maps[k][:, :R - 4])                    # columns R-4 .. R hold the direct path's residue
        assert np.unravel_index(np.argmax(m), m.shape) == (F // 2 - kd, R - delay), k
