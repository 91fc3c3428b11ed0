"""GPU parity at the shapes round 1 left untested, on both shipped paths, plus the batched entry points and the
re-entrancy the boundary promises (include/prcore.h; dask calls the operators from a thread pool, main.py:169-194).

Per-stage figures go to $PRC_PARITY_DIR/parity.json when that variable is set (tests/conftest.py:record_parity).
"""
import concurrent.futures as cf
import ctypes as C

import numpy as np
import pytest
import scipy.signal as signal

import _golden as G
import passiveradar_b200 as prb
from conftest import record_parity
from passiveradar_b200 import _lib, synth

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _sampled_columns(ref, srv, got, R, F, n, w, lags):
    """max over the sampled range columns of |gpu - oracle| / max|gpu map| (columns are independent: lag d of srv is
    lag 0 of srv rolled by -d)."""
    from oracle import xambg_oracle as xo
    peak = float(np.abs(got).max())
    worst = 0.0
    for d in lags:
        want = xo.fast_xambg_oracle(ref, np.roll(srv, -d), 0, F, n, w)
        worst = max(worst, float(np.abs(got[:, R - d, 0] - want[:, 0, 0]).max()) / peak)
    return worst


# ------------------------------------------------------------------ CAF at the config-5 corners and awkward shapes
@pytest.mark.parametrize("n,F,R,win", [
    (2 ** 22, 64, 300, True),            # D = 65536
    (2 ** 22, 1024, 300, True),          # D = 4096
    (2 ** 20, 1024, 300, True),          # D = 1024
    (2 ** 20, 64, 300, False),           # D = 16384
    (10 ** 6, 256, 300, True),           # SURVEY 8: D = 3906, 64 tail samples ignored
    (524288, 1024, 175, True),           # the reference's shipped PRconfig.yaml shape: D = 512
    (2 ** 18, 1024, 100, True),          # D = 256: one short segment per Doppler block
])
def test_xambg_large_shapes_sampled_columns(n, F, R, win, both_paths):
    ref, srv = synth.make_frame(n, "P1", frame=21)
    w = signal.get_window(("kaiser", 5.0), n) if win else None
    got = prb.fast_xambg(ref, srv, R, F, n, w)
    lags = sorted(set([0, 1, R // 3, R // 2, R - 1, R]))
    e = _sampled_columns(ref, srv, got, R, F, n, w, lags)
    record_parity(f"xambg/n{n}_F{F}_R{R}/{both_paths}", E_vs_oracle_sampled_columns=e)
    assert e <= TOL, e


@pytest.mark.parametrize("n,F,R,fl", [
    (2 ** 18, 64, 1200, 0),            # many range bins: segments of L - R samples (L = 2048 or 4096 by cost)
    (2 ** 18, 32, 700, 700),           # fused frame with R + M - 1 = 1409: 639-sample segments at L = 2048
    (2 ** 17, 16, 1500, 1500),         # L = 4096 transforms (R + M - 1 = 3009)
])
def test_long_range_and_long_filter_take_the_larger_transforms(n, F, R, fl, both_paths):
    from oracle import xambg_oracle as xo
    ref, srv = synth.make_frame(n, "P0", frame=23)
    w = signal.get_window(("kaiser", 5.0), n)
    if fl == 0:
        got = prb.fast_xambg(ref, srv, R, F, n, w)
        want = xo.fast_xambg_oracle(ref, srv, R, F, n, w)
        e = G.rel_inf(got, want)
        assert e <= TOL, e
    else:
        from passiveradar_b200.frames import FramePipeline
        got = FramePipeline(n, R, F, filter_len=fl, batch=2, nslots=1).process(ref, srv)
        want = prb.fast_xambg(ref, prb.LS_Filter(ref, srv, fl), R, F, n, w)
        e = G.rel_inf(got, want)
        assert e <= 2e-6, e
    record_parity(f"long/n{n}_F{F}_R{R}_fl{fl}/{both_paths}", E=e)


def test_ls_config4_size_and_readme_shape(both_paths):
    from oracle import clutter_oracle as co
    for n, fl in ((2 ** 21, 400), (524288, 175), (10 ** 6, 300)):
        ref, srv = synth.make_frame(n, "P1", frame=5)
        t_out, t_taps = co.ls_filter_truth(ref, srv, fl, 1.0, 10)
        out, taps = prb.LS_Filter(ref, srv, fl, 1.0, 10, True)
        e_t, e_o = G.rel_inf(taps, t_taps), G.rel_inf(out, t_out, den=float(np.abs(srv).max()))
        record_parity(f"ls/n{n}_M{fl + 10}/{both_paths}", taps_vs_truth=e_t, out_vs_truth=e_o)
        assert e_t <= TOL and e_o <= TOL, (n, e_t, e_o)


def test_frame_fused_equals_separate_operators_at_awkward_sizes(both_paths):
    """prc_frames_c64 (clutter filter applied inside the CAF kernel on the FFT path) against LS_Filter -> fast_xambg.
    Independent channels (P0): nothing cancels, the two orders of rounding agree to 2e-6.  Strong clutter (P1): the map
    is what is left after ~55 dB of cancellation, and ANY float32 evaluation differs from another at the 1e-4 level
    relative to that residual map (the reference's own complex64 map is 5e-3 from the float64 truth there, SURVEY 0.5);
    so P1 frames are held to 5e-4 and their figures are recorded."""
    from passiveradar_b200.frames import FramePipeline
    for n, F, R, fl in ((200_000, 64, 100, 100), (10 ** 6, 256, 300, 300), (524288, 1024, 175, 175), (2 ** 18, 32, 40, 64)):
        profiles = ["P0", "P1", "P0"]
        frames = [synth.make_frame(n, profiles[i], frame=30 + i) for i in range(3)]
        pipe = FramePipeline(n, R, F, filter_len=fl, batch=2, nslots=2)
        maps = pipe.run_host(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]))
        w = signal.get_window(("kaiser", 5.0), n)
        worst = {"P0": 0.0, "P1": 0.0}
        for i, (ref, srv) in enumerate(frames):
            want = prb.fast_xambg(ref, prb.LS_Filter(ref, srv, fl), R, F, n, w)
            worst[profiles[i]] = max(worst[profiles[i]], G.rel_inf(maps[i], want))
        record_parity(f"frame_fused_vs_separate/n{n}_F{F}_R{R}/{both_paths}", E_P0=worst["P0"], E_P1_strong_clutter=worst["P1"])
        assert worst["P0"] <= 2e-6 and worst["P1"] <= 5e-4, (n, worst)


# ------------------------------------------------------------------ batched entry points
def test_frames_batch_equals_single_frames_and_reports_taps(both_paths):
    import torch
    n, F, R, fl, peek = 2 ** 17, 64, 50, 50, 10
    nf = 5
    frames = [synth.make_frame(n, "P0", frame=40 + i) for i in range(nf)]      # independent channels: strict comparison
    dev = torch.device("cuda", 0)
    ref_d = torch.from_numpy(np.stack([f[0] for f in frames])).to(dev)
    srv_d = torch.from_numpy(np.stack([f[1] for f in frames])).to(dev)
    maps = torch.empty((nf, F, R + 1), dtype=torch.complex64, device=dev)
    taps = torch.empty((nf, fl + peek), dtype=torch.complex64, device=dev)
    clean = torch.empty((nf, n), dtype=torch.complex64, device=dev)
    lib = _lib.load()
    st = torch.cuda.Stream(device=dev)
    _lib.check(lib.prc_frames_c64(ref_d.data_ptr(), srv_d.data_ptr(), n, nf, n, fl, peek, 1.0, R, F, None, maps.data_ptr(),
                                  taps.data_ptr(), clean.data_ptr(), _lib.MEM_DEVICE, 0, st.cuda_stream, 0))
    status = (C.c_int * nf)()
    _lib.check(lib.prc_ls_status(0, st.cuda_stream, status, nf))
    assert not any(status)
    for i, (ref, srv) in enumerate(frames):
        c, t = prb.LS_Filter(ref, srv, fl, 1.0, peek, True)
        m = prb.fast_xambg(ref, c, R, F)
        assert G.rel_inf(taps[i].cpu().numpy(), t) <= 1e-6
        assert G.rel_inf(clean[i].cpu().numpy(), c, den=float(np.abs(srv).max())) <= 1e-6
        assert G.rel_inf(maps[i].cpu().numpy()[:, :, None], m) <= 2e-6
    # host pointers, strided frames
    big_r = np.zeros((nf, n + 64), np.complex64)
    big_s = np.zeros((nf, n + 64), np.complex64)
    for i, (ref, srv) in enumerate(frames):
        big_r[i, :n], big_s[i, :n] = ref, srv
    out = np.empty((nf, F, R + 1), np.complex64)
    _lib.check(lib.prc_frames_c64(big_r.ctypes.data, big_s.ctypes.data, n, nf, n + 64, fl, peek, 1.0, R, F, None, out.ctypes.data,
                                  None, None, _lib.MEM_HOST, 0, None, 0))
    assert G.rel_inf(out, maps.cpu().numpy()) <= 1e-6


def test_frame_pipeline_raises_on_singular_frame(both_paths):
    """ADVICE r1: the asynchronous pipeline must not hand back NaN maps silently."""
    from passiveradar_b200.frames import FramePipeline
    n, F, R = 2 ** 15, 16, 8
    ref, srv = synth.make_frame(n, "P0", frame=1)
    refs = np.stack([ref, np.zeros(n, np.complex64), ref])
    srvs = np.stack([srv, srv, srv])
    pipe = FramePipeline(n, R, F, filter_len=8, reg=0.0, peek=0, window=None, batch=2, nslots=2)
    with pytest.raises(np.linalg.LinAlgError):
        pipe.run_host(refs, srvs)
    good = FramePipeline(n, R, F, filter_len=8, reg=0.0, peek=0, window=None, batch=2, nslots=2).run_host(refs[[0, 2]], srvs[[0, 2]])
    assert np.isfinite(good).all()


def test_nlms_frames_batch_equals_single_calls():
    """The batched NLMS entry point (one CTA per frame) gives exactly what frame-by-frame calls give; config-4 taps."""
    import torch
    n, fl, peek, mu = 2 ** 16, 400, 10, 0.05
    nf = 6
    frames = [synth.make_frame(n, "P1", frame=50 + i) for i in range(nf)]
    dev = torch.device("cuda", 0)
    ref_d = torch.from_numpy(np.stack([f[0] for f in frames])).to(dev)
    srv_d = torch.from_numpy(np.stack([f[1] for f in frames])).to(dev)
    out = torch.empty((nf, n), dtype=torch.complex64, device=dev)
    taps = torch.empty((nf, fl + peek), dtype=torch.complex64, device=dev)
    lib = _lib.load()
    st = torch.cuda.Stream(device=dev)
    for block in (1, 64):
        _lib.check(lib.prc_nlms_frames_c64(ref_d.data_ptr(), srv_d.data_ptr(), n, nf, n, fl, peek, mu, block, None, out.data_ptr(),
                                           taps.data_ptr(), _lib.MEM_DEVICE, 0, st.cuda_stream, 0))
        for i, (ref, srv) in enumerate(frames):
            o, t = prb.block_NLMS(ref, srv, fl, mu, peek, block, None, True) if block > 1 else prb.NLMS_filter(ref, srv, fl, mu, peek, None, True)
            assert np.array_equal(out[i].cpu().numpy(), o), (block, i)
            assert np.array_equal(taps[i].cpu().numpy(), t), (block, i)
    # the reference-pinned C oracle on one of them (pinned to the NLMS goldens by tests/test_oracle_golden.py)
    from oracle import clutter_oracle as co
    want, _ = co.block_nlms_oracle_c(frames[2][0], frames[2][1], fl, mu, peek, 1)
    _lib.check(lib.prc_nlms_frames_c64(ref_d.data_ptr(), srv_d.data_ptr(), n, nf, n, fl, peek, mu, 1, None, out.data_ptr(),
                                       None, _lib.MEM_DEVICE, 0, st.cuda_stream, 0))
    assert G.rel_inf(out[2].cpu().numpy(), want) <= TOL
    # xambg on a batch
    maps = torch.empty((nf, 32, 41), dtype=torch.complex64, device=dev)
    _lib.check(lib.prc_xambg_frames_c64(ref_d.data_ptr(), out.data_ptr(), n, nf, n, 40, 32, None, maps.data_ptr(), _lib.MEM_DEVICE, 0,
                                        st.cuda_stream, 0))
    for i in (0, nf - 1):
        assert G.rel_inf(maps[i].cpu().numpy()[:, :, None], prb.fast_xambg(frames[i][0], out[i].cpu().numpy(), 40, 32)) <= 2e-6


# ------------------------------------------------------------------ concurrent callers (SURVEY 8b)
def test_operators_are_reentrant_under_eight_threads(both_paths):
    """8 Python threads call LS_Filter / fast_xambg / the fused frame concurrently (ctypes drops the GIL, every thread
    owns a workspace and a stream): results must equal the serial ones bit for bit."""
    n, F, R, fl = 2 ** 17, 64, 60, 60
    w = signal.get_window(("kaiser", 5.0), n)
    frames = [synth.make_frame(n, "P1", frame=60 + i) for i in range(8)]

    def work(i):
        ref, srv = frames[i % 8]
        cleaned, taps = prb.LS_Filter(ref, srv, fl, 1.0, 10, True)
        return cleaned, taps, prb.fast_xambg(ref, cleaned, R, F, n, w)

    serial = [work(i) for i in range(8)]
    with cf.ThreadPoolExecutor(8) as ex:
        for rep in range(3):
            got = list(ex.map(work, range(16)))
            for i, (c, t, m) in enumerate(got):
                sc, st, sm = serial[i % 8]
                assert np.array_equal(c, sc) and np.array_equal(t, st) and np.array_equal(m, sm), (rep, i)


def test_short_lived_threads_do_not_strand_device_memory():
    """ADVICE r1: a thread's private workspace is released when the thread exits."""
    import threading
    import torch
    n = 2 ** 16
    ref, srv = synth.make_frame(n, "P0")

    def call():
        prb.fast_xambg(ref, srv, 20, 32)

    call()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(24):
        th = threading.Thread(target=call)
        th.start()
        th.join()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 < 64 * 2 ** 20, (free0, free1)       # 24 stranded workspaces would be > 100 MB


# ------------------------------------------------------------------ config-3 staging over NCCL (needs >= 2 GPUs)
def _nccl_stream_worker(rank, world, port, q):
    import os
    import torch
    import torch.distributed as dist
    from passiveradar_b200 import distributed as D
    from passiveradar_b200.frames import FramePipeline
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        n, F, R, nframes, chunk = 2 ** 16, 32, 40, 13, 3
        frames = [synth.make_frame(n, "P0", frame=70 + i) for i in range(nframes)]       # every rank can rebuild the stream
        pipe = FramePipeline(n, R, F, filter_len=40, device=rank, batch=chunk, nslots=2)
        ids = D.shard_indices(nframes, rank, world)
        maps = torch.zeros((len(ids), F, R + 1), dtype=torch.complex64, device=dev)
        ref_all = srv_all = None
        if rank == 0:
            ref_all = torch.from_numpy(np.stack([f[0] for f in frames])).to(dev)
            srv_all = torch.from_numpy(np.stack([f[1] for f in frames])).to(dev)

        def source(gids):
            idx = torch.as_tensor(gids, device=dev)
            return ref_all.index_select(0, idx), srv_all.index_select(0, idx)

        def process(rr, ss, first):
            pipe.run_device(rr, ss, maps[first:first + rr.shape[0]])

        cnt = D.stream_frames(source, process, nframes, chunk, n, rank, world, dev, src=0)
        torch.cuda.synchronize(dev)
        worst = 0.0
        for k, f in enumerate(ids):
            ref, srv = frames[f]
            want = prb.fast_xambg(ref, prb.LS_Filter(ref, srv, 40, device=rank), R, F, n, signal.get_window(("kaiser", 5.0), n), device=rank)
            worst = max(worst, G.rel_inf(maps[k].cpu().numpy()[:, :, None], want))
        q.put((rank, cnt == len(ids), worst))
    finally:
        dist.destroy_process_group()


def test_stream_frames_over_nccl_world2():
    import socket
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_stream_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, ok, worst in res:
        assert ok and worst <= 2e-6, (rank, ok, worst)


def test_nlms_large_batch_uses_the_half_size_ctas_and_matches():
    """More frames than SMs: prc_nlms_frames_c64 switches to 512-thread CTAs (three per SM).  Same recurrence, another
    summation order of the partial dot products: compare with the single-frame kernel and with the reference-pinned C oracle."""
    import torch
    from oracle import clutter_oracle as co
    props = torch.cuda.get_device_properties(0)
    nf = props.multi_processor_count + 12
    n, fl, peek, mu = 2 ** 13, 400, 10, 0.05
    base = [synth.make_frame(n, "P1", frame=80 + i) for i in range(4)]
    dev = torch.device("cuda", 0)
    ref_d = torch.from_numpy(np.stack([base[i % 4][0] for i in range(nf)])).to(dev)
    srv_d = torch.from_numpy(np.stack([base[i % 4][1] for i in range(nf)])).to(dev)
    out = torch.empty((nf, n), dtype=torch.complex64, device=dev)
    taps = torch.empty((nf, fl + peek), dtype=torch.complex64, device=dev)
    lib = _lib.load()
    st = torch.cuda.Stream(device=dev)
    _lib.check(lib.prc_nlms_frames_c64(ref_d.data_ptr(), srv_d.data_ptr(), n, nf, n, fl, peek, mu, 1, None, out.data_ptr(),
                                       taps.data_ptr(), _lib.MEM_DEVICE, 0, st.cuda_stream, 0))
    got = out.cpu().numpy()
    gt = taps.cpu().numpy()
    for i in (0, 1, 2, 3, nf - 1):
        ref, srv = base[i % 4]
        want, ww = co.block_nlms_oracle_c(ref, srv, fl, mu, peek, 1)
        single, st1 = prb.NLMS_filter(ref, srv, fl, mu, peek, None, True)
        den = float(np.abs(want).max())
        assert G.rel_inf(got[i], want, den=den) <= TOL
        assert G.rel_inf(got[i], single, den=den) <= 2e-6
        assert G.rel_inf(gt[i], st1) <= 5e-5
    assert np.array_equal(got[0], got[4])          # same frame on another CTA: deterministic


def test_ls_multiple_frames_batch_matches_single_calls_and_reference_golden():
    """prc_ls_multiple_frames_c64 (what main.py:169-176 does per chunk, several chunks per call) against the drop-in
    LS_Filter_Multiple frame by frame, and -- through it -- against the reference's own output (golden multi_main)."""
    import torch
    g = G.load("multi_main")
    ref0, srv0 = G.inputs(g)
    n, fl, fs, bins = ref0.shape[0], int(g["filter_len"]), float(g["sample_rate"]), [float(b) for b in g["bins"]]
    others = [synth.make_frame(n, "P1", frame=90 + i) for i in range(2)]
    frames = [(ref0, srv0)] + others
    nf = len(frames)
    dev = torch.device("cuda", 0)
    stride = n + 32
    ref_d = torch.zeros((nf, stride), dtype=torch.complex64, device=dev)
    srv_d = torch.zeros((nf, stride), dtype=torch.complex64, device=dev)
    for i, (r, s) in enumerate(frames):
        ref_d[i, :n] = torch.from_numpy(r).to(dev)
        srv_d[i, :n] = torch.from_numpy(s).to(dev)
    out = torch.zeros((nf, stride), dtype=torch.complex64, device=dev)
    lib = _lib.load()
    st = torch.cuda.Stream(device=dev)
    b64 = np.ascontiguousarray(bins, dtype=np.float64)
    old = _lib.get_option("fft_min_n")
    _lib.set_option("fft_min_n", 0)
    try:
        _lib.check(lib.prc_ls_multiple_frames_c64(ref_d.data_ptr(), srv_d.data_ptr(), n, nf, stride, fl, 10, fs, b64.ctypes.data, len(bins),
                                                  out.data_ptr(), _lib.MEM_DEVICE, 0, st.cuda_stream, 0))
        got = out.cpu().numpy()[:, :n]
        for i, (r, s) in enumerate(frames):
            want = prb.LS_Filter_Multiple(r, s, fl, fs, bins)
            assert G.rel_inf(got[i], want, den=float(np.abs(s).max())) <= 2e-6, i
    finally:
        _lib.set_option("fft_min_n", old)
    assert G.rel_inf(got[0][g["out_idx"]], g["out_sub"], den=float(g["srv_absmax"])) <= TOL


def test_random_shapes_fft_path_matches_direct_path_and_oracle():
    """Randomised geometry check of the FFT-domain kernels (segment partition, circular wrap, N not a multiple of F, odd
    decimation, short last segments): 16 seeded random shapes, FFT path against the direct-form path for every stage,
    and against the CPU oracle for the CAF."""
    from oracle import xambg_oracle as xo
    rng = np.random.default_rng(20260924)
    old = (_lib.get_option("fft"), _lib.get_option("fft_min_n"))
    try:
        for case in range(16):
            n = int(rng.integers(4200, 90000))
            F = int(rng.integers(2, max(3, min(200, n // 40))))
            R = int(rng.integers(0, 260))
            fl = int(rng.integers(1, 200))
            peek = int(rng.integers(0, 12))
            reg = float(rng.choice([0.5, 1.0, 3.0]))
            use_win = bool(rng.integers(0, 2))
            ref, srv = synth.make_frame(n, "P0" if case % 2 else "P1", frame=100 + case)
            w = signal.get_window(("kaiser", 5.0), n) if use_win else None
            res = {}
            for mode in (1, 0):
                _lib.set_option("fft", mode)
                _lib.set_option("fft_min_n", 0)
                cleaned, taps = prb.LS_Filter(ref, srv, fl, reg, peek, True)
                amb = prb.fast_xambg(ref, srv, R, F, n, w)
                res[mode] = (cleaned, taps, amb)
            tag = (case, n, F, R, fl, peek)
            assert G.rel_inf(res[1][1], res[0][1]) <= 3e-6, ("taps",) + tag
            assert G.rel_inf(res[1][0], res[0][0], den=float(np.abs(srv).max())) <= 3e-6, ("cleaned",) + tag
            assert G.rel_inf(res[1][2], res[0][2]) <= 3e-6, ("map",) + tag
            if case % 4 == 0:
                assert G.rel_inf(res[1][2], xo.fast_xambg_oracle(ref, srv, R, F, n, w)) <= TOL, ("oracle",) + tag
    finally:
        _lib.set_option("fft", old[0])
        _lib.set_option("fft_min_n", old[1])
