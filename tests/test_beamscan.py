"""Beamscan of several surveillance channels (prc_beamscan_frames, csrc/beamscan.cuh, passiveradar_b200.beamforming).

CPU: the float64 oracle against a per-cell loop and hand-made power sequences, the steering conventions, the oracle's
bearing on noise-free single echoes and its interpolation bias, the ABI, the refusals, the Python checks, the launch
coverage and the ptxas log.  GPU: the kernel against the oracle for K = 1 .. 4 over grids and map shapes, the K = 1
pass-through, batching, strides, aliased channels and zero cells, and the chain FramePipeline(channels=K) ->
beamscan_frames -> bearing / os_cfar_frames / RenderPipeline on synthetic CPIs.
"""
import os
import re

import numpy as np
import pytest

import passiveradar_b200 as prb
from oracle import beam_oracle as bo
from passiveradar_b200 import _lib, synth
from passiveradar_b200.beamforming import (beamscan_frames, bearing, steering_vectors, uca_positions,
                                           ula_positions)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BEAMSCAN = os.path.join(ROOT, "passiveradar_b200", "csrc", "beamscan.cuh")
PARAMS = ("maps rows cols nframes frame_stride nchan chan_stride steering nangles wrap amp_out pos_out out_stride "
          "device stream flags")
SECTOR = np.arange(0.0, 181.0)            # 1-degree sector grid, 181 angles
CIRCLE = np.arange(0.0, 360.0)            # 1-degree full circle, 360 angles


def _cplx(rng, shape):
    return ((rng.standard_normal(shape) + 1j * rng.standard_normal(shape)) / np.sqrt(2)).astype(np.complex64)


# ------------------------------------------------------------------ CPU: oracle
def test_oracle_equals_a_per_cell_loop():
    rng = np.random.default_rng(3)
    for K, A, wrap in ((1, 1, False), (2, 2, True), (3, 7, False), (4, 9, True), (4, 5, False), (2, 1, True)):
        maps = _cplx(rng, (K, 6, 5))
        S = _cplx(rng, (A, K))
        amp, pos, a, _, _ = bo.beamscan_oracle(maps, S, wrap)
        for i in range(6):
            for j in range(5):
                m = maps[:, i, j].astype(np.complex128)
                p = [abs(sum(complex(S[q, k]) * m[k] for k in range(K))) ** 2 for q in range(A)]
                ai, d = bo.delta_of_sequence(p, wrap)
                want = ai + d
                if wrap and want >= A - 0.5:
                    want -= A
                assert a[i, j] == ai and abs(pos[i, j] - want) < 1e-12, (K, A, wrap, i, j)
                assert abs(amp[i, j] - np.sqrt(p[ai])) <= 1e-12 * max(1.0, np.sqrt(p[ai]))


@pytest.mark.parametrize("p,wrap,a,delta", [
    ([5, 3, 1], False, 0, 0.0),                   # maximum at the first end: no neighbour past it
    ([1, 3, 5], False, 2, 0.0),                   # ... at the last end
    ([5, 3, 1], True, 0, 0.5 * (1 - 3) / (1 - 10 + 3)),      # wrap: P[-1] = P[2]
    ([1, 3, 5], True, 2, 0.5 * (3 - 1) / (3 - 10 + 1)),      # wrap: P[3] = P[0]
    ([7], False, 0, 0.0), ([7], True, 0, 0.0),    # A = 1: den = 0 even with wrap
    ([2, 7], False, 1, 0.0), ([2, 7], True, 1, 0.0), ([7, 2], True, 0, 0.0),   # A = 2: P[a-1] = P[a+1]
    ([4, 4, 4, 4], False, 0, 0.0), ([4, 4, 4, 4], True, 0, 0.0),          # flat: the first maximum, den = 0
    ([1, 6, 6, 1], False, 1, 0.5), ([1, 6, 6, 2], True, 1, 0.5),          # tie with the right neighbour: +0.5
    ([6, 1, 2, 6], True, 0, -0.5),                                         # tie with the (wrapped) left one: -0.5
    ([1, 4, 9, 4, 1], False, 2, 0.0), ([1, 4, 9, 5, 1], False, 2, 0.5 * (4 - 5) / (4 - 18 + 5)),
])
def test_delta_rule_on_hand_made_sequences(p, wrap, a, delta):
    got_a, got_d = bo.delta_of_sequence(p, wrap)
    assert (got_a, got_d) == (a, pytest.approx(delta, abs=1e-15))
    amp, pos, aa, _ = bo.peak_from_powers(np.asarray(p, float)[:, None], wrap)
    want = a + delta
    if wrap and want >= len(p) - 0.5:
        want -= len(p)
    assert aa[0] == a and pos[0] == pytest.approx(want, abs=1e-15) and amp[0] == np.sqrt(max(p))


def test_delta_is_bounded_on_random_sequences():
    rng = np.random.default_rng(9)
    for wrap in (False, True):
        P = rng.exponential(1.0, (40, 5000))
        P[:, :100] = np.round(P[:, :100])                       # ties
        _, pos, a, _ = bo.peak_from_powers(P, wrap)
        d = pos - a
        if wrap:
            d = np.where(d < -1, d + 40, d)                     # a pos folded from A - 0.5 to -0.5
            assert np.all((pos >= -0.5) & (pos < 40 - 0.5))
        else:
            assert np.all((pos >= 0) & (pos <= 39))
        assert np.abs(d).max() <= 0.5


def test_steering_conventions():
    S = steering_vectors(ula_positions(4, 0.5), [90.0, 0.0, 30.0])
    assert S.shape == (3, 4) and S.dtype == np.complex64
    np.testing.assert_allclose(np.abs(S), 1.0, rtol=1e-6)
    np.testing.assert_allclose(S[0], 1.0, atol=1e-6)              # broadside of a line array along x
    np.testing.assert_allclose(S[1], [1, -1, 1, -1], atol=1e-6)   # endfire, half-wave spacing: phase pi per element
    np.testing.assert_allclose(S[2], np.exp(1j * np.pi * np.arange(4) * np.cos(np.pi / 6)), atol=1e-6)
    for K in (3, 4, 5):
        pos = uca_positions(K, 0.4)
        np.testing.assert_allclose(np.hypot(pos[:, 0], pos[:, 1]), 0.4)
        base = 17.0
        rows = steering_vectors(pos, base + 360.0 / K * np.arange(K))
        for s in range(K):                  # a_k(theta + s * 360 / K) = a_{k - s}(theta)
            np.testing.assert_allclose(rows[s], np.roll(rows[0], s), atol=2e-6)
    np.testing.assert_array_equal(steering_vectors([0.0, 0.5], [90.0]), steering_vectors(ula_positions(2), [90.0]))


@pytest.mark.parametrize("kind,K", [("ula", 2), ("ula", 3), ("ula", 4), ("uca", 3), ("uca", 4)])
def test_oracle_bearing_of_a_single_echo(kind, K):
    """Noise-free single echoes m = conj(a(theta)) * c on a 1-degree grid.  On the grid the oracle's bearing is within
    0.05 grid steps; between grid points the three-point parabola's bias, computed over a 0.01-degree sweep, stays
    under the bound the model gives:
      * ULA (half-wave), 20 .. 160 degrees: 0.0241 degrees for K = 2, 3, 4 (the bias is set by the cos(theta)
        compression of the beam away from broadside: 0.050 degrees at 10, 0.10 at 5 degrees from endfire, which is why
        the sweep stops short of it);
      * UCA of radius 0.3 wavelengths, full circle: 1.1e-4 degrees for K = 3, 4 (a two-element "circle" is a line
        with a mirror ambiguity, so K = 2 is checked as a ULA only)."""
    if kind == "ula":
        positions, grid, wrap, lo, hi, bound = ula_positions(K, 0.5), SECTOR, False, 20.0, 160.0, 0.0241
        on_lo, on_hi = 10.0, 170.0
    else:
        positions, grid, wrap, lo, hi, bound = uca_positions(K, 0.3), CIRCLE, True, 0.0, 360.0, 1.1e-4
        on_lo, on_hi = 0.0, 360.0
    S = steering_vectors(positions, grid)
    th = np.arange(lo, hi, 0.01)
    m = np.conj(steering_vectors(positions, th).astype(np.complex128)).T * (0.3 - 0.7j)
    _, pos, _, _, _ = bo.beamscan_oracle(m, S, wrap)
    err = (bearing(pos, grid, wrap=wrap) - th + 180.0) % 360.0 - 180.0
    print(f"[beamscan] {kind} K={K}: worst interpolation bias {np.abs(err).max():.2e} degrees")
    assert np.abs(err).max() <= bound
    on = np.arange(on_lo, on_hi, 1.0)
    m = np.conj(steering_vectors(positions, on).astype(np.complex128)).T
    _, pos, _, _, _ = bo.beamscan_oracle(m, S, wrap)
    err = (bearing(pos, grid, wrap=wrap) - on + 180.0) % 360.0 - 180.0
    assert np.abs(err).max() <= 0.05


def test_bearing_maps_indices_to_degrees():
    g = np.array([10.0, 20.0, 40.0])
    np.testing.assert_allclose(bearing(np.array([0.0, 0.5, 1.0, 1.25, 2.0]), g), [10, 15, 20, 25, 40])
    np.testing.assert_allclose(bearing(np.array([0.0, -0.5, 359.5, 90.25]), CIRCLE, wrap=True), [0, 359.5, 359.5, 90.25])
    np.testing.assert_allclose(bearing(np.array([0.0, 1.5]), [5.0, 95.0, 185.0, 275.0], wrap=True), [5.0, 140.0])
    assert bearing(np.array([0.0]), [42.0])[0] == 42.0
    with pytest.raises(ValueError, match="uniform with a step of 360 / A"):
        bearing(np.zeros(2), SECTOR, wrap=True)


# ------------------------------------------------------------------ CPU: ABI, refusals, build
def test_abi_entry_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "prcore.h")).read()
    m = re.search(r"\bint prc_beamscan_frames\(([^)]*)\);", header)
    assert m, "prc_beamscan_frames is not declared"
    params = [p.strip().split()[-1].lstrip("*") for p in m.group(1).split(",")]
    assert " ".join(params) == PARAMS
    assert "mem_kind" not in params
    assert len(_lib.SIGNATURES["prc_beamscan_frames"][1]) == len(params)
    assert hasattr(_lib.load(), "prc_beamscan_frames")
    names = {"steering_vectors", "ula_positions", "uca_positions", "beamscan_frames", "bearing"}
    assert names <= set(prb.__all__) and all(hasattr(prb, n) for n in names)
    src = open(os.path.join(ROOT, "passiveradar_b200", "csrc", "prcore.cu")).read()
    slots = re.search(r"kKernelNames\[K_COUNT\] = \{([^}]*)\}", src).group(1)
    assert re.findall(r'"(\w+)"', slots)[-2:] == ["frame_multi", "beamscan"]


_BUF = np.zeros(64, np.complex64)


def _call(**kw):
    args = dict(maps=_BUF.ctypes.data, rows=2, cols=3, nframes=2, frame_stride=6, nchan=2, chan_stride=12,
                steering=_BUF.ctypes.data, nangles=5, wrap=0, amp_out=_BUF.ctypes.data, pos_out=_BUF.ctypes.data,
                out_stride=6, device=0, stream=None, flags=0)
    args.update(kw)
    return _lib.load().prc_beamscan_frames(*[args[p] for p in PARAMS.split()])


REFUSALS = [
    (dict(rows=0), "rows=0 cols=3 invalid"), (dict(cols=-1), "rows=2 cols=-1 invalid"),
    (dict(nframes=-1), "nframes=-1 outside [0, 65535]"), (dict(nframes=65536), "nframes=65536 outside [0, 65535]"),
    (dict(nchan=0), "nchan=0 outside [1, 4]"), (dict(nchan=5), "nchan=5 outside [1, 4]"),
    (dict(nangles=0), "nangles=0 outside [1, 4096]"), (dict(nangles=4097), "nangles=4097 outside [1, 4096]"),
    (dict(wrap=2), "wrap=2 must be 0 or 1"), (dict(wrap=-1), "wrap=-1 must be 0 or 1"),
    (dict(chan_stride=-1), "chan_stride=-1 must be >= 0"),
    (dict(frame_stride=5), "frame_stride=5 / out_stride=6 smaller than the 6 cells"),
    (dict(out_stride=5), "frame_stride=6 / out_stride=5 smaller than the 6 cells"),
    (dict(maps=None), "maps and steering must not be NULL"), (dict(steering=None), "maps and steering must not be NULL"),
    (dict(amp_out=None, pos_out=None), "amp_out and pos_out must not both be NULL"),
    (dict(rows=1 << 30, cols=1 << 30), "exceeds the beamscan's maximum"),
]


def test_refusals_before_any_launch():
    lib = _lib.load()
    before = _lib.launch_count()
    for kw, msg in REFUSALS:
        assert _call(**kw) == _lib.PRC_E_INVALID, kw
        assert msg in lib.prc_last_error().decode(), (kw, msg, lib.prc_last_error())
    assert _lib.launch_count() == before


def test_well_formed_calls_pass_the_checks():
    """Strides below a map are fine for one frame, one output may be NULL, chan_stride may be 0; without a device such
    calls then fail with PRC_E_CUDA (with one they would read the dummy operands, so this is a CPU-only check)."""
    try:
        import torch
        if torch.cuda.is_available():
            pytest.skip("with a device the call would read the dummy operands")
    except ImportError:
        pass
    for kw in (dict(), dict(nframes=1, frame_stride=0, out_stride=0), dict(amp_out=None), dict(pos_out=None),
               dict(chan_stride=0), dict(nchan=1, nangles=1, wrap=1), dict(nchan=4, nangles=4096)):
        assert _call(**kw) == _lib.PRC_E_CUDA, kw


def test_python_argument_checks():
    before = _lib.launch_count()
    maps = np.zeros((3, 2, 4, 5), np.complex64)
    S = steering_vectors(ula_positions(3), SECTOR)
    with pytest.raises(TypeError, match="complex64"):
        beamscan_frames(maps.astype(np.complex128), S)
    with pytest.raises(ValueError, match="four-dimensional"):
        beamscan_frames(maps[0], S)
    with pytest.raises(ValueError, match="K=5 channels"):
        beamscan_frames(np.zeros((5, 2, 4, 5), np.complex64), np.ones((3, 5)))
    with pytest.raises(ValueError, match=r"steering must have shape \(A, 3\)"):
        beamscan_frames(maps, S[:, :2])
    with pytest.raises(ValueError, match="A=4097 angles"):
        beamscan_frames(maps, np.ones((4097, 3)))
    with pytest.raises(ValueError, match="A=0 angles"):
        beamscan_frames(maps, np.ones((0, 3)))
    with pytest.raises(ValueError, match="wrap must be a bool"):
        beamscan_frames(maps, S, wrap="yes")
    with pytest.raises(ValueError, match="positions must be"):
        steering_vectors(np.zeros((3, 3)), SECTOR)
    assert _lib.launch_count() == before


# every launch in beamscan.cuh -> the GPU tests of this file that reach it
COVERAGE = {f"beamscan_kernel<{K}>": ["test_kernel_matches_oracle", "test_batches_strides_aliases_and_zero_cells"]
            for K in (1, 2, 3, 4)}
COVERAGE["beamscan_kernel<1>"].append("test_one_channel_passes_through")
COVERAGE["beamscan_kernel<3>"].append("test_chain_from_frames_to_bearing_and_cfar")
COVERAGE["beamscan_kernel<4>"].append("test_chain_from_frames_to_bearing_and_cfar")


def _is_gpu_test(name):
    src = open(os.path.abspath(__file__)).read()
    i = src.index(f"\ndef {name}(")
    return "@pytest.mark.gpu" in src[src.rindex("\n\n", 0, i):i]


def test_every_beamscan_launch_has_a_covering_gpu_test():
    code = "\n".join(line.split("//", 1)[0] for line in open(BEAMSCAN).read().splitlines())
    sites = {m.group(1) + (m.group(2) or "") for m in re.finditer(r"([A-Za-z_]\w*)\s*(<[^<>;()]*>)?\s*<<<", code)}
    assert sites == set(COVERAGE), f"launch sites {sites} vs COVERAGE {set(COVERAGE)}"
    for tests in COVERAGE.values():
        for t in tests:
            assert _is_gpu_test(t), f"{t} is not a GPU test"


def test_kernel_builds_for_sm90a_without_spills():
    from passiveradar_b200 import build as b
    b.build(force=False)
    log = os.path.join(b.PKG, "libprcore.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    found = {}
    for blk in open(log).read().split("Compiling entry function")[1:]:
        head = blk.split("\n")[0]
        m = re.search(r"_ZN3prc4beam15beamscan_kernelILi(\d)EEEvNS0_10BeamParamsE", head)
        if m:
            assert "'sm_90a'" in head
            assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in blk, head
            regs = int(re.search(r"Used (\d+) registers", blk).group(1))
            assert regs <= 128, f"K={m.group(1)}: {regs} registers, fewer than two 256-thread CTAs per SM"
            found[int(m.group(1))] = regs
    assert sorted(found) == [1, 2, 3, 4], found


# ------------------------------------------------------------------ GPU
def _grid_table(K, A, rng):
    """(steering, wrap) of a test case: a ULA sector grid, a UCA circle at A = 360, random complex rows at A <= 3."""
    if A == 360:
        return steering_vectors(uca_positions(K, 0.3), CIRCLE), True
    if A <= 3:
        return _cplx(rng, (A, K)) * 1.5, A == 2
    return steering_vectors(ula_positions(K, 0.5), np.linspace(0.0, 180.0, A)), False


def _check_against_oracle(maps, S, wrap, amp, pos, what):
    """The tolerances of DESIGN.md section 21, cell by cell; returns (cells checked on pos, cells checked by beam)."""
    K, A = S.shape[1], S.shape[0]
    m = maps.reshape(K, -1)
    a_, p_ = amp.reshape(-1).astype(np.float64), pos.reshape(-1).astype(np.float64)
    absS = np.abs(S.astype(np.complex128))
    strong_n = weak_n = 0
    for c0 in range(0, m.shape[1], 8192):
        mc = m[:, c0:c0 + 8192]
        P = bo.beam_powers(mc, S)
        _, pos64, a64, den64 = bo.peak_from_powers(P, wrap)
        best = P[a64, np.arange(P.shape[1])]
        B2 = (absS @ np.abs(mc.astype(np.complex128))).max(axis=0) ** 2
        ac, pc = a_[c0:c0 + 8192], p_[c0:c0 + 8192]
        bad = np.abs(ac ** 2 - best) > 2e-6 * B2
        assert not bad.any(), (what, "amp", np.nonzero(bad)[0][:5] + c0)
        cols = np.arange(P.shape[1])
        kb = np.rint(pc).astype(np.int64)                       # the kernel's beam
        kb = kb % A if wrap else np.clip(kb, 0, A - 1)
        p_kb = P[kb, cols]
        for d in (-1, 0, 1):                                    # P of the non-adjacent beams only
            idx = a64 + d
            ok = (idx >= 0) & (idx < A) if not wrap else np.ones_like(idx, bool)
            P[idx[ok] % A, cols[ok]] = -np.inf
        strong = (best - P.max(axis=0) > 4e-6 * B2) & (np.abs(den64) >= 1e-3 * best)
        d = pc - pos64
        if wrap:
            d = (d + A / 2) % A - A / 2
        bad = strong & (np.abs(d) > 1e-3)
        assert not bad.any(), (what, "pos", np.nonzero(bad)[0][:5] + c0, pc[bad][:5], pos64[bad][:5])
        bad = ~strong & (best - p_kb > 4e-6 * B2)
        assert not bad.any(), (what, "beam", np.nonzero(bad)[0][:5] + c0)
        strong_n += int(strong.sum())
        weak_n += int((~strong).sum())
    return strong_n, weak_n


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_kernel_matches_oracle(K):
    rng = np.random.default_rng(100 + K)
    summary = []
    for A in (1, 2, 3, 181, 360, 4096):
        S, wrap = _grid_table(K, A, rng)
        for rows, cols in ((1, 1), (5, 3), (256, 301), (1024, 176)):
            T = 2 if A <= 360 else 1
            maps = _cplx(rng, (K, T, rows, cols))
            amp, pos = beamscan_frames(maps, S, wrap=wrap)
            assert amp.shape == pos.shape == (T, rows, cols) and amp.dtype == pos.dtype == np.float32
            if wrap:
                assert np.all((pos >= -0.5) & (pos < A - 0.5))
            else:
                assert np.all((pos >= 0) & (pos <= A - 1))
            s, w = _check_against_oracle(maps, S, wrap, amp, pos, f"K={K} A={A} {rows}x{cols}")
            summary.append(f"A={A} {rows}x{cols}: {s}/{s + w} on pos")
    print(f"[beamscan] K={K}: " + "; ".join(summary))


@pytest.mark.gpu
def test_one_channel_passes_through():
    """K = 1, S = [[1]]: amp = sqrtf(fmaf(re, re, im * im)), within 1 ulp of the correctly rounded |m| (float64 hypot
    rounded to float32; NumPy's complex64 abs is not correctly rounded, up to 2 ulp from that value), and pos = 0."""
    rng = np.random.default_rng(5)
    maps = _cplx(rng, (1, 3, 256, 301)) * np.float32(1e3)
    maps[0, 0, :4, :4] = 0
    amp, pos = beamscan_frames(maps, np.ones((1, 1), np.complex64))
    exact = np.hypot(maps.real.astype(np.float64), maps.imag.astype(np.float64))[0].astype(np.float32)
    ulps = np.abs(amp.astype(np.float64) - exact) / np.spacing(np.maximum(exact, np.float32(1e-30)))
    print(f"[beamscan] K=1: worst {ulps.max():.0f} ulp from the correctly rounded |m|")
    assert ulps.max() <= 1
    assert not pos.any() and not amp[0, :4, :4].any()


@pytest.mark.gpu
def test_batches_strides_aliases_and_zero_cells():
    import torch
    lib = _lib.load()
    rng = np.random.default_rng(12)
    for K, A, wrap, rows, cols in ((1, 7, False, 5, 3), (2, 181, False, 37, 29), (3, 360, True, 64, 101),
                                   (4, 4096, False, 16, 40), (4, 360, True, 256, 301)):
        S = steering_vectors(uca_positions(K, 0.3), CIRCLE) if A == 360 else _grid_table(K, A, rng)[0]
        T, cells, pad, opad = 5, rows * cols, 9, 4
        x = _cplx(rng, (K, T, cells + pad))
        x[:, 1, :cells // 3] = 0                                  # zero cells
        xd = torch.from_numpy(x).cuda()
        amp = torch.full((T, cells + opad), float("nan"), device="cuda")
        pos = torch.full((T, cells + opad), float("nan"), device="cuda")
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            _lib.check(lib.prc_beamscan_frames(xd.data_ptr(), rows, cols, T, cells + pad, K, T * (cells + pad),
                                               S.ctypes.data, A, int(wrap), amp.data_ptr(), pos.data_ptr(),
                                               cells + opad, 0, s.cuda_stream, _lib.FLAG_ASYNC))
        s.synchronize()
        ga, gp = amp.cpu().numpy(), pos.cpu().numpy()
        assert np.isnan(ga[:, cells:]).all() and np.isnan(gp[:, cells:]).all()      # the gaps are untouched
        assert not ga[1, :cells // 3].any() and not gp[1, :cells // 3].any()
        # every frame alone, through the Python layer: the same bits
        for b in range(T):
            one = np.ascontiguousarray(x[:, b:b + 1, :cells]).reshape(K, 1, rows, cols)
            a1, p1 = beamscan_frames(one, S, wrap=wrap)
            np.testing.assert_array_equal(a1.reshape(-1).view(np.uint32), ga[b, :cells].view(np.uint32))
            np.testing.assert_array_equal(p1.reshape(-1).view(np.uint32), gp[b, :cells].view(np.uint32))
        # one output only
        amp2 = torch.zeros((T, cells), device="cuda")
        _lib.check(lib.prc_beamscan_frames(xd.data_ptr(), rows, cols, T, cells + pad, K, T * (cells + pad),
                                           S.ctypes.data, A, int(wrap), amp2.data_ptr(), None, cells, 0, None, 0))
        np.testing.assert_array_equal(amp2.cpu().numpy(), ga[:, :cells])
        # chan_stride = 0 (an expanded view) equals K explicit copies of channel 0
        c0 = torch.from_numpy(np.ascontiguousarray(x[0, :, :cells]).reshape(1, T, rows, cols)).cuda()
        a0, p0 = beamscan_frames(c0.expand(K, T, rows, cols), S, wrap=wrap)
        ac, pc = beamscan_frames(c0.repeat(K, 1, 1, 1), S, wrap=wrap)
        assert a0.is_cuda and torch.equal(a0, ac) and torch.equal(p0, pc)
    # the same bits whatever the batch: 2 frames versus the same 2 frames inside 40
    x = _cplx(rng, (3, 40, 12, 10))
    S = _grid_table(3, 181, rng)[0]
    a40, p40 = beamscan_frames(x, S)
    a2, p2 = beamscan_frames(np.ascontiguousarray(x[:, 17:19]), S)
    np.testing.assert_array_equal(a40[17:19], a2)
    np.testing.assert_array_equal(p40[17:19], p2)


def _scene(K, positions, n, fs, direct, echoes, seed, frames):
    """frames CPIs of a white reference and K surveillance channels: the direct path from `direct` degrees and echoes
    (theta, delay in samples, Doppler in Hz, amplitude), each scaled by a_k(theta), plus noise of 1e-3."""
    rng = np.random.default_rng(seed)
    ref = np.stack([synth.white_iq(rng, n) for _ in range(frames)])
    t = np.arange(n) / fs
    srv = np.zeros((K, frames, n), np.complex128)
    a_d = steering_vectors(positions, [direct])[0]
    for f in range(frames):
        sig = [(a_d, ref[f])]
        for th, d, fd, amp in echoes:
            sig.append((steering_vectors(positions, [th])[0], amp * np.roll(ref[f], d) * np.exp(2j * np.pi * fd * t)))
        for k in range(K):
            srv[k, f] = sum(a[k] * s for a, s in sig) + 1e-3 * synth.white_iq(rng, n)
    return ref, srv.astype(np.complex64)


@pytest.mark.gpu
@pytest.mark.parametrize("K,kind", [(3, "uca"), (4, "ula"), (3, "ula"), (4, "uca")])
def test_chain_from_frames_to_bearing_and_cfar(K, kind):
    import torch
    from passiveradar_b200.frames import FramePipeline
    from passiveradar_b200.plotting_tools import RenderPipeline
    n, fs, R, F, T = 2 ** 18, 2.0 ** 19, 60, 64, 2
    if kind == "ula":
        positions, grid, wrap = ula_positions(K, 0.5), SECTOR, False
        direct, echoes = 150.0, [(63.4, 17, 24.0, 0.03), (101.7, 41, -14.0, 0.02)]
    else:
        positions, grid, wrap = uca_positions(K, 0.3), CIRCLE, True
        direct, echoes = 200.0, [(358.3, 17, 24.0, 0.03), (121.6, 41, -14.0, 0.02)]
    S = steering_vectors(positions, grid)
    pipe = FramePipeline(n, R, F, channels=K, batch=2, nslots=1)

    def run(echo_list, seed):
        ref, srv = _scene(K, positions, n, fs, direct, echo_list, seed, T)
        ref_d, srv_d = torch.from_numpy(ref).cuda(), torch.from_numpy(srv).cuda()
        maps_d = torch.empty((K, T, F, R + 1), dtype=torch.complex64, device="cuda")
        pipe.run_device(ref_d, srv_d, maps_d, check=True)
        return beamscan_frames(maps_d, S, wrap=wrap)

    amp, pos = run(echoes, 7)
    assert amp.is_cuda and amp.shape == (T, F, R + 1)
    deg = bearing(pos.double(), grid, wrap=wrap).cpu().numpy()
    cr = prb.os_cfar_frames(amp, 18, 4).cpu().numpy()
    data, lim = RenderPipeline().run_device(amp)
    assert data.shape == (T, R + 1, F) and torch.isfinite(data).all() and torch.isfinite(lim).all()
    for i, (th, d, fd, a) in enumerate(echoes):
        amp1, _ = run([(th, d, fd, a)], 7)                    # the echo alone: its cell
        for f in range(T):
            cell = np.unravel_index(int(torch.argmax(amp1[f])), (F, R + 1))
            err = (deg[f][cell] - th + 180.0) % 360.0 - 180.0
            p999 = np.percentile(cr[f], 99.9)
            print(f"[beamscan] {kind} K={K} echo {i} frame {f}: cell {cell}, bearing {deg[f][cell]:.3f} "
                  f"(truth {th}), CR {cr[f][cell]:.1f} vs 99.9th percentile {p999:.2f} "
                  f"(margin {cr[f][cell] / p999:.1f}x)")
            assert abs(err) <= 0.25, (th, deg[f][cell])
            assert cr[f][cell] > p999
