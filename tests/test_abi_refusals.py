"""Every C entry point that takes a mem_kind refuses a malformed call with PRC_E_INVALID and the same message whether
its operands are host or device memory, before any CUDA call (so without a GPU too) and before any launch."""
import os
import re

import numpy as np
import pytest

from passiveradar_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST, DEV = _lib.MEM_HOST, _lib.MEM_DEVICE
_BUF = np.zeros(1 << 16, np.complex128)         # operands of the calls; never read, every row is refused first
P = _BUF.ctypes.data

# parameter names of every entry point (include/prcore.h) and the values of a well-formed call
PARAMS = {
    "prc_xambg_c64": "ref srv n range_bins freq_bins window dtaps ndtaps out mem_kind device stream flags",
    "prc_xambg_frames_c64": "ref srv n nframes frame_stride range_bins freq_bins window out mem_kind device stream flags",
    "prc_direct_xambg_c64": "ref srv n range_bins freq_bins sample_rate out mem_kind device stream flags",
    "prc_ls_filter_c64": "ref srv n filter_len peek reg out taps mem_kind device stream flags",
    "prc_ls_toeplitz_c64": "ref srv n filter_len peek out taps mem_kind device stream flags",
    "prc_ls_multiple_c64": "ref srv n filter_len peek sample_rate doppler_bins nbins out taps mem_kind device stream flags",
    "prc_ls_multiple_frames_c64": "ref srv n nframes frame_stride filter_len peek sample_rate doppler_bins nbins out "
                                  "mem_kind device stream flags",
    "prc_nlms_c64": "ref srv n filter_len peek mu block_len init_taps out taps mem_kind device stream flags",
    "prc_nlms_frames_c64": "ref srv n nframes frame_stride filter_len peek mu block_len init_taps out taps mem_kind "
                           "device stream flags",
    "prc_gal_jpe_frames_c64": "ref srv n nframes frame_stride lattice_len delay_line_len mu1 mu2 peek out k_out h_out "
                              "mem_kind device stream flags",
    "prc_ls_svd_frames_c64": "ref srv n nframes frame_stride filter_len peek out taps rank_out mem_kind device stream flags",
    "prc_frame_c64": "ref srv n filter_len peek reg range_bins freq_bins window out taps cleaned_out mem_kind device "
                     "stream flags",
    "prc_frames_c64": "ref srv n nframes frame_stride filter_len peek reg range_bins freq_bins window out taps "
                      "cleaned_out mem_kind device stream flags",
    "prc_iq_mix_c64": "in_ in_kind n mode fc fs phase_offset out mem_kind device stream flags",
    "prc_frontend_c64": "in_ in_kind n mode fc fs phase_offset up down h nh out out_capacity mem_kind device stream flags",
    "prc_frontend_chunks_c64": "in_ in_kind n nchunks chunk_stride mode fc fs phase_offsets up down h nh out out_stride "
                               "out_capacity mem_kind device stream flags",
    "prc_cfar2d_f32": "x rows cols fw gw thresh cr_out det_out mem_kind device stream flags",
    "prc_cfar2d_frames": "x rows cols nframes map_stride fw gw cr_out cr_stride mem_kind device stream flags",
    "prc_persistence_frames": "x rows cols nframes map_stride n_carry hold weights pout mem_kind device stream flags",
    "prc_percentiles_frames": "x n nframes frame_stride q scale nq pout mem_kind device stream flags",
    "prc_get_measurements_frames": "maps rows cols nseq nframes seq_stride map_stride doppler_extent range_extent "
                                   "meas_capacity counts meas mem_kind device stream flags",
    "prc_multitarget_track_frames": "maps rows cols nseq nframes seq_stride map_stride doppler_extent range_extent "
                                    "n_tracks history mem_kind device stream flags",
    "prc_simple_track_frames": "maps rows cols nseq nframes seq_stride map_stride range_extent doppler_extent history "
                               "mem_kind device stream flags",
    "prc_channel_offset": "s1 dtype1 n1 s2 dtype2 n2 nd nl sos zi offset xc_abs mem_kind device stream flags",
    "prc_xcorr": "s1 dtype1 n1 s2 dtype2 n2 nlead nlag out mem_kind device stream flags",
}
VALID = dict(
    ref=P, srv=P, out=P, taps=None, n=64, nframes=2, frame_stride=64, range_bins=4, freq_bins=8, window=None,
    dtaps=None, ndtaps=0, sample_rate=1e6, filter_len=8, peek=2, reg=0.0, doppler_bins=None, nbins=1, mu=0.5,
    block_len=1, init_taps=None, lattice_len=4, delay_line_len=8, mu1=1e-3, mu2=1e-2, k_out=None, h_out=None,
    rank_out=None, cleaned_out=None, in_=P, in_kind=_lib.IQ_C64, mode=_lib.MIX_NONE, fc=0.0, fs=1e6, phase_offset=0.0,
    up=1, down=1, h=P, nh=1, out_capacity=1 << 12, nchunks=2, chunk_stride=64, phase_offsets=P, out_stride=64, x=P,
    rows=8, cols=8, fw=2, gw=1, thresh=P, cr_out=P, det_out=None, map_stride=64, cr_stride=64, n_carry=0, hold=2,
    weights=P, pout=P, q=P, scale=None, nq=1, maps=P, nseq=1, seq_stride=128, doppler_extent=256.0, range_extent=200.0,
    meas_capacity=0, counts=P, meas=None, n_tracks=1, history=P, s1=P, s2=P, dtype1=_lib.DT_C64, dtype2=_lib.DT_C64,
    n1=1 << 12, n2=1 << 12, nd=1, nl=4, sos=P, zi=P, offset=P, xc_abs=None, nlead=4, nlag=4, mem_kind=HOST, device=0,
    stream=None, flags=0,
)
REF_SRV = [e for e, p in PARAMS.items() if p.startswith("ref srv")]
FRAMES = [e for e in REF_SRV if "nframes" in PARAMS[e]]
FRONT_END = ("prc_iq_mix_c64", "prc_frontend_c64", "prc_frontend_chunks_c64")
FIRST = {e: PARAMS[e].split()[0] for e in PARAMS}
NULL_MSG = {"prc_frames_c64": "ref/srv/out_maps must not be NULL", "prc_frame_c64": "ref/srv/out_maps must not be NULL",
            "prc_iq_mix_c64": "in/out must not be NULL", "prc_frontend_c64": "in/out/h must not be NULL",
            "prc_frontend_chunks_c64": "in/out/h/phase_offsets must not be NULL",
            "prc_cfar2d_f32": "x and one of cr_out/det_out must not be NULL", "prc_cfar2d_frames": "x and cr_out must not be NULL",
            "prc_persistence_frames": "x/weights/out must not be NULL", "prc_percentiles_frames": "x/q/out must not be NULL",
            "prc_get_measurements_frames": "maps must not be NULL", "prc_multitarget_track_frames": "maps must not be NULL",
            "prc_simple_track_frames": "maps must not be NULL", "prc_channel_offset": "s1/s2 must not be NULL",
            "prc_xcorr": "s1/s2 must not be NULL"}

ROWS = []
for e in PARAMS:
    ROWS.append((e, {FIRST[e]: None}, NULL_MSG.get(e, "ref/srv/out must not be NULL")))
    if e == "prc_ls_multiple_frames_c64":
        ROWS.append((e, {"mem_kind": HOST}, "prc_ls_multiple_frames_c64 takes device pointers (mem_kind=0)"))
    else:
        ROWS.append((e, {"mem_kind": 2}, "mem_kind=2 invalid"))
for e in REF_SRV + list(FRONT_END):
    ROWS.append((e, {"n": 0}, "n=0 unsupported" if e == "prc_ls_svd_frames_c64" else "n=0 invalid"))
for e in FRAMES:
    ROWS.append((e, {"nframes": 0},
                 "nframes=0 nbins=1 invalid" if e == "prc_ls_multiple_frames_c64" else "nframes=0 invalid"))
    ROWS.append((e, {"frame_stride": 63}, "frame_stride=63 smaller than n=64"))
for e in ("prc_xambg_c64", "prc_xambg_frames_c64", "prc_frame_c64", "prc_frames_c64"):
    ROWS.append((e, {"freq_bins": 0}, "freq_bins=0 / range_bins=4 invalid"))
    ROWS.append((e, {"range_bins": -1}, "freq_bins=8 / range_bins=-1 invalid"))
ROWS.append(("prc_direct_xambg_c64", {"freq_bins": 0}, "range_bins=4 freq_bins=0 invalid"))
for e in FRONT_END:
    ROWS.append((e, {"in_kind": 3}, "in_kind=3 invalid"))
    ROWS.append((e, {"mode": 5}, "mode=5 invalid"))
    ROWS.append((e, {"mode": _lib.MIX_C64, "fs": 0.0}, "fs must not be 0"))
for e in ("prc_persistence_frames", "prc_percentiles_frames", "prc_cfar2d_frames"):
    ROWS.append((e, {"nframes": 2, "map_stride" if e != "prc_percentiles_frames" else "frame_stride": 7},
                 "frame_stride=7"))
for e in ("prc_get_measurements_frames", "prc_multitarget_track_frames", "prc_simple_track_frames"):
    ROWS.append((e, {"nframes": 0}, "nframes=0 invalid"))


def _call(entry, **kw):
    args = dict(VALID, **kw)
    return getattr(_lib.load(), entry)(*[args[p] for p in PARAMS[entry].split()])


def test_table_covers_every_entry_point_that_takes_mem_kind():
    with open(os.path.join(ROOT, "include", "prcore.h")) as f:
        decls = dict(re.findall(r"^int (prc_\w+)\(([^;]*)\);", f.read(), re.M | re.S))
    assert set(PARAMS) == {e for e, params in decls.items() if "mem_kind" in params}
    for e, names in PARAMS.items():
        assert len(names.split()) == len(decls[e].split(",")) == len(_lib.SIGNATURES[e][1]), e


@pytest.mark.parametrize("mem_kind", [HOST, DEV])
def test_malformed_calls_are_refused_before_any_launch(mem_kind):
    lib = _lib.load()
    before = _lib.launch_count()
    for entry, kw, msg in ROWS:
        if entry == "prc_ls_multiple_frames_c64" and mem_kind == HOST and "mem_kind" not in kw:
            continue            # takes device pointers only: its host refusal is a row of its own
        kw = dict({"mem_kind": mem_kind}, **kw)
        st = _call(entry, **kw)
        err = lib.prc_last_error().decode()
        assert st == _lib.PRC_E_INVALID, (entry, kw, st, err)
        assert msg in err, (entry, kw, msg, err)
    assert _lib.launch_count() == before
