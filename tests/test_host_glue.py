"""The host glue every operator module shares through ``_lib``: the dtype codes of include/prcore.h, and the stream a
device-pointer call is enqueued on when the caller is on torch's default stream."""
import os
import re

import numpy as np
import pytest

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXTENT = [256.0, 200.0]                  # [max_doppler, max_range]


def test_dtype_codes_and_tables_match_the_header():
    with open(os.path.join(ROOT, "include", "prcore.h")) as f:
        src = f.read()
    header = {name: int(v) for name, v in re.findall(r"^#define PRC_((?:DT|IQ)_\w+)\s+(\d+)\s*$", src, re.M)}
    assert sorted(header) == ["DT_C128", "DT_C64", "DT_F32", "DT_F64", "DT_I16", "DT_I8", "DT_U8",
                              "IQ_C64", "IQ_I16", "IQ_I8"]
    for name, v in header.items():
        assert getattr(_lib, name) == v, name
    dt = {"I8": np.int8, "U8": np.uint8, "I16": np.int16, "F32": np.float32, "F64": np.float64,
          "C64": np.complex64, "C128": np.complex128}
    assert _lib.DT_CODES == {np.dtype(dt[n[3:]]): v for n, v in header.items() if n.startswith("DT_")}
    # raw interleaved IQ: int8 and int16 integers, or float32 pairs read as complex64 samples
    assert _lib.IQ_KINDS == {np.dtype(np.int8): header["IQ_I8"], np.dtype(np.int16): header["IQ_I16"],
                             np.dtype(np.float32): header["IQ_C64"]}
    import torch
    for d in _lib.DT_CODES:
        assert _lib.np_dtype(_lib.torch_dtype(d)) == d
    assert _lib.np_dtype(torch.bfloat16) is None


@pytest.mark.gpu
def test_device_calls_on_the_default_stream_wait_for_its_work():
    """The library takes stream 0 for a stream of its own that does not wait for torch's default stream: work queued
    there just before the call (a copy held back by a sleep) must still be seen, with no synchronisation between."""
    import torch
    dev = torch.device("cuda", _lib.current_device())
    T, F, R1 = 24, 64, 101
    mag = synth.track_maps(910, F, R1, T, 4)
    rng = np.random.default_rng(910)
    cmaps = torch.from_numpy((mag * np.exp(1j * rng.uniform(0, 2 * np.pi, mag.shape))).astype(np.complex64)).to(dev)
    rmaps = torch.from_numpy(mag[None]).to(dev)
    torch.cuda.synchronize(dev)
    want_cfar = prb.cfar_track(cmaps, 18, 4, EXTENT, 6)
    want_track = prb.multitarget_tracker_frames(rmaps, EXTENT, 6)
    # a call that read the zeroed tensor would be seen
    assert prb.cfar_track(torch.zeros_like(cmaps), 18, 4, EXTENT, 6).tobytes() != want_cfar.tobytes()
    assert prb.multitarget_tracker_frames(torch.zeros_like(rmaps), EXTENT, 6).tobytes() != want_track.tobytes()

    def late(src):
        """A zeroed copy of src that the default stream fills after about 0.1 s of sleep."""
        dst = torch.zeros_like(src)
        torch.cuda._sleep(200_000_000)                           # cycles: 0.1 s at 2 GHz
        dst.copy_(src)
        return dst

    with torch.cuda.device(dev):
        assert torch.cuda.current_stream(dev).cuda_stream == 0
        got_cfar = prb.cfar_track(late(cmaps), 18, 4, EXTENT, 6)
        got_track = prb.multitarget_tracker_frames(late(rmaps), EXTENT, 6)
    assert got_cfar.tobytes() == want_cfar.tobytes()
    assert got_track.tobytes() == want_track.tobytes()
