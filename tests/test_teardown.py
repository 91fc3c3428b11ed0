"""The two ways a workspace is torn down (prcore.cu: Ctx::~Ctx): prc_shutdown, here with profiling records nobody
collected, and the exit of a thread that called with stream == NULL.  The next call builds new workspaces and gives the
same bits.  Device memory is not checked: other work shares the card."""
import threading

import numpy as np
import pytest

import passiveradar_b200 as prb
from passiveradar_b200 import _lib, synth

pytestmark = pytest.mark.gpu

N, R, F = 2 ** 16, 100, 64           # FFT-domain CAF (n / F = 1024)
FILTER_LEN, PEEK = 60, 10


def _inputs():
    return synth.make_frame(N, "P1", frame=7)


def _calls(ref, srv):
    """A CAF and an LS filter on the calling thread's workspace (the wrappers pass stream == NULL)."""
    caf = prb.fast_xambg(ref, srv, R, F)
    out, taps = prb.LS_Filter(ref, srv, FILTER_LEN, 1.0, PEEK, True)
    return caf, out, taps


def _same_bits(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_shutdown_with_uncollected_profile_then_the_same_call_gives_the_same_bits():
    ref, srv = _inputs()
    _lib.profile_reset()
    _lib.profile(True)
    try:
        first = _calls(ref, srv)          # leaves an event pair per launch in the workspace
    finally:
        _lib.profile(False)
    _lib.load().prc_shutdown()           # frees the workspaces with their records still pending
    _lib.profile_reset()
    again = _calls(ref, srv)
    assert _same_bits(first, again)


def test_a_thread_that_exits_frees_its_workspace_and_the_main_thread_runs_on():
    ref, srv = _inputs()
    want = _calls(ref, srv)
    res = {}

    def worker():
        try:
            res["out"] = _calls(ref, srv)
        except BaseException as exc:      # re-raised on the main thread
            res["exc"] = exc

    t = threading.Thread(target=worker)
    t.start()
    t.join()
    if "exc" in res:
        raise res["exc"]
    after = _calls(ref, srv)
    assert _same_bits(res["out"], want)
    assert _same_bits(after, want)
