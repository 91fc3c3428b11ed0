"""The committed goldens are outputs of the REFERENCE.  tests/golden/reference_digests.json holds, for a few small
cases, the sha256 of every array tests/golden/make_golden.py --only <case> produced when it was run against the
reference tree (dtype, shape and bytes; the wall-time entry excluded); that run reproduced the committed .npz files
bit for bit.  The test requires the committed arrays to still have exactly those digests, so a golden can only
change together with a fresh run of the reference."""
import hashlib
import json
import os

import numpy as np
import pytest

import _golden as G

with open(os.path.join(G.GOLDEN_DIR, "reference_digests.json")) as _f:
    DIGESTS = json.load(_f)


def _digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("name", ["xambg_small_kaiser", "ls_small", "nlms_peek0", "toep_small", "multi_fs_odd",
                                  "cfar_odd", "direct_small", "front_f32_short", "resample_c128"])
def test_committed_golden_is_what_the_reference_produces(name):
    committed = G.load(name)
    want = DIGESTS[name]
    assert set(want) == set(committed) - {"seconds"}
    for k in want:
        assert _digest(committed[k]) == want[k], f"{name}[{k}] differs from the reference's output"
