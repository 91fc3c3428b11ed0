import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "slow: takes more than a few seconds on CPU")


def pytest_collection_modifyitems(config, items):
    """GPU tests must never silently pass on a box without a GPU."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device on this machine")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(params=["fft", "direct"])
def both_paths(request):
    """Run a GPU test once on the FFT-domain kernels (csrc/fftcorr.cuh, forced for every size they accept) and once on
    the direct-form kernels (wgmma / FP32): both are shipped and selectable (include/prcore.h: prc_set_option)."""
    from passiveradar_b200 import _lib
    old = (_lib.get_option("fft"), _lib.get_option("fft_min_n"))
    if request.param == "fft":
        _lib.set_option("fft", 1)
        _lib.set_option("fft_min_n", 0)
    else:
        _lib.set_option("fft", 0)
    yield request.param
    _lib.set_option("fft", old[0])
    _lib.set_option("fft_min_n", old[1])


def record_parity(name, **values):
    """Append per-stage parity figures of a GPU test to $PRC_PARITY_DIR/parity.json (nothing is written when the
    variable is unset: the tests never write into the checkout)."""
    import json
    out_dir = os.environ.get("PRC_PARITY_DIR")
    if not out_dir:
        return
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "parity.json")
    data = {}
    if os.path.exists(path):
        try:
            with open(path) as f:
                data = json.load(f)
        except ValueError:
            data = {}
    data[name] = {k: (float(v) if isinstance(v, (int, float)) or hasattr(v, "__float__") else v) for k, v in values.items()}
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)
