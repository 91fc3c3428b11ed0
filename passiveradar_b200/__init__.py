"""passiveradar_b200 -- H100-native (sm_90a) core for the passive-radar hot path.

Drop-in operators with the reference's call signatures (Max-Manning/passiveRadar):

    from passiveradar_b200 import fast_xambg, LS_Filter, NLMS_filter, block_NLMS, GAL_JPE, LS_Filter_SVD

and a device-resident frame pipeline for streams of CPI frames
(``passiveradar_b200.frames.FramePipeline``).  All arithmetic runs in
``libprcore.so`` (hand-written CUDA, C ABI in ``include/prcore.h``); importing
this package never imports the CPU oracle and never falls back to the CPU.
"""
from .range_doppler_processing import fast_xambg, direct_xambg            # noqa: F401
from .clutter_removal import (LS_Filter, NLMS_filter, block_NLMS,            # noqa: F401
                              LS_Filter_Toeplitz, LS_Filter_Multiple, GAL_JPE, gal_jpe_frames,
                              LS_Filter_SVD, ls_filter_svd_frames)
from .signal_utils import (deinterleave_IQ, frequency_shift, resample, frontend,            # noqa: F401
                           find_channel_offset, offset_compensation, shift, xcorr, decimate,
                           channel_preprocessing, normalize)
from .target_detection import (CFAR_2D, OS_CFAR_2D, os_cfar_frames, get_measurements, multitarget_tracker, simple_target_tracker,  # noqa: F401
                               multitarget_tracker_frames, simple_tracker_frames, cfar_track, TrackerPipeline,
                               kalman_filter_dtype, target_track_dtype, target_track_dtype_simple)
from .recording import RecordingPipeline                                     # noqa: F401
from .plotting_tools import persistence, persistence_frames, RenderPipeline  # noqa: F401
from .spectrum import psd, psd_frames, SignalPreview                         # noqa: F401
from .beamforming import steering_vectors, ula_positions, uca_positions, beamscan_frames, bearing  # noqa: F401

__all__ = ["fast_xambg", "direct_xambg", "LS_Filter", "NLMS_filter", "block_NLMS", "LS_Filter_Toeplitz",
           "LS_Filter_Multiple", "GAL_JPE", "gal_jpe_frames", "LS_Filter_SVD", "ls_filter_svd_frames", "deinterleave_IQ", "frequency_shift", "resample", "frontend",
           "find_channel_offset", "offset_compensation", "shift", "xcorr", "decimate", "channel_preprocessing",
           "normalize", "CFAR_2D", "OS_CFAR_2D", "os_cfar_frames",
           "get_measurements", "multitarget_tracker", "simple_target_tracker", "multitarget_tracker_frames",
           "simple_tracker_frames", "cfar_track", "TrackerPipeline", "RecordingPipeline", "persistence", "persistence_frames",
           "RenderPipeline", "psd", "psd_frames", "SignalPreview", "steering_vectors", "ula_positions", "uca_positions",
           "beamscan_frames", "bearing"]
__version__ = "0.1.0"


def install(reference_package: str = "passiveRadar"):
    """Swap the hot-path functions of an importable copy of the reference for the GPU ones.

    ``main.py`` binds ``fast_xambg``, ``LS_Filter_Multiple``, ``NLMS_filter`` and ``find_channel_offset`` with
    ``from passiveRadar... import ...`` (main.py:10-14); calling ``install()`` before ``main.py`` is
    imported/run makes those names resolve to this package while config, I/O and the dask graph stay
    the reference's own code::

        python -c "import passiveradar_b200 as p, runpy; p.install(); runpy.run_path('main.py', run_name='__main__')" --config PRconfig.yaml

    Returns the list of ``module.attribute`` names that were replaced.
    """
    import importlib
    replaced = []
    table = {
        "range_doppler_processing": {"fast_xambg": fast_xambg, "direct_xambg": direct_xambg},
        # xcorr stays the reference's: only its LS_Filter_Toeplitz and direct_xambg call it, and both are replaced
        "signal_utils": {"deinterleave_IQ": deinterleave_IQ, "frequency_shift": frequency_shift, "resample": resample,
                         "find_channel_offset": find_channel_offset, "offset_compensation": offset_compensation,
                         "decimate": decimate, "channel_preprocessing": channel_preprocessing, "normalize": normalize},
        "target_detection": {"CFAR_2D": CFAR_2D, "get_measurements": get_measurements,
                             "multitarget_tracker": multitarget_tracker, "simple_target_tracker": simple_target_tracker},
        "clutter_removal": {"LS_Filter": LS_Filter, "NLMS_filter": NLMS_filter,
                            "LS_Filter_Toeplitz": LS_Filter_Toeplitz, "LS_Filter_Multiple": LS_Filter_Multiple},
        # the reference's plotting_tools imports matplotlib: skipped like any optional module that does not import
        "plotting_tools": {"persistence": persistence},
    }
    for modname, attrs in table.items():
        try:
            mod = importlib.import_module(f"{reference_package}.{modname}")
        except Exception:          # e.g. the reference's target_detection needs np.float (NumPy < 1.24)
            if modname in ("range_doppler_processing", "clutter_removal"):
                raise
            continue
        for name, fn in attrs.items():
            setattr(mod, name, fn)
            replaced.append(f"{reference_package}.{modname}.{name}")
        if modname == "clutter_removal" and not hasattr(mod, "block_NLMS"):
            mod.block_NLMS = block_NLMS
            replaced.append(f"{reference_package}.{modname}.block_NLMS")
    return replaced
