"""Place the UNMODIFIED reference modules of the hot path under oracle/_ref/ (git-ignored, never committed).

The reference (Max-Manning/passiveRadar) is plain Python without setup.py / pyproject.toml, so
``pip install --target oracle/_ref <reference checkout>`` has nothing to build; this recipe is the equivalent: it
copies the package's modules byte for byte and records their sha256 in oracle/_ref/MANIFEST.json.  The CPU arm of
``bench.py`` (``cpu_baseline`` and ``--impl reference``) imports ``passiveRadar.clutter_removal.LS_Filter`` /
``NLMS_filter`` / ``LS_Filter_Multiple`` and ``passiveRadar.range_doppler_processing.fast_xambg`` from there
(kind "reference"); when oracle/_ref is absent it times the oracle port instead (kind "port").

    python oracle/install_ref.py [REFERENCE_CHECKOUT]

The checkout is the argument, else $PR_REFERENCE, else a directory named ``reference`` next to the repository
checkout; without one nothing is installed and an existing oracle/_ref is left as it is.
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")
FILES = ["__init__.py", "clutter_removal.py", "range_doppler_processing.py", "signal_utils.py"]


def default_source():
    if os.environ.get("PR_REFERENCE"):
        return os.environ["PR_REFERENCE"]
    return os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference")


def install(src_root=None):
    """Copy the reference's modules to oracle/_ref/passiveRadar; returns that directory, or None without a source."""
    src = os.path.join(src_root or default_source(), "passiveRadar")
    if not os.path.isdir(src):
        return None
    dst = os.path.join(DEST, "passiveRadar")
    os.makedirs(dst, exist_ok=True)
    digest = {}
    for f in FILES:
        a = os.path.join(src, f)
        if not os.path.exists(a):
            if f == "__init__.py":
                open(os.path.join(dst, f), "w").close()
            continue
        shutil.copyfile(a, os.path.join(dst, f))
        with open(a, "rb") as fh:
            digest[f] = hashlib.sha256(fh.read()).hexdigest()
    with open(os.path.join(DEST, "MANIFEST.json"), "w") as fh:
        json.dump({"sha256": digest}, fh, indent=1)
    return dst


if __name__ == "__main__":
    out = install(sys.argv[1] if len(sys.argv) > 1 else None)
    print(out if out else "reference checkout not found; nothing installed")
