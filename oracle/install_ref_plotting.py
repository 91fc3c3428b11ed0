"""Place the reference's UNMODIFIED plotting_tools.py next to the modules oracle/install_ref.py copies (git-ignored,
never committed), for the reference column of scripts/render_bench.py.

That module imports matplotlib.pyplot at import time; it is copied byte for byte all the same, and whoever imports it
without matplotlib puts a stub in sys.modules in their own process.  Its sha256 is added to oracle/_ref/MANIFEST.json.

    python oracle/install_ref_plotting.py [REFERENCE_CHECKOUT]

Run after oracle/install_ref.py (which rewrites the manifest).  Without a reference checkout nothing is installed.
"""
import hashlib
import json
import os
import shutil
import sys

try:                                                 # same source and destination rules as install_ref
    from . import install_ref
except ImportError:                                  # run as a script
    import install_ref

FILES = ("plotting_tools.py",)


def install(src_root=None):
    """Copy the reference's plotting module to oracle/_ref/passiveRadar; returns that directory, or None."""
    src = os.path.join(src_root or install_ref.default_source(), "passiveRadar")
    dst = os.path.join(install_ref.DEST, "passiveRadar")
    if not os.path.isdir(src) or not os.path.isdir(dst):
        return None
    manifest = os.path.join(install_ref.DEST, "MANIFEST.json")
    data = {"sha256": {}}
    if os.path.exists(manifest):
        with open(manifest) as fh:
            data = json.load(fh)
    for f in FILES:
        a = os.path.join(src, f)
        if not os.path.exists(a):
            continue
        shutil.copyfile(a, os.path.join(dst, f))
        with open(a, "rb") as fh:
            data.setdefault("sha256", {})[f] = hashlib.sha256(fh.read()).hexdigest()
    with open(manifest, "w") as fh:
        json.dump(data, fh, indent=1)
    return dst


if __name__ == "__main__":
    out = install(sys.argv[1] if len(sys.argv) > 1 else None)
    print(out if out else "reference checkout (or oracle/_ref) not found; nothing installed")
