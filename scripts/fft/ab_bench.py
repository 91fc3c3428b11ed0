"""A/B of two libprcore builds on the flagship benchmark: bench.py, unmodified, in child processes.

    python scripts/fft/ab_bench.py build --base REV        # compile REV's sources and the working tree's (no GPU needed)
    python scripts/fft/ab_bench.py run --out DIR           # A, B, A, B, A, B on the GPU; DIR/ab.json

``build`` compiles every ``*.cu`` of ``passiveradar_b200/csrc`` (+ ``include``) of the commit REV (A: ``git archive``) and of
the working tree (B), each with the flags of its own passiveradar_b200/build.py, into the git-ignored
``build/ab/{A,B}/libprcore.so``.  ``run``
alternates ``bench.py --no-cpu-baseline`` between the two (each child loads its build through PRC_LIBRARY; the Python
side is the working tree's for both), so a drift of clocks or temperature over the session hits both builds alike.  The
first run of each build also writes its ``--dump-outputs`` maps, and the two are compared bit for bit.  Per run it keeps
the headline ``value``, the single-frame ``latency_us``, the ``e2e`` rate, the per-frame times of the kernels in
``KERNELS`` (``lagcorr_ls`` is empty when the one-pass frame runs: ``lagcorr_caf`` is then ``frame_pass_kernel``), the SM clocks bench.py sampled, and the card name and power limit; the summary has the median and
range per build.  On a power-capped card compare the sampled SM clocks too: a kernel that keeps more warps busy draws
more power, and the cap then lowers the clock of everything running beside it.
"""
from __future__ import annotations

import argparse
import importlib.util
import io
import json
import os
import statistics
import subprocess
import sys
import tarfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
AB = os.path.join(ROOT, "build", "ab")
KERNELS = ("lagcorr_ls", "lagcorr_caf", "caf_combine", "levinson", "doppler_fft")


def tree_flags(src_root: str) -> list:
    """NVCC_FLAGS of the tree's own build.py: a revision is compiled as it builds itself (the flags that export its C
    entry points changed when prcore.cu was split into modules)."""
    spec = importlib.util.spec_from_file_location("ab_tree_build", os.path.join(src_root, "passiveradar_b200", "build.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.NVCC_FLAGS


def compile_lib(src_root: str, out_dir: str) -> str:
    sys.path.insert(0, ROOT)
    from passiveradar_b200 import build as b
    os.makedirs(out_dir, exist_ok=True)
    lib = os.path.join(out_dir, "libprcore.so")
    csrc = os.path.join(src_root, "passiveradar_b200", "csrc")
    sources = sorted(os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith(".cu"))
    cmd = [b.find_nvcc()] + tree_flags(src_root) + ["-I", os.path.join(src_root, "include"), "-I", csrc,
                                                    "-o", lib] + sources
    res = subprocess.run(cmd, capture_output=True, text=True)
    with open(os.path.join(out_dir, "ptxas.log"), "w") as f:
        f.write(res.stdout + res.stderr)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise SystemExit(f"nvcc failed for {src_root}")
    return lib


def cmd_build(args):
    rev = subprocess.run(["git", "-C", ROOT, "rev-parse", args.base], capture_output=True, text=True, check=True).stdout.strip()
    src_a = os.path.join(AB, "A", "src")
    os.makedirs(src_a, exist_ok=True)
    tar = subprocess.run(["git", "-C", ROOT, "archive", rev, "passiveradar_b200/csrc", "passiveradar_b200/build.py",
                          "include"], capture_output=True, check=True).stdout
    with tarfile.open(fileobj=io.BytesIO(tar)) as tf:
        tf.extractall(src_a, filter="data")
    compile_lib(src_a, os.path.join(AB, "A"))
    compile_lib(ROOT, os.path.join(AB, "B"))
    dirty = subprocess.run(["git", "-C", ROOT, "status", "--porcelain", "--", "passiveradar_b200/csrc", "include"],
                           capture_output=True, text=True).stdout.strip()
    head = subprocess.run(["git", "-C", ROOT, "rev-parse", "HEAD"], capture_output=True, text=True).stdout.strip()
    with open(os.path.join(AB, "manifest.json"), "w") as f:
        json.dump({"A": {"rev": rev}, "B": {"rev": head, "uncommitted_changes": bool(dirty)}}, f, indent=1)
    print(f"A = {rev[:12]}, B = working tree ({head[:12]}{' + changes' if dirty else ''}) -> {AB}")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",", 1)]
        return {"name": name, "power_limit": power}
    except Exception as exc:       # context only
        return {"error": str(exc)}


def one_run(label, args, dump_dir=None):
    env = dict(os.environ, PRC_LIBRARY=os.path.join(AB, label, "libprcore.so"))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps),
           "--warmup", str(args.warmup), "--no-cpu-baseline"]
    if dump_dir:
        cmd += ["--dump-outputs", dump_dir]
    res = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    if res.returncode != 0:
        sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
        raise SystemExit(f"bench.py failed for build {label}")
    line = json.loads([ln for ln in res.stdout.splitlines() if ln.startswith("{")][-1])
    rec = {"build": label, "value": line["value"], "latency_us": line.get("latency_us"),
           "e2e": (line.get("e2e") or {}).get("value"), "clocks": line.get("clocks"), "card": card()}
    for k in KERNELS:
        rec[k] = line["kernels"].get(k, {}).get("us_per_frame")
    print(json.dumps(rec), flush=True)
    return rec


def summary(vals):
    vals = [v for v in vals if v is not None]
    return {"median": statistics.median(vals), "min": min(vals), "max": max(vals), "n": len(vals)} if vals else None


def cmd_run(args):
    import numpy as np
    for label in ("A", "B"):
        if not os.path.exists(os.path.join(AB, label, "libprcore.so")):
            raise SystemExit(f"{AB}/{label}/libprcore.so missing: run `ab_bench.py build` first")
    os.makedirs(args.out, exist_ok=True)
    runs = []
    for r in range(args.rounds):
        for label in ("A", "B"):
            runs.append(one_run(label, args, os.path.join(args.out, f"dump_{label}") if r == 0 else None))
    maps = {lb: np.load(os.path.join(args.out, f"dump_{lb}", "maps.npy")) for lb in ("A", "B")}
    res = {"manifest": json.load(open(os.path.join(AB, "manifest.json"))) if os.path.exists(os.path.join(AB, "manifest.json")) else None,
           "bench_args": {"steps": args.steps, "warmup": args.warmup, "no_cpu_baseline": True},
           "runs": runs,
           "maps_bit_identical": bool(np.array_equal(maps["A"], maps["B"])),
           "maps_max_abs_diff": float(np.abs(maps["A"].astype(np.float64) - maps["B"]).max()) if maps["A"].shape == maps["B"].shape else None}
    for label in ("A", "B"):
        mine = [x for x in runs if x["build"] == label]
        res[label] = {k: summary([x[k] for x in mine]) for k in ("value", "latency_us", "e2e") + KERNELS}
    a, b = res["A"]["value"], res["B"]["value"]
    res["headline_gain"] = b["median"] / a["median"] - 1.0
    res["every_B_above_every_A"] = b["min"] > a["max"]
    for k in KERNELS:
        if res["A"][k] and res["B"][k]:
            res[f"{k}_change"] = res["B"][k]["median"] / res["A"][k]["median"] - 1.0
    with open(os.path.join(args.out, "ab.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    b = sub.add_parser("build")
    b.add_argument("--base", default="HEAD", help="commit of build A (the working tree is B)")
    r = sub.add_parser("run")
    r.add_argument("--out", default=os.path.join(AB, "result"))
    r.add_argument("--rounds", type=int, default=3)
    r.add_argument("--steps", type=int, default=20)
    r.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    cmd_build(args) if args.cmd == "build" else cmd_run(args)


if __name__ == "__main__":
    main()
