"""Shared-memory traffic of the one-pass frame kernel (csrc/framepass.cuh: frame_pass_kernel<8>).

The kernel is bound by its shared-memory pipe, so what it spares there is what it gains.  Two things are held here:

* the LS lag sums accC, accX stay in registers for the CTA's whole run, and the per-block CAF sums AccP, AccQ live in
  thread-private shared slots: a block's first segment does not read them, its last does not write them back (it
  writes `acc` instead), so a block of one segment never touches them;
* pass 2 reads its twiddles from padded rows [n3][k2] (fft::Tw2Rows), two per 128-bit load, 8 loads instead of 15,
  each one wavefront as each 64-bit load of the tw2 table was.

CPU: ``scripts/fft/emul.cu rows`` pins the staged rows' values, the banks of every warp's pair loads and whole seeded
transforms with the rows against the same with the table, bit for bit; the build's ptxas log holds the kernel to two
CTAs per SM with the 16 float2 of row padding; its SASS (cuobjdump of the built library) holds the loop body to the
loads and stores above.  Both skip when the library was built elsewhere, as test_fft_residency.py does.
"""
import collections
import os
import re
import shutil
import subprocess

import pytest

import test_fft_residency as fr
from test_fft_emulation import ROOT, _nvcc

L, R3, T = 2048, 8, 128
KERNEL = "_ZN3prc4fftc17frame_pass_kernelILi8EEEvNS0_15FramePassParamsE"


@pytest.fixture(scope="module")
def rows_report(tmp_path_factory):
    if _nvcc() is None:
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("emul") / "fft_emul")
    res = subprocess.run([_nvcc(), "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-I",
                          os.path.join(ROOT, "passiveradar_b200", "csrc"), "-o", exe,
                          os.path.join(ROOT, "scripts", "fft", "emul.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    run = subprocess.run([exe, "rows"], capture_output=True, text=True)
    assert run.returncode == 0, run.stdout + run.stderr
    return {k: int(v) for k, v in (kv.split("=") for kv in run.stdout.split())}


def framepass_smem_bytes():
    """SmemSeeded<8, Tw2Rows<8>> (two padded exchange buffers + 8 rows of 18 float2) + staging L float2 + AccP, AccQ
    2 L float2 + window L float"""
    return (2 * 16 * 17 * R3 + 18 * R3 + 3 * L + L // 2) * 8


def _instr(line):
    """(address, predicate, opcode, text) of a SASS line, or None"""
    m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\w+\s+)?([A-Z][\w.]*)([^;]*);", line)
    if not m:
        return None
    return int(m.group(1), 16), (m.group(2) or "").strip(), m.group(3), m.group(3) + m.group(4)


@pytest.fixture(scope="module")
def frame_sass():
    """frame_pass_kernel<8>'s SASS: (whole kernel, loop body).  The loop body is the span of the kernel's longest
    backward branch: the walk over items, one transform per iteration."""
    from passiveradar_b200 import build as b
    b.build(force=False)
    if not os.path.exists(os.path.join(b.PKG, "libprcore.ptxas.log")):
        pytest.skip("the library was built elsewhere (no ptxas log in this tree)")
    nvcc = _nvcc()
    cuobjdump = shutil.which("cuobjdump") or (nvcc and os.path.join(os.path.dirname(nvcc), "cuobjdump"))
    if not cuobjdump or not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    res = subprocess.run([cuobjdump, "-sass", "-fun", KERNEL, b.LIB], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    ins = [x for x in map(_instr, res.stdout.splitlines()) if x]
    assert ins, "frame_pass_kernel<8> not found in the library"
    span = None
    for addr, _, op, text in ins:
        m = re.search(r"BRA\s.*?0x([0-9a-f]+)", text) if op == "BRA" else None
        if m and int(m.group(1), 16) < addr and (span is None or addr - int(m.group(1), 16) > span[1] - span[0]):
            span = (int(m.group(1), 16), addr)
    assert span is not None
    return ins, [x for x in ins if span[0] <= x[0] <= span[1]]


# ------------------------------------------------------------------ CPU
def test_tw2_rows_hold_the_table_and_load_it_in_one_wavefront_per_pair(rows_report):
    r = rows_report
    assert r["rows_values_ok"] == 1 and r["rows_loaded_ok"] == 1, r
    assert r["rows_aligned"] == 1, r                       # every pair load is one 16-byte aligned LDS.128
    assert r["rows_wavefronts"] == 1 == r["table_wavefronts"], r


def test_transforms_with_tw2_rows_are_bit_identical_to_the_table(rows_report):
    assert rows_report["rows_bit_identical"] == 1, rows_report


def test_frame_layout_grows_by_the_row_padding_and_keeps_two_ctas_per_sm(rows_report):
    assert rows_report["smem_rows_float2"] == rows_report["smem_seeded_float2"] + 2 * R3
    smem = framepass_smem_bytes()
    assert smem == 93312 == 93184 + 16 * 8
    regs, spills = fr.fftc_entries()[("frame_pass_kernel", R3, None)]
    assert regs <= 255 and spills == "0 bytes spill stores, 0 bytes spill loads", (regs, spills)
    assert fr.ctas_per_sm(regs, T, smem) == 2, f"frame_pass_kernel<8>: {regs} registers x {T} threads, {smem} B"


def test_pass_two_reads_its_twiddles_two_per_load(frame_sass):
    whole, loop = frame_sass
    # 7 pair loads per pass 2 (pair (0, 1) is one 64-bit load: k2 = 0 is not used), at the loop's transform and at the
    # closing ones
    assert sum(op == "LDS.128" for _, _, op, _ in loop) == 7
    assert sum(op == "LDS.128" for _, _, op, _ in whole) == 14


def test_loop_body_touches_the_accumulator_slots_only_for_multi_segment_blocks(frame_sass):
    _, loop = frame_sass
    count = collections.Counter((pred, op) for _, pred, op, _ in loop if op in ("LDS.64", "STS.64", "STG.E.64"))
    # unconditional: the exchanges (16 STS + 16 LDS each), the staged input (16 LDS) and pair (0, 1) of pass 2
    assert count[("", "STS.64")] == 32, count
    assert count[("", "LDS.64")] == 49, count
    # AccP, AccQ: 32 reads under one predicate (not the block's first segment), 32 slot writes under another (not its
    # last segment) and 32 writes to `acc` under its complement
    reads = [n for (pred, op), n in count.items() if op == "LDS.64" and pred]
    assert max(reads) == 32, count
    stores = {pred: n for (pred, op), n in count.items() if op == "STS.64" and pred}
    outs = {pred: n for (pred, op), n in count.items() if op == "STG.E.64"}
    assert list(stores.values()) == [32] and list(outs.values()) == [32], count
    (sp,), (gp,) = stores, outs
    assert sp.replace("!", "") == gp.replace("!", "") and sp != gp, (sp, gp)
    assert not count[("", "STG.E.64")]


def test_loop_body_keeps_its_register_copies_down(frame_sass):
    # accC, accX are updated in place: with two register sets per array ptxas copied them on every item
    _, loop = frame_sass
    copies = sum(1 for _, _, op, text in loop if op == "MOV" and re.fullmatch(r"MOV R\d+, R\d+\s*", text))
    assert copies <= 40, copies
