"""k_track2<1024, *> walks a correspondence line with a compact loop that stays out of local memory on sm_90a.

A correspondence iteration runs the line walk on 16 warps at once, beside the point warps' depth search and followed by
the serial solve. When the walk was unrolled over its 19 segments for every compile-time scale it made up almost half
of the kernel's instructions (about 8,700 of 19,000), far more than the SM's instruction caches hold, so every
iteration streamed its code in again. WalkFast now loops over the segments (two per trip) and unrolls only the samples
of a segment. The test disassembles the shipped library (cuobjdump / nvdisasm -g on the -lineinfo build) and asserts, for
both 1024-thread instantiations, that the instructions attributed to WalkFast's source lines stay below a bound and
that none of them is an LDL / STL: with 64 registers per thread and ~3 KB of L1 next to 225 KB of shared memory, a
local-memory access is an L2 round trip, and a window array indexed at run time would land there."""
import glob
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
TRACK2 = os.path.join(CSRC, "m3t_b200_track2.cuh")
KERNELS = ("_ZN4m3tb8k_track2ILi1024ELb1EEEvNS_9TrackArgsE", "_ZN4m3tb8k_track2ILi1024ELb0EEEvNS_9TrackArgsE")
# Five scale specialisations of the rolled walk, two segments per loop trip: ~1,300 instructions against the unrolled
# walk's ~8,700
MAX_WALK_INSTRUCTIONS = 1600


def _function_lines(path, name):
    """1-based line numbers of the definition of `name` in `path` (signature to matching closing brace)."""
    lines = open(path).read().splitlines()
    for i, line in enumerate(lines):
        if re.search(r"__device__.*\b%s\s*\(" % name, line):
            depth, opened = 0, False
            for j in range(i, len(lines)):
                depth += lines[j].count("{") - lines[j].count("}")
                opened = opened or "{" in lines[j]
                if opened and depth == 0:
                    return set(range(i + 1, j + 2))
    raise AssertionError(f"{name} not found in {path}")


def _attributed(so, basename, lines):
    """{kernel: [opcode, ...]} of the instructions of the two 1024-thread k_track2 instantiations whose innermost
    source location is one of `lines` of the file `basename`."""
    found = {}
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run(["cuobjdump", "-xelf", "all", so], cwd=tmp, check=True, capture_output=True)
        for cubin in glob.glob(os.path.join(tmp, "*.cubin")):
            out = subprocess.run(["nvdisasm", "-g", "-c", cubin], check=True, capture_output=True, text=True).stdout
            fn, loc = None, None
            for line in out.splitlines():
                m = re.match(r"\s*\.text\.(\S+):", line)
                if m:
                    fn, loc = m.group(1), None
                    if fn in KERNELS:
                        found.setdefault(fn, [])
                    continue
                m = re.search(r'//## File "([^"]+)", line (\d+)', line)
                if m:
                    loc = (os.path.basename(m.group(1)), int(m.group(2)))
                    continue
                m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
                if m and fn in KERNELS and loc and loc[0] == basename and loc[1] in lines:
                    found[fn].append(m.group(1))
    return found


def test_track2_line_walk_is_compact_and_register_resident(pkg):
    if not (shutil.which("cuobjdump") and shutil.which("nvdisasm")):
        pytest.skip("cuobjdump / nvdisasm not available")
    pkg._build.build_cuda()  # in-tree nvcc build (cross-compiles for sm_90a without a GPU)
    found = _attributed(os.path.join(CSRC, "libm3t_b200.so"), os.path.basename(TRACK2),
                        _function_lines(TRACK2, "WalkFast"))
    assert sorted(found) == sorted(KERNELS), sorted(found)
    for kernel, ops in found.items():
        assert ops, f"{kernel}: no instruction attributed to WalkFast (line information missing?)"
        assert len(ops) <= MAX_WALK_INSTRUCTIONS, f"{kernel}: WalkFast is {len(ops)} instructions"
        local = [op for op in ops if op.split(".")[0] in ("LDL", "STL")]
        assert not local, f"{kernel}: WalkFast touches local memory ({len(local)} x {sorted(set(local))})"
