"""k_track2<1024, *> keeps its per-update hot sections out of local memory on sm_90a.

With 64 registers per thread and ~3 KB of L1 left next to 225 KB of shared memory, every local-memory access of the
1024-thread kernel is an L2 round trip. The test disassembles the shipped library (cuobjdump / nvdisasm, -lineinfo
build) and asserts that no LDL / STL of the two 1024-thread instantiations maps to a source line of the warp
reduction of the 27 gradient / Hessian sums, of SolveAndUpdateSerial or of DepthGradient (DESIGN.md section 7 lists
what still uses local memory)."""
import glob
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
KERNELS = ("_ZN4m3tb8k_track2ILi1024ELb1EEEvNS_9TrackArgsE", "_ZN4m3tb8k_track2ILi1024ELb0EEEvNS_9TrackArgsE")


def _function_lines(path, name):
    """1-based line numbers of the definition of `name` in `path` (signature to matching closing brace)."""
    lines = open(path).read().splitlines()
    for i, line in enumerate(lines):
        if re.search(r"__device__.*\b%s\s*\(" % name, line) or (
                re.match(r"\s*__device__", lines[i - 1] if i else "") and re.search(r"\b%s\s*\(" % name, line)):
            depth, opened = 0, False
            for j in range(i, len(lines)):
                depth += lines[j].count("{") - lines[j].count("}")
                opened = opened or "{" in lines[j]
                if opened and depth == 0:
                    return set(range(i + 1, j + 2))
    raise AssertionError(f"{name} not found in {path}")


def _reduction_lines(path):
    """The recursive-halving step of the warp reduction (send / keep selects and the shuffle)."""
    lines = open(path).read().splitlines()
    hot = set()
    for i, line in enumerate(lines):
        if "__shfl_xor_sync(0xffffffffu, send," in line:
            hot |= {i - 1, i, i + 1}  # the two selects above it and the shuffle line itself
    assert hot, "warp reduction not found"
    return hot


def _local_accesses(so):
    """{kernel: [(file basename, line, opcode)]} for the LDL / STL of the two 1024-thread k_track2 instantiations."""
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
                m = re.search(r"\b(LDL|STL)\b", line)
                if m and fn in KERNELS and loc:
                    found[fn].append(loc + (m.group(1),))
    return found


def test_track2_hot_sections_do_not_touch_local_memory(pkg):
    if not (shutil.which("cuobjdump") and shutil.which("nvdisasm")):
        pytest.skip("cuobjdump / nvdisasm not available")
    pkg._build.build_cuda()  # in-tree nvcc build (cross-compiles for sm_90a without a GPU)
    track2 = os.path.join(CSRC, "m3t_b200_track2.cuh")
    kernels = os.path.join(CSRC, "m3t_b200_kernels.cuh")
    hot = {
        "warp reduction": ("m3t_b200_track2.cuh", _reduction_lines(track2)),
        "SolveAndUpdateSerial": ("m3t_b200_kernels.cuh", _function_lines(kernels, "SolveAndUpdateSerial")),
        "DepthGradient": ("m3t_b200_kernels.cuh", _function_lines(kernels, "DepthGradient")),
    }
    found = _local_accesses(os.path.join(CSRC, "libm3t_b200.so"))
    assert sorted(found) == sorted(KERNELS), sorted(found)
    bad = []
    for kernel, accesses in found.items():
        for f, line, op in accesses:
            for section, (hf, lines) in hot.items():
                if f == hf and line in lines:
                    bad.append(f"{kernel}: {op} at {f}:{line} ({section})")
    assert not bad, "\n".join(bad)
