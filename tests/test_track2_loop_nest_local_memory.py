"""k_track2<1024, *> runs its whole correspondence / update loop nest out of registers and shared memory on sm_90a.

With 64 registers per thread and ~3 KB of L1 left next to 225 KB of shared memory, every local-memory access of the
1024-thread kernel is an L2 round trip, and in the loop nest it sits on the dependent chain of every iteration (a
spilled line field before each gradient pass, the depth search state rebuilt in local memory every update iteration).
The test asserts, for both 1024-thread instantiations, that ptxas reports no spill stores or loads (build.log of the
in-tree -Xptxas -v build) and that every LDL / STL left in the shipped library (cuobjdump / nvdisasm -g) maps to a
source line of one of the rare out-of-line paths: the out-of-tile line walk (WalkSlow), the out-of-tile depth search
(DepthSearchSlow) or the large-argument reduction of sinf in the Rodrigues formula (ExpSkew, steps above 0.1 rad)."""
import os
import re
import shutil

import pytest

from test_track2_local_memory import CSRC, KERNELS, _function_lines, _local_accesses


def _ptxas_figures(log):
    """{kernel: (stack frame, spill stores, spill loads)} from the -Xptxas -v output in build.log."""
    text = open(log).read()
    pattern = (r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
               r"(\d+) bytes spill loads")
    return {m.group(1): tuple(int(x) for x in m.groups()[1:]) for m in re.finditer(pattern, text)}


def test_track2_1024_has_no_spills(pkg):
    pkg._build.build_cuda()  # in-tree nvcc build (cross-compiles for sm_90a without a GPU)
    log = os.path.join(CSRC, "build.log")
    if not os.path.exists(log):  # the library was built elsewhere: rebuild here for the ptxas report
        pkg._build.build_cuda(force=True)
    figures = _ptxas_figures(log)
    for kernel in KERNELS:
        assert kernel in figures, f"{kernel}: no ptxas -v report in build.log"
        _, stores, loads = figures[kernel]
        assert (stores, loads) == (0, 0), f"{kernel}: {stores} bytes spill stores, {loads} bytes spill loads"


def test_track2_loop_nest_does_not_touch_local_memory(pkg):
    if not (shutil.which("cuobjdump") and shutil.which("nvdisasm")):
        pytest.skip("cuobjdump / nvdisasm not available")
    pkg._build.build_cuda()
    track2 = os.path.join(CSRC, "m3t_b200_track2.cuh")
    kernels = os.path.join(CSRC, "m3t_b200_kernels.cuh")
    device = os.path.join(CSRC, "m3t_b200_device.cuh")
    source = open(device).read().splitlines()
    sinf_lines = {n for n in _function_lines(device, "ExpSkew") if "sinf(" in source[n - 1]}
    assert sinf_lines, "sinf not found in ExpSkew"
    rare = {
        ("m3t_b200_track2.cuh", n) for n in _function_lines(track2, "WalkSlow")
    } | {
        ("m3t_b200_kernels.cuh", n) for n in _function_lines(kernels, "DepthSearchSlow")
    } | {
        ("m3t_b200_device.cuh", n) for n in sinf_lines
    }
    found = _local_accesses(os.path.join(CSRC, "libm3t_b200.so"))
    assert sorted(found) == sorted(KERNELS), sorted(found)
    bad = [f"{kernel}: {op} at {f}:{line}" for kernel, accesses in found.items() for f, line, op in accesses
           if (f, line) not in rare]
    assert not bad, "\n".join(bad)
