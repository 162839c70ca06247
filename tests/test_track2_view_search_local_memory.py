"""k_track2<1024, *> keeps its closest-view search (ClosestViewPrunedGroup) out of local memory on sm_90a: the search
sits at the head of every correspondence iteration's dependent chain, and with ~3 KB of L1 next to 225 KB of shared
memory every LDL / STL there is an L2 round trip. Same disassembly as tests/test_track2_local_memory.py."""
import os
import shutil

import pytest

from test_track2_local_memory import CSRC, KERNELS, _function_lines, _local_accesses


def test_track2_view_search_does_not_touch_local_memory(pkg):
    if not (shutil.which("cuobjdump") and shutil.which("nvdisasm")):
        pytest.skip("cuobjdump / nvdisasm not available")
    pkg._build.build_cuda()  # in-tree nvcc build (cross-compiles for sm_90a without a GPU)
    lines = _function_lines(os.path.join(CSRC, "m3t_b200_views.cuh"), "ClosestViewPrunedGroup")
    found = _local_accesses(os.path.join(CSRC, "libm3t_b200.so"))
    assert sorted(found) == sorted(KERNELS), sorted(found)
    bad = [f"{kernel}: {op} at {f}:{line}" for kernel, accesses in found.items() for f, line, op in accesses
           if f == "m3t_b200_views.cuh" and line in lines]
    assert not bad, "\n".join(bad)
