"""ptxas report of k_texture_orb (m3tb_texture_detect_orb): no stack frame and no spills."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "_ZN4m3tb13k_texture_orbENS_10TexOrbArgsE"


def test_orb_kernel_has_no_local_memory(pkg):
    pkg._build.build_cuda()
    log = open(os.path.join(ROOT, "3dobjecttracking_b200", "csrc", "build.log")).read()
    m = re.search(r"Function properties for %s\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % KERNEL, log)
    if m is None:
        pytest.skip("the library was built before this run (no ptxas report in build.log)")
    assert m.groups() == ("0", "0", "0"), m.group(0)
