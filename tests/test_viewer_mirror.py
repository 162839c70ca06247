"""The C++ mirror's viewers (FullNormalRenderer, NormalColorViewer, NormalDepthViewer, Tracker::AddViewer /
UpdateViewers): the example driver's viewer mode compiles as plain C++17 (CPU), and on the GPU the overlays written by
Tracker::UpdateViewers are the bytes of the same viewers set up through the C ABI."""
import json
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3dobjecttracking_b200")


def test_viewer_mode_compiles_as_cpp17():
    if shutil.which("g++") is None:
        pytest.skip("no host C++ compiler")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(PKG, "host"), "-I", os.path.join(PKG, "synth"),
                    os.path.join(ROOT, "examples", "run_synthetic_tracker.cpp")], check=True)


@pytest.mark.gpu
def test_tracker_update_viewers_writes_the_c_abi_bytes(pkg):
    exe = pkg._build.build_host_example()
    d = tempfile.mkdtemp()
    try:
        out = subprocess.run([exe, "3", "200", "200", "2", "1", "1", "0", d], capture_output=True, text=True, check=True)
        r = json.loads(out.stdout)
        assert r["viewers_equal_c_abi"] is True
        for name in ("color_viewer.ppm", "depth_viewer.ppm"):
            with open(os.path.join(d, name), "rb") as f:
                data = f.read()
            assert data.startswith(b"P6\n640 480\n255\n") and len(data) == len(b"P6\n640 480\n255\n") + 640 * 480 * 3
    finally:
        shutil.rmtree(d, ignore_errors=True)
