"""Conventions of the C++ mirror's device ORB detection that need no device (examples/texture_orb_mirror_selftest.cpp):
plain g++ build against libm3t_b200.so, run on this machine (with or without a GPU)."""
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_orb_detection_mirror_conventions_without_device(pkg, tmp_path):
    pkg._build.build_cuda()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    exe = str(tmp_path / "texture_orb_mirror_selftest")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"),
           os.path.join(ROOT, "examples", "texture_orb_mirror_selftest.cpp"), "-o", exe, "-L", csrc, "-lm3t_b200",
           "-Wl,-rpath," + csrc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert r.returncode == 0 and out["failures"] == 0, r.stdout[-2000:]
