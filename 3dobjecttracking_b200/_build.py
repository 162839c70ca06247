"""In-tree builds: the CUDA C-ABI library (sm_90a) and the synthetic-data helper library."""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    # IEEE single-rounding arithmetic in the order written: keeps control flow (int truncations, line
    # validity) bit-identical to the reference restatement (DESIGN.md "Numerics").
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v",
    "-t", "0",  # the translation units (k_track variant groups) compile in parallel
]


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def _stale(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def build_synth(force=False):
    src = os.path.join(_HERE, "synth", "m3t_synth.cpp")
    hdr = os.path.join(_HERE, "synth", "m3t_synth.h")
    out = os.path.join(_HERE, "synth", "libm3t_synth.so")
    if force or _stale(out, [src, hdr]):
        subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-o", out, src], check=True)
    return out


def cuda_sources():
    d = os.path.join(_HERE, "csrc")
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith((".cu", ".cuh", ".h")))


def build_cuda(force=False, verbose=False):
    """nvcc -> 3dobjecttracking_b200/csrc/libm3t_b200.so (cross-compiles without a GPU)."""
    d = os.path.join(_HERE, "csrc")
    out = os.path.join(d, "libm3t_b200.so")
    srcs = [s for s in cuda_sources() if s.endswith(".cu")]
    deps = cuda_sources() + [os.path.join(_ROOT, "include", "m3t_b200.h")]
    if force or _stale(out, deps):
        cmd = ([_nvcc()] + NVCC_FLAGS + os.environ.get("M3TB_EXTRA_NVCC_FLAGS", "").split() +
               ["-I", os.path.join(_ROOT, "include"), "-o", out] + srcs)
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(os.path.join(d, "build.log"), "w") as f:
            f.write(" ".join(cmd) + "\n" + log)
        if verbose or r.returncode != 0:
            print(log)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed; see " + os.path.join(d, "build.log"))
    return out


def build_host_example(force=False):
    """g++ build of the C++ mirror's example driver (examples/run_synthetic_tracker.cpp) against the two in-tree
    libraries; proves that the header-only host mirror compiles as plain C++17 without CUDA headers."""
    src = os.path.join(_ROOT, "examples", "run_synthetic_tracker.cpp")
    hdr = os.path.join(_HERE, "host", "m3t_b200", "m3t_b200.hpp")
    out = os.path.join(_ROOT, "examples", "run_synthetic_tracker")
    csrc = os.path.join(_HERE, "csrc")
    synth = os.path.join(_HERE, "synth")
    if force or _stale(out, [src, hdr, os.path.join(csrc, "libm3t_b200.so"), os.path.join(synth, "libm3t_synth.so")]):
        cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(_ROOT, "include"), "-I", os.path.join(_HERE, "host"),
               "-I", synth, src, "-o", out, "-L", csrc, "-L", synth, "-lm3t_b200", "-lm3t_synth",
               "-Wl,-rpath," + csrc, "-Wl,-rpath," + synth, "-fopenmp"]
        subprocess.run(cmd, check=True)
    return out


def build_pose_scoring_example(force=False):
    """g++ build of examples/pose_scoring_selftest.cpp: the mirror's EvaluationModel and evaluators as plain C++17."""
    src = os.path.join(_ROOT, "examples", "pose_scoring_selftest.cpp")
    hdr = os.path.join(_HERE, "host", "m3t_b200", "m3t_b200.hpp")
    out = os.path.join(_ROOT, "examples", "pose_scoring_selftest")
    csrc = os.path.join(_HERE, "csrc")
    if force or _stale(out, [src, hdr, os.path.join(csrc, "libm3t_b200.so")]):
        subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(_ROOT, "include"), "-I",
                        os.path.join(_HERE, "host"), src, "-o", out, "-L", csrc, "-lm3t_b200", "-Wl,-rpath," + csrc],
                       check=True)
    return out


def build_all(force=False, verbose=False):
    a, b = build_synth(force), build_cuda(force, verbose)
    return a, b, build_host_example(force), build_pose_scoring_example(force)
