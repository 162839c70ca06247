"""ctypes binding of pose_score_oracle.cpp, the CPU restatement of the evaluators' pose scoring.

strict(): the -ffp-contract=off build the device results are compared with. native(): -O3 -march=native -fopenmp, the
CPU baseline of scripts/pose_score_timing.py. Both are compiled into a temporary directory, never into the tree.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pose_score_oracle.cpp")
N_CURVE_VALUES = 100
_libs = {}
_FLAGS = {"strict": ["-O2", "-ffp-contract=off", "-fopenmp"], "native": ["-O3", "-march=native", "-fopenmp"]}


def _load(kind):
    if kind in _libs:
        return _libs[kind]
    src = open(_SRC, "rb").read()
    tag = hashlib.sha1(src + " ".join(_FLAGS[kind]).encode()).hexdigest()[:16]
    out = os.path.join(tempfile.gettempdir(), f"m3tb_pose_score_oracle_{kind}_{os.getuid()}_{tag}.so")
    if not os.path.exists(out):
        tmp = out + f".{os.getpid()}"
        subprocess.run(["g++", "-std=c++17", "-fPIC", "-shared", "-Wall"] + _FLAGS[kind] + ["-o", tmp, _SRC], check=True)
        os.replace(tmp, out)
    L = C.CDLL(out)
    vp, ci, cf = C.c_void_p, C.c_int, C.c_float
    L.orc_reduce_vertices.argtypes = [vp, ci, ci, vp]
    L.orc_reduce_vertices.restype = ci
    L.orc_score_pose.argtypes = [vp, ci, vp, ci, vp, vp, vp, cf, cf, cf, cf, cf, vp, vp]
    L.orc_diameter.argtypes = [vp, ci]
    L.orc_diameter.restype = cf
    L.orc_score_poses.argtypes = [ci, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, cf, cf, cf, cf, cf, vp, vp]
    _libs[kind] = L
    return L


def strict():
    return _load("strict")


def native():
    return _load("native")


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return None if a is None else a.ctypes.data


def reduce_vertices(vertices, n_evaluation, lib=None):
    """GenderateReducedVertices: [m, 3] float32."""
    v = _f32(vertices).reshape(-1, 3)
    out = np.zeros((max(len(v), n_evaluation), 3), np.float32)
    m = (lib or strict()).orc_reduce_vertices(_p(v), len(v), int(n_evaluation), _p(out))
    return out[:m]


# defaults of m3tb_score_params_default
YCB = dict(threshold_max=0.1, curve_scale=1.0, auc_scale=1.0)
TRANSLATION_THRESHOLD = np.float32(0.05)
ROTATION_THRESHOLD = np.float32(np.float32(5.0) * np.float32(3.1415926535897) / np.float32(180.0))


def score_pose(reduced, full, body2world, gt, geometry2body=None, threshold_max=0.1, curve_scale=1.0, auc_scale=1.0,
               translation_threshold=TRANSLATION_THRESHOLD, rotation_threshold=ROTATION_THRESHOLD, lib=None):
    """One body: (result[7] in m3tb_pose_score order, add_curve[100], adds_curve[100])."""
    r, f = _f32(reduced).reshape(-1, 3), _f32(full).reshape(-1, 3)
    b, g = _f32(body2world).reshape(12), _f32(gt).reshape(12)
    g2b = None if geometry2body is None else _f32(geometry2body).reshape(12)
    res = np.zeros(7, np.float32)
    curves = np.zeros((2, N_CURVE_VALUES), np.float32)
    (lib or strict()).orc_score_pose(_p(r), len(r), _p(f), len(f), _p(b), _p(g), _p(g2b), threshold_max, curve_scale,
                                     auc_scale, translation_threshold, rotation_threshold, _p(res), _p(curves))
    return res, curves[0], curves[1]


def diameter(vertices, lib=None):
    v = _f32(vertices).reshape(-1, 3)
    return np.float32((lib or strict()).orc_diameter(_p(v), len(v)))


def score_poses(models, model_of_body, body2world, gt, geometry2body=None, threshold_max=0.1, curve_scale=1.0,
                auc_scale=1.0, lib=None):
    """Many bodies at once (OpenMP over bodies). models: list of (reduced, full); returns results [n, 7] and curves
    [n, 2, 100]."""
    reduced = [_f32(r).reshape(-1, 3) for r, _ in models]
    full = [_f32(f).reshape(-1, 3) for _, f in models]
    ro = np.cumsum([0] + [len(r) for r in reduced])[:-1].astype(np.int32)
    fo = np.cumsum([0] + [len(f) for f in full])[:-1].astype(np.int32)
    nr = np.array([len(r) for r in reduced], np.int32)
    nf = np.array([len(f) for f in full], np.int32)
    R, F = np.concatenate(reduced), np.concatenate(full)
    mb = np.ascontiguousarray(model_of_body, np.int32)
    n = len(mb)
    b, g = _f32(body2world).reshape(n, 12), _f32(gt).reshape(n, 12)
    has = np.zeros(n, np.int32) if geometry2body is None else np.ones(n, np.int32)
    g2b = np.zeros((n, 12), np.float32) if geometry2body is None else _f32(geometry2body).reshape(n, 12)
    res = np.zeros((n, 7), np.float32)
    curves = np.zeros((n, 2, N_CURVE_VALUES), np.float32)
    (lib or strict()).orc_score_poses(n, _p(mb), _p(R), _p(ro), _p(nr), _p(F), _p(fo), _p(nf), _p(b), _p(g), _p(g2b),
                                      _p(has), threshold_max, curve_scale, auc_scale, TRANSLATION_THRESHOLD,
                                      ROTATION_THRESHOLD, _p(res), _p(curves))
    return res, curves
