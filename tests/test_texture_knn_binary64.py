"""CPU checks of the BRISK / FREAK (64-byte NORM_HAMMING) texture matcher: the fixture generator
(tests/golden/make_texture_knn_binary64.py) reproduces texture_knn_binary64.npz byte for byte, the restatements
(tests/texture_reference_binary64.py, vectorised and as the row-by-row insertion) reproduce cv2.BFMatcher(NORM_HAMMING)
exactly, k_texture_knn_hamming compiles for sm_90a without local memory, and the C++ mirror's TextureModality::SetUp
takes BRISK and FREAK while it still refuses ORB_CUDA."""
import filecmp
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

import texture_reference as tr
import texture_reference_binary64 as tb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
GOLDEN = os.path.join(GOLDEN_DIR, "texture_knn_binary64.npz")
SETS = ("brisk", "brisk_large", "orb_brisk", "ties", "zero_zero", "equal_distance", "train_of_one", "empty_train",
        "float_patterns")


def test_generator_reproduces_the_fixture(tmp_path):
    pytest.importorskip("cv2")
    spec = importlib.util.spec_from_file_location("make_texture_knn_binary64",
                                                  os.path.join(GOLDEN_DIR, "make_texture_knn_binary64.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.main(str(tmp_path))
    assert filecmp.cmp(str(tmp_path / "texture_knn_binary64.npz"), GOLDEN, shallow=False)


@pytest.mark.parametrize("name", SETS)
def test_restatement_is_exact(name):
    z = np.load(GOLDEN)
    q, t = z[name + "_queries"], z[name + "_train"]
    assert q.dtype == np.uint8 and q.shape[1] == 64 and t.shape[1] == 64
    idx, dist = tb.knn2(q, t)
    assert np.array_equal(idx, z[name + "_idx"])
    assert np.array_equal(dist.view(np.uint32), z[name + "_dist"].view(np.uint32))
    if len(q) * len(t) <= 512 * 512:  # the row-by-row insertion
        loop = tb.knn2_insertion(q, t)
        assert [[j for j, _ in m] for m in loop] == [[j for j in r if j >= 0] for r in idx.tolist()]
    if name == "brisk":
        assert len(q) <= 512 and len(t) <= 512 and 20 < tb.kept(idx, dist, 0.7).sum() < len(q)
    if name == "brisk_large":
        assert len(t) > 3 * 512 and (idx[:, 0] >= 512).any()
    if name == "ties":
        assert (idx[:, 0] != 40).all() and (idx == 10).any()
    if name == "zero_zero":
        assert tuple(idx[3]) == (70, 71) and dist[3, 0] == dist[3, 1] == 0 and tb.kept(idx, dist, 0.7)[3]
    if name == "equal_distance":
        assert tuple(idx[0]) == (0, 1) and dist[0, 0] == dist[0, 1] == 1
    if name == "float_patterns":
        words = q.view(np.uint32)
        assert (words == 0xFFFFFFFF).all(1).any() and np.isnan(words.view(np.float32)).any()
        assert np.isinf(words.view(np.float32)).any() and tb.kept(idx, dist, 0.7).sum() >= 30


def test_match_ratio_test_and_small_train_sets():
    z = np.load(GOLDEN)
    q, t = z["zero_zero_queries"], z["zero_zero_train"]
    pts = np.arange(3 * len(q), dtype=np.float32).reshape(-1, 3)
    xy = np.arange(2 * len(t), dtype=np.float32).reshape(-1, 2)
    cb, cc = tb.match([(pts, q)], xy, t, 0.7)
    keep = tb.kept(z["zero_zero_idx"], z["zero_zero_dist"], 0.7)
    assert keep[3] and len(cb) == keep.sum() > 0  # 0 / 0 keeps query 3
    assert np.array_equal(cb, pts[keep]) and np.array_equal(cc, xy[z["zero_zero_idx"][keep, 0]])
    for name in ("train_of_one", "empty_train"):
        cb, _ = tb.match([(pts[:8], z[name + "_queries"])], xy[:1], z[name + "_train"], 0.7)
        assert len(cb) == 0


def test_orb_rows_agree_with_the_orb_restatement():
    """On 32-byte ORB rows the restatement here gives what tests/texture_reference.py's knn2 gives."""
    rng = np.random.default_rng(3)
    q = rng.integers(0, 256, (40, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (70, 32), dtype=np.uint8)
    idx, _ = tb.knn2(q, t)
    assert [[j for j, _ in m] for m in tr.knn2(q, t)] == idx.tolist()


def test_knn_hamming_kernel_has_no_local_memory(pkg):
    pkg._build.build_cuda()
    log = open(os.path.join(ROOT, "3dobjecttracking_b200", "csrc", "build.log")).read()
    m = re.search(r"Function properties for _ZN4m3tb21k_texture_knn_hammingENS_11TextureArgsE\n\s*(\d+) bytes stack "
                  r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    if m is None:
        pytest.skip("the library was built before this run (no ptxas report in build.log)")
    assert m.groups() == ("0", "0", "0"), m.group(0)


def test_cpp_mirror_set_up_takes_brisk_and_freak(pkg, tmp_path):
    """examples/texture_binary64_mirror_selftest.cpp: plain g++ build against libm3t_b200.so, run with or without a GPU."""
    pkg._build.build_cuda()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    exe = str(tmp_path / "texture_binary64_mirror_selftest")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"),
           os.path.join(ROOT, "examples", "texture_binary64_mirror_selftest.cpp"), "-o", exe, "-L", csrc, "-lm3t_b200",
           "-Wl,-rpath," + csrc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.stdout, r.stderr[-3000:])
    assert '"failures": 0' in r.stdout
    # the descriptor type passes SetUp's first check; the renderer that is not set up stops it
    for name in ("brisk", "freak"):
        assert "Modality %s: DescriptorType" % name not in r.stderr
    assert "Modality orb_cuda: DescriptorType::ORB_CUDA is not implemented" in r.stderr
    assert "Modality brisk: one 64-byte BRISK descriptor per keypoint" in r.stderr
