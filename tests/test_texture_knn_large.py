"""CPU checks of the large-capacity texture matchers' fixture (tests/golden/make_texture_knn_large.py): the generator
reproduces texture_knn_large.npz byte for byte, the restatements texture_reference.knn2 (NORM_HAMMING) and
texture_reference_l2.knn2_l2 (NORM_L2) reproduce its cv2.BFMatcher results, and so does the vectorised kNN the GPU
tests expand the fixture with; the pinned cases hold (0 / 0 across a 512-row chunk boundary keeps the earlier row, equal
distances keep the first two rows). Also: the texture kernels the capacity reaches compile for sm_90a without local
memory."""
import filecmp
import importlib.util
import os
import re

import numpy as np
import pytest

import texture_knn_sets
import texture_reference as tr
import texture_reference_l2 as tr2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
GOLDEN = os.path.join(GOLDEN_DIR, "texture_knn_large.npz")
SYN = [(kind, n) for kind in ("ham", "l2") for n in texture_knn_sets.SIZES]
_POPCOUNT = np.array([bin(v).count("1") for v in range(256)], np.int64)


def knn2(queries, train, hamming):
    """cv::BFMatcher knnMatch(k = 2) as (idx [n, 2], dist [n, 2]) with -1 where there is no neighbour: the two first
    train rows under (distance, index) order, which is what OpenCV's strict-less insertion in index order keeps.
    Hamming: bit counts of 32-byte rows; L2: whole-number rows, the exact int64 sum rounded to float32, then sqrt."""
    q, t = np.asarray(queries), np.asarray(train)
    idx = np.full((len(q), 2), -1, np.int32)
    dist = np.full((len(q), 2), -1.0, np.float32)
    if len(t) == 0:
        return idx, dist
    for s in range(0, len(q), 128):
        qs = q[s:s + 128]
        if hamming:
            d = _POPCOUNT[np.bitwise_xor(qs[:, None, :].astype(np.uint8), t[None, :, :].astype(np.uint8))].sum(-1)
            d = d.astype(np.float32)
        else:
            diff = qs[:, None, :].astype(np.int64) - t[None, :, :].astype(np.int64)
            d = np.sqrt((diff * diff).sum(-1).astype(np.float32))
        order = np.argsort(d, axis=1, kind="stable")[:, :2]
        k = order.shape[1]
        idx[s:s + 128, :k] = order
        dist[s:s + 128, :k] = np.take_along_axis(d, order, 1)
    return idx, dist


def ratio_keep(idx, dist, threshold=np.float32(0.7)):
    """CalculateCorrespondences' ratio test: a second neighbour, and d0 / d1 not >= threshold (0 / 0 keeps)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return (idx[:, 1] >= 0) & ~(dist[:, 0] / dist[:, 1] >= threshold)


def sift_pair(z, k):
    """(queries, train, idx, dist) of sift_pairs[k], descriptors as float32."""
    a, b = z["sift_pairs"][k]
    crops = list(z["sift_crops"])
    rows = lambda c: z["sift_desc"][z["sift_offset"][crops.index(c)]:][:z["sift_n"][c]].astype(np.float32)
    first = int(sum(z["sift_n"][z["sift_pairs"][j][0]] for j in range(k)))
    n = int(z["sift_n"][a])
    return rows(a), rows(b), z["sift_idx"][first:first + n], z["sift_dist"][first:first + n]


def test_generator_reproduces_the_fixture(tmp_path):
    pytest.importorskip("cv2")
    spec = importlib.util.spec_from_file_location("make_texture_knn_large",
                                                  os.path.join(GOLDEN_DIR, "make_texture_knn_large.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.main(str(tmp_path))
    assert filecmp.cmp(str(tmp_path / "texture_knn_large.npz"), GOLDEN, shallow=False)


def test_sift_sets_are_untruncated_whole_numbers():
    z = np.load(GOLDEN)
    assert z["sift_desc"].dtype == np.uint8 and z["sift_desc"].shape == (z["sift_n"][z["sift_crops"]].sum(), 128)
    assert z["sift_n"][3] == 2339 and set(z["sift_pairs"].ravel()) <= set(z["sift_crops"])
    assert z["sift_n"].max() == 2339 and (z["sift_n"] > 512).sum() == 5
    assert len(z["sift_idx"]) == sum(z["sift_n"][a] for a, _ in z["sift_pairs"])


@pytest.mark.parametrize("k", range(3))
def test_sift_pairs_match_the_restatement(k):
    z = np.load(GOLDEN)
    q, t, ref_idx, ref_dist = sift_pair(z, k)
    idx, dist = knn2(q, t, False)
    assert np.array_equal(idx, ref_idx) and np.array_equal(dist.view(np.uint32), ref_dist.view(np.uint32))
    for i, m in zip(range(0, len(q), 97), tr2.knn2_l2(q[::97], t)):  # the loop restatement on a sample of queries
        assert [j for j, _ in m] == [j for j in ref_idx[i] if j >= 0]
        assert np.array_equal(np.array([d for _, d in m], np.float32), ref_dist[i][ref_idx[i] >= 0])


def test_orb_4096_matches_the_restatement():
    z = np.load(GOLDEN)
    q, t = z["orb_queries"], z["orb_train"]
    assert q.shape == t.shape == (4096, 32)
    idx, dist = knn2(q, t, True)
    assert np.array_equal(idx, z["orb_idx"]) and np.array_equal(dist, z["orb_dist"])
    for i, m in zip(range(0, 4096, 257), tr.knn2(q[::257], t)):
        assert [(j, float(d)) for j, d in m] == [(int(j), float(d)) for j, d in zip(z["orb_idx"][i], z["orb_dist"][i])]
    assert 100 < ratio_keep(idx, dist).sum() < 4096


@pytest.mark.parametrize("kind,n", SYN)
def test_synthetic_sets(kind, n):
    z = np.load(GOLDEN)
    key = "syn_%s_%d" % (kind, n)
    hamming = kind == "ham"
    q, t = texture_knn_sets.synthetic(n, hamming)
    ref_idx, ref_dist = z[key + "_idx"], z[key + "_dist"]
    assert len(t) == n
    idx, dist = knn2(q, t, hamming)
    assert np.array_equal(idx, ref_idx) and np.array_equal(dist.view(np.uint32), ref_dist.view(np.uint32))
    loop = tr.knn2(q, t) if hamming else tr2.knn2_l2(q.astype(np.float32), t.astype(np.float32))
    for i, m in enumerate(loop):
        assert [j for j, _ in m] == list(ref_idx[i]), i
    keep = ratio_keep(idx, dist)
    assert tuple(idx[-1]) == (3, 10)  # equal distances: the first two marked rows
    assert dist[-1, 0] == dist[-1, 1] and not keep[-1]
    if n > 512:  # rows n - 513 and n - 1 are equal
        assert tuple(idx[-3]) == tuple(idx[-2]) == (n - 513, n - 1)
        assert dist[-3, 0] == dist[-3, 1] == 0 and keep[-3]  # 0 / 0 keeps the earlier row
        assert dist[-2, 0] == dist[-2, 1] > 0 and not keep[-2]


KERNELS = ("_ZN4m3tb16k_texture_knn_l2ENS_11TextureArgsE", "_ZN4m3tb21k_texture_knn_hammingENS_11TextureArgsE",
           "_ZN4m3tb15k_texture_matchENS_11TextureArgsE", "_ZN4m3tb18k_texture_keyframeENS_11TextureArgsE",
           "_ZN4m3tb18k_texture_featuresENS_11TexFeatArgsE")


@pytest.mark.parametrize("kernel", KERNELS)
def test_texture_kernels_have_no_local_memory(pkg, kernel):
    pkg._build.build_cuda()
    log = open(os.path.join(ROOT, "3dobjecttracking_b200", "csrc", "build.log")).read()
    m = re.search(r"Function properties for %s\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads" % kernel, log)
    if m is None:
        pytest.skip("the library was built before this run (no ptxas report in build.log)")
    assert m.groups() == ("0", "0", "0"), m.group(0)
