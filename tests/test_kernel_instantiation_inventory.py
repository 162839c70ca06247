"""Every tracking kernel the library compiles has a GPU case that runs it, and every such case names a kernel that
exists (no GPU needed). The instantiations are read from the sources: the M3TB_TRACK_GROUP_* lists of
m3t_b200_track_variants.h (k_track<T, K, LUT_SMEM, OCC, CLUSTER>) and the explicit k_track2<T, LUT_SMEM> instantiations
of m3t_b200_track2_*.cu. Each becomes the tuple m3tb_debug_last_launch reports for it, (kernel, threads,
items_per_thread, lut_smem, occ), and the set must equal the keys of test_gpu_kernel_instantiations.COVERAGE, whose
cases assert exactly that launch."""
import glob
import os
import re

from test_gpu_kernel_instantiations import CASES, COVERAGE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")

_B = r"\s*(true|false)\s*"
_X = re.compile(r"X\(\s*(\d+)\s*,\s*(\d+)\s*," + _B + "," + _B + "," + _B + r"\)")
_K2 = re.compile(r"template\s+__global__\s+void\s+k_track2<\s*(\d+)\s*," + _B + ">")


def _read(path):
    with open(path) as f:
        return f.read()


def _k_track_groups():
    """{group number: [(T, K, LUT_SMEM, OCC, CLUSTER)]} of m3t_b200_track_variants.h."""
    text = _read(os.path.join(CSRC, "m3t_b200_track_variants.h"))
    joined = text.replace("\\\n", " ")
    groups = {}
    for line in joined.splitlines():
        m = re.match(r"\s*#define\s+M3TB_TRACK_GROUP_(\d+)\(X\)(.*)", line)
        if m:
            groups[int(m.group(1))] = [(int(t), int(k), l == "true", o == "true", c == "true")
                                       for t, k, l, o, c in _X.findall(m.group(2))]
    # an X(...) outside the group lists would not be compiled where this test looks for it
    assert len(_X.findall(text)) == sum(len(v) for v in groups.values()), "X(...) entry outside M3TB_TRACK_GROUP_*"
    return groups, joined


def compiled_instantiations():
    """The set of launch tuples of every compiled k_track / k_track2 instantiation."""
    groups, header = _k_track_groups()
    assert groups, "no M3TB_TRACK_GROUP_* in m3t_b200_track_variants.h"
    # every group is in M3TB_TRACK_ALL (declared in m3t_b200.cu) and instantiated by exactly one translation unit
    m = re.search(r"#define\s+M3TB_TRACK_ALL\(X\)(.*)", header)
    assert m and sorted(int(g) for g in re.findall(r"M3TB_TRACK_GROUP_(\d+)\(X\)", m.group(1))) == sorted(groups)
    units = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "m3t_b200_track_*.cu"))):
        for g in re.findall(r"^M3TB_TRACK_GROUP_(\d+)\(M3TB_INSTANTIATE\)", _read(path), re.M):
            units.setdefault(int(g), []).append(os.path.basename(path))
    assert {g: len(u) for g, u in units.items()} == {g: 1 for g in groups}, units
    out = []
    for entries in groups.values():
        for t, k, lut, occ, cluster in entries:
            out.append(("k_track_cluster" if cluster else "k_track", t, k, int(lut), int(occ)))
    k2 = []
    for path in sorted(glob.glob(os.path.join(CSRC, "m3t_b200_track2_*.cu"))):
        k2 += [("k_track2", int(t), 1, int(lut == "true"), 0) for t, lut in _K2.findall(_read(path))]
    assert k2, "no k_track2 instantiation found"
    out += k2
    assert len(out) == len(set(out)), sorted(v for v in out if out.count(v) > 1)
    return set(out)


def test_every_instantiation_has_a_case_and_every_case_an_instantiation():
    compiled = compiled_instantiations()
    covered = set(COVERAGE)
    assert not compiled - covered, f"instantiations without a GPU case: {sorted(compiled - covered)}"
    assert not covered - compiled, f"COVERAGE rows without an instantiation: {sorted(covered - compiled)}"
    assert len(compiled) == 24, len(compiled)   # 4 x k_track2, 16 x k_track, 4 x cluster-fused k_track


def test_coverage_names_each_case_once():
    """Every case of test_gpu_kernel_instantiations sits in exactly one COVERAGE row (the launch it asserts), and every
    case a row names exists."""
    listed = [c for cases in COVERAGE.values() for c in cases]
    assert all(COVERAGE.values()), [v for v, cases in COVERAGE.items() if not cases]
    assert len(listed) == len(set(listed)), sorted(c for c in listed if listed.count(c) > 1)
    assert sorted(listed) == sorted(CASES), (sorted(set(listed) - set(CASES)), sorted(set(CASES) - set(listed)))
