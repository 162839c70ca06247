"""The C-ABI library loads and exports every symbol include/m3t_b200.h declares (no compute calls: no GPU here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    text = open(os.path.join(ROOT, "include", "m3t_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(m3tb_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(pkg, capi):
    pkg._build.build_cuda()  # in-tree nvcc build (cross-compiles for sm_90a without a GPU)
    lib = ctypes.CDLL(capi.LIB_PATH)
    declared = _header_symbols()
    assert len(declared) >= 35
    missing = [s for s in declared if not hasattr(lib, s)]
    assert not missing, missing
    assert sorted(capi.SYMBOLS) == declared, set(capi.SYMBOLS) ^ set(declared)


def test_defaults_through_the_abi_match_the_oracle(capi, oracle):
    """m3tb_*_params_default (no device needed) == the reference's defaults as restated by the oracle, field by field."""
    r1, r2 = capi.region_params(), oracle.region_params(None)
    for name, _ in r1._fields_:
        a, b = getattr(r1, name), getattr(r2, name)
        assert (list(a) == list(b)) if hasattr(a, "__len__") else (a == b), name
    d1, d2 = capi.depth_params(), oracle.depth_params(None)
    for name, _ in d1._fields_:
        a, b = getattr(d1, name), getattr(d2, name)
        assert (list(a) == list(b)) if hasattr(a, "__len__") else (a == b), name
    op = capi.OptimizerParams()
    capi.lib().m3tb_optimizer_params_default(ctypes.byref(op))
    assert (op.tikhonov_parameter_rotation, op.tikhonov_parameter_translation) == (1000.0, 30000.0)


def test_no_cpu_fallback_without_a_device(capi):
    """On a machine without a usable sm_90 device context creation fails loudly instead of computing on the CPU."""
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a CUDA device is present")
    import pytest
    with pytest.raises(capi.M3TBError):
        capi.Context(0, 1, 1, 1)


def test_cuda_library_contains_sm90a_tma_bulk_copy():
    """The shipped cubin is sm_90a and uses the TMA bulk-copy path (UBLKCP) + mbarrier (SYNCS) for staging."""
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        import pytest
        pytest.skip("cuobjdump not available")
    so = os.path.join(ROOT, "3dobjecttracking_b200", "csrc", "libm3t_b200.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert "UBLKCP" in out and "SYNCS" in out
