"""CPU tests: the C-ABI library builds for sm_90a, loads without a GPU and exports every symbol include/*.h declares."""
import ctypes
import os
import re
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(header):
    txt = open(os.path.join(ROOT, "include", header)).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b((?:b200|ggml)_[a-z0-9_]+)\s*\(", txt)))


@pytest.fixture(scope="module")
def lib():
    import ggllm_cpp_b200.binding as b
    if not os.path.exists(b.LIB_PATH):
        b.build()
    return ctypes.CDLL(b.LIB_PATH)


def test_exports_every_declared_symbol(lib):
    names = _declared("ggml_b200.h")
    assert len(names) > 40
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_cuda_surface_exports(lib):
    path = os.path.join(ROOT, "include", "ggml_b200_cuda_surface.h")
    if not os.path.exists(path):
        pytest.skip("surface header not written yet")
    names = [n for n in _declared("ggml_b200_cuda_surface.h") if n.startswith("ggml_")]
    assert len(names) >= 20
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_binding_lists_match_header():
    import ggllm_cpp_b200.binding as b
    assert sorted(b.PART_A + b.PART_B) == _declared("ggml_b200.h")


def test_no_gpu_means_loud_failure_not_fallback(lib):
    import ggllm_cpp_b200.binding as b
    lib.b200_device_count.restype = ctypes.c_int
    if lib.b200_device_count() > 0:
        pytest.skip("a GPU is visible here")
    with pytest.raises(RuntimeError):
        b.init(0)


def test_sass_is_sm90a_with_tma(lib):
    """the shipped cubin targets sm_90a only and the mat-vec stages activations with a bulk (TMA) copy"""
    import subprocess
    import ggllm_cpp_b200.binding as b
    out = subprocess.run(["cuobjdump", "-lelf", b.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out
    # one disassembly pass: the mat-vec stages activations with a TMA bulk copy; the tensor-core paths are really in the binary: wgmma
    # (prompt GEMM / attention), TMA tensor loads, and the warp-level mma.sync + cp.async rings of the long-context decode attention
    p = subprocess.Popen(["cuobjdump", "-sass", b.LIB_PATH], stdout=subprocess.PIPE, text=True)
    counts = dict.fromkeys(("UBLKCP", "HGMMA", "UTMALDG", "HMMA", "LDGSTS", "IDP.4A"), 0)
    for line in p.stdout:
        for op in counts:
            if op in line:
                counts[op] += 1
    p.wait()
    assert all(v > 0 for v in counts.values()), counts
