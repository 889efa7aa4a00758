"""The ctypes mirror in tests/ggml_abi.py has the layout of csrc/ggml_abi_mirror.h, byte for byte: a small host program compiled
against the header prints sizeof / offsetof of every field and every enum value, and the ctypes classes must agree.  (The header
itself is static_asserted against the reference headers by oracle/abi_check.cpp.)"""
import os
import shutil
import subprocess
import pytest
import ggml_abi as ga

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ggllm.cpp_b200", "csrc")
STRUCTS = {"tensor_meta": ga.TensorMeta, "tensor": ga.Tensor, "compute_params": ga.ComputeParams}
ENUMS = dict({"BACKEND_CPU": ga.BACKEND_CPU, "BACKEND_GPU": ga.BACKEND_GPU, "BACKEND_GPU_SPLIT": ga.BACKEND_GPU_SPLIT,
              "TASK_INIT": ga.TASK_INIT, "TASK_COMPUTE": ga.TASK_COMPUTE, "TASK_FINALIZE": ga.TASK_FINALIZE,
              "MAX_DIMS": ga.MAX_DIMS, "MAX_OPT": ga.MAX_OPT, "MAX_NAME": ga.MAX_NAME}, **ga.OPS)


def _program():
    lines = ['#include "ggml_abi_mirror.h"', "#include <cstdio>", "int main() {"]
    for cname, cls in STRUCTS.items():
        lines.append('    printf("sizeof %s|%%zu\\n", sizeof(abi::%s));' % (cname, cname))
        for f in cls._fields_:
            lines.append('    printf("%s.%s|%%zu %%zu\\n", offsetof(abi::%s, %s), sizeof(abi::%s::%s));' % (
                cname, f[0], cname, f[0], cname, f[0]))
    for e in ENUMS:
        lines.append('    printf("enum %s|%%d\\n", (int) abi::%s);' % (e, e))
    lines += ["    return 0;", "}"]
    return "\n".join(lines) + "\n"


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler (g++) to compile the layout probe")
def test_ctypes_mirror_matches_the_header_byte_for_byte(tmp_path):
    src, exe = tmp_path / "probe.cpp", tmp_path / "probe"
    src.write_text(_program())
    subprocess.check_call(["g++", "-std=c++17", "-I", CSRC, str(src), "-o", str(exe)])
    got = dict(line.split("|") for line in subprocess.check_output([str(exe)], text=True).splitlines())
    checked = 0
    for cname, cls in STRUCTS.items():
        assert int(got["sizeof " + cname]) == ga.C.sizeof(cls), cname
        for f in cls._fields_:
            off, size = (int(v) for v in got["%s.%s" % (cname, f[0])].split())
            desc = getattr(cls, f[0])
            assert (desc.offset, desc.size) == (off, size), ("%s.%s" % (cname, f[0]), (desc.offset, desc.size), (off, size))
            checked += 1
    for e, v in ENUMS.items():
        assert int(got["enum " + e]) == v, e
    assert checked == 9 + 20 + 5          # every field the header declares
