"""CPU tests: the environment switches the library reads are exactly the ones INTEGRATION.md section 4 documents, and every switch a
test sets still exists -- a test that sets a name the library no longer reads would quietly test the default kernel instead."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ggllm.cpp_b200", "csrc")
HEADER_MACROS = {"B200_SURFACE_TYPES_ONLY", "B200_H"}      # GGML_B200_SURFACE_TYPES_ONLY / GGML_B200_H: include guards, not switches


def _sources():
    paths = []
    for ext in ("cu", "cuh", "h", "cpp", "c"):
        paths += glob.glob(os.path.join(CSRC, "*." + ext))
    assert paths
    return {p: open(p).read() for p in sorted(paths)}


def _read_names():
    return {n for txt in _sources().values() for n in re.findall(r'\bgetenv\(\s*"([^"]*)"\s*\)', txt)}


def _documented_names():
    txt = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    m = re.search(r"^## 4\. Environment switches\n(.*?)(?=^## )", txt, flags=re.S | re.M)
    assert m, "INTEGRATION.md has no section 4"
    return set(re.findall(r"^- `([A-Z][A-Z0-9_]*)(?:=[^`]*)?`", m.group(1), flags=re.M))


def test_documented_switches_are_the_ones_read():
    read, documented = _read_names(), _documented_names()
    assert read, "no getenv literal found"
    assert read == documented, {"read, not documented": sorted(read - documented), "documented, not read": sorted(documented - read)}


def test_every_getenv_takes_a_literal():
    bad = []
    for path, txt in _sources().items():
        for m in re.finditer(r"\bgetenv\(", txt):
            if not re.match(r'\s*"[^"]*"\s*\)', txt[m.end():]):
                bad.append("%s:%d" % (os.path.basename(path), txt.count("\n", 0, m.start()) + 1))
    assert not bad, bad


def test_tests_name_only_existing_switches():
    read = _read_names()
    unknown = {}
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "*.py"))):
        for name in set(re.findall(r"B200_[A-Z0-9_]+", open(path).read())) - HEADER_MACROS - read:
            unknown.setdefault(name, []).append(os.path.basename(path))
    assert not unknown, unknown
