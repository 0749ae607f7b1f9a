"""CPU: the environment switches the package reads are exactly the ones INTEGRATION.md section 3 documents."""
import os
import re

from conftest import ROOT

PKG = os.path.join(ROOT, "llamagen_b200")


def _files(top, exts):
    for dirpath, _, files in os.walk(top):
        for f in sorted(files):
            if f.endswith(exts):
                yield os.path.join(dirpath, f)


def _read_by_package():
    names = set()
    for path in _files(os.path.join(PKG, "csrc"), (".cu", ".cuh", ".h")):
        names |= set(re.findall(r"\b(?:lg_env_flag|getenv)\s*\(\s*\"(LG_[A-Z0-9_]+)\"", open(path).read()))
    for path in _files(PKG, (".py",)):
        names |= set(re.findall(r"\bos\.(?:environ(?:\.get|\.setdefault|\.pop)?|getenv)\s*[(\[]\s*[\"'](LG_[A-Z0-9_]+)[\"']",
                                open(path).read()))
    return names


def _documented():
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    m = re.search(r"^## 3\..*?(?=^## )", text, flags=re.S | re.M)
    assert m, "INTEGRATION.md has no section 3"
    return set(re.findall(r"LG_[A-Z0-9_]*[A-Z0-9]", m.group(0)))     # also as a build define, -DLG_…


def test_documented_switches_are_the_ones_read():
    read, documented = _read_by_package(), _documented()
    assert {"LG_SPLIT", "LG_GEMM_TC", "LG_LIB_PATH"} <= read      # the scan itself finds C++ and Python reads
    assert read - documented == set(), f"read but not in INTEGRATION.md section 3: {sorted(read - documented)}"
    assert documented - read == set(), f"in INTEGRATION.md section 3 but never read: {sorted(documented - read)}"
