"""The ctypes mirrors of the host pipeline's structs (capi.HostScanSpec / HostScanResult) have the C layout of
include/obgpu_pipeline.h: a small C++ program compiled with g++ prints sizeof and offsetof of every field."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest

from oceanbase_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _c_layout(struct_name, fields):
    lines = ['#include <cstddef>', '#include <cstdio>', '#include "obgpu_pipeline.h"', "int main() {",
             f'  printf("sizeof %zu\\n", sizeof({struct_name}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({struct_name}, {f}));' for f in fields]
    lines += ["  return 0;", "}"]
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "layout.cpp"), os.path.join(d, "layout")
        with open(src, "w") as fh:
            fh.write("\n".join(lines) + "\n")
        r = subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-o", exe, src], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout
    return {k: int(v) for k, v in (line.split() for line in out.splitlines())}


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
@pytest.mark.parametrize("struct_name,mirror", [("obgpu_host_scan_spec", capi.HostScanSpec),
                                                ("obgpu_host_scan_result", capi.HostScanResult)])
def test_ctypes_mirror_matches_the_c_layout(struct_name, mirror):
    names = [f[0] for f in mirror._fields_]
    got = _c_layout(struct_name, names)
    assert got["sizeof"] == C.sizeof(mirror)
    for name in names:
        assert got[name] == getattr(mirror, name).offset, name
