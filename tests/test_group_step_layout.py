"""The ctypes mirror of lsdgpu_group_step (lsd_slam_b200/abi.py) has the C layout of include/lsdgpu.h: a C++ program compiled
against the header prints sizeof and every offsetof, which must equal the ctypes sizes and offsets.  No GPU needed."""
import ctypes
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("ctx", "kf_id", "frame_id", "gray", "stage_index", "frameToRef_init_qt", "settings", "keyframe_change")


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_group_step_matches_c_layout(tmp_path):
    from lsd_slam_b200 import abi
    src = tmp_path / "layout.cpp"
    lines = ['#include <cstddef>', '#include <cstdio>', '#include "lsdgpu.h"', "int main() {",
             '    std::printf("sizeof %zu\\n", sizeof(lsdgpu_group_step));']
    lines += [f'    std::printf("{f} %zu\\n", offsetof(lsdgpu_group_step, {f}));' for f in FIELDS]
    lines += ["    return 0;", "}"]
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    out = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    assert int(out["sizeof"]) == ctypes.sizeof(abi.GroupStep)
    assert [name for name, _ in abi.GroupStep._fields_] == list(FIELDS)
    for f in FIELDS:
        assert int(out[f]) == getattr(abi.GroupStep, f).offset, f
