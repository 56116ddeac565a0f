"""Builds tests/cpp/test_dynamic.cpp (the fuzz target's Add / Remove loop through the C++ mirror include/bvh_b200.hpp) with g++,
links libbvh_b200.so, and runs it on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    exe = os.path.join(out_dir, "test_dynamic")
    lib_dir = os.path.join(ROOT, "bvh_b200")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "test_dynamic.cpp"),
                    "-L", lib_dir, "-lbvh_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe], check=True)
    return exe


def test_cpp_dynamic_mirror_compiles_and_links(tmp_path):
    assert os.path.exists(_build(str(tmp_path)))


@pytest.mark.gpu
def test_cpp_fuzz_add_remove_loop(tmp_path):
    r = subprocess.run([_build(str(tmp_path))], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "dynamic add/remove through the C++ mirror passed" in r.stdout
