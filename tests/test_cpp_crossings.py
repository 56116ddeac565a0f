"""Builds tests/cpp/test_crossings.cpp (Bvh<T>::count_hits, contains and signed_distance of the C++ host mirror include/bvh_b200.hpp
on a fixed cube) with g++, links libbvh_b200.so, and runs it on the GPU.  The executable goes to a temporary directory: the source tree may be read-only."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    exe = os.path.join(out_dir, "test_crossings")
    lib_dir = os.path.join(ROOT, "bvh_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "test_crossings.cpp"),
           "-L", lib_dir, "-lbvh_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe]
    subprocess.run(cmd, check=True)
    return exe


def test_cpp_crossings_compiles_and_links(tmp_path):
    assert os.path.exists(_build(str(tmp_path)))


@pytest.mark.gpu
def test_cpp_crossings_fixed_scenes(tmp_path):
    r = subprocess.run([_build(str(tmp_path))], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all crossing tests passed" in r.stdout
