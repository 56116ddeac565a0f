"""Builds tests/cpp/test_triangle_pairs.cpp (Bvh<T>::triangle_pairs and triangle_pairs_with of the C++ host mirror include/bvh_b200.hpp
on two fixed tetrahedra) with g++, links libbvh_b200.so, and runs it on the GPU.  The executable goes to a temporary directory: the
source tree may be read-only."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    exe = os.path.join(out_dir, "test_triangle_pairs")
    lib_dir = os.path.join(ROOT, "bvh_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "test_triangle_pairs.cpp"),
           "-L", lib_dir, "-lbvh_b200", f"-Wl,-rpath,{lib_dir}", "-o", exe]
    subprocess.run(cmd, check=True)
    return exe


def test_cpp_triangle_pairs_compiles_and_links(tmp_path):
    assert os.path.exists(_build(str(tmp_path)))


@pytest.mark.gpu
def test_cpp_triangle_pairs_tetrahedra(tmp_path):
    r = subprocess.run([_build(str(tmp_path))], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all triangle pair tests passed" in r.stdout
