"""The compiled-language host mirror (include/laser_b200.hpp): the reference's own GEMM self-tests
re-stated in C++ (tests/cpp_host/reference_selftests.cpp) compile and link on CPU and pass on the GPU."""
import os
import subprocess

import pytest

import laser_b200 as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp_host", "reference_selftests.cpp")


CONV_SRC = os.path.join(ROOT, "tests", "cpp_host", "conv_selftests.cpp")


def build(tmp_path, src=SRC):
    exe = str(tmp_path / os.path.splitext(os.path.basename(src))[0])
    libdir = os.path.dirname(L.lib_path())
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src,
                           "-o", exe, "-L", libdir, "-llaser_b200", "-Wl,-rpath," + libdir])
    return exe


def test_cpp_mirror_compiles_and_links(tmp_path):
    out = subprocess.run([build(tmp_path), "--link-only"], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and out.stdout.startswith("laser_b200")


@pytest.mark.gpu
def test_reference_selftests_in_cpp(tmp_path):
    out = subprocess.run([build(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("SUCCESS") == 12


def test_cpp_layers_mirror_compiles_and_links(tmp_path):
    out = subprocess.run([build(tmp_path, CONV_SRC), "--link-only"], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and out.stdout.strip().endswith("workspace 243"), out.stdout + out.stderr


@pytest.mark.gpu
def test_conv_selftests_in_cpp(tmp_path):
    out = subprocess.run([build(tmp_path, CONV_SRC)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert out.stdout.count("SUCCESS") == 3
