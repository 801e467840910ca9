"""The C ABI is usable from plain C: include/laser_b200.h compiles as C11 with -Wall -Werror,
links against the in-tree library (CPU), and a C caller reproduces the reference's known
answers on the GPU (the stand-in for the Nim call site, see tests/c_harness/gemm_harness.c)."""
import os
import subprocess

import pytest

import laser_b200 as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "c_harness", "gemm_harness.c")


THREADS_SRC = os.path.join(ROOT, "tests", "c_harness", "threads_harness.c")


def build(tmp_path, src=SRC, name="gemm_harness", lib=None):
    """lib: link against this shared library by path instead of the in-tree liblaser_b200.so (the host-emulated build)"""
    exe = str(tmp_path / name)
    libdir = os.path.dirname(lib or L.lib_path())
    link = [lib] if lib else ["-L", libdir, "-llaser_b200"]
    subprocess.check_call(["/usr/bin/gcc", "-std=c11", "-O2", "-Wall", "-Werror", "-pthread", "-I", os.path.join(ROOT, "include"), src,
                           "-o", exe] + link + ["-lm", "-Wl,-rpath," + libdir])
    return exe


def test_header_is_valid_c_and_links(tmp_path):
    exe = build(tmp_path)
    out = subprocess.run([exe, "--link-only"], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0 and "version" in out.stdout


@pytest.mark.gpu
def test_c_caller_on_gpu(tmp_path):
    exe = build(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "max relative error" in out.stdout


def test_multi_gpu_harness_compiles_as_c(tmp_path):
    build(tmp_path, os.path.join(ROOT, "tests", "c_harness", "rowshard_harness.c"), "rowshard_harness")


@pytest.mark.gpu
def test_c_caller_row_shards_over_two_gpus(tmp_path):
    """laser_b200_gemm_rowsharded_f32 from plain C on 2 (and, when present, 4) GPUs of this box: NCCL bound at run time"""
    torch = pytest.importorskip("torch")
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    exe = build(tmp_path, os.path.join(ROOT, "tests", "c_harness", "rowshard_harness.c"), "rowshard_harness")
    env = dict(os.environ)
    nccl_dir = os.path.join(os.path.dirname(torch.__file__), "..", "nvidia", "nccl", "lib")
    if os.path.isdir(nccl_dir):      # a plain C process: point the loader at the NCCL torch ships if the system has none
        env["LD_LIBRARY_PATH"] = env.get("LD_LIBRARY_PATH", "") + ":" + os.path.abspath(nccl_dir)
    for g in ([2, 4] if n >= 4 else [2]):
        out = subprocess.run([exe, str(g)], capture_output=True, text=True, timeout=600, env=env)
        assert out.returncode == 0, out.stdout + out.stderr
        assert "max error relative" in out.stdout


def test_concurrent_callers_host_logic(tmp_path):
    """SURVEY.md 8(b) "Threading": four threads issue a mix of products (exact kernel, tensor cores, fp64, int64, host and
    device entries) at once and every result must be bit-identical to the serial run.  Here against the host-emulated
    build of capi.cu (tests/emu/: kernels run one at a time on the one emulated device, the host code around them --
    context creation, workspace growth, tensor-map cache, dispatch state -- runs concurrently)."""
    from emu_build import build_capi_host_emu
    emu = build_capi_host_emu()
    exe = build(tmp_path, THREADS_SRC, "threads_harness_emu", lib=emu)
    out = subprocess.run([exe, "4", "1"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    assert " 0 mismatches" in out.stdout


@pytest.mark.gpu
def test_concurrent_callers_on_gpu(tmp_path):
    """the same harness on the H100: each thread launches on its own stream (cudaStreamPerThread), so the shared workspace
    is handed from stream to stream by the library's events while kernels of different callers overlap"""
    exe = build(tmp_path, THREADS_SRC, "threads_harness")
    for argv in (["4", "3", "1"], ["6", "2", "4"]):     # scale 4: shapes up to 1200 x 1040 x 288 and 512 x 512 x 4096
        out = subprocess.run([exe] + argv, capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        assert " 0 mismatches" in out.stdout
