"""CPU-only: the WHOLE library on the CPU.  tests/emu_build.py compiles laser_b200/csrc/capi.cu -- the
complete host side: dispatch, operand classification, tensor-map construction, workspaces, the pipelined
host-pointer entry, the pre-packed API, split-K planning -- with g++ (kernel launches rewritten
textually, CUDA runtime and cuTensorMapEncodeTiled replaced by stand-ins, tests/emu/capi_host_prelude.h)
on top of the host-thread execution of every kernel, the wgmma one included (ptx_emu.h).  The ordinary
Python mirror is then loaded against that build in a subprocess (LASER_B200_LIB) and driven through the
scenarios of tests/emu_driver.py with numpy arrays as "device" memory, each checked against the oracle.
What this cannot show is listed in tests/emu/ptx_emu.h (silicon properties) -- and timing, of course."""
import os
import subprocess
import sys

import pytest

from emu_build import build_capi_host_emu, build_fake_nccl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(1200)


@pytest.fixture(scope="module")
def emulated_lib():
    return build_capi_host_emu()


def run(lib, scenario, **env):
    e = dict(os.environ, LASER_B200_LIB=lib, LASER_B200_EMU="1", PYTHONPATH=ROOT, **{k: str(v) for k, v in env.items()})
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emu_driver.py"), scenario], cwd=ROOT, env=e,
                         capture_output=True, text=True, timeout=1100)
    assert out.returncode == 0 and out.stdout.strip().startswith("OK " + scenario), out.stdout[-1500:] + out.stderr[-3000:]
    return out.stdout.strip()


@pytest.mark.parametrize("scenario", ["dispatch_and_modes", "strided_operands", "host_entry", "prepacked", "other_types",
                                      "fused_and_skinny", "tensors", "lifecycle"])
def test_scenario(emulated_lib, scenario):
    run(emulated_lib, scenario)


def test_split_k_planning_and_reduce(emulated_lib):
    assert run(emulated_lib, "split_k", LASER_B200_EMU_SMS=32).endswith("5")        # prepare A, abs-max B, split B, GEMM, reduce
    assert run(emulated_lib, "no_split_k", LASER_B200_EMU_SMS=32, LASER_B200_SPLITK=0).endswith("4")


@pytest.mark.parametrize("env", [dict(LASER_B200_PANEL_ROWS=512), dict(LASER_B200_PANEL_TAPER=1),
                                 dict(LASER_B200_PANEL_ROWS=512, LASER_B200_PANEL_TAPER=1),
                                 dict(LASER_B200_F32_MODE="tf32x3"), dict(LASER_B200_DYNSCHED=0),
                                 dict(LASER_B200_KC=64, LASER_B200_RASTER=2)],
                         ids=lambda e: ",".join("%s=%s" % (k.replace("LASER_B200_", ""), v) for k, v in e.items()))
def test_host_entry_under_configuration(emulated_lib, env):
    """the panel geometry of the pipelined host-pointer entry and the kernel configuration knobs are read
    from the environment when the library initialises: one process per configuration"""
    run(emulated_lib, "host_entry", **env)


@pytest.mark.parametrize("ndev,panels", [(2, 0), (3, 1), (2, 2), (3, 2)])
def test_rowsharded_entry_points_with_a_stand_in_nccl(emulated_lib, ndev, panels):
    """laser_b200_gemm_rowsharded_f32 / _f32_dev on 2 and 3 emulated devices (3: uneven row panels, the last rank short);
    panels >= 1: wide products in the default fp32 mode send B PREPARED in column panels, every rank multiplying its rows
    by each panel as it arrives (panels = 0: raw B in one broadcast)"""
    run(emulated_lib, "rowsharded", LASER_B200_EMU_DEVICES=ndev, LASER_B200_NCCL_LIB=build_fake_nccl(),
        LASER_B200_ROWSHARD_PANELS=panels)


def test_f16x3_mode(emulated_lib):
    """the default fp32 mode: power-of-two scaling from a device-side abs-max, two fp16 pieces, the kernel undoing the
    scales in its epilogue; range cases included.  Here on a 32-SM machine with kc = 64 (the default configuration runs the
    same assertions in test_emulated_python_mirror.py).  None of these products is split along K, on any number of SMs:
    every split keeps at least 512 K-elements and their K is at most 333; split-K in this mode is
    test_split_k_planning_and_reduce.  In the pipelined host-pointer entry every row panel of A gets its own scale"""
    run(emulated_lib, "f16x3", LASER_B200_EMU_SMS=32, LASER_B200_KC=64)
    run(emulated_lib, "host_entry", LASER_B200_F32_MODE="f16x3")


def test_the_emulated_build_is_refused_outside_these_tests(emulated_lib):
    """the Python mirror must never use the CPU test build as the product library by accident"""
    e = dict(os.environ, LASER_B200_LIB=emulated_lib, PYTHONPATH=ROOT)
    e.pop("LASER_B200_EMU", None)
    out = subprocess.run([sys.executable, "-c", "import laser_b200 as L; L.lib()"], cwd=ROOT, env=e, capture_output=True, text=True)
    assert out.returncode != 0 and "host-emulation TEST build" in out.stderr
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1"], cwd=ROOT, env=e, capture_output=True, text=True)
    assert out.returncode != 0 and "in-tree CUDA library only" in (out.stderr + out.stdout)


ASAN_DEFAULT = ["tensors", "other_types"]
ASAN_ALL = ["dispatch_and_modes", "strided_operands", "host_entry", "prepacked", "other_types", "fused_and_skinny", "tensors",
            "lifecycle"]


def test_scenarios_under_address_sanitizer():
    """the emulated library built with -fsanitize=address, loaded under LD_PRELOAD=libasan: any kernel or host
    code that reads or writes outside a buffer (numpy arrays, library workspaces) aborts -- the CPU analogue of
    compute-sanitizer memcheck.  Two quick scenarios by default, all of them (and the layer tests) with
    LASER_B200_EMU_ASAN=1 (about two minutes; clean when last run)."""
    from emu_build import asan_env
    lib = build_capi_host_emu(asan=True)
    full = os.environ.get("LASER_B200_EMU_ASAN", "0") == "1"
    for sc in (ASAN_ALL if full else ASAN_DEFAULT):
        run(lib, sc, **asan_env())
    if full:
        run(lib, "split_k", LASER_B200_EMU_SMS=32, **asan_env())
        e = dict(os.environ, LASER_B200_LIB=lib, LASER_B200_EMU="1", PYTHONPATH=ROOT, **asan_env())
        out = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_zlayers.py"), "-m", "gpu", "-q",
                              "-p", "no:cacheprovider"], cwd=ROOT, env=e, capture_output=True, text=True, timeout=2500)
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
