"""CPU-only: the two halves of tests/test_gpu_error_bounds.py that do not need an H100.

1. Its Python restatement of the split-K plan (plan()) is pinned against the library's tc_plan: through real launches of the
   tc harness (tests/test_emulated_tc.py: run_tc reports k_splits and n_direct) at small shapes, and through the harness's
   plan-only entry over a sweep of SM counts -- 132 (H100 SXM) and 114 (H100 PCIe) among them -- and shapes around every
   threshold of the plan, with tail_min_k = 2048 as the library uses it.
2. The file itself runs against the host-emulated library with 4 "SMs", where every plan class occurs at small shapes."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import test_gpu_error_bounds as G
from emu_build import build_capi_host_emu
from test_emulated_tc import emu, rnd, run_tc  # noqa: F401  (emu: the harness fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KIND = {"tf32x1": 0, "tf32x3": 1, "bf16": 2, "f16x3": 3}


def library_plan(emu, mode, M, N, K, batch, sms, enabled=1):
    out = (ctypes.c_int * 2)()
    emu.emu_tc_plan(KIND[mode], M, N, K, batch, 128, enabled, sms, 2048, out)
    return out[0], out[1]


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("shape,sms", [((637, 16, 2048), 4), ((637, 16, 2047), 4), ((893, 16, 2048), 4), ((200, 100, 1536), 4),
                                       ((300, 200, 500), 4), ((100, 100, 1536), 2), ((385, 16, 2048), 2)])
def test_plan_matches_the_launches_of_the_tc_harness(emu, mode, shape, sms):
    M, N, K = shape
    a, b = rnd((M, K), 1), rnd((K, N), 2)
    c = np.zeros(M * N, np.float32)
    _, ks, _ = run_tc(emu, mode, a, b, c, N, 1, sms=sms, tail_min_k=2048)
    assert (ks, run_tc.n_direct) == G.plan(mode, M, N, K, units=sms, kc=128, enabled=True)


def test_plan_matches_tc_plan_over_sm_counts_and_shapes(emu):
    emu.emu_tc_plan.restype = None
    emu.emu_tc_plan.argtypes = [ctypes.c_int, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    Ks = [1, 64, 500, 511, 512, 513, 1023, 1024, 1025, 1536, 2047, 2048, 2049, 4096, 8192, 65536]
    classes = set()
    checked = 0
    for sms in (1, 2, 3, 4, 8, 16, 114, 132):
        # tile counts around one wave, half a wave and the few-tiles region, in one or several problems
        counts = sorted({1, 2, 3, max(1, sms // 2), sms // 2 + 1, sms - 1, sms, sms + 1, sms + sms // 3, sms + sms // 2,
                         sms + sms // 2 + 1, 2 * sms - 1, 2 * sms, 2 * sms + 1, 3 * sms + 5})
        for tiles in (t for t in counts if t >= 1):
            for batch, nb in ((1, 1), (1, 2), (tiles, 1), (max(1, tiles // 3), 3)):
                if tiles % (batch * nb):
                    continue
                mb = tiles // (batch * nb)
                M, N = mb * 128 - 5, nb * 128 - 1
                for K in Ks:
                    for mode in ("f16x3", "tf32x3", "tf32x1", "bf16"):
                        for enabled in (1, 0):
                            want = library_plan(emu, mode, M, N, K, batch, sms, enabled)
                            got = G.plan(mode, M, N, K, batch, units=sms, kc=128, enabled=bool(enabled))
                            assert got == want, (mode, M, N, K, batch, sms, enabled)
                            checked += 1
                            t = -(-M // 128) * -(-N // 128) * batch
                            classes.add("none" if want[0] == 1 else ("few" if want[1] == 0 else "tail"))
                            if mode in ("tf32x1", "bf16"):
                                assert want[0] == 1, (mode, M, N, K, t, sms)
    assert classes == {"none", "few", "tail"} and checked > 10000


def test_error_bound_file_against_the_host_emulated_library():
    """tests/test_gpu_error_bounds.py on 4 emulated SMs (a reduced case matrix; LASER_B200_EMU_FULL=1: all of it)"""
    so = build_capi_host_emu()
    env = dict(os.environ, LASER_B200_LIB=so, LASER_B200_EMU="1", LASER_B200_EMU_SMS="4", PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_error_bounds.py"), "-m", "gpu", "-q",
                          "-p", "no:cacheprovider"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    tail = out.stdout[-4000:] + out.stderr[-2000:]
    assert out.returncode == 0 and "failed" not in out.stdout, tail
    assert int(re.search(r"(\d+) passed", out.stdout).group(1)) >= 100, tail
