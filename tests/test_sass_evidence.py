"""CPU-only: the shipped library really is a wgmma / TMA / mbarrier build (HGMMA = wgmma.mma_async, UTMALDG = TMA tile
load, SYNCS = mbarrier, USETMAXREG = setmaxnreg), for every tensor-core kernel family, and holds no mma.sync half-precision
path.  `python tests/test_sass_evidence.py DIR` writes the per-kernel counts to DIR/sass_mnemonics.txt."""
import collections
import os
import re
import shutil
import subprocess

import pytest

import laser_b200 as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MNEMONICS = ("HGMMA", "WARPGROUP", "UTMALDG", "UBLKCP", "LDGSTS", "DMMA", "HMMA", "ATOMG", "SYNCS", "STG.E.128", "USETMAXREG")


import functools


@functools.lru_cache(maxsize=1)
def sass_counts():
    """{kernel symbol: Counter(mnemonic -> count)} of the tensor-core kernels in liblaser_b200.so (one disassembly per run)"""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not installed")
    out = subprocess.run([exe, "-sass", L.lib_path()], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            res[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        for mn in MNEMONICS:
            # HMMA must not match UTCHMMA
            if re.search(r"(?<![A-Z])" + re.escape(mn), line):
                res[cur][mn] += 1
    return res


def test_tensor_core_kernels_are_wgmma_tma():
    counts = sass_counts()
    tc = {k: v for k, v in counts.items() if "gemm_tc_kernel" in k}
    # one-problem: 16-bit families (bf16, f16x3) x 4 operand major-nesses, tf32 families K-major only; batched: f16x3 x 4
    # major-nesses, tf32x3, tf32x1
    assert len(tc) == (2 * 4 + 2) + (4 + 2), sorted(tc)
    for k, c in tc.items():
        assert c["HGMMA"] >= 4 and c["WARPGROUP"] >= 2 and c["UTMALDG"] >= 2 and c["SYNCS"] >= 2, (k, dict(c))
        assert c["USETMAXREG"] == 2, k          # warp-specialised register split
    for k, c in counts.items():
        assert c["HMMA"] == 0, k                # no half-precision mma.sync anywhere in the library


def test_fp64_tensor_cores_and_bulk_copies():
    counts = sass_counts()
    dmma = [c for k, c in counts.items() if "gemm_dmma_kernel" in k]
    assert len(dmma) == 1 and dmma[0]["DMMA"] >= 32 and dmma[0]["LDGSTS"] >= 16      # mma.sync.m8n8k4.f64, cp.async staging
    ring = [c for k, c in counts.items() if "f16x2_rows_ring_kernel" in k]
    assert len(ring) == 1 and ring[0]["UBLKCP"] >= 2 and ring[0]["SYNCS"] >= 2          # cp.async.bulk rows + mbarrier


if __name__ == "__main__":
    import sys
    counts = sass_counts()
    out_dir = sys.argv[1] if len(sys.argv) > 1 else "."
    with open(os.path.join(out_dir, "sass_mnemonics.txt"), "w") as f:
        f.write("# cuobjdump -sass laser_b200/lib/liblaser_b200.so: occurrences per tensor-core kernel\n")
        f.write("# (HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / wait, UTMALDG = cp.async.bulk.tensor load, UBLKCP = cp.async.bulk,\n# LDGSTS = cp.async, SYNCS = mbarrier, DMMA = mma.sync.f64)\n")
        for k in sorted(counts):
            if "gemm_tc_kernel" in k or "gemm_dmma_kernel" in k or "f16x2_rows_ring_kernel" in k:
                f.write("%s\n    %s\n" % (k, "  ".join("%s=%d" % (m, counts[k][m]) for m in MNEMONICS if counts[k][m])))
    print("wrote", os.path.join(out_dir, "sass_mnemonics.txt"))
