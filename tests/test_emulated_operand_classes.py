"""CPU-only: the case table of tests/test_gpu_operand_classes.py pinned against the library's own operand classification, and
the file itself against the host-emulated library (every fourth case of each table; LASER_B200_EMU_FULL=1: all of them)."""
import itertools

import test_gpu_operand_classes as G
from test_emulated_python_mirror import _run_gpu_files

PAIRS = set(itertools.product((G.K_MAJOR, G.MN_MAJOR, G.GENERAL), repeat=2))


def by_mode(entry):
    out = {}
    for c in G.CASES[entry]:
        out.setdefault(c[1], []).append(c)
    return out


def test_single_product_tables_cover_every_class_pair():
    """gemm_strided and gemm_strided_fused: each layout name is, at the shape and element size of its case, in the class it
    stands for; every mode meets every class pair, every layout name on either side, every C layout and every alpha / beta"""
    for entry, shape_at in (("strided", 4), ("fused", 8)):
        for mode, cases in by_mode(entry).items():
            esz = 2 if mode == "bf16" else 4
            pairs, names_a, names_b = set(), set(), set()
            for c in cases:
                la, lb, (M, N, K) = c[2], c[3], c[shape_at]
                ca, cb = G.library_class(la, "A", M, K, esz), G.library_class(lb, "B", K, N, esz)
                assert (ca, cb) == (G.intended(la, "A"), G.intended(lb, "B")), (c, ca, cb)
                pairs.add((ca, cb))
                names_a.add(la)
                names_b.add(lb)
            if mode == "auto":
                continue
            assert pairs == PAIRS, (entry, mode, PAIRS - pairs)
            assert {c[shape_at + 2] for c in cases} == set(G.C_LAYOUTS) and {c[shape_at + 1] for c in cases} == set(G.AB)
            if entry == "strided":
                assert names_a == names_b == set(["row", "col"] + G.GEN), (mode, names_a, names_b)


def test_fused_table_puts_every_op_on_either_side_in_every_class():
    for mode, cases in by_mode("fused").items():
        if mode == "auto":
            continue
        seen = set()
        for c in cases:
            seen.add(("A", c[4], G.intended(c[2], "A")))
            seen.add(("B", c[5], G.intended(c[3], "B")))
        assert seen == set(itertools.product("AB", G.OPS, (0, 1, 2))), mode
        assert {c[6] for c in cases} == {False, True}                           # aux in the operand's layout and in another
        if mode != "simt":
            assert {c[7] for c in cases} == set(G.EPIS)                         # bias per row / column with each activation


def test_batch_tables_cover_every_class_pair_stride_kind_and_op():
    """problem 0 of each batched operand is in the class its layout stands for; every mode meets every class pair, every batch
    stride kind on A and on B and every op variant; the batch-reduced product's K is not a multiple of 4"""
    for entry in ("batched", "batch_reduce"):
        for mode, cases in by_mode(entry).items():
            pairs = set()
            for c in cases:
                la, lb, (batch, M, N, K) = c[2], c[3], c[7]
                rsa, csa, _ = G.stack_strides(la, M, K)
                rsb, csb, _ = G.stack_strides(lb, K, N)
                ca, cb = G.classify(4, 0, rsa, csa), G.classify(4, 0, csb, rsb)
                assert (ca, cb) == (G.intended(la, "A"), G.intended(lb, "B")), (c, ca, cb)
                pairs.add((ca, cb))
                if entry == "batch_reduce":
                    assert K % 4 != 0
            assert pairs == PAIRS, (entry, mode)
            assert {c[4] for c in cases} == {c[5] for c in cases} == set(G.BS_KINDS), (entry, mode)
            if mode != "auto":
                assert {c[6] for c in cases} == set(G.BOPS), (entry, mode)


def test_operand_class_file_against_the_host_emulated_library():
    """tests/test_gpu_operand_classes.py on the CPU build of the whole library, minus the cases skipped for size"""
    assert _run_gpu_files(["test_gpu_operand_classes.py"], [], 3000) >= 80
