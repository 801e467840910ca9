"""GPU: a per-element error bound for every fp32 tensor-core entry, on data that makes mix-ups visible, at the tile edges and
in every split-K plan the device's SM count leads to (the same file runs against the host-emulated library in the CPU suite,
tests/test_emulated_error_bounds.py).

Bound.  The exact result is computed in float64 and every element must satisfy

    |got - exact| <= |alpha| * (p_mode + a_mode(K, S)) * sum_k |a_ik| |b_kj|  +  EPS * (|alpha (AB)_ij| + |beta c_ij| + |bias|)

(+ the f16x3 row-norm term, + the bf16 output rounding, then through the activation: Lipschitz constant times the bound plus
a few ulps of the device's tanhf / expf).
  p_mode, the error of the operand pieces per product: 3 * 2^-22 in the three-pass modes (two pieces per operand, the lo*lo
      term dropped); 2^-9 + 2^-20 for tf32x1, whose operands the tensor core truncates to tf32 (|d| < 2^-10 each); 0 for
      bf16 inputs.
  a_mode(K, S), the accumulation error: 2e-6 in the three-pass modes (the constant of tests/test_gpu_zy_f16x3_mode.py: at
      most kc = 128 elements of K inside the tensor core, then IEEE fp32 running sums), plus one fp32 rounding (2^-24) per
      split plane the reduce kernel adds.  The one-pass modes accumulate the whole of K inside the tensor core
      (tc_params.h: kb_per_block = num_kb), so their term grows with K.  Model of one wgmma step (k = 8 tf32 or 16 bf16
      products added to the accumulator): the products are exact; they are aligned to the largest exponent and the sum is
      normalised, each with a truncation of at most one fp32 ulp (2^-23) of the largest of |acc| and the step's |products|,
      both bounded by the running sum_k |a||b|.  Over ceil(K / k) steps: a_mode = ceil(K / k) * 2 * 2^-23.
  EPS = 2^-22: the roundings of alpha * sum, the fma with beta * c and the bias add (three of 2^-24 each).
  bf16 output: round to nearest bf16 of 8 significant bits, at most 2^-8 of the magnitude (2^-9 would be half of that
      unit roundoff, which a halfway case exceeds).
  f16x3 row-norm term: an entry below 2^-17 of its row's (column's) maximum keeps absolute, not relative, precision:
      2^-36 * (max_k |a_ik| * sum_k |b_kj| + sum_k |a_ik| * max_k |b_kj|).

Data.  Signed U(-1, 1); every row of A, column of B, problem of a batch, image and output channel of a convolution scaled by
its own power of two in 2^[-12, 12].  Reading another row's, column's or problem's scale word, another problem's operand or
output, or dropping a split plane moves an element by orders of magnitude more than its bound.  Each entry also runs once
on positive data.

Plans.  plan() restates tc_plan's split-K decision (tc_params.h; pinned against the library's own in the CPU file) for the
device's SM count; the plan-class cases pick shapes that land in each class and check with launch_count() that a split
launch adds exactly one reduce kernel and that an unsplit one adds none, and that a repeated call is bit-identical.  With
LASER_B200_SPLITK=0 (a subprocess) the same cases must meet the same bound without any reduce launch.

The largest err / bound per mode and entry is printed at the end of the file."""
import os
import subprocess
import sys

import numpy as np
import pytest

from backend import EMU, dev, emu_budget, sync
from util import bf16_bits_to_f32, f32_to_bf16_bits

pytestmark = pytest.mark.gpu
import laser_b200 as L  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CHILD = os.environ.get("LASER_B200_ERRB_CHILD", "0") == "1"   # set in the subprocesses this file starts
# the CPU build runs every entry in the split classes and the plain product in all of them (LASER_B200_EMU_FULL=1: all)
FULL = not EMU or os.environ.get("LASER_B200_EMU_FULL", "0") == "1"
PATHS = {"f16x3": L.PATH_F16X3, "tf32x3": L.PATH_TF32X3, "tf32x1": L.PATH_TF32X1, "bf16": L.PATH_BF16}
f64 = np.float64

# ------------------------------------------------------------------------------------------------ error model (docstring)
P_MODE = {"f16x3": 3 * 2.0 ** -22, "tf32x3": 3 * 2.0 ** -22, "tf32x1": 2.0 ** -9 + 2.0 ** -20, "bf16": 0.0}
MMA_K = {"tf32x1": 8, "bf16": 16}
A_THREE_PASS = 2e-6
EPS = 2.0 ** -22
BF16_OUT = 2.0 ** -8
ROW_NORM = 2.0 ** -36
ACT_LIP = {"none": 1.0, "relu": 1.0, "tanh": 1.0, "sigmoid": 0.25}
ACT_ULPS = {"none": 0.0, "relu": 0.0, "tanh": 4 * 2.0 ** -23, "sigmoid": 8 * 2.0 ** -23}   # tanhf 2 ulp; expf, add, divide


def a_mode(mode, K, splits):
    if mode in ("f16x3", "tf32x3"):
        return A_THREE_PASS + (splits - 1) * 2.0 ** -24
    return -(-K // MMA_K[mode]) * 2 * 2.0 ** -23


def act_f64(name, v):
    if name == "relu":
        return np.maximum(v, 0.0)
    if name == "tanh":
        return np.tanh(v)
    if name == "sigmoid":
        with np.errstate(over="ignore"):
            return 1.0 / (1.0 + np.exp(-v))
    return v


# ------------------------------------------------------------------------------------------------ the split-K plan
def sm_count():
    if EMU:
        return int(os.environ.get("LASER_B200_EMU_SMS", "8"))
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def splitk_enabled():
    return int(os.environ.get("LASER_B200_SPLITK", "1") or 0) != 0


def kc_faithful():
    v = int(os.environ.get("LASER_B200_KC", "128") or 0)
    return v if v >= 32 else 128


def plan(mode, M, N, K, batch=1, units=None, tail_min_k=2048, kc=None, enabled=None):
    """tc_plan (tc_params.h) -> (k_splits, n_direct) of a launch of `batch` problems of M x N x K"""
    units = sm_count() if units is None else units
    kc = kc_faithful() if kc is None else kc
    enabled = splitk_enabled() if enabled is None else enabled
    block_k = 64 if mode in ("f16x3", "bf16") else 32
    num_kb = -(-K // block_k)
    kb_per_block = min(max(-(-kc // block_k) if mode in ("f16x3", "tf32x3") else num_kb, 1), num_kb)
    tiles = -(-M // 128) * -(-N // 128) * batch
    if mode == "bf16" or not enabled or units <= 0:       # bf16: the output is not fp32, never split
        return 1, tiles
    blocks = -(-num_kb // kb_per_block)
    min_blocks = -(-(512 // block_k) // kb_per_block)     # every split keeps >= 512 elements of K
    max_s = min(blocks // min_blocks, 16)
    rem = tiles if tiles < units else tiles % units
    S = min(units // rem if rem > 0 else 1, max_s)
    if S >= 2 and (tiles < units or K >= tail_min_k):
        per = -(-blocks // S)
        ks = -(-blocks // per)
        if ks >= 2:
            return ks, tiles - rem
    return 1, tiles


# ------------------------------------------------------------------------------------------------ helpers
RATIOS = {}   # (mode, entry) -> largest err / bound seen


def record(mode, entry, ratio):
    key = (mode, entry)
    RATIOS[key] = max(RATIOS.get(key, 0.0), ratio)


def mm64(x, y):
    """float64 product (batched over leading axes); on the device for large shapes"""
    if not EMU and x.shape[-2] * x.shape[-1] * y.shape[-1] * (x.shape[0] if x.ndim == 3 else 1) > 2e7:
        import torch
        return (torch.from_numpy(np.ascontiguousarray(x, f64)).cuda() @ torch.from_numpy(np.ascontiguousarray(y, f64)).cuda()).cpu().numpy()
    return np.asarray(x, f64) @ np.asarray(y, f64)


def scaled(rng, shape, rows=False, cols=False, positive=False):
    """U(-1, 1) (U(0, 1) if positive) float32, each row / column times its own 2^[-12, 12]"""
    x = rng.uniform(0.0 if positive else -1.0, 1.0, shape)
    if rows:
        x = x * 2.0 ** rng.integers(-12, 13, shape[-2])[:, None]
    if cols:
        x = x * 2.0 ** rng.integers(-12, 13, shape[-1])[None, :]
    return x.astype(np.float32)


def launches(fn):
    sync()
    n0 = L.launch_count()
    fn()
    sync()
    return L.launch_count() - n0


def at(t, off, name="f32"):
    return L.DevPtr(t.data_ptr() + off * t.element_size(), name)


C_LAYOUTS = ["even", "odd", "col", "negrow"]


def c_view(M, N, layout):
    """(buffer elements, offset of (0, 0), row stride, column stride): even / odd leading dimension, column-major with a
    padded leading dimension, rows stored bottom-up"""
    if layout == "even":
        ld = N + 2 + N % 2
        return M * ld, 0, ld, 1
    if layout == "odd":
        ld = N + 1 + (1 - N % 2)
        return M * ld, 0, ld, 1
    if layout == "col":
        return N * (M + 3), 0, 1, M + 3
    assert layout == "negrow"
    ld = N + 2
    return M * ld, (M - 1) * ld, -ld, 1


def view_index(M, N, off, rs, cs):
    return off + np.arange(M)[:, None] * rs + np.arange(N)[None, :] * cs


def bound_and_check(tag, mode, entry, got, A, B, alpha, beta=0.0, C0=None, splits=1, bias=None, act="none", extra_p=0.0):
    """the per-element check of the docstring for C = act(alpha A B + beta C0 + bias); A (..., M, K) and B (..., K, N) are the
    operands as multiplied (after any operand op), bias already broadcast to (..., M, N) or None"""
    K = A.shape[-1]
    ab = mm64(A, B)
    sab = mm64(np.abs(A), np.abs(B))
    pre = alpha * ab
    side = np.abs(alpha * ab)
    if beta != 0.0:
        pre = pre + beta * C0.astype(f64)
        side = side + np.abs(beta * C0.astype(f64))
    if bias is not None:
        pre = pre + bias
        side = side + np.abs(bias)
    bnd = abs(alpha) * (P_MODE[mode] + extra_p + a_mode(mode, K, splits)) * sab + EPS * side
    if mode == "f16x3":
        aa, bb = np.abs(A).astype(f64), np.abs(B).astype(f64)
        bnd = bnd + abs(alpha) * ROW_NORM * (aa.max(-1)[..., :, None] * bb.sum(-2)[..., None, :] +
                                             aa.sum(-1)[..., :, None] * bb.max(-2)[..., None, :])
    if mode == "bf16":
        bnd = bnd + BF16_OUT * (np.abs(pre) + bnd)
    want = act_f64(act, pre)
    bnd = ACT_LIP[act] * bnd + ACT_ULPS[act] * np.abs(want) + (2.0 ** -126 if act == "sigmoid" else 0.0)
    err = np.abs(got.astype(f64) - want)
    ok = err <= bnd
    ratio = np.where(np.isfinite(err), err / np.maximum(bnd, 1e-300), np.inf)
    worst = float(ratio.max())
    record(mode, entry, worst)
    if not ok.all():
        idx = np.unravel_index(int(np.argmax(np.where(ok, -1.0, ratio))), ratio.shape)
        pytest.fail("%s: %d of %d elements out of bound, worst err/bound %.3g at %s: got %r want %r bound %.3g" % (
            tag, int((~ok).sum()), ok.size, worst, idx, float(got[idx]), float(want[idx]), float(bnd[idx])))


# ------------------------------------------------------------------------------------------------ one product, any entry
class Single:
    """one M x N x K product with its data: A rows and B columns scaled, C0 U(-1, 1)"""

    def __init__(self, mode, M, N, K, seed, positive=False, clayout="even"):
        rng = np.random.default_rng(seed)
        self.mode, self.M, self.N, self.K = mode, M, N, K
        self.a = scaled(rng, (M, K), rows=True, positive=positive)
        self.b = scaled(rng, (K, N), cols=True, positive=positive)
        self.c0 = rng.uniform(0.0 if positive else -1.0, 1.0, (M, N)).astype(np.float32)
        self.aux_b = rng.uniform(-1.0, 1.0, (K, N)).astype(np.float32)
        self.bias_row = rng.uniform(-1.0, 1.0, M).astype(np.float32)
        self.bias_col = rng.uniform(-1.0, 1.0, N).astype(np.float32)
        if mode == "bf16":
            self.a_bits, self.b_bits = f32_to_bf16_bits(self.a).reshape(M, K), f32_to_bf16_bits(self.b).reshape(K, N)
            self.c0_bits = f32_to_bf16_bits(self.c0).reshape(M, N)
            self.a, self.b, self.c0 = bf16_bits_to_f32(self.a_bits), bf16_bits_to_f32(self.b_bits), bf16_bits_to_f32(self.c0_bits)
        self.clayout = clayout
        self.dev = {}

    def upload(self):
        if self.dev:
            return
        if self.mode == "bf16":
            self.dev["a"], self.dev["b"] = dev(self.a_bits.view(np.int16)), dev(self.b_bits.view(np.int16))
        else:
            self.dev["a"], self.dev["b"] = dev(self.a), dev(self.b)
            self.dev["aux_b"] = dev(self.aux_b)
            self.dev["bias_row"], self.dev["bias_col"] = dev(self.bias_row), dev(self.bias_col)

    def c_buffer(self, beta):
        """C's buffer: sentinels around the view, the view holds C0 (beta != 0) or NaN (beta == 0: C must not be read)"""
        size, off, rs, cs = c_view(self.M, self.N, self.clayout)
        idx = view_index(self.M, self.N, off, rs, cs)
        if self.mode == "bf16":
            buf = np.full(size + 2, 0xC2FA, np.uint16)
            buf[idx + 1] = self.c0_bits if beta != 0.0 else 0x7FC0
        else:
            buf = np.full(size + 2, -7777.0, np.float32)
            buf[idx + 1] = self.c0 if beta != 0.0 else np.nan
        return buf, off + 1, rs, cs, idx + 1

    def run(self, entry, alpha, beta, epi=None, ops=None, packs=None):
        """-> C (logical M x N, float32 values); checks that nothing outside the view changed"""
        self.upload()
        buf, off, rs, cs, idx = self.c_buffer(beta)
        name = "bf16" if self.mode == "bf16" else "f32"
        tc = dev(buf.view(np.int16) if self.mode == "bf16" else buf)
        M, N, K = self.M, self.N, self.K
        ta, tb = self.dev["a"], self.dev["b"]
        cp = at(tc, off, name)
        if entry == "strided":
            L.gemm_strided(M, N, K, alpha, at(ta, 0, name), K, 1, at(tb, 0, name), N, 1, beta, cp, rs, cs, path=PATHS[self.mode])
        elif entry == "epi":
            per_row, act = epi
            L.gemm_strided_fused(M, N, K, alpha, ta, K, 1, tb, N, 1, beta, cp, rs, cs,
                                 bias=self.dev["bias_row" if per_row else "bias_col"], bias_per_row=per_row, activation=act,
                                 path=PATHS[self.mode])
        elif entry == "fused":
            op_a, op_b = ops
            L.gemm_strided_fused(M, N, K, alpha, ta, K, 1, tb, N, 1, beta, cp, rs, cs, path=PATHS[self.mode], op_a=op_a,
                                 op_b=(op_b, self.dev["aux_b"], N, 1))
        elif entry == "packed":
            L.gemm_packed(M, N, K, alpha, packs[0], packs[1], beta, cp, rs, cs)
        else:
            assert entry == "packedB"
            L.gemm_packedB(M, N, K, alpha, ta, K, 1, packs[1], beta, cp, rs, cs)
        sync()
        after = tc.cpu().numpy().view(buf.dtype)
        mask = np.ones(buf.size, bool)
        mask[idx.reshape(-1)] = False
        assert np.array_equal(after[mask], buf[mask]), "written outside the C view"
        got = after[idx]
        return bf16_bits_to_f32(got) if self.mode == "bf16" else got

    def packs(self):
        self.upload()
        M, N, K = self.M, self.N, self.K
        pa = L.alloc_packed(L.gemm_prepackA_mem_required(M, N, K))
        pb = L.alloc_packed(L.gemm_prepackB_mem_required(M, N, K))
        L.gemm_prepackA(pa, M, N, K, self.dev["a"], K, 1)
        L.gemm_prepackB(pb, M, N, K, self.dev["b"], N, 1)
        sync()
        return pa, pb

    def operands(self, ops):
        """A and B as the kernel multiplies them, and the extra per-product error of an inexact operand op"""
        a, b, extra = self.a, self.b, 0.0
        if ops is None:
            return a, b, extra
        op_a, op_b = ops
        if op_a == "relu":
            a = np.maximum(a, np.float32(0))
        elif op_a == "tanh":
            a = np.tanh(a.astype(f64))
            extra = 4 * 2.0 ** -23          # the device's tanhf: 2 ulp
        s, one = self.aux_b, np.float32(1)
        if op_b == "relu_grad":
            b = np.where(s > 0, b, np.float32(0))
        elif op_b == "sigmoid_grad":         # every operation rounded on its own, as split.cuh: operand_op
            b = b * (s * (one - s))
        return a, b, extra


EPI_VARIANTS = {"col_none": (False, "none"), "row_relu": (True, "relu"), "col_tanh": (False, "tanh"), "row_sigmoid": (True, "sigmoid")}
OP_VARIANTS = {"relu_sigmoidgrad": ("relu", "sigmoid_grad"), "tanh_relugrad": ("tanh", "relu_grad")}


def single_case(mode, entry, variant, M, N, K, alpha, beta, seed, positive=False, clayout="even", expect=None, repeat=False):
    """run one entry on one product and hold it to the bound; expect = (k_splits, base launches): check the plan through the
    launch count"""
    emu_budget((3.0 if mode in ("f16x3", "tf32x3") else 1.0) * M * N * K)
    s = Single(mode, M, N, K, seed, positive=positive, clayout=clayout)
    epi = EPI_VARIANTS[variant] if entry == "epi" else None
    ops = OP_VARIANTS[variant] if entry == "fused" else None
    packs = s.packs() if entry in ("packed", "packedB") else None
    ks, _ = plan(mode, M, N, K)
    out = {}
    n = launches(lambda: out.__setitem__("c", s.run(entry, alpha, beta, epi, ops, packs)))
    got = out["c"]
    if expect is not None:
        assert n == expect + (1 if ks > 1 else 0), (n, expect, ks)
    if repeat:
        again = s.run(entry, alpha, beta, epi, ops, packs)
        assert np.array_equal(again.view(np.uint32), got.view(np.uint32)), "a repeated call differs"
    a, b, extra = s.operands(ops)
    bias = None
    if epi is not None:
        bias = np.broadcast_to((s.bias_row[:, None] if epi[0] else s.bias_col[None, :]).astype(f64), (M, N))
    tag = "%s %s %s M=%d N=%d K=%d alpha=%g beta=%g C=%s splits=%d" % (entry, variant, mode, M, N, K, alpha, beta, clayout, ks)
    bound_and_check(tag, mode, entry + ("" if variant is None else ":" + variant), got, a, b, alpha, beta, s.c0, ks, bias,
                    epi[1] if epi else "none", extra)
    return ks


# ------------------------------------------------------------------------------------------------ edges
MN_EDGES = [1, 127, 128, 129, 255, 256, 257]
K_EDGES = {"f16x3": [1, 63, 64, 65, 127, 128, 129, 511, 512, 513, 2047, 2048, 2049],
           "bf16": [1, 63, 64, 65, 127, 128, 129, 511, 512, 513, 2047, 2048, 2049],
           "tf32x3": [1, 31, 32, 33, 127, 128, 129, 511, 512, 513, 2047, 2048, 2049],
           "tf32x1": [1, 31, 32, 33, 127, 128, 129, 511, 512, 513, 2047, 2048, 2049]}


def edge_cases():
    """every K edge of every mode once, M, N, alpha, beta and the C layout cycled over their edges"""
    out = []
    for mode, ks in K_EDGES.items():
        for K in ks:
            j = len(out)
            M, N = MN_EDGES[j % 7], MN_EDGES[(3 * j + 2) % 7]
            alpha = (1.0, -0.5)[(j // 2) % 2]
            beta = (0.0, -1.25)[j % 2]
            out.append((mode, M, N, K, alpha, beta, C_LAYOUTS[(j // 4) % 4]))
    return out


@pytest.mark.parametrize("case", edge_cases(), ids=lambda c: "%s-M%d-N%d-K%d-a%g-b%g-%s" % c)
def test_edges(case):
    mode, M, N, K, alpha, beta, clayout = case
    single_case(mode, "strided", None, M, N, K, alpha, beta, seed=M * 7919 + N * 31 + K, clayout=clayout)


# ------------------------------------------------------------------------------------------------ plan classes
CLASSES = ["none", "few", "tail", "half", "k2047"]


def class_shape(cls, units):
    """(M, N, K) of one problem landing in plan class `cls` for a launch on `units` SMs"""
    if cls == "none":
        return 300, 200, 500                               # no mode can split K = 500
    if cls == "few":
        return (200, 100, 1536) if units >= 3 else (100, 100, 1536)   # fewer tiles than SMs, every tile split
    rem = max(1, units // 3) if cls in ("tail", "k2047") else units // 2 + 1
    tiles = units + rem
    nb = 2 if tiles % 2 == 0 and not EMU else 1
    M, N = (tiles // nb) * 128 - 3, (nb * 128 - 5 if nb == 2 else (16 if EMU else 40))
    return M, N, 2047 if cls == "k2047" else 2048


def expected_class(cls, ks, n_direct, M, N, batch=1):
    tiles = -(-M // 128) * -(-N // 128) * batch
    if not splitk_enabled():
        return ks == 1
    if cls == "few":
        return 2 <= ks <= 16 and n_direct == 0
    if cls == "tail":
        return ks >= 2 and 0 < n_direct < tiles
    return ks == 1


def base_launches(mode, entry, variant, M, N, K):
    """the launches of the same call at a K below 512, which never splits, with K's alignment (which decides whether an
    operand is read in place)"""
    s = Single(mode, M, N, 64 + K % 64, 5)
    epi = EPI_VARIANTS[variant] if entry == "epi" else None
    ops = OP_VARIANTS[variant] if entry == "fused" else None
    packs = s.packs() if entry in ("packed", "packedB") else None
    return launches(lambda: s.run(entry, 1.0, 0.0, epi, ops, packs))


def plan_cases():
    out = []
    for cls in CLASSES:
        for mode in ("f16x3", "tf32x3", "tf32x1"):
            out.append(("strided", None, mode, cls))
            if FULL or cls in (("tail",) if mode == "tf32x1" else ("few", "tail")):
                out += [("epi", v, mode, cls) for v in EPI_VARIANTS]
                out += [("fused", v, mode, cls) for v in OP_VARIANTS]
        if FULL or cls in ("few", "tail"):
            out += [("packed", None, "f16x3", cls), ("packedB", None, "f16x3", cls)]
        if cls in ("few", "tail"):
            out.append(("strided", None, "bf16", cls))
    return out


@pytest.mark.parametrize("case", plan_cases(), ids=lambda c: "%s-%s-%s-%s" % (c[0], c[1] or "plain", c[2], c[3]))
def test_plan_classes(case):
    entry, variant, mode, cls = case
    units = sm_count()
    M, N, K = class_shape(cls, units)
    ks, nd = plan(mode, M, N, K)
    if mode in ("f16x3", "tf32x3"):
        assert expected_class(cls, ks, nd, M, N), (cls, M, N, K, ks, nd)
    else:
        assert ks == 1          # tf32x1: one accumulation block (max_s = 0); bf16: not an fp32 output
    emu_budget((3.0 if mode in ("f16x3", "tf32x3") else 1.0) * M * N * K)
    base = base_launches(mode, entry, variant, M, N, K)
    i = CLASSES.index(cls)
    single_case(mode, entry, variant, M, N, K, (1.0, -0.5)[i % 2], (-1.25, 0.0)[i % 2], seed=100 + i, expect=base, repeat=True)


@pytest.mark.parametrize("entry,variant,mode", [("strided", None, "f16x3"), ("strided", None, "tf32x3"), ("strided", None, "tf32x1"),
                                                ("strided", None, "bf16"), ("epi", "row_relu", "f16x3"), ("epi", "col_none", "tf32x3"),
                                                ("fused", "relu_sigmoidgrad", "f16x3"), ("packed", None, "f16x3"),
                                                ("packedB", None, "f16x3")])
def test_positive_data(entry, variant, mode):
    single_case(mode, entry, variant, 300, 260, 700, 1.0, 0.5, seed=7, positive=True)


# ------------------------------------------------------------------------------------------------ batched
class Batch:
    """`batch` problems: A_b rows and B_b columns scaled, each problem by its own power of two too; operand X of problem b at
    base + b * bs (bs = 0: shared, bs < 0: stored last to first); C_b at b * bsC with guards between the problems"""

    def __init__(self, batch, M, N, K, seed, share_a=False, neg=False, positive=False):
        rng = np.random.default_rng(seed)
        self.batch, self.M, self.N, self.K = batch, M, N, K
        na = 1 if share_a else batch
        pa = 2.0 ** rng.integers(-12, 13, na)
        pb = 2.0 ** rng.integers(-12, 13, batch)
        self.a = np.stack([scaled(rng, (M, K), rows=True, positive=positive) * np.float32(pa[i]) for i in range(na)])
        self.b = np.stack([scaled(rng, (K, N), cols=True, positive=positive) * np.float32(pb[i]) for i in range(batch)])
        self.c0 = rng.uniform(-1.0, 1.0, (batch, M, N)).astype(np.float32)
        self.bias = rng.uniform(-1.0, 1.0, N).astype(np.float32)
        self.bias_row = rng.uniform(-1.0, 1.0, M).astype(np.float32)

        def lay(x, bs_sign):
            n, per = x.shape[0], x[0].size + 8
            buf = np.full(n * per, 5.0, np.float32)
            for i in range(n):
                slot = (n - 1 - i) if bs_sign < 0 else i
                buf[slot * per:slot * per + x[0].size] = x[i].reshape(-1)
            base = (n - 1) * per if bs_sign < 0 else 0
            return dev(buf), base, (0 if n == 1 else bs_sign * per)
        self.ta, self.oa, self.bsa = lay(self.a, -1 if neg else 1)
        self.tb, self.ob, self.bsb = lay(self.b, -1 if neg else 1)
        if share_a:
            self.bsa = 0
        self.tbias, self.tbias_row = dev(self.bias), dev(self.bias_row)
        self.ldc = N + 2 + N % 2
        self.bsc = M * self.ldc + 6

    def run(self, mode, alpha, beta, epi=None):
        M, N, K = self.M, self.N, self.K
        buf = np.full(self.batch * self.bsc + 3, -7777.0, np.float32)
        idx = (np.arange(self.batch)[:, None, None] * self.bsc + np.arange(M)[None, :, None] * self.ldc +
               np.arange(N)[None, None, :])
        buf[idx] = self.c0 if beta != 0.0 else np.nan
        tc = dev(buf)
        kw = {}
        if epi is not None:
            kw = dict(bias=self.tbias_row if epi[0] else self.tbias, bias_per_row=epi[0], activation=epi[1])
        L.gemm_strided_batched_fused(self.batch, M, N, K, alpha, at(self.ta, self.oa), K, 1, self.bsa, at(self.tb, self.ob), N, 1,
                                     self.bsb, beta, tc, self.ldc, 1, self.bsc, path=PATHS[mode], **kw)
        sync()
        after = tc.cpu().numpy()
        mask = np.ones(buf.size, bool)
        mask[idx.reshape(-1)] = False
        assert np.array_equal(after[mask].view(np.uint32), buf[mask].view(np.uint32)), "written outside the problems' C views"
        return after[idx]

    def check(self, tag, mode, entry, got, alpha, beta, splits, epi=None):
        a = np.broadcast_to(self.a, (self.batch,) + self.a.shape[1:])
        bias = None
        if epi is not None:
            bias = np.broadcast_to((self.bias_row[:, None] if epi[0] else self.bias[None, :]).astype(f64), got.shape)
        bound_and_check(tag, mode, entry, got, a, self.b, alpha, beta, self.c0, splits, bias, epi[1] if epi else "none")


BATCH_KINDS = {"own": (False, False, (False, "none")), "shared_a": (True, False, (True, "relu")), "negative": (False, True, None)}


def batch_class_shape(cls, units):
    """(batch, M, N, K) of a batched launch in class `cls`; "tail": the split tiles begin inside a problem"""
    if cls == "none":
        return 3, 200, 260, 256
    if cls == "few":
        return 2, 100, 90, 1536
    if cls == "half":
        return units + units // 2 + 1, 40, 30, 2048
    for npp in (3, 5, 7, 11, 2):              # tiles per problem: one row of npp column blocks
        batch = units // npp + 1
        rem = batch * npp - units
        if batch >= 2 and 1 <= rem <= units // 2 and (units % npp) != 0:
            return batch, 16 if EMU else 40, npp * 128 - 40, 2047 if cls == "k2047" else 2048
    pytest.skip("no batched shape splits inside a problem on %d SMs" % units)


def batched_case(mode, kind, cls, check_plan=True, positive=False):
    units = sm_count()
    batch, M, N, K = batch_class_shape(cls, units)
    share_a, neg, epi = BATCH_KINDS[kind]
    ks, nd = plan(mode, M, N, K, batch)
    if check_plan and mode in ("f16x3", "tf32x3"):
        assert expected_class(cls, ks, nd, M, N, batch), (cls, batch, M, N, K, ks, nd)
        if cls == "tail" and splitk_enabled():
            assert nd % (-(-M // 128) * -(-N // 128)) != 0        # the first split tile is not a problem's first
    emu_budget((3.0 if mode in ("f16x3", "tf32x3") else 1.0) * batch * M * N * K)
    i = CLASSES.index(cls)
    alpha, beta = (1.0, -0.5)[i % 2], (-1.25, 0.0)[i % 2]
    bt = Batch(batch, M, N, K, 200 + i, share_a=share_a, neg=neg, positive=positive)
    out = {}
    n = launches(lambda: out.__setitem__("c", bt.run(mode, alpha, beta, epi)))
    got = out["c"]
    if check_plan:
        base = launches(lambda: Batch(batch, M, N, 64 + K % 64, 9, share_a=share_a, neg=neg).run(mode, 1.0, 0.0, epi))
        assert n == base + (1 if ks > 1 else 0), (n, base, ks)
        again = bt.run(mode, alpha, beta, epi)
        assert np.array_equal(again.view(np.uint32), got.view(np.uint32)), "a repeated call differs"
    tag = "batched %s %s %s batch=%d M=%d N=%d K=%d splits=%d" % (kind, mode, cls, batch, M, N, K, ks)
    bt.check(tag, mode, "batched:" + kind, got, alpha, beta, ks, epi)


def batched_cases():
    return [(mode, kind, cls) for mode in ("f16x3", "tf32x3", "tf32x1") for kind in BATCH_KINDS for cls in CLASSES
            if FULL or cls in (("tail",) if mode == "tf32x1" else ("few", "tail"))]


@pytest.mark.parametrize("mode,kind,cls", batched_cases())
def test_batched_plan_classes(mode, kind, cls):
    batched_case(mode, kind, cls)


def test_batched_positive_data():
    batched_case("f16x3", "own", "none", positive=True)


def _child(code, **env):
    e = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]), LASER_B200_ERRB_CHILD="1", **env)
    out = subprocess.run([sys.executable] + code, cwd=ROOT, env=e, capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    return out.stdout


@pytest.mark.skipif(CHILD, reason="runs in the parent process only")
def test_batched_in_chunks_of_one_problem():
    """a 1 MB workspace cap: every problem of these batches is a chunk of its own, and the bound still holds"""
    _child(["-c", "import test_gpu_error_bounds as T\n"
                  "for mode in ('f16x3', 'tf32x3'):\n"
                  "    for kind in ('own', 'shared_a', 'negative'):\n"
                  "        T.batched_case(mode, kind, 'few', check_plan=False)\n"
                  "        T.batched_case(mode, kind, 'tail', check_plan=False)\n"], LASER_B200_BATCH_WS_MB="1")


# ------------------------------------------------------------------------------------------------ convolution
def conv_ref(x, w, padding, strides):
    """float64 direct convolution -> (n, c_out, oh * ow)"""
    n, c, h, wd = x.shape
    co, _, kh, kw = w.shape
    (ph, pw), (sh, sw) = padding, strides
    xp = np.pad(np.asarray(x, f64), ((0, 0), (0, 0), (ph, ph), (pw, pw)))
    win = np.lib.stride_tricks.sliding_window_view(xp, (kh, kw), axis=(2, 3))[:, :, ::sh, ::sw]   # n, c, oh, ow, kh, kw
    oh, ow = win.shape[2], win.shape[3]
    cols = np.ascontiguousarray(win.transpose(0, 2, 3, 1, 4, 5)).reshape(n, oh * ow, c * kh * kw)
    return np.swapaxes(cols, 1, 2), w.reshape(co, -1).astype(f64)   # B per image (K, oh*ow), A (co, K)


CONV_GEOM = ((2, 128, 6, 6), (64, 128, 3, 3)) if EMU else ((8, 256, 14, 14), (256, 256, 3, 3))   # K = 1152 / 2304


@pytest.mark.parametrize("mode,act", [("f16x3", "relu"), ("f16x3", "none"), ("tf32x3", "tanh"), ("tf32x1", "sigmoid"),
                                      ("f16x3", "positive")])
def test_conv2d_fused(mode, act):
    """images and output channels scaled by their own powers of two, a bias per output channel, K >= 1024 and few enough
    images that every tile splits"""
    ishape, kshape = CONV_GEOM
    positive = act == "positive"
    act = "none" if positive else act
    padding, strides = (1, 1), (1, 1)
    rng = np.random.default_rng(11)
    x = rng.uniform(0.0 if positive else -1.0, 1.0, ishape) * 2.0 ** rng.integers(-12, 13, ishape[0])[:, None, None, None]
    w = rng.uniform(0.0 if positive else -1.0, 1.0, kshape) * 2.0 ** rng.integers(-12, 13, kshape[0])[:, None, None, None]
    x, w = x.astype(np.float32), w.astype(np.float32)
    bias = (rng.uniform(-1.0, 1.0, kshape[0]) * 2.0 ** rng.integers(-6, 7, kshape[0])).astype(np.float32)
    oshape = tuple(L.conv2d_out_shape(ishape, kshape, padding, strides))
    M, N, K, n = kshape[0], oshape[2] * oshape[3], int(np.prod(kshape[1:])), ishape[0]
    emu_budget(3.0 * n * M * N * K)
    ks, nd = plan(mode, M, N, K, n)
    if mode != "tf32x1" and splitk_enabled():
        assert ks >= 2 and nd == 0, (ks, nd)
    tx, tw, tb = dev(x), dev(w), dev(bias)

    def run(xd, shp, wd, kshp):
        out = dev(np.full((shp[0], M) + oshape[2:], np.nan, np.float32))
        L.conv2d_fused(out, xd, shp, wd, kshp, padding, strides, bias=tb, activation=act, path=PATHS[mode])
        return out
    # the same convolution over 8 input channels (K = 72: never split) makes the launches of an unsplit call
    thin, kthin = (n, 8) + ishape[2:], (M, 8) + kshape[2:]
    assert plan(mode, M, N, 72, n)[0] == 1
    base = launches(lambda: run(dev(np.ascontiguousarray(x[:, :8])), thin, dev(np.ascontiguousarray(w[:, :8])), kthin))
    res = {}
    n_l = launches(lambda: res.__setitem__("o", run(tx, ishape, tw, kshape)))
    assert n_l == base + (1 if ks > 1 else 0), (n_l, base, ks)
    got = res["o"].cpu().numpy().reshape(n, M, N)
    b_img, a_mat = conv_ref(x, w, padding, strides)
    bound_and_check("conv2d_fused %s %s %s %s splits=%d" % (mode, act, ishape, kshape, ks), mode, "conv2d_fused", got,
                    np.broadcast_to(a_mat, (n,) + a_mat.shape), b_img, 1.0, splits=ks,
                    bias=np.broadcast_to(bias.astype(f64)[None, :, None], got.shape), act=act)


# ------------------------------------------------------------------------------------------------ split-K off
@pytest.mark.skipif(CHILD, reason="runs in the parent process only")
def test_same_cases_without_split_k():
    """LASER_B200_SPLITK=0: the plan-class cases take no reduce kernel and meet the same bound (the sums are added in
    another order, so the bits may differ)"""
    select = ("plan_classes and (few or tail) and not bf16 and not tf32x1 or conv2d" if FULL else
              "plan_classes and tail and f16x3 and not packed or conv2d and f16x3")
    out = _child(["-m", "pytest", os.path.join(HERE, "test_gpu_error_bounds.py"), "-m", "gpu", "-q", "-p", "no:cacheprovider",
                  "-k", select], LASER_B200_SPLITK="0")
    assert " passed" in out and "failed" not in out, out[-3000:]


# ------------------------------------------------------------------------------------------------ report
def test_zz_report_largest_err_over_bound(capsys):
    """the largest err / bound per mode and entry of this run (the last test of the file)"""
    if not RATIOS:
        pytest.skip("no case ran")
    lines = ["largest err / bound on %d SMs (%s):" % (sm_count(), "host-emulated library" if EMU else "device")]
    for (mode, entry), r in sorted(RATIOS.items()):
        lines.append("  %-7s %-28s %.3g" % (mode, entry, r))
    with capsys.disabled():
        print("\n" + "\n".join(lines))
