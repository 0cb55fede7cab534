"""Core kernel contracts: the wgmma GEMM / implicit-GEMM conv, flash attention forward and backward, GroupNorm and
LayerNorm, checked element by element against fp64 on the GPU (pytest -m gpu), on every instantiation their launchers
pick.

Every reference is computed in fp64 on the device from the same bf16-rounded inputs the kernel reads, and every output is
written as a view inside a larger buffer filled with a sentinel bit pattern, with sentinel columns beside the view and
sentinel rows after its last row: after the kernel, every sentinel must be bit-identical (a store masked one element too
wide, or landing in the wrong row, column or third of a fused buffer, shows up there and nowhere else).  Each GEMM case records the plan the launcher took (cl_gemm_plan) and asserts the one
it was written for, so a planner change fails here instead of moving the case to another kernel.  It also asserts the
epilogue's store path (cl_gemm_plan's fifth entry: TMA stores from shared memory, or register stores for outputs and
residuals that are not 16-byte aligned and fp32 outputs with a residual): every instantiation runs on both, and the two
must agree bit for bit.

Error bounds, per element, from the arithmetic the kernels perform (T = the fp64 sum of |terms| of the element):
  - fp32 accumulation of exact bf16 products (wgmma, fp32 FMA chains): every addition loses at most one fp32 ulp of the
    running magnitude (2^-23 of it: the tensor cores' accumulation is not documented to round to nearest, and truncation
    loses a whole ulp), so a sum of K products is within ACC * K * T, ACC = 2^-23.
  - bf16 output of a value carrying error E: |out - ref| <= 1/2 bf16 ulp(|ref| + E) + E  (assert_bf16_within).
  - GEMM: E = ACC * (K + 4) * T, T over A B^T and the epilogue inputs.  LoRA: t = x (hi + lo)^T is such a sum; s t and
    B_up are split into three bf16 parts each and the dropped cross products are below 2^-16 of s |t| |B_up|, so the rank
    update adds 2^-15 * s |t| |B_up| + |s| (|t| err) |B_up|.  fp32 outputs (out_fp32, t_out) use assert_f32_reduction with
    the same ACC * (K + 4) per element.
  - Attention forward: scores carry the fp32 error ds = ACC (d + 16) sl2 |q||k| + 2^-23 |sl2 s| (sl2 = scale * log2 e
    as the kernel's fp32 value, log2 domain).  P / l is then off by eP = ln2 (ds_ij + max_j ds_ij) + 2^-20 (ex2.approx)
    relative, and P is rounded to bf16 (unit roundoff 2^-8) for the P V product:
      o:   E = sum_j (eP_ij + 2^-8) P_ij |v_j| + ACC (Nk + 2 nkb + 8) sum_j P_ij |v_j|   (fp32 sums of P V and l, rescales)
      lse: E = max_j ds_ij + 2^-23 (|lse| + 16) + 2 (2^-21 + 2^-23 (Nk + 2 nkb))           (log2 domain)
  - Attention backward, from the kernel's own inputs (q, k, v, o, dO and the forward's lse): P = exp2(sl2 s - lse) in
    fp32 (relative eP = 2^-21 + ln2 (ds + 2^-23 |lse|)); dP = dO V^T and delta = rowsum(dO o) are fp32 sums of d
    products; dS = P (dP - delta) and P are rounded to bf16 (2^-8) before the dV, dQ and dK products:
      dS error  G = 1.01 ((eP + 2^-8) P |dP - delta| + P ACC (d + 16) (|dO||v| + |dO||o|))
      dv: E = sum_i (eP + 2^-8) P_ij |dO_i| + ACC (Nq + 8) sum_i P_ij |dO_i|
      dq: E = scale (sum_j G_ij |k_j| + ACC (Nk + 8) sum_j |dS_ij| |k_j|)   (dk likewise over the queries, with q)
    ex2.approx.ftz and the MMAs flush values below 2^-126 to zero: an absolute 2^-126 per term covers that.
  - GroupNorm / LayerNorm: fp32 partial sums over R terms carry 2^-24 R relative error of the sum of |terms|; the bounds
    of mean and rstd follow from that (the variance is E[x^2] - mu^2 in GroupNorm, two-pass in LayerNorm) and are
    propagated through y = (x - mu) rstd gamma + beta (+ SiLU with __expf / __fdividef, (2 + 1.16 |z|) and 2 ulp) and through the input
    gradient; each test states its terms.  dgamma / dbeta are fp32 reductions (assert_f32_reduction).

`test_every_gemm_instantiation_has_a_case` and `test_every_head_dim_has_a_case` (no GPU needed) parse the dispatch
tables and fail when an instantiation, or an (instantiation, store path) pair, has no case here.
"""
from __future__ import annotations

import ctypes as ct
import math
import re
import zlib
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_kernel_contracts import _bf16_ulp, _conv_fp64, assert_f32_reduction

BF16 = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
CSRC = Path(__file__).resolve().parent.parent / "controllora_b200" / "csrc"
# One fp32 accumulation step (wgmma or an FMA chain) loses at most one ulp of the running magnitude: round to nearest
# loses half of that, and the tensor cores' accumulation is not documented to round to nearest (truncation loses a whole one).
ACC = 2.0**-23
SENT = {BF16: (torch.int16, 0x5A5A), F32: (torch.int32, 0x5A5A5A5A)}   # 1.5e16 as bf16, 1.5e16 as fp32


@pytest.fixture(scope="module")
def _core_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def gpu(fn):
    return pytest.mark.gpu(pytest.mark.usefixtures("_core_gpu")(fn))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------ helpers
def _seed(*params):
    torch.manual_seed(zlib.crc32(repr(params).encode()))


def _bf(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(BF16)


def _f32(*shape, scale=1.0):
    return torch.randn(*shape, device="cuda") * scale


class Canvas:
    """A buffer filled with the sentinel; `view` is the part a kernel may write."""

    def __init__(self, shape, dtype, index):
        it, bits = SENT[dtype]
        self.buf = torch.full(shape, bits, dtype=it, device="cuda").view(dtype)
        self.view = self.buf[index]
        self.mask = torch.ones(shape, dtype=torch.bool, device="cuda")
        self.mask[index] = False

    def check(self, what):
        it, bits = SENT[self.buf.dtype]
        outside = self.buf.view(it)[self.mask]
        bad = int((outside != bits).sum())
        assert bad == 0, f"{what}: {bad} elements written outside the output view"


def _rows(B, N, width, c0, w, dtype=BF16, tail=128):
    """A [B, N, w] token-matrix view (row stride `width`, columns c0 .. c0 + w) of a [B * N + tail, width] canvas: the
    columns around it guard the column masks, the `tail` rows after the last batch guard the row masks (a row written one
    past N lands there for the last batch)."""
    c = Canvas((B * N + tail, width), dtype, (slice(0, B * N), slice(c0, c0 + w)))
    # explicit strides: a .view() would give the N = 1 dimension a stride of w, which the kernels would take for the row stride
    return c, torch.as_strided(c.buf, (B, N, w), (N * width, width, 1), c0)


def _flat(n, dtype, pad=8):
    """A contiguous [n] view with `pad` sentinel elements on either side."""
    return Canvas((n + 2 * pad,), dtype, slice(pad, pad + n))


def assert_bf16_within(out, ref64, err64, what):
    """bf16 output vs the fp64 value, given the fp64 bound E of the error before the final rounding:
    |out - ref| <= 1/2 ulp(|ref| + E) + E."""
    assert out.dtype == BF16, what
    o = out.detach().to(F64)
    r = ref64.detach().to(F64)
    e = err64.detach().to(F64).expand_as(r)
    tol = 0.5 * _bf16_ulp(r.abs() + e) + e
    err = (o - r).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = int(torch.argmax(torch.where(bad, err / tol, torch.zeros_like(err)).flatten()))
        raise AssertionError(f"{what}: {int(bad.sum())} of {o.numel()} elements beyond the bound; worst at flat index {i} "
                             f"{tuple(np.unravel_index(i, tuple(o.shape)))}: got {float(o.flatten()[i])!r}, fp64 "
                             f"{float(r.flatten()[i])!r}, bound {float(tol.flatten()[i]):.3e}")


def assert_f32_within(out, ref64, err64, what):
    o = out.detach().to(F64)
    r = ref64.detach().to(F64)
    e = err64.detach().to(F64).expand_as(r)
    err = (o - r).abs()
    bad = ~(err <= e + 1e-30)
    if bad.any():
        i = int(torch.argmax(torch.where(bad, err - e, torch.zeros_like(err)).flatten()))
        raise AssertionError(f"{what}: {int(bad.sum())} of {o.numel()} elements beyond the bound; worst at flat index {i}: "
                             f"got {float(o.flatten()[i])!r}, fp64 {float(r.flatten()[i])!r}, bound {float(e.flatten()[i]):.3e}")


def _reduction(out, ref, terms, K, what):
    """fp32 sum of K terms: per element within 2^-23 K T; the Frobenius bound follows by the triangle inequality."""
    elem = ACC * K
    rel = elem * float(terms.to(F64).norm()) / max(float(ref.to(F64).norm()), 1e-300)
    assert_f32_reduction(out, ref, terms, what, rel=max(rel, 1e-12), elem=elem)


def _f32_of(x: float) -> float:
    return float(np.float32(x))


# ====================================================================================================== GEMM
def _gemm_instantiations():
    """(BN, EXT, BK, OCC) of every launch_gemm call in dispatch_gemm."""
    src = (CSRC / "gemm_wgmma.cu").read_text()
    body = src[src.index("static int dispatch_gemm("):]
    body = body[:body.index("\n}\n")]
    return sorted({tuple(int(v) for v in m) for m in re.findall(r"launch_gemm<(\d+), (\d+), (\d+), (\d+)>", body)})


def _head_d16_cases():
    src = (CSRC / "attention_tile.cuh").read_text()
    body = src[src.index("static inline int with_head_d16("):]
    body = body[:body.index("\n}\n")]
    return sorted({int(v) for v in re.findall(r"integral_constant<int, (\d+)>", body)})


def _m2(S, n_tiles):
    """M (a multiple of 128) whose tiles fill every one of the 2 * S two-CTA slots with n_tiles column tiles."""
    return 128 * math.ceil(2 * S / n_tiles)


def _conv_n(S, per_image):
    """images of per_image 128-pixel tiles that give at least 2 * S tiles"""
    return math.ceil(2 * S / per_image)


# A case: dict(M, N, K) for a matrix A or conv=(n, H, W, C, stride, pad_lo) with N; the epilogue inputs; store = the
# epilogue's store path ("tma" unless given: the output canvas is 16-byte aligned with a 16-byte multiple pitch when N % 8
# == 0); want = the plan (BK, BN, lora, split, ctas_per_sm) where split is 1, ">1" (any split) or an exact count.
# Builders take the SM count.
def _g(name, want, **kw):
    return pytest.param(kw, want, id=name)


GEMM_INSTANTIATION_CASES = [
    # BK 32 (32- and 96-channel convs)
    _g("bk32_bn32_occ1", (32, 32, False, 1, 1), conv=lambda S: (1, 64, 64, 32, 1, 1), N=32, bias=True),
    _g("bk32_bn32_occ2", (32, 32, False, 1, 2), conv=lambda S: (_conv_n(S, 128), 128, 128, 32, 1, 1), N=32, bias=True),
    _g("bk32_bn64_occ1", (32, 64, False, 1, 1), conv=lambda S: (math.ceil(S / 32), 64, 64, 32, 1, 1), N=64, residual="alias"),
    _g("bk32_bn64_occ2", (32, 64, False, 1, 2), conv=lambda S: (_conv_n(S, 128), 128, 128, 32, 1, 1), N=64, bias=True),
    _g("bk32_bn128_occ1", (32, 128, False, 1, 1), conv=lambda S: (4, 64, 64, 96, 1, 1), N=128, bias=True, residual="sep"),
    _g("bk32_bn128_occ2", (32, 128, False, 1, 2), conv=lambda S: (_conv_n(S, 128), 128, 128, 32, 1, 1), N=128, row_bias=4096),
    # LoRA, BK 64
    _g("lora_bn64_occ1", (64, 64, True, 1, 1), M=1024, N=640, K=640, lora=4, t_out=True),
    _g("lora_bn64_occ2", (64, 64, True, 1, 2), M=lambda S: _m2(S, 3), N=192, K=320, lora=8, t_add=True, t_out=True),
    _g("lora_bn128_occ1", (64, 128, True, 1, 1), M=4096, N=384, K=640, lora=4, bias=True, residual="sep"),
    _g("lora_bn128_occ2", (64, 128, True, 1, 2), M=lambda S: _m2(S, 3), N=384, K=320, lora=8, t_out=True, residual="alias"),
    _g("lora_bn160_occ1", (64, 160, True, 1, 1), M=4096, N=320, K=320, lora=4, t_add=True, t_out=True, bias=True),
    _g("lora_bn160_occ2", (64, 160, True, 1, 2), M=lambda S: _m2(S, 2), N=320, K=320, lora=4, t_add=True, t_out=True),
    # plain, BK 64
    _g("bn64", (64, 64, False, 1, 1), M=1000, N=320, K=320, bias=True, residual="sep"),
    _g("bn128_occ1", (64, 128, False, 1, 1), M=2048, N=640, K=640, bias=True),
    _g("bn128_occ2", (64, 128, False, 1, 2), M=lambda S: _m2(S, 3), N=384, K=320, bias=True, row_bias=1000, residual="alias"),
    _g("bn160_occ1", (64, 160, False, 1, 1), M=4096, N=320, K=320, out_fp32=True, bias=True),
    _g("bn160_occ2", (64, 160, False, 1, 2), M=lambda S: _m2(S, 2), N=320, K=320, bias=True, row_bias=2000, residual="sep"),
    _g("bn256", (64, 256, False, 1, 1), M=4096, N=2560, K=320, bias=True),
]

GEMM_TAIL_CASES = [
    # M tails (M mod 128 = 1, 64, 127), N tails (no BN divides N), K tails (TMA zero fill of the last k-block)
    _g("m_tail_1", (64, 64, False, 1, 1), M=1025, N=320, K=320, bias=True, residual="alias"),
    _g("m_tail_64", (64, 64, False, 1, 1), M=1088, N=320, K=320, row_bias=100, out_fp32=True),
    _g("m_tail_127", (64, 64, False, 1, 1), M=1151, N=320, K=320, bias=True, row_bias=77, residual="sep"),
    _g("n_tail_100_k200", (64, 128, False, 1, 1), M=1001, N=100, K=200, bias=True, residual="sep", store="reg"),
    _g("n_tail_200_k72", (64, 160, False, 1, 1), M=1153, N=200, K=72, bias=True, row_bias=300),
    _g("n_tail_1000_k8", (64, 160, False, 1, 1), M=129, N=1000, K=8, out_fp32=True, bias=True),
    _g("n_tail_36", (64, 64, False, 1, 1), M=1000, N=36, K=64, residual="alias", store="reg"),
    _g("lora_r8_tails", (64, 160, True, 1, 1), M=1025, N=200, K=72, lora=8, t_add=True, t_out=True, bias=True),
    _g("lora_r4_tails", (64, 160, True, 1, 1), M=1151, N=100, K=200, lora=4, t_out=True, residual="alias", store="reg"),
    _g("lora_r4_text", (64, 64, True, 1, 1), M=154, N=768, K=768, lora=4, t_add=True, t_out=True),
    # conv pixel tiles: Wo = 1, 2, 4, 12, 24, 48, 96 (bw x bh x bn = 1x1x128, 2x2x32, 4x4x8, 4x4x8, 8x8x2, 16x8x1, 32x4x1)
    _g("conv_wo1", (64, 64, False, 1, 1), conv=lambda S: (3, 1, 1, 64, 1, 1), N=64, bias=True, residual="sep"),
    _g("conv_wo2", (32, 32, False, 1, 1), conv=lambda S: (3, 2, 2, 32, 1, 1), N=32, bias=True),
    _g("conv_wo4_c96", (32, 32, False, 1, 1), conv=lambda S: (3, 4, 4, 96, 1, 1), N=128, row_bias=16, residual="alias"),
    _g("conv_wo12", (64, 64, False, 1, 1), conv=lambda S: (2, 12, 12, 64, 1, 1), N=320, bias=True),
    _g("conv_wo24", (32, 32, False, 1, 1), conv=lambda S: (3, 24, 24, 32, 1, 1), N=64, bias=True, residual="sep"),
    _g("conv_wo48", (64, 64, False, 1, 1), conv=lambda S: (2, 48, 48, 64, 1, 1), N=128, row_bias=2304),
    _g("conv_wo96", (32, 32, False, 1, 1), conv=lambda S: (1, 96, 96, 32, 1, 1), N=32, out_fp32=True, bias=True),
    # stride 2, pad_lo 0 and 1
    _g("conv_s2_wo4_pad0", (32, 32, False, 1, 1), conv=lambda S: (3, 8, 8, 32, 2, 0), N=64, bias=True),
    _g("conv_s2_wo4_pad1", (32, 32, False, 1, 1), conv=lambda S: (3, 8, 8, 32, 2, 1), N=64, bias=True),
    _g("conv_s2_wo12_c96_pad0", (32, 32, False, 1, 1), conv=lambda S: (2, 24, 24, 96, 2, 0), N=320, residual="sep"),
    _g("conv_s2_wo12_c96_pad1", (32, 32, False, 1, 1), conv=lambda S: (2, 24, 24, 96, 2, 1), N=320, bias=True),
    _g("conv_s2_wo48_pad1", (64, 64, False, 1, 1), conv=lambda S: (2, 96, 96, 64, 2, 1), N=128, bias=True),
    _g("conv_s2_wo2_pad0", (64, 64, False, 1, 1), conv=lambda S: (3, 4, 4, 64, 2, 0), N=64, bias=True),
    _g("conv_s2_wo1_pad1", (64, 64, False, 1, 1), conv=lambda S: (3, 2, 2, 64, 2, 1), N=64, residual="alias"),
]

GEMM_SPLIT_CASES = [
    # split-K (ops.gemm splits when M <= 4096 and K >= 2048): the finishing kernel applies the epilogue in another order
    _g("split8_short_last", (64, 64, False, 8, 1), M=120, N=64, K=4160, bias=True, row_bias=50, residual="alias"),
    _g("split3_k_tail_fp32", (64, 64, False, 3, 1), M=1000, N=320, K=2120, bias=True, row_bias=300, out_fp32=True),
    _g("split16", (64, 64, False, 16, 1), M=128, N=320, K=8192, bias=True, residual="sep"),
    _g("split4_bn160", (64, 160, False, 4, 1), M=1000, N=640, K=2048, row_bias=333, residual="sep"),
    _g("split_capped_3_of_10", (64, 64, False, 3, 1), M=256, N=320, K=5120, bias=True, split_cap=3),
    _g("split2_capped", (64, 64, False, 2, 1), M=128, N=320, K=8192, residual="alias", split_cap=2),
    _g("conv_split5", (64, 64, False, 5, 1), conv=lambda S: (2, 8, 8, 320, 1, 1), N=320, bias=True, row_bias=64, residual="sep"),
    _g("conv_s2_split4", (64, 64, False, 4, 1), conv=lambda S: (2, 16, 16, 256, 2, 0), N=256, bias=True, out_fp32=True),
]

REACHED = {"gemm": set(), "gemm_store": set(), "d16": set(), "gn": set()}


def _plan_splits(rows):
    (row,) = rows
    return row[1][1]


class _CappedRecorder:
    """Records cl_gemm plans (tools.gemm_occupancy._Recorder) and optionally caps the split hint, so that split_ws
    holds fewer partials than the plan wants."""

    def __init__(self, real, cap):
        from tools.gemm_occupancy import _Recorder

        self.rec = _Recorder(real)
        self.cap = cap

    def __getattr__(self, name):
        return getattr(self.rec, name)

    def cl_gemm_split_hint(self, pargs):
        s = self.rec.real.cl_gemm_split_hint(pargs)
        return min(s, self.cap) if self.cap else s


@contextmanager
def _recording(cap=0):
    """Records the plans of the cl_gemm calls inside; split-K calls get a workspace of exactly the splits * M * N floats
    ops.gemm asks for (the capped count with `cap`), followed by sentinel floats: (plans, workspace canvases)."""
    from controllora_b200 import _lib, ops

    real = _lib.lib()
    rec = _CappedRecorder(real, cap)
    spaces = []

    def exact_ws(numel, device):
        spaces.append(_flat(numel, F32, pad=1024))
        return spaces[-1].view

    real_ws = ops._split_ws
    _lib._lib, ops._split_ws = rec, exact_ws
    try:
        yield rec.rec.rows, spaces
    finally:
        _lib._lib, ops._split_ws = real, real_ws


def _run_gemm_case(spec, want, register_store=False):
    """Runs one case and checks it against fp64; returns the output.  register_store: the output view starts 8 bytes
    into a 16-byte unit (column 4 of a bf16 canvas, 2 of an fp32 one), so the epilogue must take the register stores; the
    inputs are those of the aligned run (the seed does not depend on the store)."""
    from controllora_b200 import ops

    S = _sms()
    spec = {k: (v(S) if callable(v) else v) for k, v in spec.items()}
    store = spec.pop("store", "tma")
    _seed("gemm", sorted((k, str(v)) for k, v in spec.items()))
    N = spec["N"]
    conv = spec.get("conv")
    if conv:
        n, H, W, Cc, stride, pad_lo = conv
        K = 9 * Cc
        M = n * (H // stride) * (W // stride)
        a = _bf(n, H, W, Cc)
        kw = dict(conv_stride=stride, pad_lo=pad_lo)
    else:
        M, K = spec["M"], spec["K"]
        abuf = _bf(M, K + 16)                      # lda > K
        a = abuf[:, 8:8 + K]
        kw = {}
    b = _bf(N, K, scale=K**-0.5)
    out_fp32 = bool(spec.get("out_fp32"))
    odt = F32 if out_fp32 else BF16
    c0 = (4 if odt == BF16 else 2) if register_store else 8
    if register_store:
        store = "reg"
    cout = Canvas((M + 3, N + 24), odt, (slice(1, 1 + M), slice(c0, c0 + N)))    # ldd > N, column offset 8 (or 8 bytes)
    out = cout.view
    out0 = None
    bias = _f32(N) if spec.get("bias") else None
    rb = rpg = None
    if spec.get("row_bias"):
        rpg = spec["row_bias"]
        groups = (M + rpg - 1) // rpg
        rb_buf = _f32(groups, N + 12)
        rb = rb_buf[:, 4:4 + N]                    # ld_row_bias > N
    res = None
    if spec.get("residual") == "alias":            # the engine's accumulate: residual is the output itself
        assert not out_fp32
        out.copy_(_bf(M, N))
        out0 = out.clone()
        res = out
    elif spec.get("residual") == "sep":
        res_buf = _bf(M, N + 40)
        res = res_buf[:, 32:32 + N]                # ldr > N
    lora = spec.get("lora", 0)
    lkw = {}
    tout_c = None
    if lora:
        r = lora
        down = _f32(r, K, scale=K**-0.5)
        up = torch.zeros(N, lora, device="cuda")
        up[:, :r] = _f32(N, r, scale=0.5)
        ext = ops.split_bf16_ext(down, K)
        scale = 0.7
        lkw = dict(ext=ext, lora_up=up, lora_scale=scale)
        if spec.get("t_add"):
            lkw["t_add"] = _f32(M, lora)
        if spec.get("t_out"):
            tout_c = _flat(M * lora, F32, pad=lora * 3)
            lkw["t_out"] = tout_c.view.view(M, lora)
    runs = []
    outs = []
    for rep in range(2 if spec.get("split_cap") or want[3] != 1 else 1):
        if rep:
            if out0 is not None:
                out.copy_(out0)
        with _recording(spec.get("split_cap", 0)) as (rows, spaces):
            ops.gemm(a, b, out=out, bias=bias, row_bias=rb, rows_per_group=rpg or 0, residual=res, out_fp32=out_fp32,
                     **kw, **lkw)
            torch.cuda.synchronize()
        assert len(spaces) == (want[3] != 1), f"{len(spaces)} split-K workspaces for a case planned with splits {want[3]}"
        for ws in spaces:
            assert ws.view.numel() == _plan_splits(rows) * M * N, "workspace size"
            ws.check("split-K workspace")
        runs.append([r_[1] for r_ in rows])
        outs.append(out.clone())
    (plan,) = runs[0]
    BK = 32 if conv and conv[3] % 64 else 64
    got = (BK, plan[0], bool(lora), plan[1], plan[2])
    wsplit = want[3]
    ok = got[:3] == want[:3] and got[4] == want[4] and (got[3] == wsplit if isinstance(wsplit, int) else got[3] > 1)
    assert ok, f"planned {got}, the case was written for {want}"
    tma = {"tma": 1, "reg": 0}[store]
    assert plan[4] == tma, f"plan {got} takes the {('register', 'TMA')[plan[4]]} store, the case was written for {store}"
    REACHED["gemm"].add((BK, plan[0], bool(lora), plan[1] > 1, plan[2]))
    REACHED["gemm_store"].add((_inst_of(got), store))
    if len(outs) > 1:
        assert torch.equal(outs[0].view(torch.int16 if odt == BF16 else torch.int32),
                           outs[1].view(torch.int16 if odt == BF16 else torch.int32)), "two runs differ"
    # ---- fp64 reference
    b64 = b.to(F64)
    if conv:
        x64 = a.to(F64).permute(0, 3, 1, 2)
        w64 = b64.view(N, 3, 3, Cc).permute(0, 3, 1, 2)
        acc = _conv_fp64(x64, w64, 3, stride, pad_lo).permute(0, 2, 3, 1).reshape(M, N)
        T = _conv_fp64(x64.abs(), w64.abs(), 3, stride, pad_lo).permute(0, 2, 3, 1).reshape(M, N)
    else:
        a64 = a.to(F64)
        acc = a64 @ b64.t()
        T = a64.abs() @ b64.abs().t()
    E = torch.zeros_like(acc)
    if lora:
        e64 = ext.to(F64)
        down64 = e64[:r] + e64[8:8 + r]            # the hi + lo pair the kernel multiplies
        a2 = a.to(F64)
        t64 = a2 @ down64.t()
        tT = a2.abs() @ (e64[:r].abs() + e64[8:8 + r].abs()).t()
        if "t_add" in lkw:
            t64 = t64 + lkw["t_add"][:, :r].to(F64)
            tT = tT + lkw["t_add"][:, :r].abs().to(F64)
        terr = ACC * (K + 4) * tT
        s = _f32_of(scale)
        up64 = up[:, :r].to(F64)
        acc = acc + s * (t64 @ up64.t())
        lT = s * (t64.abs() @ up64.abs().t())
        E = E + 2.0**-15 * lT + s * (terr @ up64.abs().t())
        T = T + lT
        if tout_c is not None:
            tout = lkw["t_out"]
            _reduction(tout[:, :r], t64, tT, K + 4, "t_out vs fp64")
            tout_c.check("t_out")
    if bias is not None:
        acc = acc + bias.to(F64)
        T = T + bias.abs().to(F64)
    if rb is not None:
        g = torch.arange(M, device="cuda") // rpg
        acc = acc + rb.to(F64)[g]
        T = T + rb.abs().to(F64)[g]
    if res is not None:
        r0 = (out0 if out0 is not None else res).to(F64)
        acc = acc + r0
        T = T + r0.abs()
    E = E + ACC * (K + 4) * T
    what = f"gemm plan {got}, {store} store"
    if out_fp32:
        assert_f32_within(out, acc, E, what + " (fp32 out) vs fp64")
    else:
        assert_bf16_within(out, acc, E, what + " vs fp64")
    cout.check(what)
    return out.clone(), store


@gpu
@pytest.mark.parametrize("spec,want", GEMM_INSTANTIATION_CASES)
def test_gemm_instantiation(spec, want):
    _run_gemm_case(spec, want)


@gpu
@pytest.mark.parametrize("spec,want", GEMM_TAIL_CASES)
def test_gemm_tails(spec, want):
    _run_gemm_case(spec, want)


@gpu
@pytest.mark.parametrize("spec,want", GEMM_SPLIT_CASES)
def test_gemm_split_k(spec, want):
    _run_gemm_case(spec, want)


def _inst_of(want):
    BK, BN, lora, _, occ = want
    return (BN, 16 if lora else 0, BK, occ)


def test_every_gemm_instantiation_has_a_case():
    table = _gemm_instantiations()
    assert len(table) >= 18, table
    cased = {_inst_of(p.values[1]) for p in GEMM_INSTANTIATION_CASES}
    missing = sorted(set(table) - cased)
    assert not missing, f"launch_gemm instantiations without a case in {Path(__file__).name}: {missing}"
    extra = sorted(cased - set(table))
    assert not extra, f"cases for instantiations dispatch_gemm no longer has: {extra}"
    pairs = {(_inst_of(p.values[1]), p.values[0].get("store", "tma"))
             for p in GEMM_INSTANTIATION_CASES + GEMM_TAIL_CASES + GEMM_SPLIT_CASES + GEMM_FP32_RESIDUAL_CASES}
    pairs |= {(_inst_of(p.values[1]), "reg") for p in GEMM_REGISTER_STORE_CASES}
    missing = sorted({(i, st) for i in table for st in ("tma", "reg")} - pairs)
    assert not missing, f"(launch_gemm instantiation, store path) pairs without a case in {Path(__file__).name}: {missing}"
    assert all(p.values[1][3] == 1 for p in GEMM_REGISTER_STORE_CASES), "split-K partials always leave by TMA"


# ---- the register-store epilogue.  Every instantiation's case again, and convs with tails, LoRA tails and an M tail,
# with the output view 8 bytes off a 16-byte unit: the launch must take the register stores and give the TMA run's bits
# (both add bias, row bias and residual in the same fp32 order).  fp32 outputs with a residual always take them.
GEMM_REGISTER_STORE_CASES = GEMM_INSTANTIATION_CASES + [
    p for p in GEMM_TAIL_CASES if p.id in ("m_tail_127", "lora_r8_tails", "lora_r4_text", "conv_wo1", "conv_wo4_c96",
                                            "conv_s2_wo12_c96_pad1", "conv_s2_wo1_pad1")]
GEMM_FP32_RESIDUAL_CASES = [
    _g("fp32_residual_bn64", (64, 64, False, 1, 1), M=1000, N=320, K=320, out_fp32=True, bias=True, row_bias=300,
       residual="sep", store="reg"),
    _g("fp32_residual_bn160_occ2", (64, 160, False, 1, 2), M=lambda S: _m2(S, 2), N=320, K=320, out_fp32=True, bias=True,
       row_bias=2000, residual="sep", store="reg"),
    _g("fp32_residual_conv_bk32", (32, 32, False, 1, 1), conv=lambda S: (3, 24, 24, 32, 1, 1), N=64, out_fp32=True,
       bias=True, row_bias=576, residual="sep", store="reg"),
    _g("fp32_residual_lora", (64, 64, True, 1, 1), M=1024, N=640, K=640, lora=4, t_out=True, out_fp32=True, bias=True,
       residual="sep", store="reg"),
]


@gpu
@pytest.mark.parametrize("spec,want", GEMM_REGISTER_STORE_CASES)
def test_gemm_register_store(spec, want):
    out_a, store_a = _run_gemm_case(spec, want)
    out_r, store_r = _run_gemm_case(spec, want, register_store=True)
    assert store_r == "reg"
    it = torch.int16 if out_a.dtype == BF16 else torch.int32
    assert torch.equal(out_a.view(it), out_r.view(it)), f"the {store_a} and register stores give different bits"


@gpu
@pytest.mark.parametrize("spec,want", GEMM_FP32_RESIDUAL_CASES)
def test_gemm_fp32_output_with_residual(spec, want):
    _run_gemm_case(spec, want)


class _PlanOnly:
    """Stands in for the ctypes library: cl_gemm returns cl_gemm_plan's status and records its plan; nothing launches."""

    def __init__(self, real):
        self.real, self.plans = real, []

    def __getattr__(self, name):
        return getattr(self.real, name)

    def cl_gemm(self, pargs, stream):
        info = (ct.c_int32 * 5)()
        st = self.real.cl_gemm_plan(pargs, info)
        self.plans.append((st, tuple(info)))
        return st


def _plan_only(spec, out_fp32, split_ws=None):
    """(status, cl_gemm_plan info) of a case's shape with uninitialised operands and an aligned output."""
    from controllora_b200 import _lib, ops

    S = _sms()
    spec = {k: (v(S) if callable(v) else v) for k, v in spec.items()}
    N = spec["N"]
    kw = {}
    if spec.get("conv"):
        n, H, W, Cc, stride, pad_lo = spec["conv"]
        K = 9 * Cc
        a = torch.empty(n, H, W, Cc, device="cuda", dtype=BF16)
        kw.update(conv_stride=stride, pad_lo=pad_lo)
    else:
        K = spec["K"]
        a = torch.empty(spec["M"], K, device="cuda", dtype=BF16)
    if spec.get("lora"):
        kw.update(ext=torch.zeros(16, K, device="cuda", dtype=BF16), lora_up=torch.zeros(N, spec["lora"], device="cuda"))
    real, real_ws = _lib.lib(), ops._split_ws
    rec = _PlanOnly(real)
    _lib._lib = rec
    if split_ws is not None:
        ops._split_ws = split_ws
    try:
        ops.gemm(a, torch.empty(N, K, device="cuda", dtype=BF16), out_fp32=out_fp32, **kw)
        ((st, info),) = rec.plans
    finally:
        _lib._lib, ops._split_ws = real, real_ws
    return st, info


@gpu
@pytest.mark.parametrize("out_fp32", [False, True])
def test_gemm_staged_tile_fits_every_ring(out_fp32):
    """launch_gemm falls back to the register stores when the staged output tile (fp32 for split-K partials and fp32
    outputs) does not fit the ring.  At every instantiation's stage count it fits, so an aligned output must take TMA;
    a stage or tile change that makes the fallback reachable fails here and needs register-store cases of its own."""
    for p in GEMM_INSTANTIATION_CASES + GEMM_SPLIT_CASES:
        spec, want = p.values
        st, info = _plan_only(spec, out_fp32)
        assert st == 0, f"{p.id}: cl_gemm_plan status {st}"
        assert (info[0], info[2]) == (want[1], want[4]), f"{p.id}: plan {tuple(info)}"
        assert info[4] == 1, f"{p.id} (out_fp32 {out_fp32}): the staged tile does not fit the ring, plan {tuple(info)}"


@gpu
def test_gemm_split_k_rejects_a_misaligned_workspace():
    """The split-K finishing kernel reads the partials 16 bytes at a time: a workspace 8 bytes off is an argument
    error (checked through the plan, nothing launches)."""
    from controllora_b200 import _lib

    spec, want = next(p.values for p in GEMM_SPLIT_CASES if p.id == "split16")
    st, info = _plan_only(spec, False)
    assert st == 0 and info[1] == 16 and info[4] == 1, info
    with pytest.raises(_lib.CLError, match="split-K needs 16-byte aligned"):
        _plan_only(spec, False, split_ws=lambda numel, device: torch.empty(numel + 4, device=device)[2:2 + numel])


# ====================================================================================================== attention
D_OF_D16 = {1: 8, 2: 32, 3: 40, 4: 64, 5: 72, 6: 96, 7: 104, 8: 128, 9: 136, 10: 160, 11: 168, 12: 184}
TAIL_N = [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 77]


def _att_cases():
    cases = []
    for i, (d16, d) in enumerate(sorted(D_OF_D16.items())):     # every head dim, Nq / Nk from the tail list
        cases.append(pytest.param(2, 2, TAIL_N[i % len(TAIL_N)], TAIL_N[(i + 5) % len(TAIL_N)], d, "plain", id=f"d{d}"))
    for d in (40, 72, 160):                                     # BN 128 / BI 64, BN 64 / BI 32, and the two dK/dV CTAs
        for nq, nk in zip(TAIL_N, TAIL_N[::-1]):
            cases.append(pytest.param(1, 2, nq, nk, d, "plain", id=f"d{d}_q{nq}_k{nk}"))
    for d in (16, 192):                                         # full-width last chunks; 192: the largest tiles
        cases.append(pytest.param(2, 2, 129, 77, d, "plain", id=f"d{d}_full"))
    cases += [pytest.param(1, 2, 4096, 4096, 64, "plain", id="d64_4096"),
              pytest.param(1, 1, 77, 4096, 40, "plain", id="d40_q77_k4096"),
              pytest.param(8, 40, 130, 77, 40, "plain", id="waves_d40"),
              pytest.param(2, 8, 77, 77, 40, "qkv", id="qkv_d40"),
              pytest.param(2, 5, 150, 150, 64, "qkv", id="qkv_d64"),
              pytest.param(2, 2, 150, 150, 160, "qkv", id="qkv_d160"),
              pytest.param(2, 4, 200, 200, 64, "large", id="large_logits_d64"),
              pytest.param(1, 2, 129, 200, 160, "large", id="large_logits_d160")]
    return cases


def _attn_fwd(q, k, v, H, scale, o, lse):
    from controllora_b200 import _lib
    from controllora_b200._lib import AttnFwdArgs, check
    from controllora_b200.ops import _ptr, _stream

    B, Nq, HD = q.shape
    a = AttnFwdArgs()
    a.B, a.H, a.Nq, a.Nk, a.d = B, H, Nq, k.shape[1], HD // H
    a.q, a.ldq = _ptr(q), q.stride(1)
    a.k, a.ldk = _ptr(k), k.stride(1)
    a.v, a.ldv = _ptr(v), v.stride(1)
    a.o, a.ldo = _ptr(o), o.stride(1)
    a.lse = _ptr(lse)
    a.scale = float(scale)
    check(_lib.lib().cl_attn_fwd(ct.byref(a), _stream()), "cl_attn_fwd")


def _att_inputs(B, H, Nq, Nk, d, layout):
    HD = H * d
    if layout == "qkv":
        assert Nq == Nk
        qkv = _bf(B, Nq, 3 * HD)
        return qkv[..., :HD], qkv[..., HD:2 * HD], qkv[..., 2 * HD:]
    qb, kb, vb = _bf(B, Nq, HD + 16), _bf(B, Nk, HD + 8), _bf(B, Nk, HD + 24)   # strided rows
    q, k, v = qb[..., 8:8 + HD], kb[..., :HD], vb[..., 16:16 + HD]
    if layout == "large":
        # logits of a few hundred (the running maximum and the rescale move a lot), and one-hot rows: query i < 8 of
        # batch 0, head 0 has a score of 576 * scale with key i and 0 with every other key
        q, k = _bf(B, Nq, HD, scale=6.0), _bf(B, Nk, HD, scale=6.0)
        k[0, :, :d] = 0
        for i in range(min(8, Nq, Nk)):
            q[0, i, :d] = 0
            q[0, i, i] = 24.0
            k[0, i, i] = 24.0
    return q, k, v


def _att_ref_fwd(q, k, v, H, sl2):
    """fp64 S (raw q k^T), |q||k|, log2-domain lse, P, per head: tensors [B, H, Nq, Nk]"""
    B, Nq, HD = q.shape
    Nk = k.shape[1]
    d = HD // H
    q64 = q.to(F64).view(B, Nq, H, d).transpose(1, 2)
    k64 = k.to(F64).view(B, Nk, H, d).transpose(1, 2)
    v64 = v.to(F64).view(B, Nk, H, d).transpose(1, 2)
    S = q64 @ k64.transpose(-1, -2)
    A = q64.abs() @ k64.abs().transpose(-1, -2)
    z = S * sl2
    lse = torch.logsumexp(z * math.log(2), -1) / math.log(2)
    P = torch.exp2(z - lse[..., None])
    return q64, k64, v64, S, A, lse, P


def _unheads(x):
    B, H, N, d = x.shape
    return x.transpose(1, 2).reshape(B, N, H * d)


@gpu
@pytest.mark.parametrize("B,H,Nq,Nk,d,layout", _att_cases())
def test_attention(B, H, Nq, Nk, d, layout):
    from controllora_b200 import ops

    _seed("attn", B, H, Nq, Nk, d, layout)
    HD = H * d
    q, k, v = _att_inputs(B, H, Nq, Nk, d, layout)
    scale = d**-0.5
    sl2 = float(np.float32(np.float32(scale) * np.float32(1.4426950408889634)))
    oc, o_view = _rows(B, Nq, HD + 24, 8, HD)
    lc = _flat(B * H * Nq, F32, pad=160)
    _attn_fwd(q, k, v, H, scale, o_view, lc.view)
    o_nolse = torch.empty(B, Nq, HD, device="cuda", dtype=BF16)
    _attn_fwd(q, k, v, H, scale, o_nolse, None)
    torch.cuda.synchronize()
    REACHED["d16"].add((d + 15) // 16)
    o, lse = o_view, lc.view.view(B, H, Nq)
    oc.check("attention o")
    lc.check("attention lse (nothing may land past Nq)")
    assert torch.equal(o.view(torch.int16), o_nolse.view(torch.int16)), "need_lse=False changes o"

    q64, k64, v64, S, A, lse64, P = _att_ref_fwd(q, k, v, H, sl2)
    ds = ACC * (d + 16) * sl2 * A + 2.0**-23 * (S * sl2).abs()
    BNf = 128 if d <= 128 else 64
    nkb = (Nk + BNf - 1) // BNf
    lse_err = ds.amax(-1) + 2.0**-23 * (lse64.abs() + 16) + 2 * (2.0**-21 + 2.0**-23 * (Nk + 2 * nkb))
    assert_f32_within(lse, lse64, lse_err, "attention lse vs fp64")
    eP = 2.0**-20 + math.log(2) * (ds + ds.amax(-1, keepdim=True))    # P / l before the bf16 rounding: relative
    o64 = P @ v64
    o_err = ((eP + 2.0**-8) * P + 2.0**-126) @ v64.abs() + ACC * (Nk + 2 * nkb + 8) * (P @ v64.abs())
    assert_bf16_within(o, _unheads(o64), _unheads(o_err), "attention o vs fp64")
    if layout == "large":
        for i in range(min(8, Nq, Nk)):                             # one-hot rows: o = v of the matching key, exactly
            assert torch.equal(o[0, i, :d], v[0, i, :d]), f"one-hot row {i}"

    # ---- backward, from the kernel's own o and lse
    do = _bf(B, Nq, HD)
    if layout == "qkv":
        gc, g = _rows(B, Nq, 3 * HD + 16, 8, 3 * HD)
        dq, dk, dv = g[..., :HD], g[..., HD:2 * HD], g[..., 2 * HD:]
    else:
        qc, dq = _rows(B, Nq, HD + 16, 8, HD)
        kc, dk = _rows(B, Nk, HD + 16, 0, HD)
        vc, dv = _rows(B, Nk, HD + 24, 16, HD)
    lse_k = lse.clone()
    ops.attention_bwd(q, k, v, o, do, lse_k, H, scale, need_dq=True, need_dkv=True, dq=dq, dk=dk, dv=dv)
    torch.cuda.synchronize()
    if layout == "qkv":
        gc.check("attention_bwd dq|dk|dv")
    else:
        qc.check("attention_bwd dq")
        kc.check("attention_bwd dk")
        vc.check("attention_bwd dv")
    do64 = do.to(F64).view(B, Nq, H, d).transpose(1, 2)
    o_in = o.to(F64).view(B, Nq, H, d).transpose(1, 2)
    lk = lse_k.to(F64)
    Pb = torch.exp2(S * sl2 - lk[..., None])
    eP = 2.0**-21 + math.log(2) * (ds + 2.0**-23 * lk.abs()[..., None])       # fp32 P, relative
    dP = do64 @ v64.transpose(-1, -2)
    Bt = do64.abs() @ v64.abs().transpose(-1, -2)
    delta = (do64 * o_in).sum(-1)
    Dt = (do64.abs() * o_in.abs()).sum(-1)
    dS = Pb * (dP - delta[..., None])
    G = 1.01 * ((eP + 2.0**-8 + 2.0**-23) * Pb * (dP - delta[..., None]).abs() + Pb * ACC * (d + 16) * (Bt + Dt[..., None])
                + 2.0**-126 * ((dP - delta[..., None]).abs() + 1))             # flush to zero below 2^-126
    sc = _f32_of(scale)
    dv64 = Pb.transpose(-1, -2) @ do64
    dv_err = ((eP + 2.0**-8) * Pb + 2.0**-126).transpose(-1, -2) @ do64.abs() + ACC * (Nq + 8) * (Pb.transpose(-1, -2) @ do64.abs())
    dq64 = sc * (dS @ k64)
    dq_err = sc * (G @ k64.abs() + ACC * (Nk + 8) * (dS.abs() @ k64.abs())) + 2.0**-23 * dq64.abs() + 2.0**-125 * (Nk + 8)
    dk64 = sc * (dS.transpose(-1, -2) @ q64)
    dk_err = sc * (G.transpose(-1, -2) @ q64.abs() + ACC * (Nq + 8) * (dS.abs().transpose(-1, -2) @ q64.abs())) + 2.0**-23 * dk64.abs() + 2.0**-125 * (Nq + 8)
    assert_bf16_within(dv, _unheads(dv64), _unheads(dv_err), "attention_bwd dv vs fp64")
    assert_bf16_within(dq, _unheads(dq64), _unheads(dq_err), "attention_bwd dq vs fp64")
    assert_bf16_within(dk, _unheads(dk64), _unheads(dk_err), "attention_bwd dk vs fp64")

    if layout == "qkv":                 # need_dq=False / need_dkv=False leave the other thirds of the buffer untouched
        for need_dq, need_dkv in ((False, True), (True, False)):
            gc2, g2 = _rows(B, Nq, 3 * HD + 16, 8, 3 * HD)
            ops.attention_bwd(q, k, v, o, do, lse_k, H, scale, need_dq=need_dq, need_dkv=need_dkv,
                              dq=g2[..., :HD], dk=g2[..., HD:2 * HD], dv=g2[..., 2 * HD:])
            torch.cuda.synchronize()
            gc2.check("attention_bwd partial")
            it = torch.int16
            if need_dq:
                assert torch.equal(g2[..., :HD].view(it), dq.view(it)), "dq differs with need_dkv=False"
                assert bool((g2[..., HD:].view(it) == SENT[BF16][1]).all()), "need_dkv=False wrote dk / dv"
            else:
                assert torch.equal(g2[..., HD:].view(it), g[..., HD:].view(it)), "dk / dv differ with need_dq=False"
                assert bool((g2[..., :HD].view(it) == SENT[BF16][1]).all()), "need_dq=False wrote dq"


def test_every_head_dim_has_a_case():
    table = _head_d16_cases()
    assert table == list(range(1, 13)), table
    cased = {(p.values[4] + 15) // 16 for p in _att_cases()}
    missing = sorted(set(table) - cased)
    assert not missing, f"with_head_d16 cases without an attention case in {Path(__file__).name}: {missing}"
    assert all(D_OF_D16[k] % 8 == 0 and (D_OF_D16[k] + 15) // 16 == k for k in D_OF_D16)


# ====================================================================================================== GroupNorm
def gn_plan(n, HW, C, G, S, max_cluster=16):
    """gn_cluster_launch's choice, restated: (cl = CTAs per image, cs = channel ranges, shared-memory bytes)."""
    cpg = C // G
    cs = 1
    while G % (2 * cs) == 0 and C // (2 * cs) >= 128 and ((G // (2 * cs)) * cpg) % 8 == 0 and n * 16 * cs < 2 * S:
        cs *= 2
    Cl, Gl = C // cs, G // cs
    rows_par = 512 // (Cl // 8)
    part, gsum = 4 * 2 * rows_par * Cl, 8 * 2 * Gl
    smem = gsum + 4 * 4 * Cl + max(part, gsum)
    cl = 8 if (smem > 100 * 1024 and max_cluster > 8) else max_cluster
    while cl > 1 and (n * cl * cs > 3 * S or HW // cl < rows_par):
        cl //= 2
    return cl, cs, smem, rows_par


# (n, H, W, C, G): the comment gives (cl, cs) at 132 SMs
GN_CASES = [
    (1, 64, 64, 320, 32),     # cl 16, cs 2, groups of 10 channels
    (8, 32, 32, 640, 32),     # cl 8, cs 4 (batch 8, the UNet's 32 x 32 level), groups of 20
    (2, 15, 20, 320, 32),     # cl 8, HW = 300 not divisible by 8
    (2, 10, 15, 320, 32),     # cl 4, HW = 150
    (2, 6, 10, 320, 32),      # cl 2, HW = 60
    (2, 5, 6, 320, 32),       # cl 1, HW = 30
    (3, 16, 16, 128, 32),     # cl 8, cs 1 (C / 2 < 128), groups of 4
    (17, 8, 8, 4096, 4096),   # cl 8, cs 1: > 100 KiB of shared memory caps the cluster at 8; cpg = 1
    (1, 7, 9, 96, 96),        # cl 1, cs 1, cpg 1
    (2, 32, 32, 1280, 32),    # cl 16, cs 8, groups of 40
]


@gpu
@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("n,H,W,C,G", GN_CASES)
def test_groupnorm(n, H, W, C, G, silu):
    from controllora_b200 import ops

    _seed("gn", n, H, W, C, G, silu)
    HW = H * W
    cl, cs, smem, rows_par = gn_plan(n, HW, C, G, _sms())
    REACHED["gn"].add((cl, cs))
    x = (_f32(n, HW, C) + 0.5).to(BF16)                        # a mean offset exercises E[x^2] - mu^2
    gamma, beta = 1 + _f32(C, scale=0.3), _f32(C, scale=0.3)
    eps = 1e-6
    yc = _flat(n * HW * C, BF16, pad=64)
    y_full = yc.view.view(n, HW, C)
    sc_ = _flat(n * G * 2, F32, pad=32)
    ops._call("cl_groupnorm_fwd", ops._p(x), ops._p(gamma), ops._p(beta), ops._p(y_full), ops._p(sc_.view), n, HW, C, G,
              ct.c_float(eps), int(silu))
    torch.cuda.synchronize()
    yc.check("groupnorm y")
    sc_.check("groupnorm stats")
    stats = sc_.view.view(n, G, 2)
    cpg = C // G
    m = HW * cpg
    x64 = x.to(F64).view(n, HW, G, cpg)
    mu = x64.mean((1, 3))
    ex2 = (x64**2).mean((1, 3))
    var = (ex2 - mu**2).clamp_min(0)
    rs = 1 / torch.sqrt(var + _f32_of(eps))
    R = math.ceil(math.ceil(HW / cl) / rows_par) + rows_par + 2       # fp32 additions per channel partial sum
    e_mu = 2.0**-24 * R * x64.abs().mean((1, 3))
    e_var = 2.0**-24 * (R + 1) * ex2 + 2 * mu.abs() * e_mu
    rho = 0.5 * e_var / (var + _f32_of(eps)) + 2.0**-23
    assert_f32_within(stats[..., 0], mu, e_mu + 2.0**-24 * mu.abs(), "groupnorm mean vs fp64")
    assert_f32_within(stats[..., 1], rs, rho * rs, "groupnorm rstd vs fp64")
    g64, b64 = gamma.to(F64).view(G, cpg), beta.to(F64).view(G, cpg)
    xh = (x64 - mu[:, None, :, None]) * rs[:, None, :, None]
    z = xh * g64 + b64
    s_ = rs[:, None, :, None] * g64.abs()
    e_z = (xh.abs() * g64.abs() * rho[:, None, :, None] + s_ * e_mu[:, None, :, None]
           + 2.0**-22 * (x64.abs() * s_ + mu.abs()[:, None, :, None] * s_ + b64.abs()))
    if silu:                                                    # __expf: 2 + 1.16 |z| ulp, __fdividef: 2 ulp
        y64 = z * torch.sigmoid(z)
        e_y = 1.1 * e_z + 2.0**-22 * (6 + 1.2 * z.abs()) * y64.abs()
    else:
        y64, e_y = z, e_z
    assert_bf16_within(y_full.view(n, HW, G, cpg), y64, e_y, f"groupnorm y (cl {cl}, cs {cs}) vs fp64")

    # ---- backward from the kernel's stats
    dy = _bf(n, HW, C)
    for accumulate in (False, True):
        dxc = _flat(n * HW * C, BF16, pad=64)
        dx = dxc.view.view(n, HW, C)
        prev = _bf(n, HW, C) if accumulate else None
        if accumulate:
            dx.copy_(prev)
        dgc, dbc = _flat(C, F32, pad=8), _flat(C, F32, pad=8)
        dg0, db0 = _f32(C), _f32(C)
        dgc.view.copy_(dg0)
        dbc.view.copy_(db0)
        ops.groupnorm_bwd(x, dy, gamma, beta, stats, G, silu, dx=dx, accumulate=accumulate, dgamma=dgc.view, dbeta=dbc.view)
        torch.cuda.synchronize()
        dxc.check("groupnorm dx")
        dgc.check("groupnorm dgamma")
        dbc.check("groupnorm dbeta")
        mu_k, rs_k = stats[..., 0].to(F64)[:, None, :, None], stats[..., 1].to(F64)[:, None, :, None]
        dy64 = dy.to(F64).view(n, HW, G, cpg)
        xhk = (x64 - mu_k) * rs_k
        zk = xhk * g64 + b64
        if silu:
            sg = torch.sigmoid(zk)
            dz = dy64 * sg * (1 + zk * (1 - sg))
            e_zk = 2.0**-22 * ((x64.abs() + mu_k.abs()) * rs_k * g64.abs() + b64.abs())
            e_dz = dy64.abs() * (2.0**-22 * (6 + 1.2 * zk.abs()) * (2 + zk.abs()) + 0.5 * e_zk)
        else:
            dz, e_dz = dy64, torch.zeros_like(dy64)
        Rb = math.ceil(math.ceil(HW / cl) / rows_par) + rows_par + 4
        # per channel: a1 = sum dz, dzxh = rs (sum dz x - mu a1)
        a1 = dz.sum(1)
        t_a1 = dz.abs().sum(1)
        dzxh = (dz * xhk).sum(1)
        t_dzxh = rs_k[:, 0] * ((dz.abs() * x64.abs()).sum(1) + mu_k[:, 0].abs() * t_a1)
        e_a1 = 2.0**-24 * Rb * t_a1 + e_dz.sum(1)
        e_dzxh = 2.0**-24 * (Rb + 2) * t_dzxh + (e_dz * xhk.abs()).sum(1)
        dgam = dg0.to(F64) + dzxh.sum(0).reshape(C)
        dbet = db0.to(F64) + a1.sum(0).reshape(C)
        t_g = dg0.abs().to(F64) + t_dzxh.sum(0).reshape(C)
        t_b = db0.abs().to(F64) + t_a1.sum(0).reshape(C)
        assert_f32_within(dgc.view, dgam, e_dzxh.sum(0).reshape(C) + 2.0**-24 * (n * cl + 2) * t_g, "groupnorm dgamma vs fp64")
        assert_f32_within(dbc.view, dbet, e_a1.sum(0).reshape(C) + 2.0**-24 * (n * cl + 2) * t_b, "groupnorm dbeta vs fp64")
        Sg = (g64 * a1).sum(-1, keepdim=True)                   # [n, G, 1]: sum over the group of gamma dz
        Sgx = (g64 * dzxh).sum(-1, keepdim=True)                # sum of gamma dz xhat
        eSg = (g64.abs() * e_a1).sum(-1, keepdim=True) + 2.0**-23 * cpg * (g64.abs() * t_a1).sum(-1, keepdim=True)
        eSgx = (g64.abs() * e_dzxh).sum(-1, keepdim=True) + 2.0**-23 * cpg * (g64.abs() * t_dzxh).sum(-1, keepdim=True)
        Sg, Sgx, eSg, eSgx = (t_[:, None, :, :] for t_ in (Sg, Sgx, eSg, eSgx))
        dx64 = rs_k * g64 * dz - rs_k / m * Sg - xhk * rs_k / m * Sgx
        tdx = rs_k * g64.abs() * dz.abs() + rs_k / m * ((g64.abs() * t_a1).sum(-1)[:, None, :, None]) \
            + xhk.abs() * rs_k / m * ((g64.abs() * t_dzxh).sum(-1)[:, None, :, None])
        e_dx = rs_k * g64.abs() * e_dz + rs_k / m * eSg + (xhk.abs() + 2.0**-22 * (x64.abs() + mu_k.abs()) * rs_k) * rs_k / m * (Sgx.abs() + eSgx) \
            + 2.0**-21 * tdx
        if accumulate:
            p64 = prev.to(F64).view(n, HW, G, cpg)
            dx64 = dx64 + p64
            e_dx = e_dx + 2.0**-24 * p64.abs()
        assert_bf16_within(dx.view(n, HW, G, cpg), dx64, e_dx, f"groupnorm dx (silu {silu}, accumulate {accumulate}) vs fp64")


def test_groupnorm_cases_reach_every_cluster_choice():
    """The case list reaches every cluster size, channel ranges > 1, the > 100 KiB path, HW not divisible by the
    cluster, 10-channel groups and cpg = 1, at the H100 SXM's 132 SMs (the rule is restated in gn_plan)."""
    plans = [(gn_plan(n, H * W, C, G, 132), n, H * W, C, G) for n, H, W, C, G in GN_CASES]
    assert {p[0][0] for p in plans} == {1, 2, 4, 8, 16}, plans
    assert any(p[0][1] > 1 for p in plans)
    assert any(p[0][2] > 100 * 1024 and p[0][0] == 8 for p in plans)
    assert any(hw % p[0] for p, n, hw, c, g in plans)
    assert any(c // g == 10 for *_, c, g in plans) and any(c == g for *_, c, g in plans)


# ====================================================================================================== LayerNorm
LN_C = [8, 72, 512, 520, 768, 776, 1280, 1288, 2560]   # the four template variants (<= 512, <= 768, <= 1280, <= 2560)
LN_T = [1, 7, 17, 154]                                 # not multiples of the 16 (C <= 768) or 8 rows per block


@gpu
@pytest.mark.parametrize("T", LN_T)
@pytest.mark.parametrize("Cc", LN_C)
def test_layernorm(Cc, T):
    from controllora_b200 import ops

    _seed("ln", Cc, T)
    x = (_f32(T, Cc) + 0.25).to(BF16)
    gamma, beta = 1 + _f32(Cc, scale=0.3), _f32(Cc, scale=0.3)
    eps = 1e-5
    yc = _flat(T * Cc, BF16, pad=64)
    stc = _flat(T * 2, F32, pad=16)
    ops._call("cl_layernorm_fwd", ops._p(x), ops._p(gamma), ops._p(beta), ops._p(yc.view), ops._p(stc.view), T, Cc,
              ct.c_float(eps))
    torch.cuda.synchronize()
    yc.check("layernorm y")
    stc.check("layernorm stats")
    y, st = yc.view.view(T, Cc), stc.view.view(T, 2)
    x64 = x.to(F64)
    mu = x64.mean(-1, keepdim=True)
    var = ((x64 - mu) ** 2).mean(-1, keepdim=True)
    rs = 1 / torch.sqrt(var + _f32_of(eps))
    R = Cc // 32 + 8                                    # per-lane chain of C / 32 + 5 shuffle levels
    e_mu = 2.0**-24 * R * x64.abs().mean(-1, keepdim=True)
    rho = 0.5 * (2.0**-23 * R + e_mu**2 / (var + _f32_of(eps))) + 2.0**-21
    assert_f32_within(st[:, :1], mu, e_mu + 2.0**-24 * mu.abs(), "layernorm mean vs fp64")
    assert_f32_within(st[:, 1:], rs, rho * rs, "layernorm rstd vs fp64")
    g64, b64 = gamma.to(F64), beta.to(F64)
    xh = (x64 - mu) * rs
    y64 = xh * g64 + b64
    e_y = xh.abs() * g64.abs() * (rho + 2.0**-22) + rs * g64.abs() * e_mu + 2.0**-23 * ((x64.abs() + mu.abs()) * rs * g64.abs() + b64.abs())
    assert_bf16_within(y, y64, e_y, "layernorm y vs fp64")

    dy = _bf(T, Cc)
    for accumulate in (False, True):
        dxc = _flat(T * Cc, BF16, pad=64)
        prev = _bf(T, Cc)
        if accumulate:
            dxc.view.copy_(prev.flatten())
        ops.layernorm_bwd(x, dy, gamma, st, dx=dxc.view.view(T, Cc), accumulate=accumulate)
        torch.cuda.synchronize()
        dxc.check("layernorm dx")
        mk, rk = st[:, :1].to(F64), st[:, 1:].to(F64)
        xhk = (x64 - mk) * rk
        dg = dy.to(F64) * g64
        s1 = dg.mean(-1, keepdim=True)
        s2 = (dg * xhk).mean(-1, keepdim=True)
        dx64 = rk * (dg - s1 - xhk * s2)
        e_xh = 2.0**-23 * (x64.abs() + mk.abs()) * rk
        e_s1 = 2.0**-24 * (R + 1) * dg.abs().mean(-1, keepdim=True)
        e_s2 = 2.0**-24 * (R + 2) * (dg.abs() * xhk.abs()).mean(-1, keepdim=True) + (dg.abs() * e_xh).mean(-1, keepdim=True)
        e_dx = rk * (2.0**-21 * (dg.abs() + s1.abs() + xhk.abs() * s2.abs()) + e_s1 + xhk.abs() * e_s2 + e_xh * s2.abs())
        if accumulate:
            dx64 = dx64 + prev.to(F64)
            e_dx = e_dx + 2.0**-24 * prev.to(F64).abs()
        assert_bf16_within(dxc.view.view(T, Cc), dx64, e_dx, f"layernorm dx (accumulate {accumulate}) vs fp64")


# ====================================================================================================== coverage report
@gpu
def test_zz_report_reached_instantiations(record_property):
    """Runs last in this file: the GEMM plans (BK, BN, lora, split > 1, CTAs per SM), attention D16s and GroupNorm
    (cl, cs) the cases above reached on this device."""
    reached = {k: sorted(v) for k, v in REACHED.items()}
    print("reached:", reached)
    record_property("reached", repr(reached))
