"""Side-kernel contracts: the LoRA side path (lora.cu), the UNet-edge kernels (smallops.cu) and the glue kernels
(elementwise.cu), checked element by element against fp64 on the GPU (pytest -m gpu), at every launch branch.

Every output is a view inside a sentinel-filled canvas (tests/test_core_kernel_contracts.Canvas).  Each raw stride and
offset the C ABI takes is given a gap (so_j / so_c, ldo / col_off / lo_off, lda / ldb / ldt, the pack descriptors' ld /
row_off, the slice destination), and after the kernel every sentinel must be bit-identical.  Accumulating kernels
start from non-zero contents.

Two kinds of input per branch:
  - exact inputs: small integers (|v| <= 4) and power-of-two alpha / mul, so that every fp32 product and partial sum is
    an integer or half-integer below 2^24 and no rounding happens in any order of summation or of the atomics.  The
    kernel must then equal fp64 bit for bit, which is the only way to see one dropped, doubled or misplaced row of a
    32768-row reduction (a worst-case rounding bound over such a sum is 4e-3 of it, one row is 3e-5);
  - random inputs, with a per-element bound from the kernel's arithmetic (T = fp64 sum of |terms| of the element,
    ACC = 2^-23: one fp32 rounding of the running magnitude per operation, as in the core suite):
      skinny_atb / skinny_atb_batch / skinny_small: M fp32 products (fp32 x bf16: one rounding each) summed per thread,
        across the CTA's row groups and by one atomic per CTA, into a non-zero output: ACC (M + rows_par + CTAs + 4) T;
      rowdot: ACC (N + 8) T;  rank_update: ACC (rp + 3) T before the bf16 rounding;  rowmat: ACC (J + 2) T;
      small_matmul: ACC (J + 8) T;  conv_in: ACC (9 Cin + 2) T;  conv_out: ACC (9 C + 40) T;  conv_out_bwd: ACC 40 T;
      small_linear: ACC (K + 8) T over the (SiLU'd) inputs, plus the input SiLU's error carried through |W|;
      mse_loss: per-thread chains of L = ceil(n / threads) squares, 5 shuffle levels, 8 warps and one atomic per CTA:
        ACC (L + 16 + CTAs) T, with T = sum d^2 / n;  dpred is three fp32 roundings of the same order, restated bit for bit.
    Transcendentals (CUDA Math API, no fast-math flags in the build): erff, expf, sinf, cosf within 2 ulp; __expf within
    2 + floor(1.173 |x|) ulp.  SiLU z / (1 + __expf(-z)) (IEEE division): relative (4 + 1.2 |z|) 2^-23.  GELU:
    u = fp32(g / sqrt 2) is off by 2^-23 |u|, so erff(u) by 2^-23 (0.82 |g| + 2) and the GELU by 1/2 |g| 2^-23
    (0.82 |g| + 3) + 2^-24 |gelu|; its derivative adds the __expf term |g| 0.4 e^(-g^2/2) 2^-23 (6 + 0.9 g^2) (the 2^-24 rounding of -g^2/2 included).
    timestep_embedding: f = expf(fp32(fp32(-ln 1e4 j) / half)) within 2 ulp of exp of that fp32 argument, so
    a = fp32(t f) within 3 2^-23 |a| of t exp(.); sin / cos add 2 ulp of the result.
  - pure data movement (pack, upsample, zero insertion, concat, slice, layout changes) and the kernels whose fp32
    arithmetic has a fixed order (add, upsample2x_bwd, slice and nhwc_to_nchw_f32 accumulation) are restated in that
    order and must match bit for bit.

The CPU guards parse the launchers (every launch_k<...> instantiation, SK_CASE and CONV_IN_CASE) and restate their
runtime branch rules (skinny_atb's rows_par classes, skinny_atb_batch's template and vectorised-a choice, rank_update's
vectorised t, v2_inject_bwd's templates by C), and fail when a case list misses a branch.
"""
from __future__ import annotations

import ctypes as ct
import math
import re
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_core_kernel_contracts import Canvas, _reduction, assert_bf16_within, assert_f32_within
from tests.test_kernel_contracts import _bf16_ulp, _conv_fp64, assert_f32_reduction  # noqa: F401

BF16 = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
CSRC = Path(__file__).resolve().parent.parent / "controllora_b200" / "csrc"
ACC = 2.0**-23
H100_SMS = 132
REACHED: dict[str, set] = {}


@pytest.fixture(scope="module")
def _side_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def gpu(fn):
    return pytest.mark.gpu(pytest.mark.usefixtures("_side_gpu")(fn))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _reach(kind, key):
    REACHED.setdefault(kind, set()).add(key)


# ------------------------------------------------------------------------------------------------------------ helpers
def _seed(*params):
    torch.manual_seed(zlib.crc32(repr(params).encode()))


def _ints(*shape, lo=-4, hi=4, dtype=F32):
    return torch.randint(lo, hi + 1, shape, device="cuda").to(dtype)


def _rand(*shape, dtype=F32, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(dtype)


def _inp(exact, *shape, dtype=F32, scale=1.0):
    return _ints(*shape, dtype=dtype) if exact else _rand(*shape, dtype=dtype, scale=scale)


def _flat(n, dtype, pad=8):
    return Canvas((n + 2 * pad,), dtype, slice(pad, pad + n))


class _Strided(Canvas):
    """An as_strided view (offset, strides with gaps) of a sentinel buffer."""

    def __init__(self, shape, strides, dtype, offset=16, pad=16):
        span = offset + sum((s - 1) * st for s, st in zip(shape, strides)) + 1 + pad
        super().__init__((span,), dtype, slice(0, 0))
        self.view = torch.as_strided(self.buf, shape, strides, offset)
        torch.as_strided(self.mask, shape, strides, offset).fill_(False)


def _in_canvas(t, rows_gap=0, col_off=0, col_gap=0):
    """t [M, C] copied into a wider buffer: a view with row stride C + col_off + col_gap starting at column col_off."""
    M, Cc = t.shape
    buf = torch.zeros(M + rows_gap, Cc + col_off + col_gap, device="cuda", dtype=t.dtype)
    v = buf[:M, col_off:col_off + Cc]
    v.copy_(t)
    return v


def _exact_equal(out, ref64, what):
    """Exact inputs: every fp32 operation is exact, so the output is the fp64 value (rounded once to bf16 for bf16 outputs)."""
    if out.dtype == BF16:
        assert torch.equal(ref64.to(F32).to(F64), ref64), f"{what}: the exact inputs leave the fp32 range"
        ref64 = ref64.to(BF16).to(F64)
    o = out.to(F64)
    bad = o != ref64
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {o.numel()} elements differ from the exact fp64 value; first at flat "
                             f"index {i}: got {float(o.flatten()[i])!r}, exact {float(ref64.flatten()[i])!r}")


def _bits_equal(out, ref, what):
    it = {BF16: torch.int16, F32: torch.int32}[out.dtype]
    assert ref.dtype == out.dtype, what
    bad = out.contiguous().view(it) != ref.contiguous().view(it)
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {out.numel()} elements differ bitwise; first at flat index {i}: "
                             f"got {float(out.flatten()[i])!r}, want {float(ref.flatten()[i])!r}")


def _ulp32(x64):
    m = x64.abs().clamp_min(2.0**-126)
    _, e = torch.frexp(m)
    return torch.ldexp(torch.ones_like(m), e - 24)


def _call(name, *args):
    from controllora_b200 import ops

    ops._call(name, *args)


def _p(t):
    from controllora_b200 import ops

    return ops._p(t)


def _i64(v):
    return ct.c_int64(int(v))


def _f(v):
    return ct.c_float(float(v))


# ====================================================================================================== skinny_atb
def skinny_atb_plan(M, C, S):
    """cl_skinny_atb's launch, restated: (rows_par, threads, rows_per_cta, grid)."""
    chunks = C // 8
    rows_par = max(512 // chunks, 1)
    threads = (rows_par * chunks + 31) // 32 * 32
    if threads > 512:
        rows_par, threads = 1, (chunks + 31) // 32 * 32
    rpc = max((M + S - 1) // S, rows_par * 16)
    return rows_par, threads, rpc, (M + rpc - 1) // rpc


SKINNY_R = [1, 2, 3, 4, 8]
SKINNY_C = [8, 24, 320, 768, 800, 1280, 4096]


def _skinny_M(C, S=H100_SMS):
    rows_par = skinny_atb_plan(1, C, S)[0]
    one = max(rows_par * 16 - 5, 1)                     # one CTA
    big = min(32768, (1 << 25) // C) + 37               # a tail slab; up to 8 * 64^2 rows
    return [one, big]


def _skinny_cases():
    cases = []
    for r in SKINNY_R:
        for C in SKINNY_C:
            for M in _skinny_M(C):
                cases.append(pytest.param(r, C, M, id=f"r{r}_C{C}_M{M}"))
    return cases


def _skinny_ref(a, b, r, alpha, out0):
    a64, b64 = a[:, :r].to(F64), b.to(F64)
    return out0.to(F64) + alpha * (a64.t() @ b64), abs(alpha) * (a64.abs().t() @ b64.abs()) + out0.to(F64).abs()


@gpu
@pytest.mark.parametrize("r,C,M", _skinny_cases())
def test_skinny_atb(r, C, M):
    rows_par, threads, rpc, grid = skinny_atb_plan(M, C, _sms())
    _reach("skinny_atb", (r, rows_par == 1, (rows_par * (C // 8)) % 32 != 0, grid == 1, M % rpc != 0))
    for exact in (True, False):
        _seed("skinny", r, C, M, exact)
        a = _in_canvas(_inp(exact, M, r), col_off=1, col_gap=2)               # lda = r + 3, offset 1
        b = _in_canvas(_inp(exact, M, C, dtype=BF16), col_off=8, col_gap=8)   # ldb = C + 16
        alpha = 0.5 if exact else 0.37
        for so_j, so_c in ((C + 5, 1), (1, r + 3)):
            oc = _Strided((r, C), (so_j, so_c), F32)
            out0 = _inp(exact, r, C)
            oc.view.copy_(out0)
            _call("cl_skinny_atb", _p(a), a.stride(0), r, _p(b), _i64(b.stride(0)), _p(oc.view), _i64(so_j), _i64(so_c),
                  _f(alpha), M, C)
            torch.cuda.synchronize()
            what = f"skinny_atb<{r}> C {C} M {M} (so_j, so_c) = ({so_j}, {so_c}) {'exact' if exact else 'random'}"
            oc.check(what)
            ref, T = _skinny_ref(a, b, r, alpha, out0)
            if exact:
                _exact_equal(oc.view, ref, what)
            else:
                _reduction(oc.view, ref, T, M + rows_par + grid + 4, what)


# ====================================================================================================== skinny_atb_batch
def _batch_templates():
    src = (CSRC / "lora.cu").read_text()
    return sorted({(int(a), int(b)) for a, b in re.findall(r"launch_k\(skinny_atb_batch_kernel<(\d+), (\d+)>", src)})


def batch_plan(descs, S, templates=None):
    """cl_skinny_atb_batch's launch, restated: ((RT, U), slabs, [vec_a per descriptor]).  A descriptor is
    (M, C, r, col, lda, orient) with `a` a column view at `col` of a 16-byte aligned [M, lda] table."""
    templates = templates or _batch_templates()
    max_r = max(d[2] for d in descs)
    RT, U = min((t for t in templates if t[0] >= max_r), key=lambda t: t[0])
    max_m = max(d[0] for d in descs)
    slabs = max(min(S // len(descs), (max_m + 63) // 64), 1)
    vec = [(4 * col) % 16 == 0 and lda % 4 == 0 and lda >= RT for (M, C, r, col, lda, o) in descs]
    return (RT, U), slabs, vec


# (M, C, r, col, lda, orient): orient "dB" writes out[c, j] (so_j, so_c) = (1, r + 1), "dA" writes out[j, c] = (C + 3, 1)
SKINNY_BATCH_CASES = {
    # rank <= 4: <4, 8>.  t_out[:, col:] views of [M, 8] tables (col 0, 4: vectorised), col 1 / 2 (scalar), lda 3 < RT
    "r4_engine_views": [(32768, 320, 4, 0, 8, "dB"), (32768, 320, 4, 4, 8, "dA"), (32768, 320, 2, 1, 8, "dB"),
                        (32768, 320, 3, 2, 8, "dA"), (4096 + 77, 768, 3, 0, 3, "dB"), (1000, 1280, 1, 0, 4, "dA")],
    # rank 8 next to lower ranks: <8, 4>.  r < RT with vectorised a (lda 8 / 12 >= RT, aligned) and scalar a (col 1, lda 4 < RT)
    "r8_mixed": [(8192 + 5, 320, 8, 0, 8, "dA"), (8192 + 5, 320, 4, 4, 8, "dB"), (8192 + 5, 768, 3, 0, 12, "dA"),
                 (8192 + 5, 1280, 2, 1, 8, "dB"), (4099, 640, 4, 0, 4, "dA"), (333, 8, 8, 0, 8, "dB")],
    # M differing by 100x in one batch
    "m_ratio_100": [(32768, 320, 4, 0, 8, "dA"), (327, 320, 4, 4, 8, "dB"), (331, 1280, 2, 0, 4, "dA")],
    # max_m small: slabs clamped to ceil(max_m / 64)
    "slabs_clamped": [(200, 320, 4, 0, 8, "dA"), (150, 768, 8, 0, 8, "dB"), (3, 1280, 1, 1, 8, "dA")],
    "n1": [(32768 + 3, 1280, 4, 0, 8, "dA")],
    "n16": [(2048 + 17 * i, (320, 768, 1280, 40)[i % 4], 1 + i % 4, (0, 4, 1, 0)[i % 4], 8, ("dA", "dB")[i % 2])
            for i in range(16)],
    # 17 descriptors: the queue flushes 16 by itself, the 17th on flush()
    "n17_autoflush": [(1024 + 31 * i, (320, 768, 1280)[i % 3], (4, 8, 2)[i % 3], (0, 0, 4)[i % 3], 8, ("dA", "dB")[i % 2])
                      for i in range(17)],
}


def _batches(descs, max_n=16):
    return [descs[i:i + max_n] for i in range(0, len(descs), max_n)]


@gpu
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "random"])
@pytest.mark.parametrize("name", list(SKINNY_BATCH_CASES))
def test_skinny_atb_batch(name, exact):
    from controllora_b200 import ops

    descs = SKINNY_BATCH_CASES[name]
    S = _sms()
    _seed("skinny_batch", name, exact)
    q = ops.SkinnyQueue()
    runs = []
    for (M, C, r, col, lda, orient) in descs:
        tab = torch.zeros(M, lda, device="cuda")
        tab[:, col:col + r] = _inp(exact, M, r)
        a = tab[:, col:]                                          # what the engine passes: t_out[:, col:]
        b = _in_canvas(_inp(exact, M, C, dtype=BF16), col_off=8, col_gap=8)
        so_j, so_c = (1, r + 1) if orient == "dB" else (C + 3, 1)
        oc = _Strided((r, C), (so_j, so_c), F32)
        out0 = _inp(exact, r, C)
        oc.view.copy_(out0)
        alpha = 0.5 if exact else -0.61
        q.add(a, r, b, oc.view, so_j, so_c, alpha)
        runs.append((M, C, r, a, b, oc, out0, alpha))
    assert len(q.descs) == len(descs) % 16, "the queue flushes at 16 descriptors"
    q.flush()
    torch.cuda.synchronize()
    for batch in _batches(descs):
        (RT, U), slabs, vec = batch_plan(batch, S)
        for d, v in zip(batch, vec):
            M, C, r = d[0], d[1], d[2]
            rows_par = 512 // (C // 8)
            rpc = (M + slabs - 1) // slabs
            _reach("skinny_batch", (RT, U, v, r < RT))
            _reach("skinny_batch_C_idle", (C, (512 // (C // 8)) * (C // 8) < 512))
            _reach("skinny_batch_tail", rpc % (U * rows_par) != 0)
        _reach("skinny_batch_slabs", (len(batch), slabs < S // len(batch)))
    for i, (M, C, r, a, b, oc, out0, alpha) in enumerate(runs):
        what = f"skinny_atb_batch {name} descriptor {i} (M {M}, C {C}, r {r}, lda {a.stride(0)}) {'exact' if exact else 'random'}"
        oc.check(what)
        ref, T = _skinny_ref(a, b, r, alpha, out0)
        if exact:
            _exact_equal(oc.view, ref, what)
        else:
            rows_par = 512 // (C // 8)
            _reduction(oc.view, ref, T, M + rows_par + S + 4, what)


# ====================================================================================================== rowdot / rank_update
ROWDOT_CASES = [(rp, N, M) for rp in (4, 8) for N, M in ((8, 77), (320, 32768 + 5), (1000, 4097), (1536 if rp == 8 else 3072, 5000))]


@gpu
@pytest.mark.parametrize("rp,N,M", ROWDOT_CASES)
def test_rowdot(rp, N, M):
    assert N * rp * 4 <= 48 * 1024
    _reach("rowdot", (rp, N % 256 != 0, N * rp * 4 == 48 * 1024, M > _sms() * 4 * 8))
    for exact in (True, False):
        _seed("rowdot", rp, N, M, exact)
        a = _in_canvas(_inp(exact, M, N, dtype=BF16), col_gap=8)             # lda = N + 8
        u = _inp(exact, N, rp)
        ec = _flat(M * rp, F32, pad=64)
        _call("cl_rowdot", _p(a), _i64(a.stride(0)), _p(u), rp, _p(ec.view), M, N)
        torch.cuda.synchronize()
        what = f"rowdot<{rp}> N {N} M {M} {'exact' if exact else 'random'}"
        ec.check(what)
        e = ec.view.view(M, rp)
        ref = a.to(F64) @ u.to(F64)
        if exact:
            _exact_equal(e, ref, what)
        else:
            _reduction(e, ref, a.to(F64).abs() @ u.to(F64).abs(), N + 8, what)


def rank_update_vec_t(col, ldt):
    """rank_update's vectorised-t rule for a column view at `col` of a 16-byte aligned table with row stride ldt."""
    return (4 * col) % 16 == 0 and ldt % 4 == 0


# (rp, C, M, t layout (col, ldt), in_place)
RANK_UPDATE_CASES = [
    (4, 320, 32768, (0, 4), False), (4, 320, 32768, (1, 5), True), (4, 8, 77, (0, 8), False), (4, 3072, 300, (1, 7), False),
    (8, 1280, 8192 + 3, (0, 8), True), (8, 1280, 8192 + 3, (1, 9), False), (8, 1536, 513, (4, 12), False),
    (8, 768, 4096, (3, 11), True),
]


@gpu
@pytest.mark.parametrize("rp,C,M,tl,in_place", RANK_UPDATE_CASES)
def test_rank_update(rp, C, M, tl, in_place):
    col, ldt = tl
    _reach("rank_update", (rp, rank_update_vec_t(col, ldt), C * rp * 4 == 48 * 1024, in_place))
    for exact in (True, False):
        _seed("rank_update", rp, C, M, tl, in_place, exact)
        x0 = _inp(exact, M, C, dtype=BF16)
        tbuf = torch.zeros(M, ldt, device="cuda")
        tbuf[:, col:col + rp] = _ints(M, rp, lo=-2, hi=2) if exact else _rand(M, rp)
        t = tbuf[:, col:]
        tab = _ints(C, rp, lo=-2, hi=2) if exact else _rand(C, rp, scale=0.3)
        alpha = 0.5 if exact else 0.77
        oc = _flat(M * C, BF16, pad=64)
        out = oc.view.view(M, C)
        if in_place:
            out.copy_(x0)
            x = out
        else:
            x = x0
        _call("cl_rank_update", _p(x), _p(t), ldt, _p(tab), rp, _f(alpha), _p(out), _i64(M), C)
        torch.cuda.synchronize()
        what = f"rank_update<{rp}> C {C} M {M} t (col {col}, ldt {ldt}){' in place' if in_place else ''} {'exact' if exact else 'random'}"
        oc.check(what)
        t64, tab64 = t[:, :rp].to(F64), tab.to(F64)
        ref = x0.to(F64) + alpha * (t64 @ tab64.t())
        if exact:
            _exact_equal(out, ref, what)
        else:
            E = ACC * (rp + 3) * (x0.to(F64).abs() + abs(alpha) * (t64.abs() @ tab64.abs().t()))
            assert_bf16_within(out, ref, E, what)


# ====================================================================================================== rowmat
ROWMAT_IJ = [(1, 1), (1, 8), (3, 3), (3, 8), (8, 1), (8, 3), (8, 8), (3, 1), (1, 3)]


def _rowmat_cases():
    cases = []
    for k, (I, J) in enumerate(ROWMAT_IJ):
        for mode in ("f32", "f32_acc", "hilo"):
            cases.append(pytest.param(I, J, mode, k % 2 == 1, 1000 + 13 * k, id=f"I{I}_J{J}_{mode}_{'wT' if k % 2 else 'w'}"))
    cases.append(pytest.param(8, 8, "f32_acc", False, 300007, id="I8_J8_f32_acc_waves"))
    cases.append(pytest.param(3, 8, "hilo", True, 300007, id="I3_J8_hilo_waves"))
    return cases


@gpu
@pytest.mark.parametrize("I,J,mode,wT,M", _rowmat_cases())
def test_rowmat(I, J, mode, wT, M):
    _reach("rowmat", (mode, wT))
    for exact in (True, False):
        _seed("rowmat", I, J, mode, wT, M, exact)
        a = _in_canvas(_inp(exact, M, J), col_off=1, col_gap=1)             # lda = J + 2
        w = _inp(exact, I, J, scale=0.5)
        if wT:                                                               # w stored [J, I + 1]: sw_i = 1, sw_j = I + 1
            wb = torch.zeros(J, I + 1, device="cuda")
            wb[:, :I] = w.t()
            sw_i, sw_j, wp = 1, I + 1, wb
        else:
            wb = torch.zeros(I, J + 2, device="cuda")
            wb[:, :J] = w
            sw_i, sw_j, wp = J + 2, 1, wb
        alpha = 2.0 if exact else 0.43
        a64, w64 = a.to(F64), w.to(F64)
        s64 = alpha * (a64 @ w64.t())
        E = ACC * (J + 2) * abs(alpha) * (a64.abs() @ w64.abs().t())
        what = f"rowmat I {I} J {J} {mode} {'sw transposed' if wT else ''} M {M} {'exact' if exact else 'random'}"
        if mode.startswith("f32"):
            ldo = I + 3
            oc = Canvas((M + 2, ldo), F32, (slice(1, 1 + M), slice(0, I)))
            acc = mode == "f32_acc"
            o0 = _inp(exact, M, I)
            oc.view.copy_(o0)
            _call("cl_rowmat", _p(a), a.stride(0), _p(wp), sw_i, sw_j, I, J, _f(alpha), _p(oc.view), ldo, 0, 0, 0, int(acc), M)
            torch.cuda.synchronize()
            oc.check(what)
            ref = s64 + (o0.to(F64) if acc else 0)
            if exact:
                _exact_equal(oc.view, ref, what)
            else:
                assert_f32_within(oc.view, ref, E + (2.0**-24 * ref.abs() + ACC * o0.to(F64).abs() if acc else 0), what)
        else:
            ldo, col_off, lo_off = 24, 1, 9
            oc = Canvas((M + 2, ldo), BF16, (slice(1, 1 + M), slice(col_off, col_off + I)))
            oc.mask[1:1 + M, col_off + lo_off:col_off + lo_off + I] = False
            base = oc.buf[1:]
            _call("cl_rowmat", _p(a), a.stride(0), _p(wp), sw_i, sw_j, I, J, _f(alpha), _p(base), ldo, 1, col_off, lo_off, 0, M)
            torch.cuda.synchronize()
            oc.check(what)
            hi = base[:M, col_off:col_off + I]
            lo = base[:M, col_off + lo_off:col_off + lo_off + I]
            if exact:
                s32 = s64.to(F32) + 0.0                       # the kernel's sum starts from +0: no -0 results
                assert torch.equal(s32.to(F64), s64), "exact inputs must give an fp32-exact sum"
                h = s32.to(BF16)
                _bits_equal(hi, h, what + " hi")
                _bits_equal(lo, (s32 - h.to(F32)).to(BF16), what + " lo")
            else:
                assert_bf16_within(hi, s64, E, what + " hi")
                assert_bf16_within(lo, s64 - hi.to(F64), E, what + " lo")


# ====================================================================================================== skinny_small / small_matmul
SKINNY_SMALL_CASES = [(I, (3 * I) % 8 + 1, M) for I in range(1, 9) for M in (1000,)] + [(8, 8, 100003), (2, 7, 100003)]


@gpu
@pytest.mark.parametrize("I,J,M", SKINNY_SMALL_CASES)
def test_skinny_small(I, J, M):
    _reach("skinny_small", (I, J, M > _sms() * 256))
    for exact in (True, False):
        _seed("skinny_small", I, J, M, exact)
        a = _in_canvas(_inp(exact, M, I), col_off=2, col_gap=1)
        b = _in_canvas(_inp(exact, M, J), col_off=1, col_gap=3)
        oc = _flat(I * J, F32, pad=32)
        o0 = _inp(exact, I * J)
        oc.view.copy_(o0)
        alpha = 0.5 if exact else 1.3
        _call("cl_skinny_small", _p(a), a.stride(0), I, _p(b), b.stride(0), J, _p(oc.view), _f(alpha), M)
        torch.cuda.synchronize()
        what = f"skinny_small I {I} J {J} M {M} {'exact' if exact else 'random'}"
        oc.check(what)
        ref = o0.to(F64).view(I, J) + alpha * (a.to(F64).t() @ b.to(F64))
        if exact:
            _exact_equal(oc.view.view(I, J), ref, what)
        else:
            T = o0.to(F64).abs().view(I, J) + abs(alpha) * (a.to(F64).abs().t() @ b.to(F64).abs())
            _reduction(oc.view.view(I, J), ref, T, M + 2 * _sms() + 16, what)


# (I, J, K, transposed a, transposed b, transposed out)
SMALL_MATMUL_CASES = [(1, 1, 1, False, False, False), (3, 5, 7, True, False, True), (8, 31, 8, False, True, False),
                      (8, 100, 320, True, True, True), (4, 33, 4000, False, False, True), (320, 8, 40, True, False, False),
                      (5, 64, 3, False, True, True)]


@gpu
@pytest.mark.parametrize("I,J,K,ta,tb,to", SMALL_MATMUL_CASES)
def test_small_matmul(I, J, K, ta, tb, to):
    _reach("small_matmul", (J < 32, J % 32 != 0, I * K > _sms() * 64, ta, tb, to))
    for exact in (True, False):
        for acc in (False, True):
            _seed("small_matmul", I, J, K, ta, tb, to, exact, acc)
            A, B = _inp(exact, I, J), _inp(exact, J, K)
            ab = torch.zeros((J, I + 3) if ta else (I, J + 2), device="cuda")
            (ab[:, :I] if ta else ab[:, :J]).copy_(A.t() if ta else A)
            sa_i, sa_j = (1, I + 3) if ta else (J + 2, 1)
            bb = torch.zeros((K, J + 1) if tb else (J, K + 5), device="cuda")
            (bb[:, :J] if tb else bb[:, :K]).copy_(B.t() if tb else B)
            sb_j, sb_k = (1, J + 1) if tb else (K + 5, 1)
            so_i, so_k = (1, I + 2) if to else (K + 3, 1)
            oc = _Strided((I, K), (so_i, so_k), F32)
            o0 = _inp(exact, I, K)
            oc.view.copy_(o0)
            alpha = 0.25 if exact else -0.9
            _call("cl_small_matmul", _p(ab), _i64(sa_i), _i64(sa_j), _p(bb), _i64(sb_j), _i64(sb_k), _p(oc.view), _i64(so_i),
                  _i64(so_k), I, J, K, _f(alpha), int(acc))
            torch.cuda.synchronize()
            what = f"small_matmul I {I} J {J} K {K} ({ta}, {tb}, {to}) accumulate {acc} {'exact' if exact else 'random'}"
            oc.check(what)
            p64 = alpha * (A.to(F64) @ B.to(F64))
            ref = p64 + (o0.to(F64) if acc else 0)
            if exact:
                _exact_equal(oc.view, ref, what)
            else:
                T = abs(alpha) * (A.to(F64).abs() @ B.to(F64).abs()) + (o0.to(F64).abs() if acc else 0)
                assert_f32_within(oc.view, ref, ACC * (J + 8) * T, what)


# ====================================================================================================== lora_pack_batch
@gpu
@pytest.mark.parametrize("mul", [1.0, 0.5, 1 / 0.7])
def test_lora_pack_batch(mul):
    """kinds 0 (hi/lo rows of ext), 1 (fp32 table columns) and 2 (bf16 transposed hi | hi columns), with row_off != 0,
    transposed source strides, r K > 16 * 256 (the grid-stride loop wraps), and sentinels in every row and column no
    descriptor covers; the result is pure rounding, so it is restated bit for bit."""
    from controllora_b200 import ops

    _seed("pack", mul)
    plan = ops.PackPlan(torch.device("cuda"))
    checks = []
    # kind 0: ext [16, K + 8]: rows 0..3 from src [4, K], rows 5..7 from a transposed [K, 3] source
    K0 = 1288
    ext = Canvas((16, K0 + 8), BF16, (slice(0, 0), slice(0, 0)))
    s0 = _rand(4, K0)
    s0t = _rand(K0 + 2, 5)[:K0, 1:4]                            # [K, 3] view, s_j = 1, s_k = 5
    plan.add(s0, ext.buf, 0, 4, K0, s0.stride(0), 1, K0 + 8, 0, unscaled=mul != 1.0)
    plan.add(s0t, ext.buf, 0, 3, K0, 1, s0t.stride(0), K0 + 8, 5, unscaled=mul != 1.0)
    for rows, src in ((slice(0, 4), s0), (slice(5, 8), s0t.t())):
        ext.mask[rows, :K0] = False
        ext.mask[rows.start + 8:rows.stop + 8, :K0] = False
        checks.append(("ext", ext, rows, src, 0))
    # kind 1: table [N + 3, 12] fp32, columns 2..9 from a transposed source (down.weight [8, N]) and 10..11 from up [N, 2]
    N1 = 1280
    tab = Canvas((N1 + 3, 12), F32, (slice(0, 0), slice(0, 0)))
    s1 = _rand(8, N1)                                           # r = 8, K = N: r K = 10240 > 4096
    s1u = _rand(N1, 2)
    plan.add(s1, tab.buf, 1, 8, N1, s1.stride(0), 1, 12, 2)
    plan.add(s1u, tab.buf, 1, 2, N1, 1, s1u.stride(0), 12, 10, unscaled=mul != 1.0)
    tab.mask[:N1, 2:12] = False
    # kind 2: bf16 [K + 2, 20]: columns 1..4 and 9..12 both hi(src)
    K2 = 777
    tb = Canvas((K2 + 2, 20), BF16, (slice(0, 0), slice(0, 0)))
    s2 = _rand(4, K2)
    plan.add(s2, tb.buf, 2, 4, K2, s2.stride(0), 1, 20, 1, unscaled=mul != 1.0)
    tb.mask[:K2, 1:5] = False
    tb.mask[:K2, 9:13] = False
    plan.set_unscaled_mul(mul)
    plan.run()
    torch.cuda.synchronize()
    m = torch.tensor(mul, dtype=F32).item()
    ext.check("pack kind 0")
    tab.check("pack kind 1")
    tb.check("pack kind 2")
    v0 = s0 * m if mul != 1.0 else s0
    v0t = s0t.t() * m if mul != 1.0 else s0t.t()
    for rows, v in ((slice(0, 4), v0), (slice(5, 8), v0t)):
        hi = v.to(BF16)
        _bits_equal(ext.buf[rows, :K0], hi, f"pack kind 0 hi rows {rows}")
        _bits_equal(ext.buf[rows.start + 8:rows.stop + 8, :K0], (v - hi.to(F32)).to(BF16), f"pack kind 0 lo rows {rows}")
    _bits_equal(tab.buf[:N1, 2:10], s1.t().contiguous(), "pack kind 1 (mul 1)")
    _bits_equal(tab.buf[:N1, 10:12], s1u * m if mul != 1.0 else s1u, "pack kind 1 unscaled")
    h2 = (s2 * m if mul != 1.0 else s2).t().to(BF16)
    _bits_equal(tb.buf[:K2, 1:5], h2, "pack kind 2 hi")
    _bits_equal(tb.buf[:K2, 9:13], h2, "pack kind 2 hi (second slot)")
    _reach("pack", (0, 1, 2, mul != 1.0))


# ====================================================================================================== conv_in / conv_out
CONV_IN_CASES = [(n, Cin, H, W, Cout, bias) for (n, Cin, H, W, Cout, bias) in [
    (1, 3, 5, 7, 8, True), (2, 4, 9, 11, 40, False), (1, 4, 64, 64, 320, True), (2, 3, 13, 1, 72, True),
    (1, 4, 1, 17, 320, False), (3, 4, 16, 16, 96, True), (1, 3, 23, 29, 328, False), (2, 3, 31, 33, 320, True)]]


@gpu
@pytest.mark.parametrize("n,Cin,H,W,Cout,bias", CONV_IN_CASES)
def test_conv_in(n, Cin, H, W, Cout, bias):
    _reach("conv_in", (Cin, Cout % 32 != 0, bias, (n * H * W) % 256 != 0))
    for exact in (True, False):
        _seed("conv_in", n, Cin, H, W, Cout, bias, exact)
        x = _inp(exact, n, Cin, H, W) if exact else _rand(n, Cin, H, W) * 1.3      # fp32, rounded to bf16 by the kernel
        w = _inp(exact, Cout, 9 * Cin, dtype=BF16, scale=0.3)
        b = _inp(exact, Cout) if bias else None
        yc = _flat(n * H * W * Cout, BF16, pad=64)
        _call("cl_conv_in", _p(x), _p(w), _p(b), _p(yc.view), n, Cin, H, W, Cout)
        torch.cuda.synchronize()
        what = f"conv_in Cin {Cin} Cout {Cout} {n}x{H}x{W} bias {bias} {'exact' if exact else 'random'}"
        yc.check(what)
        x64 = x.to(BF16).to(F64)
        w64 = w.to(F64).view(Cout, 3, 3, Cin).permute(0, 3, 1, 2)
        ref = _conv_fp64(x64, w64, 3, 1, 1)
        T = _conv_fp64(x64.abs(), w64.abs(), 3, 1, 1)
        if b is not None:
            ref = ref + b.to(F64)[:, None, None]
            T = T + b.to(F64).abs()[:, None, None]
        y = yc.view.view(n, H, W, Cout).permute(0, 3, 1, 2)
        if exact:
            _exact_equal(y, ref, what)
        else:
            assert_bf16_within(y, ref, ACC * (9 * Cin + 2) * T, what)


CONV_OUT_C_MAX = (200 * 1024) // (4 * 9 * 2) // 8 * 8      # 2840: the [4][9][C] bf16 weights fill 200 KB
CONV_OUT_CASES = [(1, 1, 1, 8), (2, 1, 37, 320), (2, 29, 1, 320), (2, 64, 64, 320), (1, 7, 5, CONV_OUT_C_MAX), (3, 9, 11, 40),
                  (1, 32, 32, 1280)]


@gpu
@pytest.mark.parametrize("n,H,W,C", CONV_OUT_CASES)
def test_conv_out(n, H, W, C):
    waves = n * H * W > _sms() * 4 * 8
    _reach("conv_out", (C == CONV_OUT_C_MAX, H == 1 or W == 1, waves))
    for exact in (True, False):
        _seed("conv_out", n, H, W, C, exact)
        x = _inp(exact, n, H, W, C, dtype=BF16)
        w = _inp(exact, 4, 9 * C, dtype=BF16, scale=C**-0.5)
        b = _inp(exact, 4)
        yc = _flat(n * 4 * H * W, F32, pad=64)
        _call("cl_conv_out", _p(x), _p(w), _p(b), _p(yc.view), n, H, W, C, 4)
        torch.cuda.synchronize()
        what = f"conv_out C {C} {n}x{H}x{W} {'exact' if exact else 'random'}"
        yc.check(what)
        x64 = x.to(F64).permute(0, 3, 1, 2)
        w64 = w.to(F64).view(4, 3, 3, C).permute(0, 3, 1, 2)
        ref = _conv_fp64(x64, w64, 3, 1, 1) + b.to(F64)[:, None, None]
        T = _conv_fp64(x64.abs(), w64.abs(), 3, 1, 1) + b.to(F64).abs()[:, None, None]
        y = yc.view.view(n, 4, H, W)
        if exact:
            _exact_equal(y, ref, what)
        else:
            assert_f32_within(y, ref, ACC * (9 * C + 40) * T, what)

        dy = _inp(exact, n, 4, H, W)
        dc = _flat(n * H * W * C, BF16, pad=64)
        _call("cl_conv_out_bwd", _p(dy), _p(w), _p(dc.view), n, H, W, C, 4)
        torch.cuda.synchronize()
        what = f"conv_out_bwd C {C} {n}x{H}x{W} {'exact' if exact else 'random'}"
        dc.check(what)
        dx = dc.view.view(n, H, W, C).permute(0, 3, 1, 2)
        dref = F.conv_transpose2d(dy.to(F64), w64, padding=1)
        dT = F.conv_transpose2d(dy.to(F64).abs(), w64.abs(), padding=1)
        if exact:
            _exact_equal(dx, dref, what)
        else:
            assert_bf16_within(dx, dref, ACC * 40 * dT, what)


# ====================================================================================================== small_linear
SMALL_LINEAR_K_MAX = 48 * 1024 // (8 * 4)     # 1536: eight batch rows of fp32 inputs in 48 KB
SMALL_LINEAR_CASES = [(Bt, N, K) for Bt, N, K in [(1, 1280, 320), (8, 1283, 1280), (9, 1283, SMALL_LINEAR_K_MAX), (17, 77, 8),
                                                    (2, 3, 1536)]]


def _silu_err(z):
    """|fp32 SiLU(z) - silu(z)| for an exact fp32 input z (z / (1 + __expf(-z)), IEEE division)."""
    return (4 + 1.2 * z.abs()) * ACC * (z * torch.sigmoid(z)).abs() + 2.0**-140


@gpu
@pytest.mark.parametrize("silu_in,silu_out", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("Bt,N,K", SMALL_LINEAR_CASES)
def test_small_linear(Bt, N, K, silu_in, silu_out):
    _reach("small_linear", (Bt > 8, N % 8 != 0, K == SMALL_LINEAR_K_MAX, silu_in, silu_out))
    for exact in ((True, False) if not (silu_in or silu_out) else (False,)):
        _seed("small_linear", Bt, N, K, silu_in, silu_out, exact)
        x = _inp(exact, Bt, K, scale=2.0)
        w = _inp(exact, N, K, dtype=BF16, scale=K**-0.5)
        b = _inp(exact, N)
        oc = _flat(Bt * N, F32, pad=64)
        _call("cl_small_linear", _p(x), _p(w), _p(b), _p(oc.view), Bt, N, K, int(silu_in), int(silu_out))
        torch.cuda.synchronize()
        what = f"small_linear Bt {Bt} N {N} K {K} silu ({silu_in}, {silu_out}) {'exact' if exact else 'random'}"
        oc.check(what)
        x64, w64, b64 = x.to(F64), w.to(F64), b.to(F64)
        xin = x64 * torch.sigmoid(x64) if silu_in else x64
        ein = _silu_err(x64) if silu_in else torch.zeros_like(x64)
        s = xin @ w64.t() + b64
        Es = ACC * (K + 8) * ((xin.abs() + ein) @ w64.abs().t() + b64.abs()) + ein @ w64.abs().t()
        out = oc.view.view(Bt, N)
        if silu_out:
            ref = s * torch.sigmoid(s)
            E = 1.1 * Es + _silu_err(s) * 1.01
        else:
            ref, E = s, Es
        if exact:
            _exact_equal(out, ref, what)
        else:
            assert_f32_within(out, ref, E, what)


# ====================================================================================================== timestep_embedding / mse
@gpu
@pytest.mark.parametrize("dim", [320, 322, 2, 1280])
def test_timestep_embedding(dim):
    """diffusers get_timestep_embedding (flip_sin_to_cos, freq_shift 0) restated in fp64 from the fp32 argument of exp."""
    half = dim // 2
    _reach("timestep_embedding", half % 2 == 1)
    _seed("temb", dim)
    t = torch.cat([torch.tensor([0.0, 1.0, 999.0, 500.0, 998.5], device="cuda"), torch.rand(300, device="cuda") * 999])
    B = t.numel()
    oc = _flat(B * dim, F32, pad=32)
    _call("cl_timestep_embedding", _p(t), _p(oc.view), B, dim)
    torch.cuda.synchronize()
    oc.check("timestep_embedding")
    # the fp32 argument of exp in the kernel's order, with IEEE division (numpy: torch divides by a scalar through its
    # reciprocal, which is up to an ulp away)
    expo = (np.float32(-9.210340371976184) * np.arange(half, dtype=np.float32)) / np.float32(half)
    f64 = torch.exp(torch.from_numpy(expo.astype(np.float64)).cuda())
    a64 = t.to(F64)[:, None] * f64[None, :]
    Ea = 3 * ACC * a64.abs() + 2.0**-149
    out = oc.view.view(B, dim)
    for part, ref in ((out[:, :half], torch.cos(a64)), (out[:, half:], torch.sin(a64))):
        E = Ea + 2 * _ulp32(ref.abs() + Ea) * 2
        assert_f32_within(part, ref, E, f"timestep_embedding dim {dim}")


MSE_CASES = [(1, 1.0, True), (65536, 1.0, True), (65536, 0.25, True), (1000003, 3.0, True), (1000003, 1.0, False),
             (4 * 4 * 64 * 64 + 5, 65536.0, True)]


@gpu
@pytest.mark.parametrize("n,gscale,need_grad", MSE_CASES)
def test_mse_loss(n, gscale, need_grad):
    S = _sms()
    blocks = min((n + 255) // 256, S * 4)
    _reach("mse", (n % 256 != 0, (n + 255) // 256 > S * 4, gscale != 1.0, need_grad))
    for exact in ((True, False) if n & (n - 1) == 0 else (False,)):
        _seed("mse", n, gscale, need_grad, exact)
        pred, target = _inp(exact, n), _inp(exact, n)
        lc = _flat(1, F32, pad=4)
        lc.view.fill_(123.0)                                   # the launcher clears the loss
        dc = _flat(n, F32, pad=64) if need_grad else None
        _call("cl_mse_loss", _p(pred), _p(target), _p(lc.view), _p(dc.view if dc else None), _i64(n), _f(gscale))
        torch.cuda.synchronize()
        what = f"mse_loss n {n} gscale {gscale} {'exact' if exact else 'random'}"
        lc.check(what)
        d64 = pred.to(F64) - target.to(F64)
        ref = (d64**2).sum() / n
        if exact:
            _exact_equal(lc.view, ref.view(1), what)
        else:
            L = math.ceil(n / (blocks * 256))
            _reduction(lc.view, ref.view(1), ref.view(1), L + 16 + blocks, what + " loss")
        if need_grad:
            dc.check(what + " dpred")
            inv = torch.tensor(1.0, dtype=F32, device="cuda") / torch.tensor(float(n), dtype=F32, device="cuda")
            d32 = pred - target
            _bits_equal(dc.view, ((2.0 * d32) * inv) * torch.tensor(gscale, dtype=F32, device="cuda"), what + " dpred")


# ====================================================================================================== GEGLU / add
GEGLU_CASES = [(1, 8), (77, 8), (4096 + 5, 1280), (300, 1280), (33, 640)]


def _gelu_terms(g64):
    erf = torch.erf(g64 / math.sqrt(2))
    gelu = 0.5 * g64 * (1 + erf)
    e_gelu = 0.5 * g64.abs() * ACC * (0.82 * g64.abs() + 3) + 2.0**-24 * gelu.abs()
    dens = g64 / math.sqrt(2 * math.pi) * torch.exp(-0.5 * g64 * g64)
    ggrad = 0.5 * (1 + erf) + dens
    e_ggrad = 0.5 * ACC * (0.82 * g64.abs() + 3) + dens.abs() * ACC * (6 + 0.9 * g64 * g64) + ACC * ggrad.abs()
    return gelu, e_gelu, ggrad, e_ggrad


@gpu
@pytest.mark.parametrize("T,Fd", GEGLU_CASES)
def test_geglu(T, Fd):
    _reach("geglu", (Fd, T * Fd // 8 > _sms() * 16 * 256))
    _seed("geglu", T, Fd)
    p = _rand(T, 2 * Fd, dtype=BF16, scale=2.0)
    oc = _flat(T * Fd, BF16, pad=64)
    _call("cl_geglu_fwd", _p(p), _p(oc.view), _i64(T), Fd)
    dout = _rand(T, Fd, dtype=BF16)
    dc = _flat(T * 2 * Fd, BF16, pad=64)
    _call("cl_geglu_bwd", _p(p), _p(dout), _p(dc.view), _i64(T), Fd)
    torch.cuda.synchronize()
    oc.check("geglu_fwd")
    dc.check("geglu_bwd")
    a64, g64, d64 = p[:, :Fd].to(F64), p[:, Fd:].to(F64), dout.to(F64)
    gelu, e_gelu, ggrad, e_ggrad = _gelu_terms(g64)
    out = a64 * gelu
    assert_bf16_within(oc.view.view(T, Fd), out, 1.01 * (a64.abs() * e_gelu + 2.0**-24 * out.abs()), f"geglu_fwd T {T} F {Fd}")
    dp = dc.view.view(T, 2 * Fd)
    da = d64 * gelu
    assert_bf16_within(dp[:, :Fd], da, 1.01 * (d64.abs() * e_gelu + 2.0**-24 * da.abs()), f"geglu_bwd da T {T} F {Fd}")
    dg = d64 * a64 * ggrad
    assert_bf16_within(dp[:, Fd:], dg, 1.01 * ((d64 * a64).abs() * e_ggrad + 2.0**-23 * dg.abs()), f"geglu_bwd dg T {T} F {Fd}")


@gpu
@pytest.mark.parametrize("n", [8, 8 * 1001, H100_SMS * 16 * 256 * 8 + 24])
def test_add(n):
    _seed("add", n)
    a, b = _rand(n, dtype=BF16), _rand(n, dtype=BF16, scale=100.0)
    oc = _flat(n, BF16, pad=16)
    _call("cl_add", _p(a), _p(b), _p(oc.view), _i64(n))
    torch.cuda.synchronize()
    oc.check("add")
    _bits_equal(oc.view, (a.to(F32) + b.to(F32)).to(BF16), f"add n {n}")


# ====================================================================================================== upsample / zero insertion
UPS_CASES = [(1, 1, 1, 8), (2, 3, 5, 8), (1, 7, 9, 40), (2, 64, 64, 320), (1, 16, 16, 1280)]


@gpu
@pytest.mark.parametrize("n,H,W,C", UPS_CASES)
def test_upsample2x(n, H, W, C):
    _reach("upsample", (C == 8, H % 2 == 1 or W % 2 == 1, n * 4 * H * W * C // 8 > _sms() * 16 * 256))
    _seed("ups", n, H, W, C)
    x = _rand(n, H, W, C, dtype=BF16)
    yc = _flat(n * 4 * H * W * C, BF16, pad=64)
    _call("cl_upsample2x_fwd", _p(x), _p(yc.view), n, H, W, C)
    torch.cuda.synchronize()
    yc.check("upsample2x_fwd")
    _bits_equal(yc.view.view(n, 2 * H, 2 * W, C), x.repeat_interleave(2, 1).repeat_interleave(2, 2), f"upsample2x_fwd {n}x{H}x{W}x{C}")
    dy = _rand(n, 2 * H, 2 * W, C, dtype=BF16)
    for acc in (False, True):
        dc = _flat(n * H * W * C, BF16, pad=64)
        d0 = _rand(n, H, W, C, dtype=BF16)
        dc.view.copy_(d0.flatten())
        _call("cl_upsample2x_bwd", _p(dy), _p(dc.view), n, H, W, C, int(acc))
        torch.cuda.synchronize()
        dc.check("upsample2x_bwd")
        s = d0.to(F32) if acc else torch.zeros(n, H, W, C, device="cuda")
        d = dy.to(F32)
        for yy in range(2):
            for xx in range(2):
                s = s + d[:, yy::2, xx::2]
        _bits_equal(dc.view.view(n, H, W, C), s.to(BF16), f"upsample2x_bwd {n}x{H}x{W}x{C} accumulate {acc}")
    for off in (0, 1):
        zc = _flat(n * 4 * H * W * C, BF16, pad=64)
        _call("cl_zero_insert2x", _p(x), _p(zc.view), n, H, W, C, off)
        torch.cuda.synchronize()
        zc.check("zero_insert2x")
        z = torch.zeros(n, 2 * H, 2 * W, C, device="cuda", dtype=BF16)
        z[:, off::2, off::2] = x
        _bits_equal(zc.view.view(n, 2 * H, 2 * W, C), z, f"zero_insert2x {n}x{H}x{W}x{C} off {off}")


# ====================================================================================================== concat / slice
CONCAT_CASES = [(1, 8, 8), (77, 8, 320), (4096 + 3, 320, 640), (300, 1280, 8), (H100_SMS * 16 * 256 // 8 + 5, 64, 8)]


@gpu
@pytest.mark.parametrize("M,Ca,Cb", CONCAT_CASES)
def test_concat_and_slice(M, Ca, Cb):
    _reach("concat_slice", (min(Ca, Cb) == 8,))
    _seed("concat", M, Ca, Cb)
    a, b = _rand(M, Ca, dtype=BF16), _rand(M, Cb, dtype=BF16)
    oc = _flat(M * (Ca + Cb), BF16, pad=64)
    _call("cl_concat_channels", _p(a), _p(b), _p(oc.view), _i64(M), Ca, Cb)
    torch.cuda.synchronize()
    oc.check("concat_channels")
    cat = oc.view.view(M, Ca + Cb)
    _bits_equal(cat, torch.cat([a, b], 1), f"concat M {M} Ca {Ca} Cb {Cb}")
    for c_off, Cd in ((0, Ca), (Ca, Cb), (8, Ca + Cb - 8) if Ca + Cb > 8 else (0, 8)):
        for acc in (False, True):
            sc = _flat(M * Cd, BF16, pad=64)
            d0 = _rand(M, Cd, dtype=BF16)
            sc.view.copy_(d0.flatten())
            _call("cl_slice_channels", _p(cat), _p(sc.view), _i64(M), Ca + Cb, c_off, Cd, int(acc))
            torch.cuda.synchronize()
            sc.check("slice_channels")
            want = cat[:, c_off:c_off + Cd]
            want = (want.to(F32) + d0.to(F32)).to(BF16) if acc else want
            _bits_equal(sc.view.view(M, Cd), want, f"slice M {M} [{c_off}, {c_off + Cd}) accumulate {acc}")


# ====================================================================================================== layout changes
LAYOUT_CASES = [(1, 8, 1, 1), (2, 8, 7, 9), (1, 40, 5, 13), (2, 320, 32, 32), (1, 4, 64, 64), (3, 33, 3, 11)]


@gpu
@pytest.mark.parametrize("n,C,H,W", LAYOUT_CASES)
def test_layout_changes(n, C, H, W):
    _reach("layout", ((H * W) % 32 != 0, C % 32 != 0))
    _seed("layout", n, C, H, W)
    for dt in (F32, BF16):
        x = _rand(n, C, H, W, dtype=dt)
        yc = _flat(n * H * W * C, BF16, pad=64)
        _call("cl_nchw_to_nhwc", _p(x), int(dt == F32), _p(yc.view), n, C, H * W)
        torch.cuda.synchronize()
        yc.check("nchw_to_nhwc")
        _bits_equal(yc.view.view(n, H, W, C), x.permute(0, 2, 3, 1).to(BF16), f"nchw_to_nhwc {dt} {n}x{C}x{H}x{W}")
        _reach("nchw_to_nhwc", str(dt))
    xh = _rand(n, H, W, C, dtype=BF16)
    for acc in (False, True):
        yc = _flat(n * C * H * W, F32, pad=64)
        y0 = _rand(n, C, H, W)
        yc.view.copy_(y0.flatten())
        _call("cl_nhwc_to_nchw_f32", _p(xh), _p(yc.view), n, C, H * W, int(acc))
        torch.cuda.synchronize()
        yc.check("nhwc_to_nchw_f32")
        want = xh.permute(0, 3, 1, 2).to(F32)
        _bits_equal(yc.view.view(n, C, H, W), y0 + want if acc else want.contiguous(), f"nhwc_to_nchw_f32 accumulate {acc}")
    n8 = n * C * H * W
    f = _rand(n8)
    bc = _flat(n8, BF16, pad=16)
    _call("cl_f32_to_bf16", _p(f), _p(bc.view), _i64(n8))
    fc = _flat(n8, F32, pad=16)
    _call("cl_bf16_to_f32", _p(bc.view), _p(fc.view), _i64(n8))
    torch.cuda.synchronize()
    bc.check("f32_to_bf16")
    fc.check("bf16_to_f32")
    _bits_equal(bc.view, f.to(BF16), "f32_to_bf16")
    _bits_equal(fc.view, f.to(BF16).to(F32), "bf16_to_f32")


# ====================================================================================================== CPU guards
SIDE_FILES = ("lora.cu", "smallops.cu", "elementwise.cu")
# kernels of these files whose fp64 cases live in tests/test_kernel_contracts.py (V2 injection, weight-space and VAE /
# CLIP helpers) or in the sampler suites
ELSEWHERE = {"v2_inject_fwd_kernel", "v2_inject_bwd_kernel", "hilo_combine_kernel", "cast_matrix_kernel",
             "axpy_matrix_kernel", "softmax_rows_kernel", "channel_affine_nchw_kernel", "clip_embed_kernel",
             "quick_gelu_kernel", "causal_attention_small_kernel", "cfg_ddim_kernel", "cfg_dpmpp_kernel",
             "sampler_prep_kernel", "cfg_solver_dev_kernel", "counter_advance_kernel"}


def _launched(fname):
    """(kernel, template arguments) of every launch_k in a source file, with SK_CASE / CONV_IN_CASE expanded."""
    src = (CSRC / fname).read_text()
    out = set()
    for name, targs in re.findall(r"launch_k\((?:clb::)?(\w+)(?:<([^>]*)>)?\s*,", src):
        targs = targs.replace(" ", "")
        if targs in ("R", "CI"):
            continue                                             # the macro bodies: expanded below
        out.add((name, targs))
    sk = [int(v) for v in re.findall(r"SK_CASE\((\d+)\)", src)]
    out |= {("skinny_atb_kernel", str(r)) for r in sk}
    ci = [int(v) for v in re.findall(r"CONV_IN_CASE\((\d+)\)", src)]
    out |= {("conv_in_kernel", str(c)) for c in ci}
    return out


def _cased_instantiations():
    cased = {("skinny_atb_kernel", str(r)) for r in SKINNY_R}
    for descs in SKINNY_BATCH_CASES.values():
        for batch in _batches(descs):
            (RT, U), _, _ = batch_plan(batch, H100_SMS)
            cased.add(("skinny_atb_batch_kernel", f"{RT},{U}"))
    cased |= {("rowdot_kernel", str(rp)) for rp, _, _ in ROWDOT_CASES}
    cased |= {("rank_update_kernel", str(c[0])) for c in RANK_UPDATE_CASES}
    cased |= {("conv_in_kernel", str(c[1])) for c in CONV_IN_CASES}
    cased |= {("conv_out_kernel", "4"), ("conv_out_bwd_kernel", "4")}
    cased |= {("nchw_to_nhwc_kernel", "float"), ("nchw_to_nhwc_kernel", "__nv_bfloat16")}
    cased |= {(k, "") for k in ("lora_pack_kernel", "rowmat_kernel", "skinny_small_kernel", "small_matmul_kernel",
                                "timestep_embedding_kernel", "small_linear_kernel", "mse_kernel", "geglu_fwd_kernel",
                                "geglu_bwd_kernel", "add_kernel", "upsample2x_kernel", "upsample2x_bwd_kernel",
                                "zero_insert2x_kernel", "concat_kernel", "slice_kernel", "nhwc_to_nchw_f32_kernel",
                                "f32_to_bf16_kernel", "bf16_to_f32_kernel")}
    return cased


def test_every_side_kernel_instantiation_has_a_case():
    launched = set().union(*(_launched(f) for f in SIDE_FILES))
    assert ("skinny_atb_batch_kernel", "4,8") in launched and ("skinny_atb_kernel", "8") in launched, launched
    mine = {k for k in launched if k[0] not in ELSEWHERE}
    cased = _cased_instantiations()
    missing = sorted(mine - cased)
    assert not missing, f"side-kernel instantiations without a case in {Path(__file__).name}: {missing}"
    extra = sorted(cased - mine)
    assert not extra, f"cases for instantiations the launchers no longer have: {extra}"


def test_skinny_atb_cases_reach_every_rows_par_class():
    """rows_par 512 (C 8) and 1 (C 4096), blocks with idle threads (C 24, 800), one CTA and a tail slab, every rank."""
    reached = set()
    for r in SKINNY_R:
        for C in SKINNY_C:
            for M in _skinny_M(C):
                rows_par, threads, rpc, grid = skinny_atb_plan(M, C, H100_SMS)
                reached.add((rows_par, threads > rows_par * (C // 8), grid == 1, M % rpc != 0))
    rp = {x[0] for x in reached}
    assert {512, 1} <= rp, rp
    assert any(x[1] for x in reached), "no C leaves threads of a CTA inactive"
    assert any(x[2] for x in reached) and any(not x[2] and x[3] for x in reached), reached
    src = (CSRC / "lora.cu").read_text()
    assert sorted(int(v) for v in re.findall(r"SK_CASE\((\d+)\)", src)) == SKINNY_R


def test_skinny_batch_cases_reach_every_branch():
    """Both templates, with r < RT through the vectorised and the scalar `a` loads; C 320 / 768 / 1280 (32 idle threads);
    M not a multiple of U rows_par; a 100x M ratio in one batch; clamped slabs; n = 1, 16 and 17."""
    templates = _batch_templates()
    assert len(templates) >= 2, templates
    reached, cs, tails, clamped, ns, ratio = set(), set(), False, False, set(), False
    for descs in SKINNY_BATCH_CASES.values():
        ns.add(len(descs))
        for batch in _batches(descs):
            (RT, U), slabs, vec = batch_plan(batch, H100_SMS)
            clamped |= slabs < H100_SMS // len(batch)
            ms = [d[0] for d in batch]
            ratio |= max(ms) >= 100 * min(ms)
            for d, v in zip(batch, vec):
                M, C, r = d[0], d[1], d[2]
                rows_par = 512 // (C // 8)
                reached.add((RT, U, v, r < RT))
                cs.add(C)
                tails |= ((M + slabs - 1) // slabs) % (U * rows_par) != 0
    for RT, U in templates:
        for v in (True, False):
            assert (RT, U, v, True) in reached, f"skinny_atb_batch_kernel<{RT}, {U}>: no r < RT case with vec_a {v}"
    assert {320, 768, 1280} <= cs and tails and clamped and ratio, (cs, tails, clamped, ratio)
    assert {1, 16, 17} <= ns, ns


def test_rank_update_and_rowdot_cases_reach_every_branch():
    src = (CSRC / "lora.cu").read_text()
    rps = {int(v) for v in re.findall(r"launch_k\(rank_update_kernel<(\d+)>", src)}
    reached = {(rp, rank_update_vec_t(*tl)) for rp, C, M, tl, _ in RANK_UPDATE_CASES}
    assert reached >= {(rp, v) for rp in rps for v in (True, False)}, reached
    assert {rp for rp, C, *_ in RANK_UPDATE_CASES if C * rp * 4 == 48 * 1024} == rps, "C rp at the 48 KB limit"
    assert any(ip for *_, ip in RANK_UPDATE_CASES)
    rd = {int(v) for v in re.findall(r"launch_k\(rowdot_kernel<(\d+)>", src)}
    assert {rp for rp, N, M in ROWDOT_CASES if N * rp * 4 == 48 * 1024} == rd
    assert all(any(r == rp and N % 256 for r, N, _ in ROWDOT_CASES) for rp in rd)


def test_v2_inject_bwd_templates_have_cases():
    """v2_inject_bwd picks its template by C (`Ccols <= X`); the V2 contract cases must reach every one."""
    from tests.test_kernel_contracts import BWD_C

    src = (CSRC / "lora.cu").read_text()
    body = src[src.index('extern "C" int cl_v2_inject_bwd('):]
    body = body[:body.index("\n}\n")]
    branches = re.findall(r"(?:if \(Ccols <= (\d+)\) |else )launch_k\(v2_inject_bwd_kernel<(\d+), (\d+)>", body)
    assert len(branches) >= 3, branches
    bounds = [int(b) if b else 1 << 30 for b, *_ in branches]
    for i, (hi, (_, it, r)) in enumerate(zip(bounds, branches)):
        lo = bounds[i - 1] if i else 0
        assert any(lo < C <= hi for C in BWD_C), f"v2_inject_bwd_kernel<{it}, {r}> (C in ({lo}, {hi}]) has no case in BWD_C"


def test_conv_in_and_glue_cases_reach_every_branch():
    src = (CSRC / "smallops.cu").read_text()
    ci = {int(v) for v in re.findall(r"CONV_IN_CASE\((\d+)\)", src)}
    for c in ci:
        assert any(cin == c and cout % 32 for _, cin, _, _, cout, _ in CONV_IN_CASES), f"conv_in Cin {c}: no Cout % 32 != 0 case"
        assert any(cin == c and cout % 32 == 0 for _, cin, _, _, cout, _ in CONV_IN_CASES)
    assert {b for *_, b in CONV_IN_CASES} == {True, False}
    assert any((n * H * W) % 256 for n, _, H, W, _, _ in CONV_IN_CASES)
    assert CONV_OUT_C_MAX in [c[3] for c in CONV_OUT_CASES] and 8 in [c[3] for c in CONV_OUT_CASES]
    assert any(H == 1 and W == 1 for _, H, W, _ in CONV_OUT_CASES)
    assert any(H == 1 and W > 1 for _, H, W, _ in CONV_OUT_CASES) and any(W == 1 and H > 1 for _, H, W, _ in CONV_OUT_CASES)
    assert {b > 8 for b, *_ in SMALL_LINEAR_CASES} == {True, False}
    assert any(N % 8 for _, N, _ in SMALL_LINEAR_CASES) and any(K == SMALL_LINEAR_K_MAX for *_, K in SMALL_LINEAR_CASES)
    assert {8, 1280} <= {f for _, f in GEGLU_CASES}
    assert any(c == 8 and (h % 2 or w % 2) for _, h, w, c in UPS_CASES)
    assert any((h * w) % 32 and c % 32 for _, c, h, w in LAYOUT_CASES)


# ====================================================================================================== coverage report
@gpu
def test_zz_report_reached_branches(record_property):
    """Runs last in this file: the launch branches the cases above reached on this device."""
    reached = {k: sorted(v, key=repr) for k, v in sorted(REACHED.items())}
    print("reached:", reached)
    record_property("reached", repr(reached))
