"""Kernel contracts: every kernel that tests/emu_ops.py restates on the CPU, checked on the GPU against an independent fp64
reference and against that restatement (pytest -m gpu).

The host-logic suite swaps each `controllora_b200.ops` wrapper for its torch restatement in tests/emu_ops.py; its results
mean something only if each restatement computes what its kernel computes.  Each case below runs the real kernel on CUDA
tensors, recomputes the operation in fp64 from the same (bf16-rounded) inputs, and runs the emulator function on `.cpu()`
clones of the same inputs.  Shapes come from the code paths that pick tiles, template instantiations and thread layouts.

Tolerances (see the helpers below):
  - pure data movement is bit-exact;
  - fp32 reductions of bf16 inputs: relative Frobenius error <= 1e-4, and every element within 2e-5 of the fp64 sum of
    |terms| (products of bf16 values are exact in fp32, so only the summation order remains);
  - bf16 outputs: at most one bf16 ulp from the fp64 result rounded to bf16; against the emulator at most one ulp, on at
    most 0.1 % of the elements (plus the Poisson spread of that count, which matters only for tensors of a few thousand
    elements).  Where an output is a small difference of large terms, the ulp is taken at 2^-12 of the
    magnitude of the terms (fp32 arithmetic cannot resolve below that).

`test_every_emulated_kernel_has_a_contract_case` (no GPU needed) fails when an emulated kernel has no case here.
"""
from __future__ import annotations

import ctypes as C
import math
import re
import zlib
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from tests import emu_ops as E

BF16 = torch.bfloat16
F64 = torch.float64

# ------------------------------------------------------------------------------------------------------------ registry
CONTRACTS: dict[str, list[str]] = {}
# kernels whose kernel-vs-restatement case lives in another test file: name -> (file under tests/, test function)
CROSS_REFERENCED = {"add_noise": ("test_gpu_parity.py", "test_add_noise_matches_oracle_restatement")}


def contract(*names):
    """Registers the decorated test as the kernel-vs-emulator case of the named `emu_ops` entries."""

    def deco(fn):
        for n in names:
            CONTRACTS.setdefault(n, []).append(fn.__name__)
        return fn

    return deco


@pytest.fixture(scope="module")
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def gpu(fn):
    return pytest.mark.gpu(pytest.mark.usefixtures("_need_gpu")(fn))


def test_every_emulated_kernel_has_a_contract_case():
    required = set(E._FUNCS) | {"PackPlan.run", "SkinnyQueue"}
    missing = sorted(required - set(CONTRACTS) - set(CROSS_REFERENCED))
    assert not missing, f"emulated kernels without a kernel-vs-emulator case in {Path(__file__).name}: {missing}"
    for name, (fname, test) in CROSS_REFERENCED.items():
        src = (Path(__file__).parent / fname).read_text()
        assert re.search(rf"^def {test}\(", src, re.M), f"{name}: {fname}::{test} does not exist"


# ------------------------------------------------------------------------------------------------------------ helpers
def _seed(*params):
    torch.manual_seed(zlib.crc32(repr(params).encode()))


def _bf(*shape, scale=1.0):
    return (torch.randn(*shape, device="cuda") * scale).to(BF16)


def _f32(*shape, scale=1.0):
    return torch.randn(*shape, device="cuda") * scale


def _cpu(t):
    return None if t is None else t.detach().cpu()


def _sync():
    torch.cuda.synchronize()


def _f32_of(x: float) -> float:
    """The value a C `float` parameter carries."""
    return float(torch.tensor(x, dtype=torch.float32))


def _bf16_ulp(x64: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp at |x| (8 significant bits); normal range only."""
    m = x64.abs().clamp_min(2.0**-126)
    _, e = torch.frexp(m)
    return torch.ldexp(torch.ones_like(m), e - 8)


def assert_f32_reduction(out, ref64, terms64, what, rel=1e-4, elem=2e-5):
    """fp32 result of a reduction vs its fp64 value: relative Frobenius error, and per element against the fp64 sum of
    |terms| (a dropped or doubled block of terms shows up in both)."""
    o = out.detach().to("cpu", F64)
    r = ref64.detach().to("cpu", F64)
    t = terms64.detach().to("cpu", F64)
    err = (o - r).abs()
    fro = float(err.norm() / r.norm().clamp_min(1e-300))
    assert fro <= rel, f"{what}: relative Frobenius error {fro:.3e} > {rel:.0e}"
    bad = err > elem * t + 1e-30
    if bad.any():
        i = int(torch.argmax((err - elem * t).flatten()))
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond {elem:.0e} * sum|terms|; worst at flat index {i}: "
                             f"got {float(o.flatten()[i])!r}, fp64 {float(r.flatten()[i])!r}, sum|terms| {float(t.flatten()[i])!r}")


def assert_bf16_vs_ref(out, ref64, what, floor=None):
    """bf16 output within one bf16 ulp of the fp64 result rounded to bf16 (ulp taken at max(|ref|, floor))."""
    assert out.dtype == BF16, what
    o = out.detach().to("cpu", F64)
    r = ref64.detach().to("cpu", F64).to(BF16).to(F64)
    mag = r.abs() if floor is None else torch.maximum(r.abs(), floor.detach().to("cpu", F64).expand_as(r))
    tol = _bf16_ulp(mag)
    err = (o - r).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = int(torch.argmax(torch.where(bad, err / tol, torch.zeros_like(err)).flatten()))
        raise AssertionError(f"{what}: {int(bad.sum())} of {o.numel()} elements more than 1 bf16 ulp from fp64; worst at flat "
                             f"index {i}: got {float(o.flatten()[i])!r}, fp64->bf16 {float(r.flatten()[i])!r}")


def assert_bf16_vs_emu(out, emu, what, floor=None, max_frac=1e-3):
    """kernel vs emulator, both bf16: at most one ulp apart, and at most max_frac of the elements differ at all."""
    assert out.dtype == BF16 and emu.dtype == BF16, what
    o = out.detach().to("cpu", F64)
    e = emu.detach().to("cpu", F64)
    assert o.shape == e.shape, (what, o.shape, e.shape)
    mag = e.abs() if floor is None else torch.maximum(e.abs(), floor.detach().to("cpu", F64).expand_as(e))
    err = (o - e).abs()
    bad = ~(err <= _bf16_ulp(mag))
    assert not bad.any(), f"{what}: kernel and emulator differ by more than 1 bf16 ulp at {int(bad.sum())} elements"
    frac = float((err > 0).double().mean())
    expect = max_frac * err.numel()                   # rounding flips are rare events: allow the Poisson spread on small tensors
    assert int((err > 0).sum()) <= expect + 3 * math.sqrt(expect) + 2, f"{what}: kernel and emulator differ at {100 * frac:.3f} % of the elements (> {100 * max_frac:.1f} %)"


def assert_f32_close(out, other, what, rtol, scale=None):
    """fp32 vs fp32 (or fp64) within rtol of max(|other|, scale) per element."""
    o = out.detach().to("cpu", F64)
    r = other.detach().to("cpu", F64)
    assert o.shape == r.shape, (what, o.shape, r.shape)
    mag = r.abs() if scale is None else torch.maximum(r.abs(), scale.detach().to("cpu", F64).expand_as(r))
    err = (o - r).abs()
    bad = ~(err <= rtol * mag + 1e-38)
    if bad.any():
        i = int(torch.argmax(torch.where(bad, err, torch.zeros_like(err)).flatten()))
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond rtol {rtol:.1e}; worst at flat index {i}: "
                             f"got {float(o.flatten()[i])!r}, expected {float(r.flatten()[i])!r}")


def _floor(terms64, rel=2.0**-12):
    return rel * terms64


# ------------------------------------------------------------------------------------------------------------ conv_wgrad
def _conv_fp64(x, w, k, stride, pad_lo):
    """x NCHW, w [Cout, Cin, k, k]; the hint encoder's convolutions written with explicit padding."""
    if k == 1:
        return F.conv2d(x, w)
    if stride == 1:
        return F.conv2d(F.pad(x, (1, 1, 1, 1)), w)
    return F.conv2d(F.pad(x, (pad_lo, 1 - pad_lo, pad_lo, 1 - pad_lo)), w, stride=2)


def _wgrad_fp64(dy, x, k, stride, pad_lo, Cout, Cin):
    """dW = d/dW sum(dY * conv(X, W)) in fp64, on the device; dy / x NHWC."""
    xin = x.to(F64).permute(0, 3, 1, 2)
    w = torch.zeros(Cout, Cin, k, k, dtype=F64, device=x.device, requires_grad=True)
    with torch.enable_grad():
        (g,) = torch.autograd.grad(_conv_fp64(xin, w, k, stride, pad_lo), w, dy.to(F64).permute(0, 3, 1, 2))
    return g


WGRAD_CASES = [
    # (n, H, W, Cin, Cout, k, stride, pad_lo)                    pixel tile bw x bh x bn (from Wo, Ho)
    (1, 64, 64, 32, 32, 3, 1, 1),       # 64 x 2 x 1
    (2, 64, 64, 64, 64, 3, 1, 1),
    (3, 24, 24, 128, 128, 3, 1, 1),     # 8 x 8 x 2: batch 3 is not a multiple of bn
    (2, 24, 24, 96, 320, 3, 1, 1),      # Cin not a multiple of 64, Cout not a multiple of 128
    (1, 24, 24, 32, 32, 3, 1, 1),       # image box 2 > 1 image
    (2, 24, 40, 64, 64, 3, 1, 1),
    (3, 8, 8, 256, 256, 3, 1, 1),       # Wo*Ho = 64 < 128
    (3, 4, 4, 64, 64, 3, 1, 1),         # 4 x 4 x 8
    (2, 4, 4, 96, 320, 3, 1, 1),
    (4, 256, 256, 32, 32, 3, 1, 1),     # 2048 pixel blocks over ~86 splits, the last one short
    (2, 64, 64, 32, 64, 3, 2, 0),       # stride 2: the 5-D strided view, pad_lo 0 and 1
    (2, 64, 64, 32, 64, 3, 2, 1),
    (2, 64, 64, 96, 320, 3, 2, 0),
    (2, 64, 64, 96, 320, 3, 2, 1),
    (2, 16, 16, 32, 64, 3, 2, 0),
    (2, 16, 16, 32, 64, 3, 2, 1),
    (2, 16, 16, 96, 320, 3, 2, 0),
    (2, 16, 16, 96, 320, 3, 2, 1),
    (2, 8, 8, 32, 64, 3, 2, 0),
    (2, 8, 8, 32, 64, 3, 2, 1),
    (3, 8, 8, 96, 320, 3, 2, 0),
    (3, 8, 8, 96, 320, 3, 2, 1),
    (2, 32, 32, 320, 320, 1, 1, 0),     # 1x1
    (1, 24, 24, 64, 320, 1, 1, 0),
    (3, 8, 8, 1280, 640, 1, 1, 0),
]
# the concat-hidden control LoRA's dA / dB as 1x1 "dY^T X" on (1, 1, T, C) views: (T, Cout of dy, Cin of x)
LORA_T = [8192, 144 * 2, 77 * 3, 4225]
LORA_PAIRS = [(320, 8), (8, 320), (640, 16), (16, 640), (1280, 256), (256, 1280), (8, 256), (256, 256)]
WGRAD_CASES += [(1, 1, T, cx, cy, 1, 1, 0) for T in LORA_T for (cy, cx) in LORA_PAIRS]


@gpu
@contract("conv_wgrad")
@pytest.mark.parametrize("n,H,W,Cin,Cout,k,stride,pad_lo", WGRAD_CASES)
def test_conv_wgrad(n, H, W, Cin, Cout, k, stride, pad_lo):
    from controllora_b200 import ops

    _seed("wgrad", n, H, W, Cin, Cout, k, stride, pad_lo)
    x = _bf(n, H, W, Cin)
    dy = _bf(n, H // stride, W // stride, Cout)
    dw0 = _f32(Cout, Cin, k, k)
    alpha = 0.7
    dw = dw0.clone()
    ops.conv_wgrad(dy, x, dw, k, stride, pad_lo, alpha)
    g = _wgrad_fp64(dy, x, k, stride, pad_lo, Cout, Cin)
    ga = _wgrad_fp64(dy.abs(), x.abs(), k, stride, pad_lo, Cout, Cin)
    _sync()
    a = _f32_of(alpha)
    ref = dw0.to(F64) + a * g
    terms = dw0.abs().to(F64) + a * ga
    assert_f32_reduction(dw, ref, terms, "conv_wgrad vs fp64")
    dw_e = _cpu(dw0).clone()
    E.conv_wgrad(_cpu(dy), _cpu(x), dw_e, k, stride, pad_lo, alpha)
    assert_f32_reduction(dw_e, ref, terms, "emulated conv_wgrad vs fp64")
    assert_f32_reduction(dw, dw_e.to(F64), terms, "conv_wgrad vs emulator")


# ------------------------------------------------------------------------------------------------------------ conv_in_wgrad
@gpu
@contract("conv_in_wgrad")
@pytest.mark.parametrize("n,Cin,H,W,Cout", [(1, 3, 17, 23, 32), (2, 4, 31, 33, 320), (1, 3, 9, 7, 20), (2, 4, 5, 5, 20),
                                           (3, 4, 13, 11, 32), (2, 3, 512, 512, 32)])
def test_conv_in_wgrad(n, Cin, H, W, Cout):
    from controllora_b200 import ops

    _seed("conv_in_wgrad", n, Cin, H, W, Cout)
    x = _f32(n, Cin, H, W)                                   # fp32 guide: the kernel rounds it to bf16
    assert not torch.equal(x, x.to(BF16).float())
    dy = _bf(n, H, W, Cout)
    dw0 = _f32(Cout, Cin, 3, 3)
    dw = dw0.clone()
    ops.conv_in_wgrad(x, dy, dw)
    xb = x.to(BF16).permute(0, 2, 3, 1)
    g = _wgrad_fp64(dy, xb, 3, 1, 1, Cout, Cin)
    ga = _wgrad_fp64(dy.abs(), xb.abs(), 3, 1, 1, Cout, Cin)
    _sync()
    ref = dw0.to(F64) + g
    terms = dw0.abs().to(F64) + ga
    assert_f32_reduction(dw, ref, terms, "conv_in_wgrad vs fp64")
    dw_e = _cpu(dw0).clone()
    E.conv_in_wgrad(_cpu(x), _cpu(dy), dw_e)
    assert_f32_reduction(dw_e, ref, terms, "emulated conv_in_wgrad vs fp64")
    assert_f32_reduction(dw, dw_e.to(F64), terms, "conv_in_wgrad vs emulator")


# ------------------------------------------------------------------------------------------------------------ colsum
@gpu
@contract("colsum")
@pytest.mark.parametrize("C", [8, 32, 320, 1280, 2048])
@pytest.mark.parametrize("M", [1, 7, 100003])
def test_colsum(C, M):
    from controllora_b200 import ops

    _seed("colsum", C, M)
    x = _bf(M, C)
    out0 = _f32(C)
    alpha = 0.7
    out = out0.clone()
    ops.colsum(x, out, alpha)
    _sync()
    a = _f32_of(alpha)
    x64 = x.to(F64)
    ref = out0.to(F64) + a * x64.sum(0)
    terms = out0.abs().to(F64) + a * x64.abs().sum(0)
    assert_f32_reduction(out, ref, terms, "colsum vs fp64")
    out_e = _cpu(out0).clone()
    E.colsum(_cpu(x), out_e, alpha)
    assert_f32_reduction(out_e, ref, terms, "emulated colsum vs fp64")
    assert_f32_reduction(out, out_e.to(F64), terms, "colsum vs emulator")


# ------------------------------------------------------------------------------------------------------------ conv_weight_prep
@gpu
@contract("conv_weight_prep")
@pytest.mark.parametrize("Cout,Cin,k,with_wd", [(320, 96, 3, True), (32, 4, 3, False), (64, 320, 1, True), (20, 3, 3, True)])
def test_conv_weight_prep(Cout, Cin, k, with_wd):
    from controllora_b200 import ops

    _seed("prep", Cout, Cin, k, with_wd)
    w = _f32(Cout, Cin, k, k)
    wf = torch.full((Cout * k * k * Cin + 8,), 7.0, device="cuda", dtype=BF16)
    wd = torch.full((Cout * k * k * Cin + 8,), 7.0, device="cuda", dtype=BF16) if with_wd else None
    ops.conv_weight_prep(w, wf, wd)
    _sync()
    n = Cout * k * k * Cin
    want_f = w.permute(0, 2, 3, 1).to(BF16).flatten()                  # [Cout][ky][kx][Cin]
    assert torch.equal(wf[:n], want_f) and torch.equal(wf[n:], torch.full((8,), 7.0, device="cuda", dtype=BF16))
    if with_wd:
        want_d = w.flip(2, 3).permute(1, 2, 3, 0).to(BF16).flatten()   # [Cin][taps flipped][Cout]
        assert torch.equal(wd[:n], want_d) and torch.equal(wd[n:], torch.full((8,), 7.0, device="cuda", dtype=BF16))
    wf_e = torch.full((n + 8,), 7.0, dtype=BF16)
    wd_e = torch.full((n + 8,), 7.0, dtype=BF16) if with_wd else None
    E.conv_weight_prep(_cpu(w), wf_e, wd_e)
    assert torch.equal(_cpu(wf), wf_e)
    if with_wd:
        assert torch.equal(_cpu(wd), wd_e)


# ------------------------------------------------------------------------------------------------------------ V2 side path
def _uc_variants(M):
    """(label, uc view or None, rc): contiguous-column views for rc 1..3, a 4-column view with ldu % 4 != 0 (scalar path)
    and a 16-byte aligned one with ldu % 4 == 0 (vector path)."""
    w8 = _f32(M, 8)
    w7 = _f32(M, 7)
    w12 = _f32(M, 12)
    return [("none", None, 4), ("rc1", w8[:, :1], 1), ("rc2", w8[:, :2], 2), ("rc3", w8[:, :3], 3),
            ("rc4_scalar", w7[:, 1:5], 4), ("rc4_vector", w12[:, 4:8], 4)]


def _th16(M):
    hi = _f32(M, 8)
    lo = _f32(M, 8, scale=2.0**-9)
    return torch.cat([hi, lo], 1).contiguous()                          # [hi0..3 | hi4..7 | lo0..3 | lo4..7]


@gpu
@contract("v2_inject_fwd")
@pytest.mark.parametrize("C", [8, 320, 1280])
@pytest.mark.parametrize("M", [1, 4097])
def test_v2_inject_fwd(C, M):
    from controllora_b200 import ops

    _seed("v2fwd", C, M)
    x = _bf(M, C)
    th16 = _th16(M)
    tab = _f32(C, 4, scale=0.5)
    alpha = 0.6
    a = _f32_of(alpha)
    for label, uc, rc in _uc_variants(M):
        y, t = ops.v2_inject_fwd(x, th16, uc, rc, tab, alpha)
        _sync()
        what = f"v2_inject_fwd[{label}]"
        th = th16.to(F64)
        t64 = th[:, :8] + th[:, 8:]
        tterm = th[:, :8].abs() + th[:, 8:].abs()
        if uc is not None:
            t64[:, :rc] += uc[:, :rc].to(F64)
            tterm[:, :rc] += uc[:, :rc].abs().to(F64)
        assert_f32_close(t, t64, what + " t vs fp64", 2.0**-22, tterm)
        assert torch.equal(t[:, 4:8], th16[:, 4:8] + th16[:, 12:16]), what + ": t[:, 4:8] is not the upper hi/lo combine"
        y64 = x.to(F64) + a * (t64[:, :4] @ tab.to(F64).t())
        yterm = x.abs().to(F64) + a * (t64[:, :4].abs() @ tab.abs().to(F64).t())
        assert_bf16_vs_ref(y, y64, what + " y vs fp64", _floor(yterm))
        y_e, t_e = E.v2_inject_fwd(_cpu(x), _cpu(th16), _cpu(uc), rc, _cpu(tab), alpha)
        assert torch.equal(_cpu(t), t_e), what + ": t differs from the emulator"
        assert_bf16_vs_emu(y, y_e, what + " y vs emulator", _floor(yterm))


BWD_C = [8, 512, 520, 768, 776, 1280]          # at and just past the template boundaries (<= 512, <= 768, <= 1280)
BWD_M = [1, 3, 5, 4097]                        # not multiples of the 4 or 2 rows a warp handles


@gpu
@contract("v2_inject_bwd")
@pytest.mark.parametrize("C", BWD_C)
@pytest.mark.parametrize("M", BWD_M)
@pytest.mark.parametrize("need_dh", [True, False])
def test_v2_inject_bwd(C, M, need_dh):
    from controllora_b200 import ops

    _seed("v2bwd", C, M, need_dh)
    dy = _bf(M, C)
    up = _f32(C, 4, scale=0.5)
    down = _f32(C, 4, scale=0.5) if need_dh else None
    alpha = 0.6
    dt, dh = ops.v2_inject_bwd(dy, up, down, alpha, need_dh)
    _sync()
    d64 = dy.to(F64)
    dt64 = d64 @ up.to(F64)
    dterm = d64.abs() @ up.abs().to(F64)
    assert_f32_reduction(dt, dt64, dterm, "v2_inject_bwd dt vs fp64")
    dt_e, dh_e = E.v2_inject_bwd(_cpu(dy), _cpu(up), _cpu(down), alpha, need_dh)
    assert_f32_reduction(dt, dt_e.to(F64), dterm, "v2_inject_bwd dt vs emulator")
    if not need_dh:
        assert dh is None and dh_e is None
        return
    a = _f32_of(alpha)
    dh64 = d64 + a * (dt64 @ down.to(F64).t())
    hterm = d64.abs() + a * (dterm @ down.abs().to(F64).t())
    assert_bf16_vs_ref(dh, dh64, "v2_inject_bwd dh vs fp64", _floor(hterm))
    assert_bf16_vs_emu(dh, dh_e, "v2_inject_bwd dh vs emulator", _floor(hterm))


@gpu
@contract("rank4_project_update")
@pytest.mark.parametrize("C", BWD_C)
@pytest.mark.parametrize("M", BWD_M)
def test_rank4_project_update(C, M):
    from controllora_b200 import ops

    _seed("rank4", C, M)
    x = _bf(M, C)
    proj = _f32(C, 4, scale=0.5)
    upd = _f32(C, 4, scale=0.5)
    alpha = 0.6
    a = _f32_of(alpha)
    w8 = _f32(M, 8)
    variants = _uc_variants(M)[1:] + [("none", None, 0), ("rc0", w8[:, :4], 0)]
    for label, uc, rc in variants:
        what = f"rank4_project_update[{label}]"
        y, t = ops.rank4_project_update(x, proj, upd, uc, rc, alpha)
        _sync()
        x64 = x.to(F64)
        t64 = x64 @ proj.to(F64)
        tterm = x64.abs() @ proj.abs().to(F64)
        if uc is not None and rc:
            t64[:, :rc] += uc[:, :rc].to(F64)
            tterm[:, :rc] += uc[:, :rc].abs().to(F64)
        assert_f32_reduction(t, t64, tterm, what + " t vs fp64")
        y64 = x64 + a * (t64 @ upd.to(F64).t())
        yterm = x64.abs() + a * (tterm @ upd.abs().to(F64).t())
        assert_bf16_vs_ref(y, y64, what + " y vs fp64", _floor(yterm))
        y_e, t_e = E.rank4_project_update(_cpu(x), _cpu(proj), _cpu(upd), _cpu(uc), rc, alpha)
        assert_f32_reduction(t, t_e.to(F64), tterm, what + " t vs emulator")
        assert_bf16_vs_emu(y, y_e, what + " y vs emulator", _floor(yterm))


@gpu
@contract("hilo_combine")
@pytest.mark.parametrize("nb", [1, 2, 3])
def test_hilo_combine(nb):
    from controllora_b200 import ops

    _seed("hilo", nb)
    M = 1003
    src = _f32(M, 16 * nb)
    out = ops.hilo_combine(src, nb)
    _sync()
    s = src.to(F64).view(M, nb, 2, 8)
    ref = (s[:, :, 0] + s[:, :, 1]).reshape(M, 8 * nb).float()          # one correctly rounded fp32 add
    assert torch.equal(out, ref)
    assert torch.equal(_cpu(out), E.hilo_combine(_cpu(src), nb))


# ------------------------------------------------------------------------------------------------------------ strided weight helpers
@gpu
@contract("cast_matrix")
@pytest.mark.parametrize("form", ["plain", "transposed", "sliced", "sliced_transposed", "strided_out"])
@pytest.mark.parametrize("alpha", [1.0, 0.7])
def test_cast_matrix(form, alpha):
    from controllora_b200 import ops

    _seed("cast", form, alpha)
    base = _f32(40, 96)                                   # an fp32 master, e.g. Bc [C, R] or Ac [R, C + cc]
    if form == "plain":
        src, I, J, s_i, s_j, off = base, 40, 96, 96, 1, 0
    elif form == "transposed":
        src, I, J, s_i, s_j, off = base, 96, 40, 1, 96, 0
    elif form == "sliced":
        src, I, J, s_i, s_j, off = base[:, 32:], 40, 64, 96, 1, 32
    elif form == "sliced_transposed":
        src, I, J, s_i, s_j, off = base[:, 32:], 64, 40, 1, 96, 32
    else:
        src, I, J, s_i, s_j, off = base, 96, 40, 1, 96, 0
    out_base = torch.full((I, J + 24), 3.0, device="cuda", dtype=BF16)
    out = ops.cast_matrix(src, I, J, s_i, s_j, alpha, out=out_base[:, :J] if form == "strided_out" else None)
    _sync()
    view = torch.as_strided(base, (I, J), (s_i, s_j), off)
    ref = (view.to(F64) * _f32_of(alpha)).float().to(BF16)             # fp32 product, rounded to bf16
    assert torch.equal(out, ref)
    if form == "strided_out":
        assert torch.equal(out_base[:, J:], torch.full((I, 24), 3.0, device="cuda", dtype=BF16)), "wrote past J"
    base_c = _cpu(base)
    out_e = E.cast_matrix(base_c[:, off:] if off else base_c, I, J, s_i, s_j, alpha)
    assert torch.equal(_cpu(out), out_e)


@gpu
@contract("axpy_matrix")
@pytest.mark.parametrize("alpha", [1.0, -0.3])
def test_axpy_matrix(alpha):
    from controllora_b200 import ops

    _seed("axpy", alpha)
    R, C, cc = 16, 320, 256
    g0 = _f32(R, C + cc)                                  # gAc = [dAc_h | dAc_c]
    src = _f32(R, cc)
    g = g0.clone()
    ops.axpy_matrix(src, g[:, C:], alpha)
    _sync()
    a = _f32_of(alpha)
    assert torch.equal(g[:, :C], g0[:, :C]), "axpy_matrix wrote outside its column slice"
    ref = g0[:, C:].to(F64) + a * src.to(F64)
    terms = g0[:, C:].abs().to(F64) + abs(a) * src.abs().to(F64)
    assert_f32_close(g[:, C:], ref, "axpy_matrix vs fp64", 2.0**-23, terms)
    g_e = _cpu(g0).clone()
    E.axpy_matrix(_cpu(src), g_e[:, C:], alpha)
    assert_f32_close(g[:, C:], g_e[:, C:], "axpy_matrix vs emulator", 2.0**-22, terms)


# ------------------------------------------------------------------------------------------------------------ VAE / CLIP helpers
@gpu
@contract("softmax_rows")
@pytest.mark.parametrize("cols", [4, 4096, 12288])
def test_softmax_rows(cols):
    from controllora_b200 import ops

    _seed("softmax", cols)
    scale = 0.5
    rows = [_f32(cols, scale=3.0),
            torch.linspace(-110.0, 10.0, cols, device="cuda")[torch.randperm(cols, device="cuda")],   # e^-60 .. 1
            torch.full((cols,), 7.25, device="cuda"),                                                 # all equal
            1000.0 + _f32(cols),                                                                      # large offset
            _f32(cols, scale=0.01)]
    s = torch.stack(rows).contiguous()
    p = ops.softmax_rows(s, scale)
    _sync()
    ref = torch.softmax(_f32_of(scale) * s.to(F64), -1)
    assert_bf16_vs_ref(p, ref, "softmax_rows vs fp64")
    p64 = p.to(F64)
    assert torch.all((p64.sum(-1) - 1).abs() <= _bf16_ulp(p64).sum(-1)), "softmax rows do not sum to 1 within bf16 rounding"
    assert torch.equal(p[2], torch.full((cols,), 1.0 / cols, device="cuda").to(BF16))
    assert_bf16_vs_emu(p, E.softmax_rows(_cpu(s), scale), "softmax_rows vs emulator")


@gpu
@contract("causal_attention_small")
@pytest.mark.parametrize("T", [1, 77, 128])
@pytest.mark.parametrize("d", [40, 64])
def test_causal_attention_small(T, d):
    from controllora_b200 import ops

    _seed("causal", T, d)
    B, H = 2, 12
    Cc = H * d
    qkv = _bf(B * T, 3 * Cc)
    scale = d**-0.5
    out = ops.causal_attention_small(qkv, B, T, H, scale)
    _sync()
    q, k, v = (t.to(F64).reshape(B, T, H, d).permute(0, 2, 1, 3) for t in qkv.split(Cc, 1))
    s = (q @ k.transpose(-1, -2)) * _f32_of(scale)
    s = s.masked_fill(torch.ones(T, T, dtype=torch.bool, device="cuda").triu(1), float("-inf"))
    p = torch.softmax(s, -1)
    ref = (p @ v).permute(0, 2, 1, 3).reshape(B * T, Cc)
    terms = (p @ v.abs()).permute(0, 2, 1, 3).reshape(B * T, Cc)
    assert_bf16_vs_ref(out, ref, "causal_attention_small vs fp64", _floor(terms))
    assert_bf16_vs_emu(out, E.causal_attention_small(_cpu(qkv), B, T, H, scale), "causal_attention_small vs emulator", _floor(terms))
    # softmax rows sum to one: with v = 1 every output is 1
    ones = qkv.clone()
    ones[:, 2 * Cc:] = 1.0
    o1 = ops.causal_attention_small(ones, B, T, H, scale)
    _sync()
    assert torch.equal(o1, torch.ones_like(o1)), "causal attention weights do not sum to 1"


@gpu
@contract("clip_embed")
def test_clip_embed():
    from controllora_b200 import ops

    _seed("clip_embed")
    vocab, T, Cc = 1000, 77, 768
    tok = _bf(vocab, Cc)
    pos = _bf(T, Cc)
    ids = torch.randint(0, vocab, (3, T), device="cuda")
    ids[0, 0], ids[0, -1], ids[1, :5], ids[2, 40:] = 0, vocab - 1, vocab - 1, 0
    out = ops.clip_embed(ids, tok, pos)
    _sync()
    ref = (tok.to(F64)[ids] + pos.to(F64)[None]).float().to(BF16)
    assert torch.equal(out, ref)
    assert torch.equal(_cpu(out), E.clip_embed(_cpu(ids), _cpu(tok), _cpu(pos)))


@gpu
@contract("quick_gelu_")
@pytest.mark.parametrize("numel", [8, 8 * 4097])
def test_quick_gelu(numel):
    from controllora_b200 import ops

    _seed("qgelu", numel)
    edge = torch.tensor([20.0, -20.0, 8.0, -8.0, 0.0, -0.5, 1e-3, -3.0], device="cuda")
    x = torch.cat([edge, _f32(numel - 8, scale=4.0)]).to(BF16)
    x0 = x.clone()
    ops.quick_gelu_(x)
    _sync()
    x64 = x0.to(F64)
    ref = x64 * torch.sigmoid(1.702 * x64)
    assert_bf16_vs_ref(x, ref, "quick_gelu_ vs fp64")
    assert_bf16_vs_emu(x, E.quick_gelu_(_cpu(x0).clone()), "quick_gelu_ vs emulator")


@gpu
@contract("channel_affine_nchw")
def test_channel_affine_nchw():
    from controllora_b200 import ops

    _seed("affine")
    x = _f32(2, 4, 33, 17)
    shift = _f32(4)
    mul = 1 / 0.18215
    y = ops.channel_affine_nchw(x, mul, shift)
    _sync()
    m = _f32_of(mul)
    ref = m * x.to(F64) + shift.to(F64).view(1, 4, 1, 1)
    assert_f32_close(y, ref, "channel_affine_nchw vs mul * x + shift", 2.0**-24 * (1 + 1e-9))
    terms = (m * x.abs().to(F64) + shift.abs().to(F64).view(1, 4, 1, 1))
    assert_f32_close(y, E.channel_affine_nchw(_cpu(x), mul, _cpu(shift)), "channel_affine_nchw vs emulator", 2.0**-22, terms)


@gpu
@contract("f32_to_bf16", "bf16_to_f32")
def test_f32_bf16_conversions():
    from controllora_b200 import ops

    _seed("convert")
    n = 100003
    bits = torch.randint(-2**31, 2**31 - 1, (n,), dtype=torch.int32)
    bits[:1000] = (bits[:1000] & ~0xFFFF) | 0x8000                     # exact ties: round to even
    x = bits.view(torch.float32)
    x = torch.where(torch.isnan(x), torch.zeros_like(x), x)
    x[1000:1006] = torch.tensor([float("inf"), float("-inf"), 0.0, -0.0, 3.4e38, 1e-40])
    x = x.cuda()
    y = ops.f32_to_bf16(x)
    _sync()
    assert torch.equal(y.view(torch.int16), x.to(BF16).view(torch.int16))
    assert torch.equal(_cpu(y).view(torch.int16), E.f32_to_bf16(_cpu(x)).view(torch.int16))
    z = torch.empty(n, device="cuda")
    ops._call("cl_bf16_to_f32", ops._p(y), ops._p(z), C.c_int64(n))
    _sync()
    assert torch.equal(z.view(torch.int32), y.float().view(torch.int32))


# ------------------------------------------------------------------------------------------------------------ sampler step program
def _solver_tables(kind, S):
    ac = torch.linspace(0.999, 0.05, S + 1, dtype=F64)
    coef = torch.zeros(S, 8, dtype=torch.float32)
    host = []
    for s in range(S):
        a_t, a_p = float(ac[s + 1]), float(ac[s])
        if kind == 0:
            coef[s, :4] = torch.tensor([a_t**0.5, (1 - a_t) ** 0.5, a_p**0.5, (1 - a_p) ** 0.5], dtype=F64).float()
            host.append((a_t, a_p))
        else:
            c = (a_t**0.5, (1 - a_t) ** 0.5, 0.9 - 0.01 * s, 0.3 + 0.02 * s, -0.05 * s)
            c = tuple(_f32_of(v) for v in c)
            coef[s, :5] = torch.tensor(c)
            host.append(c)
    return coef.cuda(), host


@gpu
@contract("sampler_prep", "cfg_solver_step_dev")
@pytest.mark.parametrize("kind", [0, 1])
def test_sampler_step_program(kind):
    """sampler_prep + cfg_solver_step_dev over a whole coefficient table equal the host-parameter solver steps bit for bit
    (those are pinned to the oracle in test_gpu_parity.py), and the device step counter advances once per step."""
    from controllora_b200 import ops

    _seed("sampler", kind)
    S, g = 10, 7.5
    coef, host = _solver_tables(kind, S)
    ts_table = torch.linspace(981, 1, S, device="cuda")
    lat = _f32(2, 4, 9, 7)
    lat_h = lat.clone()
    x0p = torch.zeros_like(lat)
    x0p_h = torch.zeros_like(lat)
    x2 = torch.empty(4, 4, 9, 7, device="cuda")
    tt = torch.empty(4, device="cuda")
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    for s in range(S):
        pre = (_cpu(lat).clone(), _cpu(x0p).clone(), _cpu(ctr).clone())
        ops.sampler_prep(lat, x2, tt, ts_table, ctr)
        _sync()
        assert torch.equal(x2, torch.cat([lat, lat])) and torch.equal(tt, ts_table[s].expand(4))
        x2_e, tt_e = torch.empty(4, 4, 9, 7), torch.empty(4)
        E.sampler_prep(pre[0], x2_e, tt_e, _cpu(ts_table), pre[2])
        assert torch.equal(_cpu(x2), x2_e) and torch.equal(_cpu(tt), tt_e)
        eps2 = _f32(4, 4, 9, 7)
        ops.cfg_solver_step_dev(eps2, lat, x0p, coef, ctr, g, kind)
        if kind == 0:
            ops.cfg_ddim_step(eps2, lat_h, g, *host[s])
        else:
            ops.cfg_dpmpp_step(eps2, lat_h, x0p_h, g, *host[s])
        _sync()
        assert int(ctr) == s + 1, "the device step counter did not advance"
        assert torch.equal(lat, lat_h), f"step {s}: device-table step differs from the host-parameter step"
        if kind == 1:
            assert torch.equal(x0p, x0p_h)
        lat_e, x0p_e, ctr_e = pre
        E.cfg_solver_step_dev(_cpu(eps2), lat_e, x0p_e, _cpu(coef), ctr_e, g, kind)
        assert int(ctr_e) == s + 1
        scale = pre[0].abs() + _cpu(eps2).abs().view(2, -1).amax(0).view_as(lat_e) * 10 + pre[1].abs()
        assert_f32_close(lat, lat_e, f"cfg_solver_step_dev kind {kind} step {s} vs emulator", 1e-5, scale)
        if kind == 1:
            assert_f32_close(x0p, x0p_e, f"cfg_solver_step_dev x0 step {s} vs emulator", 1e-5, scale * 5)


@gpu
@contract("cfg_ddim_step", "cfg_dpmpp_step")
def test_host_parameter_solver_steps_match_emulator():
    from controllora_b200 import ops

    _seed("host_solver")
    g = 7.5
    eps2 = _f32(4, 4, 16, 16)
    lat = _f32(2, 4, 16, 16)
    x0p = _f32(2, 4, 16, 16)
    scale = lat.abs() + 10 * eps2.abs().view(2, -1).amax(0).view_as(lat) + x0p.abs()
    l1, l1e = lat.clone(), _cpu(lat).clone()
    ops.cfg_ddim_step(eps2, l1, g, 0.3, 0.5)
    E.cfg_ddim_step(_cpu(eps2), l1e, g, 0.3, 0.5)
    l2, x2, l2e, x2e = lat.clone(), x0p.clone(), _cpu(lat).clone(), _cpu(x0p).clone()
    c = (0.55, 0.83, 0.7, 0.4, -0.1)
    ops.cfg_dpmpp_step(eps2, l2, x2, g, *c)
    E.cfg_dpmpp_step(_cpu(eps2), l2e, x2e, g, *c)
    _sync()
    assert_f32_close(l1, l1e, "cfg_ddim_step vs emulator", 1e-5, scale)
    assert_f32_close(l2, l2e, "cfg_dpmpp_step vs emulator", 1e-5, scale * 4)
    assert_f32_close(x2, x2e, "cfg_dpmpp_step x0 vs emulator", 1e-5, scale * 4)


# ------------------------------------------------------------------------------------------------------------ optimizer
@gpu
@contract("step_begin", "adamw_dev", "sumsq")
@pytest.mark.parametrize("n,max_norm,grad_scale,zero_grad", [(1001, 1.0, 1.0, True),       # clipping active
                                                             (1001, 1e6, 0.25, False),      # clipping inactive
                                                             (100003, 2.0, 0.125, True),
                                                             (4097, 0.0, 2.0, True)])       # no clipping at all
def test_step_begin_adamw_dev(n, max_norm, grad_scale, zero_grad):
    """The captured step's optimizer tail (step_begin, sumsq, adamw_dev) over 4 steps vs torch.optim.AdamW with
    clip_grad_norm_ on the scaled gradient, in fp64."""
    from controllora_b200 import ops

    _seed("adamw_dev", n, max_norm, grad_scale, zero_grad)
    lr, b1, b2, eps, wd = 1e-3, 0.9, 0.999, 1e-8, 1e-2
    # the kernel gets these as C floats (1 - 0.999f is 1.3e-5 away from 1e-3): the fp64 reference uses the same values
    lr32, b1_32, b2_32, eps32, wd32 = (_f32_of(v_) for v_ in (lr, b1, b2, eps, wd))
    p = _f32(n)
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    gn = torch.full((1,), 123.0, device="cuda")
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    p_ref = p.to("cpu", F64).requires_grad_(True)
    opt = torch.optim.AdamW([p_ref], lr=lr32, betas=(b1_32, b2_32), eps=eps32, weight_decay=wd32)
    pe, ge, me, ve = _cpu(p).clone(), None, torch.zeros(n), torch.zeros(n)
    gne, stepe = torch.full((1,), 123.0), torch.zeros(1, dtype=torch.int64)
    for k in range(1, 5):
        g = _f32(n, scale=3.0 * k)
        g0 = g.clone()
        ge = _cpu(g).clone()
        ops.step_begin(gn, step)
        ops.sumsq(g, gn)
        ops.adamw_dev(p, g, m, v, lr, b1, b2, eps, wd, step, gnorm_sq=gn, max_norm=max_norm, grad_scale=grad_scale,
                      zero_grad=zero_grad)
        _sync()
        assert int(step) == k
        gsq = float((g0.to(F64) ** 2).sum())
        assert abs(float(gn) - gsq) <= 1e-5 * gsq, "sumsq"
        p_ref.grad = g0.to("cpu", F64) * _f32_of(grad_scale)
        if max_norm > 0:
            torch.nn.utils.clip_grad_norm_([p_ref], max_norm)
        opt.step()
        st = opt.state[p_ref]
        what = f"adamw_dev step {k}"
        assert_f32_close(p, p_ref.detach(), what + " p vs torch.optim.AdamW (fp64)", 1e-6, torch.full((1,), 30 * lr))
        # moments: fp32 rounding of terms as large as the largest moment
        assert_f32_close(m, st["exp_avg"], what + " m vs fp64", 1e-6, st["exp_avg"].abs().amax().expand(1))
        assert_f32_close(v, st["exp_avg_sq"], what + " v vs fp64", 1e-6, st["exp_avg_sq"].abs().amax().expand(1))
        assert torch.equal(g, torch.zeros_like(g) if zero_grad else g0), "zero_grad"
        # the restatement, on the same inputs
        E.step_begin(gne, stepe)
        E.sumsq(ge, gne)
        E.adamw_dev(pe, ge, me, ve, lr, b1, b2, eps, wd, stepe, gnorm_sq=gne, max_norm=max_norm, grad_scale=grad_scale,
                    zero_grad=zero_grad)
        assert int(stepe) == k
        assert_f32_close(gn, gne, what + " sumsq vs emulator", 1e-5)
        assert_f32_close(p, pe, what + " p vs emulator", 1e-6, torch.full((1,), 30 * lr))
        assert_f32_close(m, me, what + " m vs emulator", 1e-6, me.abs().amax().expand(1))
        assert_f32_close(v, ve, what + " v vs emulator", 1e-6, ve.abs().amax().expand(1))
        assert torch.equal(_cpu(g), ge)


@gpu
@contract("adamw")
def test_adamw_host_step_matches_emulator():
    from controllora_b200 import ops

    _seed("adamw")
    n = 10007
    p, g = _f32(n), _f32(n, scale=3.0)
    m, v = _f32(n, scale=0.1), _f32(n, scale=0.1).abs()
    pe, ge, me, ve = (_cpu(t).clone() for t in (p, g, m, v))
    gn = (g.to(F64) ** 2).sum().float().reshape(1)
    for step in (1, 3):
        ops.adamw(p, g, m, v, 1e-3, 0.9, 0.999, 1e-8, 1e-2, step, gnorm_sq=gn, max_norm=1.0, grad_scale=0.5, zero_grad=False)
        E.adamw(pe, ge, me, ve, 1e-3, 0.9, 0.999, 1e-8, 1e-2, step, gnorm_sq=_cpu(gn), max_norm=1.0, grad_scale=0.5, zero_grad=False)
    _sync()
    assert_f32_close(p, pe, "adamw p vs emulator", 1e-6, torch.full((1,), 3e-2))
    assert_f32_close(m, me, "adamw m vs emulator", 1e-6, me.abs().amax().expand(1))
    assert_f32_close(v, ve, "adamw v vs emulator", 1e-6, ve.abs().amax().expand(1))


# ------------------------------------------------------------------------------------------------------------ GEMM, attention, norms:
# kernel vs emulator only here; their per-element fp64 contracts are in tests/test_core_kernel_contracts.py
def _max_floor(e, rel=2.0**-12):
    return e.detach().abs().float().amax().to(F64).reshape(1) * rel


@gpu
@contract("gemm")
@pytest.mark.parametrize("form", ["epilogue", "lora", "conv1", "conv2_pad0", "conv2_pad1", "fp32_out"])
def test_gemm_matches_emulator(form):
    from controllora_b200 import ops

    _seed("gemm", form)
    kw = {}
    if form.startswith("conv"):
        a = _bf(2, 16, 16, 64)
        b = _bf(128, 9 * 64, scale=0.05)
        kw["conv_stride"] = 1 if form == "conv1" else 2
        kw["pad_lo"] = 0 if form == "conv2_pad0" else 1
        kw["bias"] = _f32(128)
    else:
        M, N, K = 300, 320, 640
        a = _bf(M, K)
        b = _bf(N, K, scale=0.05)
        kw.update(bias=_f32(N), residual=_bf(M, N))
        if form == "lora":
            kw.update(ext=ops.split_bf16_ext(_f32(4, K, scale=0.05), K), lora_up=_f32(N, 4), lora_scale=0.8,
                      t_add=_f32(M, 4), t_out=torch.empty(M, 4, device="cuda"))
        if form == "fp32_out":
            kw["out_fp32"] = True
            del kw["residual"]
    out = ops.gemm(a, b, **kw)
    _sync()
    kwe = {k_: (_cpu(v_) if isinstance(v_, torch.Tensor) else v_) for k_, v_ in kw.items()}
    if "t_out" in kwe:
        kwe["t_out"] = torch.empty(300, 4)
    out_e = E.gemm(_cpu(a), _cpu(b), **kwe)
    if form == "fp32_out":
        terms = a.abs().to(F64) @ b.abs().to(F64).t() + kw["bias"].abs().to(F64)
        assert_f32_reduction(out, out_e.to(F64), terms, "gemm fp32 out vs emulator")
    else:
        assert_bf16_vs_emu(out, out_e, f"gemm[{form}] vs emulator", _max_floor(out_e))
    if form == "lora":
        e16 = a.abs().to(F64) @ kw["ext"].abs().to(F64).t()
        terms = e16[:, :4] + e16[:, 8:12] + kw["t_add"].abs().to(F64)
        assert_f32_reduction(kw["t_out"], kwe["t_out"].to(F64), terms, "gemm t_out vs emulator")


@gpu
@contract("attention_fwd", "attention_bwd")
@pytest.mark.parametrize("Nq,Nk,d", [(64, 77, 40), (256, 256, 64), (100, 100, 80)])
def test_attention_matches_emulator(Nq, Nk, d):
    from controllora_b200 import ops

    _seed("attn", Nq, Nk, d)
    B, H = 2, 8
    q, k, v, do = _bf(B, Nq, H * d), _bf(B, Nk, H * d), _bf(B, Nk, H * d), _bf(B, Nq, H * d)
    scale = d**-0.5
    o, lse = ops.attention_fwd(q, k, v, H, scale)
    dq, dk, dv = ops.attention_bwd(q, k, v, o, do, lse, H, scale)
    _sync()
    # the kernels round the probabilities to bf16 for the P V (and dS) products, as flash attention does; the restatement
    # keeps them in fp32, so the two agree to the bf16 precision of P rather than to one ulp of the output
    o_e, lse_e = E.attention_fwd(_cpu(q), _cpu(k), _cpu(v), H, scale)
    rel = lambda x_, e_: float((x_.cpu().double() - e_.double()).norm() / e_.double().norm())
    assert rel(o, o_e) <= 5e-3, f"attention_fwd vs emulator: relative error {rel(o, o_e):.2e}"
    dq_e, dk_e, dv_e = E.attention_bwd(_cpu(q), _cpu(k), _cpu(v), o_e, _cpu(do), lse_e, H, scale)
    for name, x_, e_ in (("dq", dq, dq_e), ("dk", dk, dk_e), ("dv", dv, dv_e)):
        assert rel(x_, e_) <= 1e-2, f"attention_bwd {name} vs emulator: relative error {rel(x_, e_):.2e}"


@gpu
@contract("groupnorm_fwd", "groupnorm_bwd", "layernorm_fwd", "layernorm_bwd")
def test_norms_match_emulator():
    from controllora_b200 import ops

    _seed("norms")
    x = _bf(2, 8, 8, 320)
    gamma, beta = 1 + _f32(320, scale=0.1), _f32(320, scale=0.1)
    y, st = ops.groupnorm_fwd(x, gamma, beta, 32, 1e-6, True)
    dy = _bf(2, 8, 8, 320)
    dgam, dbet = torch.zeros(320, device="cuda"), torch.zeros(320, device="cuda")
    dx = ops.groupnorm_bwd(x, dy, gamma, beta, st, 32, True, dgamma=dgam, dbeta=dbet)
    _sync()
    y_e, st_e = E.groupnorm_fwd(_cpu(x), _cpu(gamma), _cpu(beta), 32, 1e-6, True)
    assert_bf16_vs_emu(y, y_e, "groupnorm_fwd vs emulator", _max_floor(y_e))
    dg_e, db_e = torch.zeros(320), torch.zeros(320)
    dx_e = E.groupnorm_bwd(_cpu(x), _cpu(dy), _cpu(gamma), _cpu(beta), st_e, 32, True, dgamma=dg_e, dbeta=db_e)
    assert_bf16_vs_emu(dx, dx_e, "groupnorm_bwd dx vs emulator", _max_floor(dx_e, 2.0**-10), max_frac=1e-2)
    assert_f32_close(dgam, dg_e, "groupnorm_bwd dgamma vs emulator", 1e-4, _max_floor(dg_e, 1e-3))
    assert_f32_close(dbet, db_e, "groupnorm_bwd dbeta vs emulator", 1e-4, _max_floor(db_e, 1e-3))

    xl = _bf(2, 77, 768)
    gl, bl = 1 + _f32(768, scale=0.1), _f32(768, scale=0.1)
    yl, stl = ops.layernorm_fwd(xl, gl, bl)
    dyl = _bf(2, 77, 768)
    dxl = ops.layernorm_bwd(xl, dyl, gl, stl)
    _sync()
    yl_e, stl_e = E.layernorm_fwd(_cpu(xl), _cpu(gl), _cpu(bl))
    assert_bf16_vs_emu(yl, yl_e, "layernorm_fwd vs emulator", _max_floor(yl_e))
    dxl_e = E.layernorm_bwd(_cpu(xl), _cpu(dyl), _cpu(gl), stl_e)
    assert_bf16_vs_emu(dxl, dxl_e, "layernorm_bwd vs emulator", _max_floor(dxl_e, 2.0**-10), max_frac=1e-2)


@gpu
@contract("geglu_fwd", "geglu_bwd", "add", "upsample2x_fwd", "upsample2x_bwd", "zero_insert2x", "concat_channels",
          "slice_channels", "nchw_to_nhwc", "nhwc_to_nchw_f32")
def test_elementwise_and_layout_match_emulator():
    from controllora_b200 import ops

    _seed("elementwise")
    p = _bf(154, 2 * 1280, scale=2.0)
    # the kernel's and torch's erf differ by a few fp32 ulps: within one bf16 ulp everywhere, more rounding flips than 0.1 %
    assert_bf16_vs_emu(ops.geglu_fwd(p), E.geglu_fwd(_cpu(p)), "geglu_fwd vs emulator", _max_floor(E.geglu_fwd(_cpu(p))), max_frac=2e-2)
    dout = _bf(154, 1280)
    gb, gb_e = ops.geglu_bwd(p, dout), E.geglu_bwd(_cpu(p), _cpu(dout))
    assert_bf16_vs_emu(gb, gb_e, "geglu_bwd vs emulator", _max_floor(gb_e), max_frac=2e-2)
    a, b = _bf(4096), _bf(4096)
    assert torch.equal(_cpu(ops.add(a, b)), E.add(_cpu(a), _cpu(b)))
    x = _bf(2, 8, 6, 320)
    assert torch.equal(_cpu(ops.upsample2x_fwd(x)), E.upsample2x_fwd(_cpu(x)))
    dy = _bf(2, 16, 12, 320)
    assert_bf16_vs_emu(ops.upsample2x_bwd(dy), E.upsample2x_bwd(_cpu(dy)), "upsample2x_bwd vs emulator")
    acc, acc_e = x.clone(), _cpu(x).clone()
    ops.upsample2x_bwd(dy, acc, accumulate=True)
    E.upsample2x_bwd(_cpu(dy), acc_e, accumulate=True)
    assert_bf16_vs_emu(acc, acc_e, "upsample2x_bwd (accumulate) vs emulator", _max_floor(acc_e))
    for off in (0, 1):
        assert torch.equal(_cpu(ops.zero_insert2x(x, off)), E.zero_insert2x(_cpu(x), off))
    c2 = _bf(2, 8, 6, 64)
    assert torch.equal(_cpu(ops.concat_channels(x, c2)), E.concat_channels(_cpu(x), _cpu(c2)))
    assert torch.equal(_cpu(ops.slice_channels(x, 64, 128)), E.slice_channels(_cpu(x), 64, 128))
    dst, dst_e = c2.clone(), _cpu(c2).clone()
    ops.slice_channels(x, 256, 64, dst, accumulate=True)
    E.slice_channels(_cpu(x), 256, 64, dst_e, accumulate=True)
    assert torch.equal(_cpu(dst), dst_e)
    for xin in (_f32(2, 320, 7, 9), _bf(2, 320, 7, 9)):
        assert torch.equal(_cpu(ops.nchw_to_nhwc(xin)), E.nchw_to_nhwc(_cpu(xin)))
    assert torch.equal(_cpu(ops.nhwc_to_nchw_f32(x)), E.nhwc_to_nchw_f32(_cpu(x)))
    o, o_e = _f32(2, 320, 8, 6), None
    o_e = _cpu(o).clone()
    ops.nhwc_to_nchw_f32(x, o, accumulate=True)
    E.nhwc_to_nchw_f32(_cpu(x), o_e, accumulate=True)
    _sync()
    assert torch.equal(_cpu(o), o_e)


@gpu
@contract("conv_in", "conv_out", "conv_out_bwd", "timestep_embedding", "small_linear", "mse_loss")
def test_unet_edges_match_emulator():
    from controllora_b200 import ops

    _seed("edges")
    x = _f32(2, 4, 16, 12)
    w = _bf(320, 3, 3, 4, scale=0.2)
    bias = _f32(320, scale=0.1)
    y, y_e = ops.conv_in(x, w, bias, 320), E.conv_in(_cpu(x), _cpu(w), _cpu(bias), 320)
    assert_bf16_vs_emu(y, y_e, "conv_in vs emulator", _max_floor(y_e))
    h = _bf(2, 16, 12, 320)
    wo = _bf(4, 3, 3, 320, scale=0.05)
    bo = _f32(4)
    co, co_e = ops.conv_out(h, wo, bo), E.conv_out(_cpu(h), _cpu(wo), _cpu(bo))
    co_terms = F.conv2d(h.abs().to(F64).permute(0, 3, 1, 2), wo.abs().to(F64).permute(0, 3, 1, 2), bo.abs().to(F64), padding=1)
    assert_f32_reduction(co, co_e.to(F64), co_terms, "conv_out vs emulator")
    dyo = _f32(2, 4, 16, 12)
    db, db_e = ops.conv_out_bwd(dyo, wo, 320), E.conv_out_bwd(_cpu(dyo), _cpu(wo), 320)
    assert_bf16_vs_emu(db, db_e, "conv_out_bwd vs emulator", _max_floor(db_e))
    t = torch.tensor([0.0, 1.0, 500.0, 999.0], device="cuda")
    te, te_e = ops.timestep_embedding(t, 320), E.timestep_embedding(_cpu(t), 320)
    assert_f32_close(te, te_e, "timestep_embedding vs emulator", 5e-4, torch.ones(1))        # angles up to 999 rad
    xs = _f32(4, 320)
    ws = _bf(1280, 320, scale=0.05)
    bs = _f32(1280, scale=0.1)
    for si, so in ((False, False), (True, True)):
        sl, sl_e = ops.small_linear(xs, ws, bs, si, so), E.small_linear(_cpu(xs), _cpu(ws), _cpu(bs), si, so)
        sl_terms = (F.silu(xs) if si else xs).abs().to(F64) @ ws.abs().to(F64).t() + bs.abs().to(F64)
        assert_f32_reduction(sl, sl_e.to(F64), sl_terms, f"small_linear silu {si}/{so} vs emulator")
    pred, tgt = _f32(2, 4, 8, 8), _f32(2, 4, 8, 8)
    (loss, gr), (loss_e, gr_e) = ops.mse_loss(pred, tgt, 0.5), E.mse_loss(_cpu(pred), _cpu(tgt), 0.5)
    _sync()
    assert_f32_close(loss, loss_e, "mse_loss vs emulator", 1e-5)
    assert_f32_close(gr, gr_e, "mse_loss grad vs emulator", 1e-6, _max_floor(gr_e, 1e-6))


@gpu
@contract("skinny_atb", "rowdot", "rowmat", "skinny_small", "small_matmul", "rank_update", "PackPlan.run", "SkinnyQueue")
def test_lora_side_kernels_match_emulator():
    from controllora_b200 import ops

    _seed("lora_side")
    M, K, N = 3000, 320, 640
    a, b = _f32(M, 8), _bf(M, K)
    out0 = _f32(4, K)
    out, out_e = out0.clone(), _cpu(out0).clone()
    ops.skinny_atb(a, 4, b, out, K, 1, 0.5)
    E.skinny_atb(_cpu(a), 4, _cpu(b), out_e, K, 1, 0.5)
    terms = out0.abs().to(F64) + 0.5 * (a[:, :4].abs().to(F64).t() @ b.abs().to(F64))
    _sync()
    assert_f32_reduction(out, out_e.to(F64), terms, "skinny_atb vs emulator")
    u = _f32(K, 4)
    e, e_e = ops.rowdot(b, u), E.rowdot(_cpu(b), _cpu(u))
    _sync()
    assert_f32_reduction(e, e_e.to(F64), b.abs().to(F64) @ u.abs().to(F64), "rowdot vs emulator")
    w = _f32(4, 8)
    ro, ro_e = torch.empty(M, 4, device="cuda"), torch.empty(M, 4)
    ops.rowmat(a, w, 8, 1, 4, 8, 0.7, ro, 4)
    E.rowmat(_cpu(a), _cpu(w), 8, 1, 4, 8, 0.7, ro_e, 4)
    ob, ob_e = torch.zeros(M, 128, device="cuda", dtype=BF16), torch.zeros(M, 128, dtype=BF16)
    ops.rowmat(a, w, 8, 1, 4, 8, 0.7, ob, 128, out_mode=1, col_off=8, lo_off=64)
    E.rowmat(_cpu(a), _cpu(w), 8, 1, 4, 8, 0.7, ob_e, 128, out_mode=1, col_off=8, lo_off=64)
    _sync()
    rterm = 0.7 * (a.abs().to(F64) @ w.abs().to(F64).t())
    assert_f32_reduction(ro, ro_e.to(F64), rterm, "rowmat vs emulator")
    assert_f32_reduction(ob[:, 8:12].float() + ob[:, 72:76].float(), (ob_e[:, 8:12].float() + ob_e[:, 72:76].float()).to(F64), rterm,
                         "rowmat hi/lo vs emulator")
    b4 = _f32(M, 4)
    ss, ss_e = torch.zeros(4, 4, device="cuda"), torch.zeros(4, 4)
    ops.skinny_small(a, 4, b4, 4, ss, 2.0)
    E.skinny_small(_cpu(a), 4, _cpu(b4), 4, ss_e, 2.0)
    down = _f32(4, K)
    sm, sm_e = torch.zeros(K, 4, device="cuda"), torch.zeros(K, 4)
    ops.small_matmul(down, 1, K, w, 8, 1, sm, 4, 1, K, 4, 4, alpha=1.5)
    E.small_matmul(_cpu(down), 1, K, _cpu(w), 8, 1, sm_e, 4, 1, K, 4, 4, alpha=1.5)
    x = _bf(M, N)
    t = _f32(M, 8)
    tab = _f32(N, 4, scale=0.5)
    ru, ru_e = ops.rank_update(x, t, tab, 0.6), E.rank_update(_cpu(x), _cpu(t), _cpu(tab), 0.6)
    _sync()
    assert_f32_reduction(ss, ss_e.to(F64), 2.0 * (a[:, :4].abs().to(F64).t() @ b4.abs().to(F64)), "skinny_small vs emulator")
    assert_f32_reduction(sm, sm_e.to(F64), 1.5 * (down.abs().to(F64).t() @ w[:, :4].abs().to(F64)), "small_matmul vs emulator")
    assert_bf16_vs_emu(ru, ru_e, "rank_update vs emulator", _floor(x.abs().to(F64) + 0.6 * (t[:, :4].abs().to(F64) @ tab.abs().to(F64).t())))

    # PackPlan: hi/lo ext rows, tables, transposed forms, kind 2 and an unscaled descriptor
    def plan_on(dev, src_down, src_up):
        bufs = (torch.zeros(16, K, device=dev, dtype=BF16), torch.zeros(N, 8, device=dev), torch.zeros(16, N, device=dev, dtype=BF16),
                torch.zeros(K, 4, device=dev), torch.zeros(K, 16, device=dev, dtype=BF16))
        plan = ops.PackPlan(dev)
        plan.add_ext(src_down, bufs[0], row_off=2)
        plan.add_table(src_up, bufs[1], col_off=4)
        plan.add_ext(src_up, bufs[2], transposed=True, unscaled=True)
        plan.add_table(src_down, bufs[3], transposed=True)
        plan.add(src_down, bufs[4], 2, 4, K, src_down.stride(0), src_down.stride(1), 16, 1)
        plan.set_unscaled_mul(2.5)
        return plan, bufs

    dn, upm = _f32(4, K, scale=0.3), _f32(N, 4, scale=0.3)
    plan, bufs = plan_on("cuda", dn, upm)
    plan.run()
    plan_e, bufs_e = plan_on("cpu", _cpu(dn), _cpu(upm))
    E._pack_run(plan_e)
    _sync()
    for i, (x_, e_) in enumerate(zip(bufs, bufs_e)):
        assert torch.equal(_cpu(x_), e_), f"PackPlan buffer {i} differs from the emulator"

    # SkinnyQueue: mixed ranks and widths in one batch, plus the flush
    specs = [(1, 320), (4, 1280), (8, 1280), (3, 8), (2, 640)]
    ops_in = [(_f32(M, 8), r, _bf(M, Cc), _f32(r, Cc), 0.5 + 0.1 * i) for i, (r, Cc) in enumerate(specs)]
    q, qe = ops.SkinnyQueue(), ops.SkinnyQueue()
    outs, outs_e = [], []
    for a_, r, b_, o0, al in ops_in:
        o, oe = o0.clone(), _cpu(o0).clone()
        q.add(a_, r, b_, o, b_.shape[1], 1, al)
        E._skinny_add(qe, _cpu(a_), r, _cpu(b_), oe, b_.shape[1], 1, al)
        outs.append(o)
        outs_e.append(oe)
    q.flush()
    E._skinny_flush(qe)
    _sync()
    for (a_, r, b_, o0, al), o, oe in zip(ops_in, outs, outs_e):
        terms = o0.abs().to(F64) + al * (a_[:, :r].abs().to(F64).t() @ b_.abs().to(F64))
        assert_f32_reduction(o, oe.to(F64), terms, f"SkinnyQueue r={r} C={b_.shape[1]} vs emulator")
