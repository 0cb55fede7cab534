"""The two-CTA short-K GEMM tiles (pytest -m gpu for the kernels; the ptxas check needs only nvcc).

GPU: every two-CTA instantiation, at census shapes and with M and N tails, with each epilogue input (bias, per-image row
bias, residual read from its own buffer or from the output itself, LoRA t_add / t_out, fp32 output).  Each case runs M rows
planned at two CTAs per SM and its first M1 rows planned at one, into outputs that sit inside sentinel-filled buffers: no
byte outside an output may change, and the two plans must give the same bits, since they issue the same MMA sequence and
the same epilogue arithmetic.

CPU: ptxas must keep the wgmma groups of every GEMM instantiation in flight (no C7515 / C7518 / C7519 serialisation) and
spill nothing.
"""
from __future__ import annotations

import re
import shutil
import subprocess
import zlib
from pathlib import Path

import pytest
import torch

from tools.gemm_occupancy import _Recorder

CSRC = Path(__file__).resolve().parent.parent / "controllora_b200" / "csrc"
SENT = {torch.bfloat16: (torch.int16, 0x5A5A), torch.float32: (torch.int32, 0x5A5A5A5A)}
TAIL_ROWS, PAD_COLS = 64, 8


def _plans(fn):
    """Run fn with every cl_gemm call recorded; returns the plans (block_n, splits, ctas_per_sm, resident_per_sm)."""
    from controllora_b200 import _lib

    rec = _Recorder(_lib.lib())
    _lib._lib = rec
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        _lib._lib = rec.real
    return [r[1] for r in rec.rows]


class _Canvas:
    """A [M + TAIL_ROWS, N + 2 * pad] sentinel buffer whose rows 0..M, columns pad..pad + N are the output."""

    def __init__(self, M, N, dtype, pad=PAD_COLS):
        it, bits = SENT[dtype]
        self.buf = torch.full((M + TAIL_ROWS, N + 2 * pad), bits, dtype=it, device="cuda").view(dtype)
        self.view = self.buf[:M, pad:pad + N]
        self.mask = torch.ones(self.buf.shape, dtype=torch.bool, device="cuda")
        self.mask[:M, pad:pad + N] = False

    def check(self, what):
        it, bits = SENT[self.buf.dtype]
        bad = int((self.buf.view(it)[self.mask] != bits).sum())
        assert bad == 0, f"{what}: {bad} elements written outside the output"


# (name, block_n, lora, conv channels (0: plain matrix), N, K, images or rows at two CTAs per SM, the same at one)
INSTANTIATIONS = [
    ("bn160", 160, False, 0, 320, 320, 32768, 8192),
    ("bn128", 128, False, 0, 384, 320, 16384, 8192),
    ("lora_bn64", 64, True, 0, 320, 320, 8192, 4096),
    ("lora_bn128", 128, True, 0, 384, 320, 16384, 8192),
    ("lora_bn160", 160, True, 0, 320, 320, 32768, 8192),
    ("conv_bk32_bn32", 32, False, 32, 32, 288, 4, 2),
    ("conv_bk32_bn64", 64, False, 32, 64, 288, 4, 2),
    ("conv_bk32_bn128", 128, False, 32, 128, 288, 4, 2),
    ("conv_bn128", 128, False, 64, 128, 576, 4, 2),
]
EPILOGUES = ["plain", "bias_rowbias_residual", "residual_aliased", "fp32_bias"]
CONV_SIDE = 128


@pytest.mark.gpu
@pytest.mark.parametrize("tail", [False, True], ids=["exact", "tails"])
@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("name,bn,lora,conv_c,N,K,big,small", INSTANTIATIONS, ids=[i[0] for i in INSTANTIATIONS])
def test_two_cta_tile_matches_one_cta_plan(name, bn, lora, conv_c, N, K, big, small, epi, tail):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from controllora_b200 import ops

    if tail and conv_c:
        N -= 4                                       # an N tail only: the images set the conv's M
    elif tail:
        N, big, small = N + 16, big - 68, small - 68
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(repr((name, epi, tail)).encode()))
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    if conv_c:
        x = rnd(big, CONV_SIDE, CONV_SIDE, conv_c).to(torch.bfloat16)
        rows_per_img = CONV_SIDE * CONV_SIDE
        M, M1 = big * rows_per_img, small * rows_per_img
        a_of = lambda m: x[: m // rows_per_img]
        conv = {"conv_stride": 1}
    else:
        x = rnd(big, K).to(torch.bfloat16)
        M, M1 = big, small
        a_of = lambda m: x[:m]
        conv = {}
    w = (rnd(N, K) / K**0.5).to(torch.bfloat16)
    fp32 = epi == "fp32_bias"
    kw = {"block_n": bn, "out_fp32": fp32}
    if epi in ("bias_rowbias_residual", "residual_aliased", "fp32_bias"):
        kw["bias"] = rnd(N)
    row_bias = rnd(8, N) if epi == "bias_rowbias_residual" else None
    res = rnd(M, N).to(torch.bfloat16) if epi in ("bias_rowbias_residual", "residual_aliased") else None
    rp = 8 if bn == 128 else 4
    if lora:
        down = rnd(rp, K) / K**0.5
        up = rnd(N, rp) * 0.5
        kw.update(ext=ops.split_bf16_ext(down, K), lora_up=up, lora_scale=0.7)
        t_add = rnd(M, rp)

    outs, t_outs, plans = [], [], []
    for m in (M, M1):
        c = _Canvas(m, N, torch.float32 if fp32 else torch.bfloat16)
        extra = {}
        if row_bias is not None:
            # groups of the M rows: each of the first M1 rows is in the same group in both runs
            extra.update(row_bias=row_bias, rows_per_group=(M + 7) // 8)
        if res is not None:
            if epi == "residual_aliased":
                c.view.copy_(res[:m])
                extra["residual"] = c.view
            else:
                extra["residual"] = res[:m]
        if lora:
            tc = _Canvas(m, rp, torch.float32, pad=0)     # t_out is a contiguous [m, rp]: sentinel rows after it
            t_out = tc.view
            extra.update(t_add=t_add[:m], t_out=t_out)
        plans += _plans(lambda: ops.gemm(a_of(m), w, out=c.view, **conv, **kw, **extra))
        c.check(f"{name} {epi} M={m}")
        if lora:
            tc.check(f"{name} {epi} t_out M={m}")
        outs.append(c.view)
        if lora:
            t_outs.append(t_out)
    assert [(p[0], p[1], p[2]) for p in plans] == [(bn, 1, 2), (bn, 1, 1)], plans
    assert plans[0][3] == 2, f"the device keeps {plans[0][3]} CTAs of this kernel resident per SM"
    assert torch.equal(outs[0][:M1], outs[1]), f"{name} {epi}: two-CTA and one-CTA outputs differ"
    if lora:
        assert torch.equal(t_outs[0][:M1], t_outs[1]), f"{name} {epi}: t_out differs"


def test_gemm_wgmma_groups_stay_in_flight(tmp_path):
    """ptxas -v over gemm_wgmma.cu: no instantiation serialises its wgmma groups and none spills."""
    from controllora_b200 import build

    if shutil.which(build.NVCC) is None and not Path(build.NVCC).exists():
        pytest.skip("nvcc not found")
    cmd = [build.NVCC, *build.FLAGS, "-Xptxas", "-v", "-c", str(CSRC / "gemm_wgmma.cu"), "-o", str(tmp_path / "g.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    assert "gemm_wgmma_kernel" in log, "ptxas printed no per-kernel report"
    serialised = [l for l in log.splitlines() if re.search(r"\(C75(15|18|19)\)|wgmma\.mma_async instructions are serialized", l)]
    assert not serialised, "\n".join(serialised)
    spills = [l for l in log.splitlines() if re.search(r"[1-9]\d* bytes spill (stores|loads)", l)]
    assert not spills, "\n".join(spills)
