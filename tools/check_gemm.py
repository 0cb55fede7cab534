"""GPU bring-up check for cl_gemm: each case runs in its own subprocess (a trapped kernel kills only its case).

usage: python tools/check_gemm.py            # run all cases
       python tools/check_gemm.py CASE_NAME  # run one case in-process
"""
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

CASES = {}


def case(fn):
    CASES[fn.__name__] = fn
    return fn


def _setup():
    import torch

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)
    return torch


def _rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-30))


def _gemm_ref(a, b):
    return a.float() @ b.float().t()


def _run_plain(M, N, K, block_n=0, tol=4e-3):
    torch = _setup()
    from controllora_b200 import ops

    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
    out = ops.gemm(a, b, block_n=block_n)
    torch.cuda.synchronize()
    ref = _gemm_ref(a, b)
    err = _rel(out, ref)
    print(f"plain M={M} N={N} K={K} bn={block_n}: rel={err:.3e} maxabs={float((out.float()-ref).abs().max()):.3e}")
    assert err < tol, err


@case
def plain_1tile():
    _run_plain(128, 128, 64, 128)


@case
def plain_k320():
    _run_plain(256, 128, 320, 128)


@case
def plain_bn64():
    _run_plain(384, 64, 128, 64)


@case
def plain_bn160_tail():
    _run_plain(1000, 320, 320, 160)


@case
def plain_bn256():
    _run_plain(4096, 2560, 320, 256)


@case
def plain_bn320():
    """requested 320-column tiles (not an instantiated width: cl_gemm falls back to its tail-tile choice), M tails included."""
    _run_plain(4096, 640, 2560, 320)
    _run_plain(32768, 320, 2880, 320)
    _run_plain(1000, 320, 2048, 320)      # M tail


@case
def plain_big():
    _run_plain(32768, 320, 320)
    _run_plain(8192, 640, 2560)
    _run_plain(616, 1280, 768)


@case
def epilogue_all():
    torch = _setup()
    from controllora_b200 import ops

    M, N, K = 2048, 640, 640
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda")
    rb = torch.randn(8, N, device="cuda")
    res = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    ref = _gemm_ref(a, b) + bias + rb.repeat_interleave(M // 8, 0) + res.float()
    out = ops.gemm(a, b, bias=bias, row_bias=rb, rows_per_group=M // 8, residual=res)
    out32 = ops.gemm(a, b, bias=bias, row_bias=rb, rows_per_group=M // 8, residual=res, out_fp32=True)
    torch.cuda.synchronize()
    print(f"epilogue bf16 rel={_rel(out, ref):.3e}  fp32 rel={_rel(out32, ref):.3e}")
    assert _rel(out, ref) < 4e-3 and _rel(out32, ref) < 1e-5
    # in-place accumulate (residual aliases out)
    acc = res.clone()
    ops.gemm(a, b, residual=acc, out=acc)
    torch.cuda.synchronize()
    ref2 = _gemm_ref(a, b) + res.float()
    print(f"accumulate rel={_rel(acc, ref2):.3e}")
    assert _rel(acc, ref2) < 4e-3


def _run_lora(M, N, K, r, rp, with_tadd):
    torch = _setup()
    from controllora_b200 import ops

    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
    down = torch.randn(r, K, device="cuda") / r
    up = torch.zeros(N, rp, device="cuda")
    up[:, :r] = torch.randn(N, r, device="cuda") * 0.5
    scale = 0.7
    ext = ops.split_bf16_ext(down, K)
    t_add = torch.zeros(M, rp, device="cuda")
    if with_tadd:
        t_add[:, :r] = torch.randn(M, r, device="cuda")
    t_out = torch.empty(M, rp, device="cuda")
    out = ops.gemm(a, b, ext=ext, lora_up=up, lora_scale=scale, t_add=t_add if with_tadd else None, t_out=t_out,
                   out_fp32=True)
    torch.cuda.synchronize()
    t_ref = a.float() @ down.t()
    if with_tadd:
        t_ref = t_ref + t_add[:, :r]
    base = _gemm_ref(a, b)
    lora = scale * (t_ref @ up[:, :r].t())
    ref = base + lora
    e_all = _rel(out, ref)
    e_lora = _rel(out - base, lora)
    e_t = _rel(t_out[:, :r], t_ref)
    print(f"lora M={M} N={N} K={K} r={r} rp={rp} tadd={with_tadd}: rel={e_all:.3e} lora-term rel={e_lora:.3e} t rel={e_t:.3e}")
    assert e_all < 1e-4 and e_lora < 1e-3 and e_t < 1e-4


@case
def lora_r4():
    _run_lora(4096, 320, 320, 4, 4, False)


@case
def lora_r4_tadd():
    _run_lora(1000, 640, 640, 4, 4, True)


@case
def lora_r8_cross():
    _run_lora(616, 1280, 768, 8, 8, False)


@case
def resident_short_k():
    """M large enough for the smem-resident-weights mode (per-lane store epilogue): the bf16 transpose path (nothing added to the
    accumulator), the fp32 transpose path with bias + residual, and the LoRA epilogue (rank 4 and stacked rank 8) with bf16 output."""
    torch = _setup()
    from controllora_b200 import ops

    _run_plain(32768, 320, 320)
    _run_plain(16384 + 64, 640, 320)
    M, N, K = 32768, 320, 320
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda")
    res = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    base = _gemm_ref(a, b)
    out = ops.gemm(a, b, bias=bias, residual=res)
    torch.cuda.synchronize()
    e = _rel(out, base + bias + res.float())
    print(f"resident bias+residual: rel={e:.3e}")
    assert e < 4e-3
    for r, rp in ((4, 4), (8, 8)):
        down = torch.randn(r, K, device="cuda") / r
        up = torch.randn(N, rp, device="cuda") * 0.5
        t_add = torch.randn(M, rp, device="cuda")
        t_out = torch.empty(M, rp, device="cuda")
        out = ops.gemm(a, b, ext=ops.split_bf16_ext(down, K), lora_up=up, lora_scale=0.7, t_add=t_add, t_out=t_out, bias=bias, residual=res)
        torch.cuda.synchronize()
        t_ref = a.float() @ down.t() + t_add[:, :r]
        ref = base + 0.7 * (t_ref @ up[:, :r].t()) + bias + res.float()
        e, e_t = _rel(out, ref), _rel(t_out[:, :r], t_ref)
        lora_only = _rel(out.float() - base - bias - res.float(), 0.7 * (t_ref @ up[:, :r].t()))
        print(f"resident lora r={r}: rel={e:.3e} lora-term rel={lora_only:.3e} t rel={e_t:.3e}")
        assert e < 4e-3 and e_t < 1e-4 and lora_only < 3e-2


@case
def two_cta_plain():
    """short-K shapes the planner runs two CTAs per SM (BN 128), one with an M that is not a multiple of 128"""
    _run_plain(16384, 384, 320)
    _run_plain(32700, 384, 320)


@case
def two_cta_epilogue():
    """two CTAs per SM with bias + row bias + residual, in bf16 and fp32 output"""
    torch = _setup()
    from controllora_b200 import ops

    M, N, K = 16384, 384, 320
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda")
    rb = torch.randn(8, N, device="cuda")
    res = torch.randn(M, N, device="cuda").to(torch.bfloat16)
    ref = _gemm_ref(a, b) + bias + rb.repeat_interleave(M // 8, 0) + res.float()
    out = ops.gemm(a, b, bias=bias, row_bias=rb, rows_per_group=M // 8, residual=res)
    out32 = ops.gemm(a, b, bias=bias, row_bias=rb, rows_per_group=M // 8, residual=res, out_fp32=True)
    torch.cuda.synchronize()
    print(f"two-CTA epilogue bf16 rel={_rel(out, ref):.3e}  fp32 rel={_rel(out32, ref):.3e}")
    assert _rel(out, ref) < 4e-3 and _rel(out32, ref) < 1e-5


@case
def two_cta_conv():
    """hint-encoder 3x3 convs at two CTAs per SM: 32 channels (BK 32) at BN 32 and 64, 64 channels at BN 128, stride 2"""
    _conv_case(2, 256, 256, 32, 32, 1, 1, True)
    _conv_case(2, 256, 256, 32, 64, 1, 1, False)
    _conv_case(8, 128, 128, 64, 128, 1, 1, True)
    _conv_case(2, 512, 512, 32, 32, 2, 0, False)


def _conv_case(n, H, W, Cc, N, stride, pad_lo, with_epi):
    torch = _setup()
    import torch.nn.functional as F
    from controllora_b200 import ops

    x = torch.randn(n, H, W, Cc, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, 3, 3, Cc, device="cuda") / (9 * Cc) ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda") if with_epi else None
    rb = torch.randn(n, N, device="cuda") if with_epi else None
    Ho, Wo = H // stride, W // stride
    out = ops.gemm(x, w.view(N, 9 * Cc), conv_stride=stride, pad_lo=pad_lo, bias=bias, row_bias=rb,
                   rows_per_group=Ho * Wo)
    torch.cuda.synchronize()
    xn = x.float().permute(0, 3, 1, 2)
    wn = w.float().permute(0, 3, 1, 2)
    if stride == 1:
        ref = F.conv2d(xn, wn, padding=1)
    elif pad_lo == 1:
        ref = F.conv2d(xn, wn, stride=2, padding=1)
    else:
        ref = F.conv2d(F.pad(xn, (0, 1, 0, 1)), wn, stride=2, padding=0)
    if with_epi:
        ref = ref + bias[None, :, None, None] + rb[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1)
    err = _rel(out, ref)
    print(f"conv n={n} {H}x{W} C={Cc} N={N} stride={stride} pad_lo={pad_lo}: rel={err:.3e}")
    assert err < 4e-3, err


@case
def conv_s1_64():
    _conv_case(2, 64, 64, 320, 320, 1, 1, True)


@case
def conv_s1_small():
    _conv_case(4, 8, 8, 1280, 1280, 1, 1, False)
    _conv_case(3, 16, 16, 640, 1280, 1, 1, True)
    _conv_case(2, 32, 32, 960, 640, 1, 1, False)


@case
def conv_s2():
    _conv_case(2, 64, 64, 320, 320, 2, 1, True)
    _conv_case(2, 64, 64, 64, 64, 2, 0, False)
    _conv_case(4, 16, 16, 1280, 1280, 2, 1, False)


@case
def conv_bn320():
    """deep-K convs whose N is a multiple of 320, with the fused epilogue operands"""
    _conv_case(8, 64, 64, 320, 320, 1, 1, True)
    _conv_case(8, 32, 32, 640, 640, 1, 1, True)
    _conv_case(8, 32, 32, 1280, 640, 1, 1, False)


@case
def conv_96():
    _conv_case(1, 96, 96, 320, 320, 1, 1, False)
    _conv_case(2, 24, 24, 1280, 1280, 1, 1, False)


@case
def split_k():
    """Few output tiles + deep K: ops.gemm cuts K across CTAs (fp32 partial tiles + finishing kernel).  Checks the
    epilogue (bias / row_bias / residual, bf16 and fp32 out), an uneven split and run-to-run bit stability."""
    torch = _setup()
    from controllora_b200 import ops

    for (M, N, K) in [(512, 1280, 5120), (200, 640, 2112), (128, 320, 11520)]:
        a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
        b = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
        bias = torch.randn(N, device="cuda")
        rb = torch.randn(8, N, device="cuda")
        res = torch.randn(M, N, device="cuda").to(torch.bfloat16)
        rpg = (M + 7) // 8
        grp = torch.arange(M, device="cuda") // rpg
        ref = _gemm_ref(a, b) + bias + rb[grp] + res.float()
        out = ops.gemm(a, b, bias=bias, row_bias=rb, rows_per_group=rpg, residual=res)
        out_b = ops.gemm(a, b, bias=bias, row_bias=rb, rows_per_group=rpg, residual=res)
        out32 = ops.gemm(a, b, bias=bias, row_bias=rb, rows_per_group=rpg, residual=res, out_fp32=True)
        torch.cuda.synchronize()
        print(f"split-K M={M} N={N} K={K}: bf16 rel={_rel(out, ref):.3e} fp32 rel={_rel(out32, ref):.3e}")
        assert _rel(out, ref) < 4e-3 and _rel(out32, ref) < 1e-5
        assert torch.equal(out, out_b)
    _conv_case(8, 8, 8, 2560, 1280, 1, 1, True)
    _conv_case(8, 8, 8, 1280, 1280, 1, 1, True)


@case
def perf():
    torch = _setup()
    from controllora_b200 import ops

    shapes = [
        (32768, 320, 320), (8192, 640, 640), (2048, 1280, 1280), (32768, 2560, 320), (32768, 320, 1280),
        (8192, 5120, 640), (8192, 640, 2560), (2048, 10240, 1280), (2048, 1280, 5120), (8192, 8192, 8192),
    ]
    for (M, N, K) in shapes:
        a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
        b = (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        for _ in range(3):
            ops.gemm(a, b, out=out)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 20
        e0.record()
        for _ in range(iters):
            ops.gemm(a, b, out=out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        # cuBLAS for context (not part of the product path)
        for _ in range(3):
            torch.matmul(a, b.t())
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            torch.matmul(a, b.t())
        e1.record()
        torch.cuda.synchronize()
        ms_ref = e0.elapsed_time(e1) / iters
        fl = 2.0 * M * N * K
        by = 2.0 * (M * K + N * K + M * N)
        print(f"perf M={M:6d} N={N:6d} K={K:5d}: {ms*1e3:8.1f} us {fl/ms/1e9:8.1f} TFLOP/s {by/ms/1e6:7.1f} GB/s | cuBLAS {ms_ref*1e3:8.1f} us {fl/ms_ref/1e9:8.1f} TFLOP/s")
    # conv perf (last row: the hint encoder's 32-channel level at 512 x 512)
    for (n, H, Cc, N) in [(8, 64, 320, 320), (8, 32, 640, 640), (8, 16, 1280, 1280), (8, 8, 1280, 1280), (8, 512, 32, 32)]:
        x = torch.randn(n, H, H, Cc, device="cuda").to(torch.bfloat16)
        w = (torch.randn(N, 9 * Cc, device="cuda") / (9 * Cc) ** 0.5).to(torch.bfloat16)
        out = torch.empty(n, H, H, N, device="cuda", dtype=torch.bfloat16)
        for _ in range(3):
            ops.gemm(x, w, out=out, conv_stride=1)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            ops.gemm(x, w, out=out, conv_stride=1)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        fl = 2.0 * n * H * H * N * 9 * Cc
        print(f"perf conv n={n} {H}x{H} C={Cc} N={N}: {ms*1e3:8.1f} us {fl/ms/1e9:8.1f} TFLOP/s")


def main():
    if len(sys.argv) > 1:
        CASES[sys.argv[1]]()
        print("CASE_OK")
        return
    results = {}
    for name in CASES:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, __file__, name], capture_output=True, text=True, timeout=150)
            ok = r.returncode == 0 and "CASE_OK" in r.stdout
            out = r.stdout + r.stderr
        except subprocess.TimeoutExpired as e:
            ok, out = False, f"TIMEOUT {e}"
        results[name] = ok
        print(f"=== {name}: {'PASS' if ok else 'FAIL'} ({time.time()-t0:.1f}s)")
        tail = out.strip().splitlines()
        for line in (tail if ok else tail[-25:]):
            print("    " + line)
        sys.stdout.flush()
    print("SUMMARY", results)
    sys.exit(0 if all(results.values()) else 1)


if __name__ == "__main__":
    main()
