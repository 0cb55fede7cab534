"""Tile-width sweep of cl_gemm on the short-K / small-M UNet shapes: python tools/gemm_bn_sweep.py"""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch
from controllora_b200 import ops

shapes = [(32768, 320, 320), (8192, 640, 640), (2048, 1280, 1280), (512, 1280, 1280), (2048, 1280, 5120), (8192, 640, 2560), (32768, 320, 1280), (2048, 10240, 1280)]
for (M, N, K) in shapes:
    a = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda") / K ** 0.5).to(torch.bfloat16)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    res = []
    for bn in (0, 64, 128, 160, 256):
        if bn and N % bn:
            continue
        try:
            for _ in range(10):
                ops.gemm(a, b, out=out, block_n=bn)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                ops.gemm(a, b, out=out, block_n=bn)
            e1.record()
            torch.cuda.synchronize()
            res.append(f"bn={bn}: {e0.elapsed_time(e1) / 20 * 1e3:6.1f} us")
        except Exception as ex:
            res.append(f"bn={bn}: {type(ex).__name__}")
    print(f"M={M} N={N} K={K}:  " + "  ".join(res), flush=True)
