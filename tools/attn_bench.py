"""Attention kernel timing at the SD-1.5 shapes of the bs-8 train step (CUDA events, 20 launches after 3 warm-up launches),
with torch's scaled_dot_product_attention on the same tensors beside it for context, and the achieved rate of the QK^T + PV
matmuls (4 B H Nq Nk d FLOP forward, 2.5x that backward).

usage: python tools/attn_bench.py [--dump DIR]

--dump DIR: instead of timing, writes o, lse, dq, dk and dv of every shape, from the same seeded inputs, as
DIR/<shape>_<name>.npy, so two builds of the library (CLB_LIB) can be compared bit for bit."""
import argparse
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch
import torch.nn.functional as F

from controllora_b200 import ops

SHAPES = [  # (B, Nq, Nk, heads, d): self-attention at 64² / 32² / 16² latents, cross-attention to 77 text tokens
    (8, 4096, 4096, 8, 40), (8, 1024, 1024, 8, 80), (8, 256, 256, 8, 160), (8, 4096, 77, 8, 40), (8, 1024, 77, 8, 80),
]


def timed(fn, n=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def inputs(B, Nq, Nk, H, d):
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(B, Nq, H * d, device="cuda", generator=g).to(torch.bfloat16)
    k = torch.randn(B, Nk, H * d, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn(B, Nk, H * d, device="cuda", generator=g).to(torch.bfloat16)
    do = torch.randn(B, Nq, H * d, device="cuda", generator=g).to(torch.bfloat16)
    return q, k, v, do


def dump(out_dir):
    import numpy as np

    out = Path(out_dir)
    out.mkdir(parents=True, exist_ok=True)
    for B, Nq, Nk, H, d in SHAPES:
        q, k, v, do = inputs(B, Nq, Nk, H, d)
        scale = d ** -0.5
        o, lse = ops.attention_fwd(q, k, v, H, scale)
        dq, dk, dv = ops.attention_bwd(q, k, v, o, do, lse, H, scale)
        tag = f"B{B}_Nq{Nq}_Nk{Nk}_H{H}_d{d}"
        for name, t in (("o", o), ("lse", lse), ("dq", dq), ("dk", dk), ("dv", dv)):
            t = t.view(torch.int16) if t.dtype == torch.bfloat16 else t   # numpy has no bf16: keep the raw bits
            np.save(out / f"{tag}_{name}.npy", t.cpu().numpy())
    print(f"dumped o, lse, dq, dk, dv of {len(SHAPES)} shapes to {out}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dump", default=None, metavar="DIR")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attn_bench: needs a CUDA device")
    print(torch.cuda.get_device_name(0))
    if a.dump:
        dump(a.dump)
        return
    for B, Nq, Nk, H, d in SHAPES:
        q, k, v, do = inputs(B, Nq, Nk, H, d)
        scale = d ** -0.5
        o, lse = ops.attention_fwd(q, k, v, H, scale)
        t_f = timed(lambda: ops.attention_fwd(q, k, v, H, scale))
        t_b = timed(lambda: ops.attention_bwd(q, k, v, o, do, lse, H, scale))
        sp = lambda t, n: t.view(B, n, H, d).transpose(1, 2)
        qt, kt, vt = (sp(t, n).detach().requires_grad_(True) for t, n in ((q, Nq), (k, Nk), (v, Nk)))
        ot = F.scaled_dot_product_attention(qt, kt, vt, scale=scale)
        dot = sp(do, Nq)
        t_tf = timed(lambda: F.scaled_dot_product_attention(qt, kt, vt, scale=scale))
        t_tb = timed(lambda: torch.autograd.grad(ot, (qt, kt, vt), dot, retain_graph=True))
        ref = ot.detach().transpose(1, 2).reshape(B, Nq, H * d).float()
        err = float((o.float() - ref).norm() / ref.norm())
        fl = 4.0 * B * H * Nq * Nk * d
        print(f"B={B} Nq={Nq} Nk={Nk} H={H} d={d}: fwd {t_f * 1e3:8.1f} us ({fl / t_f / 1e9:6.1f} TFLOP/s)  bwd {t_b * 1e3:8.1f} us "
              f"({2.5 * fl / t_b / 1e9:6.1f} TFLOP/s) | torch sdpa fwd {t_tf * 1e3:8.1f} us bwd {t_tb * 1e3:8.1f} us | rel err vs sdpa {err:.1e}",
              flush=True)


if __name__ == "__main__":
    main()
