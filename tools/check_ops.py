"""GPU bring-up checks for attention / norm / elementwise / edge kernels against torch fp32 references.
Each case runs in its own subprocess.  usage: python tools/check_ops.py [CASE]"""
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


def _attn_ref(q, k, v, H, scale):
    import torch

    B, Nq, HD = q.shape
    d = HD // H
    qf = q.float().view(B, Nq, H, d).transpose(1, 2)
    kf = k.float().view(B, -1, H, d).transpose(1, 2)
    vf = v.float().view(B, -1, H, d).transpose(1, 2)
    s = (qf @ kf.transpose(-1, -2)) * scale
    p = s.softmax(-1)
    o = (p @ vf).transpose(1, 2).reshape(B, Nq, HD)
    lse = torch.logsumexp(s, -1) * 1.4426950408889634
    return o, lse


def _attn_case(B, H, Nq, Nk, d, tol=6e-3):
    torch = _setup()
    from controllora_b200 import ops

    q = torch.randn(B, Nq, H * d, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, Nk, H * d, device="cuda").to(torch.bfloat16)
    v = torch.randn(B, Nk, H * d, device="cuda").to(torch.bfloat16)
    scale = d**-0.5
    o, lse = ops.attention_fwd(q, k, v, H, scale)
    torch.cuda.synchronize()
    ro, rl = _attn_ref(q, k, v, H, scale)
    eo, el = _rel(o, ro), float((lse - rl).abs().max())
    print(f"attn B={B} H={H} Nq={Nq} Nk={Nk} d={d}: o rel={eo:.3e} lse maxabs={el:.3e}")
    assert eo < tol and el < 2e-2, (eo, el)


@case
def attn_d64_one_block():
    _attn_case(1, 1, 128, 128, 64)


@case
def attn_d40():
    _attn_case(2, 8, 1024, 1024, 40)


@case
def attn_cross77():
    _attn_case(2, 8, 1024, 77, 40)
    _attn_case(2, 8, 256, 77, 160)


@case
def attn_d80_d160():
    _attn_case(2, 8, 1024, 1024, 80)
    _attn_case(2, 8, 256, 256, 160)
    _attn_case(2, 8, 64, 64, 160)


@case
def attn_small_d():
    _attn_case(2, 4, 256, 256, 16)
    _attn_case(1, 2, 200, 300, 32)


@case
def attn_paired():
    """Paired-tile forward kernel (d <= 64, Nq > 128): ragged query/key counts (second tile partly / fully out of
    range), many key blocks, and keys whose magnitude jumps in later blocks so that the lazy O rescale (row max
    growing by more than 2^8) actually runs."""
    torch = _setup()
    from controllora_b200 import ops

    _attn_case(1, 2, 200, 300, 40)
    _attn_case(2, 3, 300, 77, 64)
    _attn_case(1, 2, 640, 1000, 8)
    B, H, N, d = 2, 4, 512, 40
    q = torch.randn(B, N, H * d, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, N, H * d, device="cuda")
    k[:, 128:256] *= 6.0
    k[:, 384:] *= 30.0
    k = k.to(torch.bfloat16)
    v = torch.randn(B, N, H * d, device="cuda").to(torch.bfloat16)
    o, lse = ops.attention_fwd(q, k, v, H, d**-0.5)
    torch.cuda.synchronize()
    ro, rl = _attn_ref(q, k, v, H, d**-0.5)
    eo, el = _rel(o, ro), float((lse - rl).abs().max())
    print(f"attn growing-max: o rel={eo:.3e} lse maxabs={el:.3e}")
    assert eo < 6e-3 and el < 5e-2, (eo, el)


@case
def attn_perf():
    torch = _setup()
    from controllora_b200 import ops

    for (B, H, N, Nk, d) in [(8, 8, 4096, 4096, 40), (8, 8, 4096, 77, 40), (8, 8, 1024, 1024, 80), (8, 8, 256, 256, 160)]:
        q = torch.randn(B, N, H * d, device="cuda").to(torch.bfloat16)
        k = torch.randn(B, Nk, H * d, device="cuda").to(torch.bfloat16)
        v = torch.randn(B, Nk, H * d, device="cuda").to(torch.bfloat16)
        o = torch.empty_like(q)
        for _ in range(3):
            ops.attention_fwd(q, k, v, H, d**-0.5, out=o)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.attention_fwd(q, k, v, H, d**-0.5, out=o)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        fl = 4.0 * B * H * N * Nk * d
        print(f"attn perf B={B} N={N} Nk={Nk} d={d}: {ms*1e3:.1f} us  {fl/ms/1e9:.1f} TFLOP/s")


@case
def groupnorm():
    torch = _setup()
    import torch.nn.functional as F
    from controllora_b200 import ops

    # incl. batch 8 (16-CTA clusters), HW not divisible by the cluster size (10x10), hint-encoder channel counts, 2x2 maps, and
    # wide shapes: group totals larger than the partial-sum area (C = G = 2056), more than 100 KiB of shared memory per CTA
    # (8-CTA clusters), and the largest shared-memory footprint (C = G = 4096)
    for (n, H, C, G, silu, eps) in [(2, 64, 320, 32, True, 1e-5), (3, 16, 1280, 32, False, 1e-6), (2, 32, 2560, 32, True, 1e-5),
                                    (2, 64, 64, 32, True, 1e-6), (8, 32, 320, 32, True, 1e-5), (2, 10, 640, 32, True, 1e-5),
                                    (1, 128, 32, 32, True, 1e-6), (3, 2, 128, 32, False, 1e-5), (16, 16, 1920, 32, True, 1e-5),
                                    (1, 4, 2056, 2056, True, 1e-5), (17, 2, 4096, 512, False, 1e-5), (17, 4, 4096, 4096, True, 1e-6)]:
        x = (torch.randn(n, H, H, C, device="cuda") * 1.5 + 0.3).to(torch.bfloat16)
        g = 1 + 0.1 * torch.randn(C, device="cuda")
        b = 0.1 * torch.randn(C, device="cuda")
        y, stats = ops.groupnorm_fwd(x, g, b, G, eps, silu)
        xr = x.float().permute(0, 3, 1, 2).requires_grad_(True)
        gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
        z = F.group_norm(xr, G, gr, br, eps)
        yr = F.silu(z) if silu else z
        dy = torch.randn_like(yr).to(torch.bfloat16)
        yr.backward(dy.float())
        dg = torch.zeros(C, device="cuda")
        db = torch.zeros(C, device="cuda")
        dyc = dy.permute(0, 2, 3, 1).contiguous()
        dx = ops.groupnorm_bwd(x, dyc, g, b, stats, G, silu, dgamma=dg, dbeta=db)
        acc = dx.clone()
        ops.groupnorm_bwd(x, dyc, g, b, stats, G, silu, dx=acc, accumulate=True)
        torch.cuda.synchronize()
        mean_ref = x.float().view(n, H * H, G, C // G).mean(dim=(1, 3))
        assert _rel(stats[..., 0], mean_ref) < 1e-3 and _rel(acc, 2 * xr.grad.permute(0, 2, 3, 1)) < 8e-3
        e1 = _rel(y, yr.permute(0, 2, 3, 1))
        e2 = _rel(dx, xr.grad.permute(0, 2, 3, 1))
        e3, e4 = _rel(dg, gr.grad), _rel(db, br.grad)
        print(f"groupnorm n={n} H={H} C={C} silu={silu}: y rel={e1:.3e} dx rel={e2:.3e} dgamma rel={e3:.3e} dbeta rel={e4:.3e}")
        assert e1 < 4e-3 and e2 < 4e-3 and e3 < 1e-3 and e4 < 1e-3


@case
def layernorm():
    torch = _setup()
    import torch.nn.functional as F
    from controllora_b200 import ops

    for (T, C) in [(1000, 320), (512, 640), (300, 1280), (64, 128), (40, 2560)]:
        x = (torch.randn(T, C, device="cuda") * 2 + 0.5).to(torch.bfloat16)
        g = 1 + 0.1 * torch.randn(C, device="cuda")
        b = 0.1 * torch.randn(C, device="cuda")
        y, stats = ops.layernorm_fwd(x, g, b, 1e-5)
        xr = x.float().requires_grad_(True)
        yr = F.layer_norm(xr, (C,), g, b, 1e-5)
        dy = torch.randn_like(yr).to(torch.bfloat16)
        yr.backward(dy.float())
        dx = ops.layernorm_bwd(x, dy, g, stats)
        acc = dx.clone()
        ops.layernorm_bwd(x, dy, g, stats, dx=acc, accumulate=True)
        torch.cuda.synchronize()
        e1, e2, e3 = _rel(y, yr), _rel(dx, xr.grad), _rel(acc, 2 * xr.grad)
        print(f"layernorm T={T} C={C}: y rel={e1:.3e} dx rel={e2:.3e} acc rel={e3:.3e}")
        assert e1 < 4e-3 and e2 < 4e-3 and e3 < 6e-3


@case
def elementwise():
    torch = _setup()
    import torch.nn.functional as F
    from controllora_b200 import ops

    p = torch.randn(1000, 2560, device="cuda").to(torch.bfloat16)
    pr = p.float().requires_grad_(True)
    a, g = pr.chunk(2, -1)
    outr = a * F.gelu(g)
    out = ops.geglu_fwd(p)
    do = torch.randn_like(outr).to(torch.bfloat16)
    outr.backward(do.float())
    dp = ops.geglu_bwd(p, do)
    print(f"geglu fwd rel={_rel(out, outr):.3e} bwd rel={_rel(dp, pr.grad):.3e}")
    assert _rel(out, outr) < 4e-3 and _rel(dp, pr.grad) < 4e-3
    x = torch.randn(2, 8, 8, 64, device="cuda").to(torch.bfloat16)
    up = ops.upsample2x_fwd(x)
    upr = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(up.float(), upr)
    dyu = torch.randn(2, 16, 16, 64, device="cuda").to(torch.bfloat16)
    dxu = ops.upsample2x_bwd(dyu)
    ref = dyu.float().view(2, 8, 2, 8, 2, 64).sum((2, 4))
    assert _rel(dxu, ref) < 4e-3
    zi = ops.zero_insert2x(x, 1)
    zr = torch.zeros(2, 16, 16, 64, device="cuda")
    zr[:, 1::2, 1::2] = x.float()
    assert torch.equal(zi.float(), zr)
    a_ = torch.randn(100, 64, device="cuda").to(torch.bfloat16)
    b_ = torch.randn(100, 128, device="cuda").to(torch.bfloat16)
    cat = ops.concat_channels(a_, b_)
    assert torch.equal(cat, torch.cat([a_, b_], -1))
    sl = ops.slice_channels(cat, 64, 128)
    assert torch.equal(sl, b_)
    ops.slice_channels(cat, 64, 128, dst=sl, accumulate=True)
    assert _rel(sl, 2 * b_.float()) < 4e-3
    s = ops.add(a_, a_)
    assert _rel(s, 2 * a_.float()) < 1e-6
    xn = torch.randn(2, 70, 9, 9, device="cuda")
    nh = ops.nchw_to_nhwc(xn)
    assert torch.equal(nh, xn.permute(0, 2, 3, 1).to(torch.bfloat16))
    back = ops.nhwc_to_nchw_f32(nh)
    assert torch.equal(back, nh.float().permute(0, 3, 1, 2))
    print("elementwise ok")


@case
def edges():
    torch = _setup()
    import torch.nn.functional as F
    from controllora_b200 import ops

    x = torch.randn(2, 4, 64, 64, device="cuda")
    w = (torch.randn(320, 3, 3, 4, device="cuda") / 6).to(torch.bfloat16)
    bias = torch.randn(320, device="cuda") * 0.1
    y = ops.conv_in(x, w, bias, 320)
    yr = F.conv2d(x.to(torch.bfloat16).float(), w.float().permute(0, 3, 1, 2), bias, padding=1).permute(0, 2, 3, 1)
    print(f"conv_in rel={_rel(y, yr):.3e}")
    assert _rel(y, yr) < 4e-3
    g3 = torch.randn(2, 3, 32, 32, device="cuda")
    w3 = (torch.randn(64, 3, 3, 3, device="cuda") / 5).to(torch.bfloat16)
    y3 = ops.conv_in(g3, w3, None, 64)
    y3r = F.conv2d(g3.to(torch.bfloat16).float(), w3.float().permute(0, 3, 1, 2), None, padding=1).permute(0, 2, 3, 1)
    assert _rel(y3, y3r) < 4e-3
    h = torch.randn(2, 64, 64, 320, device="cuda").to(torch.bfloat16)
    wo = (torch.randn(4, 3, 3, 320, device="cuda") / 54).to(torch.bfloat16)
    bo = torch.randn(4, device="cuda") * 0.1
    o = ops.conv_out(h, wo, bo)
    hr = h.float().permute(0, 3, 1, 2).requires_grad_(True)
    orf = F.conv2d(hr, wo.float().permute(0, 3, 1, 2), bo, padding=1)
    print(f"conv_out rel={_rel(o, orf):.3e}")
    assert _rel(o, orf) < 1e-4
    do = torch.randn_like(orf)
    orf.backward(do)
    dh = ops.conv_out_bwd(do, wo, 320)
    print(f"conv_out_bwd rel={_rel(dh, hr.grad.permute(0, 2, 3, 1)):.3e}")
    assert _rel(dh, hr.grad.permute(0, 2, 3, 1)) < 4e-3
    t = torch.tensor([0.0, 1.0, 500.0, 999.0], device="cuda")
    te = ops.timestep_embedding(t, 320)
    import math
    half = 160
    ex = torch.exp(-math.log(10000.0) * torch.arange(half, device="cuda").float() / half)
    em = t[:, None] * ex[None]
    ter = torch.cat([torch.cos(em), torch.sin(em)], -1)
    print(f"timestep_embedding maxabs={float((te - ter).abs().max()):.3e}")
    assert float((te - ter).abs().max()) < 2e-3
    xs = torch.randn(11, 1280, device="cuda")
    ws = (torch.randn(700, 1280, device="cuda") / 36).to(torch.bfloat16)
    bs = torch.randn(700, device="cuda")
    ys = ops.small_linear(xs, ws, bs, silu_in=True, silu_out=True)
    ysr = F.silu(F.silu(xs) @ ws.float().t() + bs)
    print(f"small_linear rel={_rel(ys, ysr):.3e}")
    assert _rel(ys, ysr) < 1e-4
    pred, tgt = torch.randn(8, 4, 64, 64, device="cuda"), torch.randn(8, 4, 64, 64, device="cuda")
    loss, dpred = ops.mse_loss(pred, tgt)
    lr = F.mse_loss(pred, tgt)
    assert abs(float(loss) - float(lr)) < 1e-5 * float(lr) + 1e-6
    assert _rel(dpred, 2 * (pred - tgt) / pred.numel()) < 1e-6
    print("edges ok")


@case
def conv_dgrad():
    """dX of the 3x3 convs through the same implicit-GEMM kernel on flipped/transposed weights (+ zero insertion)."""
    torch = _setup()
    import torch.nn.functional as F
    from controllora_b200 import ops

    for (n, H, Cin, Cout, stride, pad_lo) in [(2, 32, 128, 192, 1, 1), (2, 32, 128, 128, 2, 1), (2, 32, 64, 128, 2, 0)]:
        x = torch.randn(n, Cin, H, H, device="cuda").to(torch.bfloat16).float().requires_grad_(True)
        w = (torch.randn(Cout, Cin, 3, 3, device="cuda") / (9 * Cin) ** 0.5).to(torch.bfloat16).float()
        if stride == 1:
            y = F.conv2d(x, w, padding=1)
        elif pad_lo == 1:
            y = F.conv2d(x, w, stride=2, padding=1)
        else:
            y = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2)
        dy = torch.randn_like(y).to(torch.bfloat16)
        y.backward(dy.float())
        # dgrad weights: Wd[ci][ky'][kx'][co] = W[co][ci][2-ky'][2-kx']
        wd = w.flip(2, 3).permute(1, 2, 3, 0).contiguous().to(torch.bfloat16).view(Cin, 9 * Cout)
        dyn = dy.permute(0, 2, 3, 1).contiguous()
        if stride == 2:
            dyn = ops.zero_insert2x(dyn, 0 if pad_lo == 1 else 1)
        dx = ops.gemm(dyn, wd, conv_stride=1)
        torch.cuda.synchronize()
        e = _rel(dx, x.grad.permute(0, 2, 3, 1))
        print(f"conv dgrad n={n} H={H} {Cin}->{Cout} stride={stride} pad_lo={pad_lo}: rel={e:.3e}")
        assert e < 4e-3


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
