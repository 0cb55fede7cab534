"""Where the wgmma GEMM's time goes in one bench step, per launch shape, and what its occupancy plan is.

usage: python tools/gemm_occupancy.py [--config diffusiondb-canny-v2] [--batch 8] [--json OUT.json] [--dump OUT.npz]

1. Runs one eager (no CUDA graph) Trainer step of the bench workload (hint encoder + UNet fwd/bwd + optimizer) and records
   every cl_gemm launch: shape, k-blocks per tile, the planner's block_n / splits / CTAs per SM (cl_gemm_plan), the CTAs
   of that kernel the device keeps resident per SM at its launch's shared-memory size
   (cudaOccupancyMaxActiveBlocksPerMultiprocessor), and its CUDA-event time (each launch bracketed, so serialised).
2. Times each distinct launch configuration of that step ALONE, with operands rotated through > 200 MB so L2 does not
   hold them, and prints a per-shape table and the step total of the launches with at most 20 k-blocks per tile.
3. --dump: runs seeded cases at the census shapes and saves every output (D, t_out, fp32 and residual outputs) so two
   builds of the library (CLB_LIB) can be compared bit for bit.
"""
import argparse
import ctypes as C
import json
import sys
from collections import OrderedDict
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import torch

SHORT_K = 20   # k-blocks per tile at or below which a launch counts as short-K


def _plan(lib, args):
    """(block_n, splits, ctas_per_sm, resident_per_sm, tma_store), or None for a library without cl_gemm_plan."""
    if not hasattr(lib, "cl_gemm_plan"):
        return None
    info = (C.c_int32 * 5)()
    if lib.cl_gemm_plan(C.byref(args), info) != 0:
        return None
    return tuple(info)


class _Recorder:
    """Stands in for the ctypes library: every cl_gemm call is planned, bracketed with CUDA events and recorded."""

    def __init__(self, real):
        self.real = real
        self.rows = []

    def __getattr__(self, name):
        return getattr(self.real, name)

    def cl_gemm(self, pargs, stream):
        a = pargs._obj
        key = OrderedDict(M=a.M, N=a.N, K=a.K, a_mode=a.a_mode, n_img=a.n_img, H=a.H, W=a.W, C=a.C, pad_lo=a.pad_lo,
                          lora_rp=a.lora_rp if a.lora_up else 0, t_add=bool(a.t_add), t_out=bool(a.t_out),
                          bias=bool(a.bias), row_bias=bool(a.row_bias), residual=bool(a.residual), out_fp32=a.out_fp32,
                          split_k=a.split_k)
        plan = _plan(self.real, a)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        st = self.real.cl_gemm(pargs, stream)
        e1.record()
        self.rows.append((key, plan, e0, e1))
        return st


def _kb_per_tile(key, plan):
    bk = 32 if key["a_mode"] != 0 and key["C"] % 64 != 0 else 64
    nkb = (key["K"] + bk - 1) // bk
    splits = plan[1] if plan else max(1, key["split_k"])
    return (nkb + splits - 1) // splits


def record_step(config, batch):
    import bench
    import controllora_b200 as cb
    from controllora_b200 import _lib
    from controllora_b200.configs import NAMED, wire_processors
    from controllora_b200.trainer import Trainer

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    unet = cb.UNet2DConditionModel.synthetic(dev, seed=0)
    cl = cb.ControlLoRA.from_config(NAMED[config]).to(dev)
    wire_processors(unet, cl)
    tr = Trainer(unet, cl, lr=1e-4, cuda_graph=False)
    x, t, e, guide, tgt = (h.to(dev) for h in bench.synth_inputs(torch, batch))
    e = e.to(torch.bfloat16)
    for _ in range(2):
        tr.step(x, t, e, guide, tgt)
    torch.cuda.synchronize()
    rec = _Recorder(_lib.lib())
    _lib._lib = rec
    try:
        tr.step(x, t, e, guide, tgt)
        torch.cuda.synchronize()
    finally:
        _lib._lib = rec.real
    out = []
    for key, plan, e0, e1 in rec.rows:
        out.append({"key": dict(key), "plan": plan, "kb_per_tile": _kb_per_tile(key, plan), "us": e0.elapsed_time(e1) * 1e3})
    del tr, unet, cl
    torch.cuda.empty_cache()
    return out


def _operands(key, nsets, dev="cuda"):
    """Seeded operand sets for one recorded launch configuration, and a function launching set i."""
    from controllora_b200 import ops

    M, N, K = key["M"], key["N"], key["K"]
    g = torch.Generator(device=dev).manual_seed(1234 + M + 7 * N + 13 * K)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    if key["a_mode"] == 0:
        As = [rnd(M, K).to(torch.bfloat16) for _ in range(nsets)]
        conv = {}
    else:
        s = 1 if key["a_mode"] == 1 else 2
        As = [rnd(key["n_img"], key["H"], key["W"], key["C"]).to(torch.bfloat16) for _ in range(nsets)]
        conv = {"conv_stride": s, "pad_lo": key["pad_lo"]}
    Wt = (rnd(N, K) / K ** 0.5).to(torch.bfloat16)
    dt = torch.float32 if key["out_fp32"] else torch.bfloat16
    Ds = [torch.empty(M, N, device=dev, dtype=dt) for _ in range(nsets)]
    kw = {"out_fp32": bool(key["out_fp32"])}
    if key["bias"]:
        kw["bias"] = rnd(N)
    if key["row_bias"]:
        kw["row_bias"] = rnd(8, N)
        kw["rows_per_group"] = (M + 7) // 8
    res = [rnd(M, N).to(torch.bfloat16) for _ in range(nsets)] if key["residual"] else None
    rp = key["lora_rp"]
    if rp:
        r = 4 if rp == 4 else 8
        down = rnd(r, K) / r
        up = torch.zeros(N, rp, device=dev)
        up[:, :r] = rnd(N, r) * 0.5
        kw.update(ext=ops.split_bf16_ext(down, K), lora_up=up, lora_scale=0.7)
        if key["t_add"]:
            kw["t_add"] = rnd(M, rp)
    t_outs = [torch.empty(M, rp, device=dev) for _ in range(nsets)] if rp and key["t_out"] else None

    def run(i):
        extra = {}
        if res is not None:
            extra["residual"] = res[i]
        if t_outs is not None:
            extra["t_out"] = t_outs[i]
        out = Ds[i].view(-1, N) if not conv else Ds[i]
        return ops.gemm(As[i], Wt, out=out, **conv, **kw, **extra)

    return run, Ds, t_outs


def time_alone(key, iters=10):
    per = 2 * (key["M"] * key["K"] // (9 if key["a_mode"] else 1) + key["M"] * key["N"]) * (2 if key["out_fp32"] else 1)
    nsets = max(2, min(16, int(200e6 // per) + 1))
    run, _, _ = _operands(key, nsets)
    for i in range(nsets):
        run(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        for i in range(nsets):
            run(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (iters * nsets)


# Census shapes (SURVEY 8a) plus the epilogue variants the short-K launches use; seeded, for bit-for-bit comparisons.
def _census():
    base = dict(a_mode=0, n_img=0, H=0, W=0, C=0, pad_lo=1, lora_rp=0, t_add=False, t_out=False, bias=False, row_bias=False,
                residual=False, out_fp32=0, split_k=0)
    cases = []
    for M, N, K in [(32768, 320, 320), (32768, 2560, 320), (32768, 320, 1280), (8192, 640, 640), (8192, 5120, 640),
                    (2048, 1280, 1280), (32768, 1280, 320), (1000, 320, 320), (32768, 640, 320)]:
        cases.append(dict(base, M=M, N=N, K=K))
    cases.append(dict(base, M=32768, N=320, K=320, lora_rp=4, t_add=True, t_out=True))
    cases.append(dict(base, M=8192, N=640, K=640, lora_rp=8, t_out=True))
    cases.append(dict(base, M=32768, N=320, K=320, bias=True, row_bias=True, residual=True))
    cases.append(dict(base, M=32768, N=320, K=320, out_fp32=1, bias=True))
    for n, H, Cc, N in [(8, 64, 320, 320), (8, 512, 32, 32), (8, 256, 32, 64), (8, 128, 64, 96)]:
        cases.append(dict(base, M=n * H * H, N=N, K=9 * Cc, a_mode=1, n_img=n, H=H, W=H, C=Cc))
    return cases


def dump(path):
    arrays = {}
    for ci, key in enumerate(_census()):
        run, Ds, t_outs = _operands(key, 1)
        run(0)
        torch.cuda.synchronize()
        arrays[f"c{ci}_D"] = Ds[0].view(torch.int16 if Ds[0].dtype == torch.bfloat16 else torch.int32).cpu().numpy()
        if t_outs is not None:
            arrays[f"c{ci}_t_out"] = t_outs[0].view(torch.int32).cpu().numpy()
    import numpy as np

    np.savez(path, **arrays)
    print(f"dumped {len(arrays)} arrays of {len(_census())} census cases to {path}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="diffusiondb-canny-v2")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--json", default=None)
    ap.add_argument("--dump", default=None, metavar="OUT.npz")
    ap.add_argument("--census-only", action="store_true", help="time the census shapes alone, skip the step")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_occupancy: needs a CUDA device")
    from controllora_b200 import _lib

    if a.dump:
        dump(a.dump)
        return
    rows = [] if a.census_only else record_step(a.config, a.batch)
    distinct = OrderedDict()
    for r in rows:
        k = json.dumps(r["key"], sort_keys=True)
        d = distinct.setdefault(k, {"key": r["key"], "plan": r["plan"], "kb_per_tile": r["kb_per_tile"], "count": 0, "step_us": 0.0})
        d["count"] += 1
        d["step_us"] += r["us"]
    for key in _census():
        k = json.dumps(key, sort_keys=True)
        if k not in distinct:
            distinct[k] = {"key": key, "plan": None, "kb_per_tile": None, "count": 0, "step_us": 0.0}
    lib = _lib.lib()
    for d in distinct.values():
        key = d["key"]
        if d["plan"] is None or d["kb_per_tile"] is None:
            run, _, _ = _operands(key, 1)      # plan through a real argument block: run once under the recorder
            rec = _Recorder(lib)
            _lib._lib = rec
            try:
                run(0)
                torch.cuda.synchronize()
            finally:
                _lib._lib = lib
            d["plan"] = rec.rows[-1][1]
            d["kb_per_tile"] = _kb_per_tile(key, d["plan"])
        d["alone_us"] = time_alone(key)
    total = sum(d["step_us"] for d in distinct.values())
    short = sum(d["step_us"] for d in distinct.values() if d["kb_per_tile"] <= SHORT_K)
    print(f"{'M':>7} {'N':>6} {'K':>6} {'mode':>4} {'lora':>4} {'kb/tile':>7} {'bn':>4} {'spl':>3} {'cta/SM':>6} {'resident':>8} "
          f"{'count':>5} {'step us':>9} {'alone us':>9}")
    for d in sorted(distinct.values(), key=lambda d: -d["step_us"]):
        k, p = d["key"], d["plan"] or (0, 0, 0, 0, 0)
        print(f"{k['M']:7d} {k['N']:6d} {k['K']:6d} {k['a_mode']:4d} {k['lora_rp']:4d} {d['kb_per_tile']:7d} {p[0]:4d} {p[1]:3d} "
              f"{p[2]:6d} {p[3]:8d} {d['count']:5d} {d['step_us']:9.1f} {d['alone_us']:9.1f}")
    print(f"GEMM launches in one step: {len(rows)}, {total / 1e3:.3f} ms (serialised event timing); "
          f"with <= {SHORT_K} k-blocks per tile: {short / 1e3:.3f} ms")
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps({"launches": len(rows), "total_us": total, "short_k_us": short,
                                            "shapes": list(distinct.values())}, indent=1))


if __name__ == "__main__":
    main()
