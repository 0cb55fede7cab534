"""SD-2.x next to SD-1.5 on synthetic weights, the two models alternated in the same process:

  sample   GraphedSampler at the SD-2.1 shape: 768², batch 4 (UNet batch 8), CFG 7.5, DDIM 50 and DPM-Solver++ 25, with and
           without a ControlLoRA (configs/mpii-pose.json v1 flavour).  SD-2 runs v-prediction, SD-1.5 epsilon.  At 768² the
           first level's self-attention has 9216 tokens: head dim 64 with 5 heads on SD-2, head dim 40 with 8 heads on SD-1.5.
  train    one captured Trainer step at the SD-2-base shape: 512², batch 8, diffusiondb-canny-v2 (its cross-attention LoRAs at
           the model's text width: 1024 on SD-2, 768 on SD-1.5).

Every number is CUDA-event time over a whole call after a warm-up call, repeated `--runs` times with the models alternated; the
card's name and power limit are printed with them.  Prints one JSON line per measurement and a summary line.

usage: python tools/sd2_bench.py [--runs 3] [--what sample,train]"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _randomize_up(torch, module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in module.named_parameters():
            if n.endswith("up.weight"):
                p.copy_((0.02 * torch.randn(p.shape, generator=g)).to(p.device))


def _model(cb, torch, name):
    from controllora_b200 import unet as U

    cfg = U.SD21_CONFIG if name == "sd2" else U.SD15_CONFIG
    return cb.UNet2DConditionModel.synthetic("cuda", cfg), cfg["cross_attention_dim"]


def _control(cb, torch, unet, xd, config_name):
    from controllora_b200.configs import NAMED, wire_processors

    cfg = dict(NAMED[config_name])
    cfg["lora_cross_attention_dims"] = ([None, xd] * 5, [None, xd] * 5, [None, xd] * 5, [None, xd])
    cl = cb.ControlLoRA(**cfg).to("cuda")
    _randomize_up(torch, cl, 3)
    wire_processors(unet, cl)
    return cl


def _plain(unet):
    from controllora_b200.unet_module import _DefaultProcessor

    unet.set_attn_processor(_DefaultProcessor())


def bench_sample(torch, cb, name, unet, xd, scheduler, steps, control):
    from controllora_b200.sampler import GraphedSampler

    _plain(unet)
    cl = _control(cb, torch, unet, xd, "mpii-pose") if control else None
    B, size = 4, 768
    g = torch.Generator().manual_seed(11)
    guide = (torch.rand(B, 3, size, size, generator=g) * 2 - 1).cuda() if control else None
    cond = torch.randn(B, 77, xd, generator=g).cuda().to(torch.bfloat16)
    unc = torch.randn(B, 77, xd, generator=g).cuda().to(torch.bfloat16)
    pt = "v_prediction" if name == "sd2" else "epsilon"
    gs = GraphedSampler(unet, cl, B, size, size, scheduler=scheduler, num_inference_steps=steps, prediction_type=pt)
    gs(guide, cond, unc, seed=0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    lat = gs(guide, cond, unc, seed=1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    out = dict(what="sample", model=name, prediction_type=pt, scheduler=scheduler, steps=steps, control=control, image=size, batch=B,
               ms_total=round(ms, 2), ms_per_step=round(ms / steps, 3), finite=bool(torch.isfinite(lat).all()))
    del gs, cl
    torch.cuda.empty_cache()
    return out


def bench_train(torch, cb, name, unet, xd, steps=10):
    from controllora_b200.trainer import Trainer

    _plain(unet)
    cl = _control(cb, torch, unet, xd, "diffusiondb-canny-v2")
    B = 8
    tr = Trainer(unet, cl, lr=1e-4, cuda_graph=True, prediction_type="v_prediction" if name == "sd2" else "epsilon")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 4, 64, 64, generator=g).cuda()
    t = torch.randint(0, 1000, (B,), generator=g).float().cuda()
    e = torch.randn(B, 77, xd, generator=g).cuda().to(torch.bfloat16)
    guide = ((torch.rand(B, 3, 512, 512, generator=g) > 0.92).float() * 2 - 1).cuda()
    tgt = torch.randn(B, 4, 64, 64, generator=g).cuda()
    for _ in range(4):                                   # eager warm-ups, capture, first replay
        loss = tr.step(x, t, e, guide, tgt)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = tr.step(x, t, e, guide, tgt)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    out = dict(what="train", model=name, config="diffusiondb-canny-v2", cross_dim=xd, image=512, batch=B, ms_per_step=round(ms, 3),
               images_per_s=round(B / ms * 1e3, 2), loss_finite=bool(torch.isfinite(torch.as_tensor(float(loss)))))
    del tr, cl
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--what", default="sample,train")
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("sd2_bench.py measures on the GPU: no CUDA device")
    import controllora_b200 as cb

    card = _card()
    print(json.dumps({"card": card}), flush=True)
    what = a.what.split(",")
    rows = []
    models = {name: _model(cb, torch, name) for name in ("sd2", "sd15")}     # both resident: alternated inside every run
    for run in range(a.runs):
        for name in ("sd2", "sd15"):
            unet, xd = models[name]
            if "sample" in what:
                for sched, steps in (("ddim", 50), ("dpmpp", 25)):
                    for control in (False, True):
                        r = dict(run=run, **bench_sample(torch, cb, name, unet, xd, sched, steps, control))
                        rows.append(r)
                        print(json.dumps(r), flush=True)
            if "train" in what:
                r = dict(run=run, **bench_train(torch, cb, name, unet, xd))
                rows.append(r)
                print(json.dumps(r), flush=True)
    summary = {}
    for r in rows:
        key = (r["what"], r.get("scheduler", ""), str(r.get("control", "")), r["model"])
        summary.setdefault("/".join(key), []).append(r["ms_per_step"])
    print(json.dumps({"card": card, "runs": a.runs, "ms_per_step": {k: sorted(v) for k, v in summary.items()}}), flush=True)


if __name__ == "__main__":
    main()
