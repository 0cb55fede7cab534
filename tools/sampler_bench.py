"""PNDM against DDIM on GraphedSampler at the C3 shape (512x512, batch 8, UNet batch 16 under CFG 7.5, SD-1.5 UNet with seeded
synthetic weights): 50 PNDM steps (51 UNet calls: the second timestep runs twice) against 50 DDIM steps, with the
configs/mpii-pose.json v1 ControlLoRA (config C3) and without a ControlLoRA (the base model, as for DreamBooth class images).
The four samplers are warmed up (capture included), then their whole calls are timed with CUDA events, alternated round by
round so that drift on a shared card hits all of them alike.  Also timed: the fused CFG + update kernels alone (PLMS against
the DDIM form of cl_cfg_solver_step_dev, 200 launches each at n = 8 x 4 x 64 x 64, issued one by one from Python, so the
per-launch figure is bounded by the Python call, not by the kernel), and sample_class_images for 16 images
at sample_batch_size 8 with synthetic SD-1.5-shape VAE and text encoder (PNDM, 50 steps; decode and JPEG writing included).
Prints one JSON line with the card's name and power limit.   usage: python tools/sampler_bench.py [--rounds R]"""
import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch

import controllora_b200 as cb
from controllora_b200 import ops
from controllora_b200.configs import NAMED, wire_processors
from controllora_b200.sampler import GraphedSampler, ddim_coeffs, ddim_timesteps, pndm_rows, sample_class_images, sd15_alphas_cumprod


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:   # the timing stands without the label; say why it is missing
        return torch.cuda.get_device_name(0), f"unknown ({exc})"


def timed_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def kernel_us(dev, n_launch=200):
    """Per-launch time of the two update kernels on C3-sized latents (tables long enough for every launch)."""
    B = 8
    eps2 = torch.randn(2 * B, 4, 64, 64, device=dev)
    lat = torch.randn(B, 4, 64, 64, device=dev)
    ring, saved, x0p = torch.zeros(3, B, 4, 64, 64, device=dev), torch.zeros_like(lat), torch.zeros_like(lat)
    ac = sd15_alphas_cumprod()
    rows = pndm_rows(50, ac)
    prow = torch.tensor((rows * (n_launch // len(rows) + 2))[: n_launch + 20], dtype=torch.float32, device=dev)
    drow = [[a ** 0.5, (1 - a) ** 0.5, p ** 0.5, (1 - p) ** 0.5, 0, 0, 0, 0] for a, p in (ddim_coeffs(t, 50, ac) for t in ddim_timesteps(50))]
    dtab = torch.tensor((drow * (n_launch // len(drow) + 2))[: n_launch + 20], dtype=torch.float32, device=dev)
    ctr = torch.zeros(1, dtype=torch.int64, device=dev)
    out = {}
    for name, fn in (("plms", lambda: ops.cfg_plms_step_dev(eps2, lat, ring, saved, prow, ctr, 7.5)),
                     ("ddim", lambda: ops.cfg_solver_step_dev(eps2, lat, x0p, dtab, ctr, 7.5, 0))):
        for _ in range(2):                            # warm-up, then timed; the counter restarts so rows stay in the table
            ctr.zero_()
            lat.normal_()
            ms = timed_ms(lambda: [fn() for _ in range(n_launch)])
        out[name] = ms * 1e3 / n_launch
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampler_bench needs a CUDA device: there is no CPU measurement")
    dev = torch.device("cuda", 0)
    name, power = card()
    B, size, steps = 8, 512, 50
    # two UNets with the same synthetic weights: one with the ControlLoRA's processors wired, one without processors (the
    # base model); a captured step keeps reading the processor set it was captured with
    unet_c = cb.UNet2DConditionModel.synthetic(dev, seed=0)
    unet_b = cb.UNet2DConditionModel.synthetic(dev, seed=0)
    g = torch.Generator().manual_seed(11)
    cl = cb.ControlLoRA.from_config(NAMED["mpii-pose"]).to(dev)
    with torch.no_grad():
        for n_, p_ in cl.named_parameters():
            if n_.endswith("up.weight"):
                p_.copy_((0.02 * torch.randn(p_.shape, generator=g)).to(dev))
    wire_processors(unet_c, cl)
    guide = (torch.rand(B, 3, size, size, generator=g) * 2 - 1).to(dev)
    cond = torch.randn(B, 77, 768, generator=g).to(dev).to(torch.bfloat16)
    unc = torch.randn(B, 77, 768, generator=g).to(dev).to(torch.bfloat16)

    def run(sampler, with_control, seed):
        return sampler(guide if with_control else None, cond, unc, seed=seed)

    samplers = {}
    for ctl in (True, False):
        for sched in ("pndm", "ddim"):
            gs = GraphedSampler(unet_c if ctl else unet_b, cl if ctl else None, B, size, size, scheduler=sched,
                                num_inference_steps=steps, guidance_scale=7.5)
            samplers[f"{sched}_{'control' if ctl else 'nocontrol'}"] = (gs, ctl)
            run(gs, ctl, 0)                             # warm-up: eager step, capture, full loop
            torch.cuda.synchronize()
    times = {k: [] for k in samplers}
    finite = True
    for r in range(a.rounds):
        for k, (gs, ctl) in samplers.items():
            holder = {}
            times[k].append(timed_ms(lambda: holder.setdefault("lat", run(gs, ctl, 1 + r))))
            finite = finite and bool(torch.isfinite(holder["lat"]).all())
    res = {"device": name, "power_limit": power, "image": size, "batch": B, "unet_batch": 2 * B, "steps": steps, "rounds": a.rounds}
    for k, v in times.items():
        gs = samplers[k][0]
        res[k] = {"ms_median": sorted(v)[len(v) // 2], "ms_all": v, "unet_calls": gs.calls, "launches_per_step": gs.launches_per_step}
    for ctl in ("control", "nocontrol"):
        res[f"pndm_over_ddim_{ctl}"] = res[f"pndm_{ctl}"]["ms_median"] / res[f"ddim_{ctl}"]["ms_median"]
    res["unet_call_ratio"] = 51 / 50
    res["update_kernel_us"] = kernel_us(dev)
    # class images: base model, PNDM 50 steps, 16 images at sample_batch_size 8 (warm-up call first, into a separate directory)
    vae, clip = cb.AutoencoderKL.synthetic(dev), cb.CLIPTextModel.synthetic(dev)
    ids = torch.randint(0, 49408, (77,), generator=g).to(dev)
    neg = torch.randint(0, 49408, (77,), generator=g).to(dev)
    gs = samplers["pndm_nocontrol"][0]
    with tempfile.TemporaryDirectory() as d:
        sample_class_images(unet_b, vae, clip, ids, neg, B, Path(d, "warm"), sample_batch_size=B, sampler=gs)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        paths = sample_class_images(unet_b, vae, clip, ids, neg, 16, Path(d, "timed"), sample_batch_size=B, sampler=gs)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    res["class_images"] = {"images": len(paths), "seconds": dt, "images_per_s": len(paths) / dt,
                           "what": "sample_class_images: CLIP + 51 UNet calls (graph replays) + VAE decode + uint8 + JPEG, per batch of 8"}
    res["latents_finite"] = finite
    res["not_measured"] = "the reference's fp16 diffusers pipeline generating the same class images (not runnable here)"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
