"""Denoise-loop timing on the CUDA UNet for the two inference call patterns of the reference (synthetic weights / inputs):

  c3   SURVEY §8(d) config 3: v1 ControlLoRA (mpii-pose architecture), 512x512, batch 8 (UNet batch 16 under CFG),
       50-step DDIM, guidance 7.5                                  (apps/gradio_*2image.py, train_...:829-843)
  mix  config 5 = mix_lora_and_control_lora.py: v1 ControlLoRA + a rank-4 plain LoRA stacked as pre_lora on every
       processor (:94-121), 768x768 (latent 96x96, 9216 tokens at level 0), batch 4 (UNet batch 8), 30 steps of
       DPMSolverMultistepScheduler (:80,153-164)

usage: python tools/denoise_demo.py [c3|mix] [--steps N]      -> one JSON line (UNet evaluations per second)
"""
import argparse
import json
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import torch

import controllora_b200 as cb
from controllora_b200.configs import NAMED, wire_processors
from controllora_b200.sampler import ddim_sample, dpmpp_sample


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("which", nargs="?", default="c3", choices=["c3", "mix"])
    ap.add_argument("--steps", type=int, default=0)
    a = ap.parse_args()
    dev = "cuda"
    unet = cb.UNet2DConditionModel.synthetic(dev, seed=0)
    cl = cb.ControlLoRA.from_config(NAMED["mpii-pose"]).to(dev)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for n_, p_ in cl.named_parameters():
            if n_.endswith("up.weight"):
                p_.copy_((0.02 * torch.randn(p_.shape, generator=g)).to(dev))
    procs = wire_processors(unet, cl)
    if a.which == "mix":
        for name, p in procs.items():                       # mix_lora_and_control_lora.py:113-121
            pre = cb.LoRACrossAttnProcessor(p.hidden_size, p.cross_attention_dim, rank=4)
            with torch.no_grad():
                for n_, q_ in pre.named_parameters():
                    if n_.endswith("up.weight"):
                        q_.copy_(0.02 * torch.randn(q_.shape, generator=g))
            p.inject_pre_lora(pre.to(dev))
        B, size, steps, fn, name = 4, 768, a.steps or 30, dpmpp_sample, "DPM-Solver++(2M)"
    else:
        B, size, steps, fn, name = 8, 512, a.steps or 50, ddim_sample, "DDIM"
    guide = (torch.rand(B, 3, size, size, generator=g) * 2 - 1).to(dev)
    cond = torch.randn(B, 77, 768, generator=g).to(dev).to(torch.bfloat16)
    unc = torch.randn(B, 77, 768, generator=g).to(dev).to(torch.bfloat16)
    fn(unet, cl, guide, cond, unc, num_inference_steps=3, guidance_scale=7.5, seed=0)       # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    lat = fn(unet, cl, guide, cond, unc, num_inference_steps=steps, guidance_scale=7.5, seed=1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    print(json.dumps({"case": a.which, "sampler": name, "image": size, "batch": B, "unet_batch": 2 * B, "steps": steps,
                      "ms_total": ms, "denoise_steps_per_s": steps / ms * 1e3, "latents_finite": bool(torch.isfinite(lat).all()),
                      "latents_std": float(lat.std())}))


if __name__ == "__main__":
    main()
