"""The reference's algorithm run the way the reference runs it — eager PyTorch on the GPU (cuBLAS / cuDNN / ATen), frozen
UNet in bf16, trainable ControlLoRA in fp32 under bf16 autocast (accelerate's mixed_precision="bf16",
train_text_to_image_control_lora.py:437-447) — using the oracle restatement (oracle/), because diffusers itself is not
installable here.  SURVEY.md §8(d) calls this "the real bar": the reference has no kernels of its own.

This is a measurement script kept with the tests (it executes the oracle, which only tests/, smoke() and the CPU arm of
bench.py may do); it is not collected by pytest, not part of the product path and not part of bench.py's JSON line.  It
prints one JSON line.   usage: python tests/perf_eager_gpu_baseline.py [--batch 8] [--steps 5] [--config diffusiondb-canny-v2]
"""
import argparse
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import torch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--config", default="diffusiondb-canny-v2")
    a = ap.parse_args()
    from oracle import models_ref as MR
    from oracle import unet_ref as UR
    from controllora_b200.configs import NAMED
    import bench

    dev = "cuda"
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    unet = UR.UNet2DConditionModel()
    UR.init_synthetic_(unet, seed=1)
    unet.requires_grad_(False)
    unet.to(dev).to(torch.bfloat16)                    # weight_dtype = bf16 for the frozen network
    cl = MR.ControlLoRA.from_config(NAMED[a.config])
    MR.randomize_lora_up_(cl, seed=3)
    cl.to(dev)                                         # trainable parameters stay fp32
    MR.wire_processors(unet, cl)
    opt = torch.optim.AdamW(cl.parameters(), lr=1e-4, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    x, t, e, guide, tgt = (v.to(dev) for v in bench.synth_inputs(torch, a.batch))

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            cl(guide)
            pred = unet(x.to(torch.bfloat16), t.long(), e.to(torch.bfloat16)).sample
            loss = torch.nn.functional.mse_loss(pred.float(), tgt)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(cl.parameters(), 1.0)
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss

    for _ in range(3):
        loss = step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.time()
    e0.record()
    for _ in range(a.steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    wall = (time.time() - t0) / a.steps * 1e3
    print(json.dumps({
        "what": "oracle restatement of the reference step, eager PyTorch on the GPU (cuBLAS/cuDNN/ATen), bf16 autocast",
        "config": a.config, "batch": a.batch, "steps": a.steps, "ms_per_step": ms, "wall_ms_per_step": wall,
        "images_per_s": a.batch / ms * 1e3, "final_loss": float(loss),
        "max_mem_gb": torch.cuda.max_memory_allocated() / 2**30, "torch": torch.__version__}))


if __name__ == "__main__":
    main()
