"""Canny annotator timing: controllora_b200.canny_batch (edges + guide + pixel_values, the per-batch work of the canny
configs' dataset) at B = 8, 512x512 RGB and at B = 1, 1024x1024 RGB, with CUDA events over 50 calls after 5 warm-up calls,
eager and as one replayed CUDA graph.  Algorithmic bytes per pixel: 3 (uint8 RGB in) + 24 (guide + pixel_values, fp32
[3, H, W] each) + 12 (int32 label table written once, read by the mark and resolve passes) = 39.  Where cv2 is installed,
cv2.Canny over the same images on the host is timed for context.  Prints one JSON line with the card's name and power
limit.   usage: python tools/canny_bench.py"""
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
import torch

from controllora_b200 import canny_batch
from tests.golden.make_canny_golden import shapes, smooth_noise

BYTES_PER_PIXEL = 3 + 24 + 12
CONFIGS = [(8, 512, 512), (1, 1024, 1024)]


def timed(fn, n=50, warmup=5):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3     # us per call


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:   # the timing stands without the label; say why it is missing
        return torch.cuda.get_device_name(0), f"unknown ({exc})"


def main():
    assert torch.cuda.is_available(), "canny_bench needs a GPU"
    name, power = card()
    rng = np.random.default_rng(0)
    result = {"device": name, "power_limit": power, "bytes_per_pixel": BYTES_PER_PIXEL, "configs": []}
    for B, H, W in CONFIGS:
        imgs = np.stack([shapes(rng, H, W) if b % 2 else smooth_noise(rng, H, W, 3, cell=8, noise=4) for b in range(B)])
        x = torch.from_numpy(imgs).cuda()
        thr_np = rng.integers(1, 255, (B, 2)).astype(np.float32)
        thr = torch.from_numpy(thr_np).cuda()
        eager_us = timed(lambda: canny_batch(x, thr))
        graph = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            canny_batch(x, thr)
        torch.cuda.current_stream().wait_stream(s)
        with torch.cuda.graph(graph):
            canny_batch(x, thr)
        graph_us = timed(graph.replay)
        nbytes = B * H * W * BYTES_PER_PIXEL
        row = {"B": B, "H": H, "W": W, "algorithmic_bytes": nbytes, "eager_us": round(eager_us, 2), "graph_us": round(graph_us, 2),
               "graph_GBps": round(nbytes / graph_us / 1e3, 1)}
        try:
            import cv2

            t0 = time.perf_counter()
            reps = 3
            for _ in range(reps):
                for b in range(B):
                    cv2.Canny(imgs[b], float(thr_np[b, 0]), float(thr_np[b, 1]))
            row["cv2_host_us"] = round((time.perf_counter() - t0) / reps * 1e6, 1)
            row["cv2_threads"] = cv2.getNumThreads()
        except ImportError:
            row["cv2_host_us"] = None
        result["configs"].append(row)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
