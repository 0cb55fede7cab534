"""Pose renderer timing: controllora_b200.pose_batch for 8 canvases of 512x512 with 3 persons each (the guides of one
mpii-pose training batch) and pose_control for one app-sized call (detect and image resolution 512, 3 persons), with
CUDA events after warm-up.  Reported with host work (the whole Python call: limb parameters, descriptors, one upload,
two launches) and without it (a PoseBuffers call captured in a CUDA graph and replayed: upload plus the two kernels).
Algorithmic bytes: the fp32 guide written (12 B per output pixel), plus the uint8 canvas written and the background
read (3 B each) where a call has them.  For context the same drawing is timed with host cv2 calls (the reference's call
sequence: circle, ellipse2Poly, copy, fillConvexPoly, addWeighted per limb) on this machine's CPU.  Prints one JSON line
with the card's name and power limit.   usage: python tools/pose_bench.py"""
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
import torch

from controllora_b200 import pose as PZ
from controllora_b200.transforms import resize_image_size
from tests.golden.make_pose_golden import skeleton


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:   # the timing stands without the label; say why it is missing
        return torch.cuda.get_device_name(0), f"unknown ({exc})"


def device_us(fn, n=200, warmup=10):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


def host_us(fn, n=50, warmup=5):
    """Wall time per call including the host work, ending in a device synchronise."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e6


def cv2_draw(cv2, H, W, candidate, subset):
    """The reference's draw_bodypose call sequence with cv2 (limb parameters from pose.limb_params, which the CPU tests
    pin to the reference's own expressions)."""
    canvas = np.zeros((H, W, 3), np.uint8)
    for i in range(18):
        for n in range(len(subset)):
            index = int(subset[n][i])
            if index == -1:
                continue
            x, y = candidate[index][0:2]
            cv2.circle(canvas, (int(x), int(y)), 4, PZ.COLORS[i], thickness=-1)
    for i in range(17):
        for n in range(len(subset)):
            index = subset[n][np.array(PZ.LIMB_SEQ[i]) - 1]
            if -1 in index:
                continue
            a, b = index.astype(int)
            cx, cy, half, angle = PZ.limb_params(*candidate[a][0:2], *candidate[b][0:2])
            cur = canvas.copy()
            cv2.fillConvexPoly(cur, cv2.ellipse2Poly((cx, cy), (half, PZ.STICKWIDTH), angle, 0, 360, 1), PZ.COLORS[i])
            canvas = cv2.addWeighted(canvas, 0.4, cur, 0.6, 0)
    return canvas


def dense(skels, P):
    kp = np.zeros((len(skels), P, 18, 3))
    for b, (cand, sub) in enumerate(skels):
        for p in range(len(sub)):
            for k in range(18):
                if sub[p, k] >= 0:
                    kp[b, p, k] = (*cand[int(sub[p, k]), :2], 1.0)
    return kp


def main():
    assert torch.cuda.is_available(), "pose_bench needs a GPU"
    name, power = card()
    rng = np.random.default_rng(0)
    result = {"device": name, "power_limit": power, "configs": []}

    B, H, W, P = 8, 512, 512, 3
    skels = [skeleton(rng, H, W, P, missing=0.05) for _ in range(B)]
    kp = dense(skels, P)
    n_limbs = sum(len(PZ._prims_from_dense(kp[b], "bench")[1]) for b in range(B))
    with_host = host_us(lambda: PZ.pose_batch(kp, (H, W)))
    buf = PZ.PoseBuffers(B, P, (H, W))
    buf.stage(kp)
    buf.launch()
    torch.cuda.synchronize()
    assert torch.equal(buf.guide, PZ.pose_batch(kp, (H, W)))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        buf.launch()
    graph_dev = device_us(graph.replay)
    nbytes = B * H * W * 12
    row = {"call": "pose_batch", "B": B, "H": H, "W": W, "persons": P, "limbs": n_limbs, "algorithmic_bytes": nbytes,
           "with_host_us": round(with_host, 1), "device_graph_us": round(graph_dev, 1),
           "device_GBps": round(nbytes / graph_dev / 1e3, 1)}
    try:
        import cv2

        t0 = time.perf_counter()
        reps = 3
        for _ in range(reps):
            for cand, sub in skels:
                cv2_draw(cv2, H, W, cand, sub)
        row["cv2_host_us"] = round((time.perf_counter() - t0) / reps * 1e6, 1)
        row["cv2_threads"] = cv2.getNumThreads()
    except ImportError:
        row["cv2_host_us"] = None
    result["configs"].append(row)

    h, w = 768, 1024
    dh, dw, _ = resize_image_size(h, w, 512)
    ih, iw, _ = resize_image_size(h, w, 512)
    cand, sub = skeleton(rng, dh, dw, 3, missing=0.05)
    with_host = host_us(lambda: PZ.pose_control(cand, sub, (h, w), 512, 512))
    row = {"call": "pose_control", "input": [h, w], "detect": [dh, dw], "image": [ih, iw], "persons": 3,
           "algorithmic_bytes": ih * iw * 12, "with_host_us": round(with_host, 1)}
    try:
        import cv2

        t0 = time.perf_counter()
        reps = 10
        for _ in range(reps):
            m = cv2.resize(cv2_draw(cv2, dh, dw, cand, sub), (iw, ih), interpolation=cv2.INTER_NEAREST)
            torch.from_numpy(m[..., ::-1].copy().transpose([2, 0, 1])).float()[None] / 127.5 - 1
        row["cv2_host_us"] = round((time.perf_counter() - t0) / reps * 1e6, 1)
    except ImportError:
        row["cv2_host_us"] = None
    result["configs"].append(row)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
