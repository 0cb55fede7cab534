"""PNG decode + transform timing (cl_png_decode through controllora_b200.png, then cl_resample / cl_canny), against the
reference's host pipeline on the same machine's CPU, single-threaded (the training scripts' --dataloader_num_workers 0).
  fill50k:     8 image + guide pairs at 512x512 (a filled circle and its outline, written by Pillow), decode_png +
               train_transform at 512  vs  Image.open + convert("RGB") + Resize / ToTensor / Normalize + the crop
  diffusiondb: 8 photo-like PNGs at 512x512 and 768x768 (Pillow, default level), decode_png + canny_batch  vs
               np.asarray(Image.open) + cv2.Canny + the dataset's arithmetic
  flat_4096 / noise_4096 / zfixed / single_block: decode only (the block discovery's worst cases)
Sources are synthetic, from seeds (tests/golden/make_png_golden.py), encoded at run time.  Per workload: ms per call from
a host clock around a synchronised call (host parsing, packing and the upload included), alternated with the Pillow path,
three repeats of 5 calls each, reported as a range; kernel time per phase from torch.profiler over one call in a separate
run; deflate blocks per stream from the oracle's block walker and how many the chain took from confirmed candidates.
Prints one JSON line with the card's name and power limit.
    usage: python tools/png_bench.py"""
import io
import json
import sys
import time
import zlib
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
import torch

from controllora_b200 import canny_batch, ops, reference_crops, train_transform
from controllora_b200 import png as P
from oracle import png_ref
from tests.golden import make_png_golden as G
from tools.canny_bench import card

RES = 512
REPEATS, CALLS = 3, 5


def alternated(gpu_fn, cpu_fn):
    """ms per call of gpu_fn (synchronised) and cpu_fn, alternated repeat by repeat."""
    gpu_fn()
    torch.cuda.synchronize()
    g, c = [], []
    for _ in range(REPEATS):
        t0 = time.perf_counter()
        for _ in range(CALLS):
            gpu_fn()
            torch.cuda.synchronize()
        g.append((time.perf_counter() - t0) / CALLS * 1e3)
        if cpu_fn is not None:
            t0 = time.perf_counter()
            cpu_fn()
            c.append((time.perf_counter() - t0) * 1e3)
    return g, c


def phases(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    groups = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        n = e.name
        key = next((k for k in ("find", "count", "walk", "write", "jump", "gather", "unfilter", "unpack", "init", "resample",
                                "canny") if f"{k}" in n), "scan" if "Scan" in n else "memset" if "emset" in n else
                   "copy" if "emcpy" in n else "other")
        groups[key] = groups.get(key, 0.0) + e.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(groups.items())}


def blocks(files):
    """(oracle blocks per stream, blocks the device chain took from confirmed candidates per stream)."""
    p = P.pack([P.parse(f) for f in files], 3)
    out = torch.empty(max(p.out_bytes, 1), dtype=torch.uint8, device="cuda")
    status, counts, table = ops.png_decode(p, torch.from_numpy(p.host.copy()).cuda(), out, 3)
    t = table.cpu().numpy()
    taken = [int(((t[d.blk0:d.blk0 + n, 2] >> 35) & 1).sum()) for d, n in zip(p.images, counts)]
    return [len(png_ref.block_table(P.parse(f).zdata)) for f in files], taken


def workload(name, files, gpu_fn, cpu_fn):
    from PIL import Image

    px = sum(int(np.prod(Image.open(io.BytesIO(s)).size)) for s in files)
    nbytes = sum(len(s) for s in files)
    dec, _ = alternated(lambda: P.decode_png(files), None)
    full, ref = alternated(gpu_fn, cpu_fn)
    n_blocks, taken = blocks(files)
    return {"what": name, "images": len(files), "compressed_bytes": nbytes, "bits_per_pixel": round(8 * nbytes / px, 3),
            "ms_per_call": [round(min(full), 2), round(max(full), 2)],
            "decode_ms_per_call": [round(min(dec), 2), round(max(dec), 2)],
            "decode_Mpix_per_s": [round(px / max(dec) / 1e3, 1), round(px / min(dec) / 1e3, 1)],
            "pillow_ms": [round(min(ref), 1), round(max(ref), 1)],
            "blocks_per_stream": [min(n_blocks), max(n_blocks)], "blocks_from_candidates": [min(taken), max(taken)],
            "phases_ms": phases(gpu_fn)}


def main():
    assert torch.cuda.is_available(), "png_bench needs a GPU"
    import cv2
    from PIL import Image
    from torchvision import transforms

    torch.set_num_threads(1)
    cv2.setNumThreads(1)
    name, power = card()
    rng = np.random.default_rng(0)
    result = {"device": name, "power_limit": power, "configs": []}

    pairs = [G.fill50k_pair(rng, 512) for _ in range(8)]
    imgs, guides = [a for a, _ in pairs], [g for _, g in pairs]
    crops = reference_crops([(512, 512)] * 8, RES)
    tf = transforms.Compose([transforms.Resize(RES, interpolation=transforms.InterpolationMode.BILINEAR),
                             transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])

    def fill_cpu():
        for s in imgs + guides:
            tf(Image.open(io.BytesIO(s)).convert("RGB"))[:, :RES, :RES]

    result["configs"].append(workload("fill50k", imgs + guides,
                                      lambda: train_transform(P.decode_png(imgs), P.decode_png(guides), RES, crops=crops), fill_cpu))

    db = [G.photo_png(rng, 512, 512) for _ in range(4)] + [G.photo_png(rng, 768, 768) for _ in range(4)]

    def db_gpu():
        out = P.decode_png(db)
        for k in (0, 4):
            canny_batch(torch.stack(out[k:k + 4]), (100, 200))

    def db_cpu():
        for s in db:
            a = np.asarray(Image.open(io.BytesIO(s)))
            edges = cv2.Canny(a, 100, 200)
            (a.astype(np.float32) / 127.5 - 1, edges.astype(np.float32) / 127.5 - 1)

    result["configs"].append(workload("diffusiondb", db, db_gpu, db_cpu))

    flat = np.zeros((4096, 4096 * 3), np.uint8)
    flat[:, 0::3], flat[:, 1::3], flat[:, 2::3] = 200, 30, 90
    noise = rng.integers(0, 256, (4096, 4096 * 3), dtype=np.uint8)
    a = G.scanlines(rng, 1024, 1024, 2, 8, "smooth")
    for nm, f in (("flat_4096", G.build_png(flat, 4096, 2, 8, filters=(1,))),
                  ("noise_4096", G.build_png(noise, 4096, 2, 8, filters=(0,), level=1)),
                  ("zfixed_1024", G.build_png(a, 1024, 2, 8, filters=(4,), strategy=zlib.Z_FIXED)),
                  ("single_block_1024", G.build_png(a, 1024, 2, 8, filters=(4,), level=9, mem_level=9))):
        result["configs"].append(workload(nm, [f], lambda f=f: P.decode_png([f]),
                                          lambda f=f: np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
