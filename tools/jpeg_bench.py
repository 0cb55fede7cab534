"""JPEG decode + transform timing (cl_jpeg_decode through controllora_b200.jpeg, then cl_resample), against the
reference's host pipeline on the same machine's CPU, single-threaded (the training scripts' --dataloader_num_workers 0).
  dreambooth: 4 instance images of 4032x3024 (4:2:0, quality 92) and 4 class images of 512x512 written as
              sample_class_images writes them (Image.save defaults: quality 75, 4:2:0), decode_jpeg + dreambooth_transform
              at 512 (random crop)  vs  Image.open + convert("RGB") + Resize / RandomCrop / ToTensor / Normalize
  pose:       8 images of 1280x720 (quality 90) and their 8 guides, decode_jpeg + train_transform at 512  vs
              Image.open + convert("RGB") + Resize / ToTensor / Normalize + the crop, for images and guides
  sync_flat / sync_striped: the 4096x4096 flat and striped images alone, decode_jpeg only (the windows' worst cases)
Sources are synthetic photo-like content from seeds (tests/golden/make_jpeg_golden.py), encoded by Pillow at run time;
bits per pixel are printed so the content can be judged.  Per workload: ms per call from a host clock around a
synchronised call (host parsing, packing and the upload included), three repeats of 5 calls each, reported as a range;
kernel time per phase from torch.profiler over one call; compressed MB/s and output Mpixel/s of the decode; the rounds the
window states took to reach their fixpoint.  Prints one JSON line with the card's name and power limit.
    usage: python tools/jpeg_bench.py"""
import io
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np
import torch

from controllora_b200 import jpeg as J
from controllora_b200 import ops, reference_crops, train_transform
from tests.golden import make_jpeg_golden as G
from tools.canny_bench import card

RES = 512
REPEATS, CALLS = 3, 5


def host_ms(fn, calls=CALLS):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(REPEATS):
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
            torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) / calls * 1e3)
    return out


def phases(fn):
    """Kernel time per phase (ms) of one call, from torch.profiler."""
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
        key = ("sync" if "jpeg_sync" in n else "write" if "jpeg_write" in n else "idct" if "jpeg_idct" in n else
               "color" if "jpeg_color" in n else "scan" if "Scan" in n else "memset" if "emset" in n else
               "resample" if "resample" in n else "copy" if "emcpy" in n else "other")
        groups[key] = groups.get(key, 0.0) + e.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(groups.items())}


def rounds_of(streams):
    p = J.pack([J.parse(s) for s in streams])
    staged = torch.from_numpy(p.host.copy()).pin_memory()
    out = torch.empty(max(p.out_bytes, 1), dtype=torch.uint8, device="cuda")
    return ops.jpeg_decode(p, staged.cuda(), out)[1]


def host_reference(streams, fn, calls=1):
    t = []
    for _ in range(REPEATS):
        t0 = time.perf_counter()
        for _ in range(calls):
            for s in streams:
                fn(s)
        t.append((time.perf_counter() - t0) / calls * 1e3)
    return t


def workload(name, streams, gpu_fn, cpu_fn=None):
    from PIL import Image

    px = sum(int(np.prod(Image.open(io.BytesIO(s)).size)) for s in streams)
    nbytes = sum(len(s) for s in streams)
    dec = host_ms(lambda: J.decode_jpeg(streams))
    full = host_ms(gpu_fn) if gpu_fn is not None else dec
    row = {"what": name, "images": len(streams), "compressed_bytes": nbytes, "bits_per_pixel": round(8 * nbytes / px, 3),
           "ms_per_call": [round(min(full), 2), round(max(full), 2)],
           "decode_ms_per_call": [round(min(dec), 2), round(max(dec), 2)],
           "decode_MBps": [round(nbytes / max(dec) / 1e3, 1), round(nbytes / min(dec) / 1e3, 1)],
           "decode_Mpix_per_s": [round(px / max(dec) / 1e3, 1), round(px / min(dec) / 1e3, 1)],
           "phases_ms": phases(gpu_fn if gpu_fn is not None else (lambda: J.decode_jpeg(streams))),
           "sync_rounds": rounds_of(streams)}
    if cpu_fn is not None:
        ref = cpu_fn()
        row["pillow_torchvision_ms"] = [round(min(ref), 1), round(max(ref), 1)]
    return row


def main():
    assert torch.cuda.is_available(), "jpeg_bench needs a GPU"
    from PIL import Image
    from torchvision import transforms

    torch.set_num_threads(1)
    name, power = card()
    rng = np.random.default_rng(0)
    result = {"device": name, "power_limit": power, "configs": []}

    inst = [G.pil_jpeg(G.photo(rng, 3024, 4032), quality=92) for _ in range(4)]
    cls = [G.pil_jpeg(G.photo(rng, 512, 512)) for _ in range(4)]
    db = inst + cls
    tv = transforms.Compose([transforms.Resize(RES, interpolation=transforms.InterpolationMode.BILINEAR),
                             transforms.RandomCrop(RES), transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])
    result["configs"].append(workload(
        "dreambooth", db, lambda: J.dreambooth_transform(J.decode_jpeg(db), RES),
        lambda: host_reference(db, lambda s: tv(Image.open(io.BytesIO(s)).convert("RGB")))))

    imgs = [G.pil_jpeg(G.photo(rng, 720, 1280), quality=90) for _ in range(8)]
    guides = [G.pil_jpeg(G.photo(rng, 720, 1280, cell=16, edges=40), quality=90) for _ in range(8)]
    crops = reference_crops([(720, 1280)] * 8, RES)
    tf = transforms.Compose([transforms.Resize(RES, interpolation=transforms.InterpolationMode.BILINEAR),
                             transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])

    def pose_cpu(s):
        return tf(Image.open(io.BytesIO(s)).convert("RGB"))[:, :RES, :RES]

    result["configs"].append(workload(
        "pose", imgs + guides, lambda: train_transform(J.decode_jpeg(imgs), J.decode_jpeg(guides), RES, crops=crops),
        lambda: host_reference(imgs + guides, pose_cpu)))

    for nm, s in (("sync_flat", G.pil_jpeg(G.flat(4096, 4096))), ("sync_striped", G.pil_jpeg(G.striped(4096, 4096)))):
        result["configs"].append(workload(nm, [s], None,
                                          lambda s=s: host_reference([s], lambda x: np.asarray(Image.open(io.BytesIO(x))))))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
