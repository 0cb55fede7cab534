"""Generates tests/golden/pose_golden.npz: seeded OpenPose skeletons and the canvases the reference's draw_bodypose
(annotator/openpose/util.py:37-70, imported unmodified) draws from them, so that the oracle (oracle/pose_ref.py) and the
CUDA kernel are pinned to the reference where the reference tree is not present.

    python -m tests.golden.make_pose_golden        (needs cv2 and the reference tree)

The skeleton constructors are also used by tests/test_pose.py; only main() needs cv2.
"""
import importlib.util
import sys
import types
from pathlib import Path

import numpy as np

from tests.golden.reference_import import REFERENCE_ROOT

OUT = Path(__file__).resolve().parent / "pose_golden.npz"


def import_reference_util():
    """The reference's annotator/openpose/util.py, unmodified.  It imports matplotlib (for draw_handpose's colours,
    never reached by draw_bodypose), which is not installed: a bare stand-in module is registered while it loads."""
    path = REFERENCE_ROOT / "annotator" / "openpose" / "util.py"
    saved = sys.modules.get("matplotlib")
    sys.modules["matplotlib"] = types.ModuleType("matplotlib")
    try:
        spec = importlib.util.spec_from_file_location("_reference_openpose_util", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is None:
            del sys.modules["matplotlib"]
        else:
            sys.modules["matplotlib"] = saved
    return mod


def skeleton(rng, H, W, persons, *, integer=False, outside=0.0, missing=0.15):
    """(candidate [N, 4] float64 (x, y, score, id), subset [P, 20] float64) in body.py's layout: people built around a
    random centre and scale, some keypoints missing, some pushed outside the canvas."""
    cand, subset = [], []
    for _ in range(persons):
        row = -np.ones(20)
        cx, cy = rng.uniform(-0.1, 1.1) * W, rng.uniform(-0.1, 1.1) * H
        s = rng.uniform(0.05, 0.6) * min(H, W)
        pts = np.stack([cx + s * rng.normal(0, 0.5, 18), cy + s * rng.normal(0, 0.7, 18)], 1)
        for k in range(18):
            if rng.uniform() < missing:
                continue
            x, y = pts[k]
            if rng.uniform() < outside:
                x, y = x + rng.choice([-1, 1]) * rng.uniform(0.5, 1.5) * W, y + rng.uniform(-1, 1) * H
            if integer:
                x, y = float(np.round(x)), float(np.round(y))
            row[k] = len(cand)
            cand.append([x, y, rng.uniform(0.2, 1.0), len(cand)])
        row[18], row[19] = rng.uniform(5, 20), float((row[:18] >= 0).sum())
        subset.append(row)
    return np.array(cand, np.float64).reshape(-1, 4), np.array(subset, np.float64).reshape(-1, 20)


def background(rng, H, W):
    return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)


def cases():
    """[(name, canvas, candidate, subset)]: zero and non-zero backgrounds, 0-6 persons, square and non-square canvases."""
    rng = np.random.default_rng(2024)
    sizes = [(512, 512), (384, 512), (512, 384), (97, 131), (768, 512), (64, 640), (300, 300), (1, 1), (40, 7), (512, 768)]
    out = []
    for i, (H, W) in enumerate(sizes):
        P = i % 7
        cand, sub = skeleton(rng, H, W, P, integer=i % 2 == 0, outside=0.2 if i % 3 == 0 else 0.0)
        bg = background(rng, H, W) if i % 4 == 3 else np.zeros((H, W, 3), np.uint8)
        out.append((f"pose{i}_{H}x{W}_p{P}", bg, cand, sub))
    return out


def main():
    util = import_reference_util()
    arrays = {"names": np.array([c[0] for c in cases()])}
    for name, bg, cand, sub in cases():
        arrays[f"bg_{name}"] = bg
        arrays[f"cand_{name}"] = cand
        arrays[f"subset_{name}"] = sub
        arrays[f"out_{name}"] = util.draw_bodypose(bg.copy(), cand, sub)
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    sys.exit(main())
