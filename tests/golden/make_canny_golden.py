"""Generates tests/golden/canny_golden.npz: seeded images, a (lo, hi) threshold pair per image and cv2.Canny's output for
each, so that the oracle (oracle/annotator_ref.py) and the CUDA kernel are pinned to OpenCV where OpenCV is not installed.

    python -m tests.golden.make_canny_golden        (needs cv2)

The image constructors are also used by tests/test_annotator.py; only main() needs cv2.
"""
import sys
from pathlib import Path

import numpy as np

OUT = Path(__file__).resolve().parent / "canny_golden.npz"


def smooth_noise(rng, H, W, C, cell=8, noise=6):
    """Bilinearly upsampled coarse noise plus fine noise: edges of every orientation, some long chains."""
    gh, gw = H // cell + 2, W // cell + 2
    coarse = rng.uniform(0, 255, (gh, gw, C))
    ys = np.arange(H) / cell
    xs = np.arange(W) / cell
    y0, x0 = ys.astype(int), xs.astype(int)
    fy, fx = (ys - y0)[:, None, None], (xs - x0)[None, :, None]
    a = coarse[y0][:, x0]
    b = coarse[y0][:, x0 + 1]
    c = coarse[y0 + 1][:, x0]
    d = coarse[y0 + 1][:, x0 + 1]
    img = (a * (1 - fy) * (1 - fx) + b * (1 - fy) * fx + c * fy * (1 - fx) + d * fy * fx)
    img = img + rng.normal(0, noise, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def shapes(rng, H, W, C=3, n=60, patch=96):
    """Random flat rectangles and discs over a vertical colour ramp, with one patch of smooth noise: long edges of every
    orientation, T-junctions and corners, and a file that compresses."""
    ramp = np.linspace(rng.uniform(0, 255, C), rng.uniform(0, 255, C), H)
    img = np.repeat(ramp[:, None, :], W, axis=1)
    y, x = np.mgrid[0:H, 0:W]
    for k in range(n):
        colour = rng.uniform(0, 255, C)
        cy, cx = rng.uniform(0, H), rng.uniform(0, W)
        r = rng.uniform(4, max(4.0, min(H, W) / 5))
        if k % 2:
            mask = (y - cy) ** 2 + (x - cx) ** 2 < r * r
        else:
            mask = (abs(y - cy) < r) & (abs(x - cx) < r * rng.uniform(0.3, 3))
        img[mask] = colour
    py, px = int(rng.integers(0, max(1, H - patch))), int(rng.integers(0, max(1, W - patch)))
    ph, pw = min(patch, H - py), min(patch, W - px)
    img[py:py + ph, px:px + pw] = smooth_noise(rng, ph, pw, C, cell=6, noise=4)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def checkerboard(H, W, square=7):
    y, x = np.mgrid[0:H, 0:W]
    return np.where(((y // square) + (x // square)) % 2 == 0, 40, 215).astype(np.uint8)


def spiral(n=1024, spacing=8, weak=40):
    """A one-pixel-wide square spiral of value `weak` on black, wound outwards from the centre, whose centre pixel is 255:
    with thresholds (100, 300) only the gradients around the centre are strong, so every edge pixel far away is reached
    by hysteresis along the whole spiral, across every 32x32 tile border."""
    img = np.zeros((n, n), np.uint8)
    y = x = n // 2
    dirs = [(0, 1), (1, 0), (0, -1), (-1, 0)]
    step, d = spacing, 0
    while True:
        for _ in range(2):
            dy, dx = dirs[d % 4]
            for _ in range(step):
                if not (2 <= y + dy < n - 2 and 2 <= x + dx < n - 2):
                    img[n // 2, n // 2] = 255
                    return img
                y, x = y + dy, x + dx
                img[y, x] = weak
            d += 1
        step += spacing


def cases():
    """(name, image, (lo, hi)) of the golden file, seeded."""
    rng = np.random.default_rng(20240531)
    out = [
        ("smooth_rgb", smooth_noise(rng, 192, 256, 3), (60.0, 140.0)),
        ("smooth_grey", smooth_noise(rng, 160, 120, 1)[:, :, 0], (150.0, 50.0)),          # swapped
        ("smooth_rgb_frac", smooth_noise(rng, 96, 130, 3, cell=5), (33.5, 87.25)),        # fractional
        ("constant", np.full((64, 80, 3), 117, np.uint8), (10.0, 20.0)),
        ("checkerboard", checkerboard(100, 90), (50.0, 100.0)),
        ("spiral", spiral(), (100.0, 300.0)),
        ("odd_517x333", shapes(rng, 333, 517), (80.75, 40.5)),        # swapped + fractional
        # integer thresholds in the dataset's range randint(1, 255), one pair in each order
        ("rgb512_a", shapes(rng, 512, 512), (9.0, 104.0)),
        ("rgb512_b", shapes(rng, 512, 512, patch=160), (181.0, 37.0)),
        ("equal_thr", smooth_noise(rng, 70, 70, 3), (90.0, 90.0)),
    ]
    return [(n, img, (float(lo), float(hi))) for n, img, (lo, hi) in out]


def main():
    import cv2

    arrays = {}
    names = []
    for name, img, (lo, hi) in cases():
        names.append(name)
        arrays[f"img_{name}"] = img
        arrays[f"thr_{name}"] = np.array([lo, hi], np.float64)
        arrays[f"edges_{name}"] = cv2.Canny(img, lo, hi)
    arrays["names"] = np.array(names)
    np.savez_compressed(OUT, **arrays)
    print(f"{OUT}: {OUT.stat().st_size} bytes, cv2 {cv2.__version__}, {len(names)} images")


if __name__ == "__main__":
    sys.exit(main())
