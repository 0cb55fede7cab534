"""ORACLE (tests only): cv2.Canny(img, low, high) with the defaults the reference uses (aperture 3, L2gradient=False),
restated in numpy, and the float32 arithmetic that turns an image and its Canny map into the `pixel_values` / `guide`
tensors of process/diffusiondb_canny.py:35-45 and apps/gradio_canny2image.py:71-74.

Rules (OpenCV 4.x canny.cpp):
  1. per channel, integer 3x3 Sobel dx / dy with a replicate border;
  2. m = |dx| + |dy|; with several channels each pixel keeps the channel of largest m (first one on a tie) and its dx, dy;
  3. thresholds are swapped when lo > hi, then floored;
  4. non-maximum suppression along the quantised gradient direction (tan 22.5 deg = 13573 / 2^15), neighbours outside
     the image have m = 0; a candidate is a kept pixel with m > low, a strong pixel a candidate with m > high;
  5. hysteresis: an edge is a candidate 8-connected, through candidates, to a strong pixel.
Hysteresis is written as a 3x3 dilation of the edge set restricted to candidates, repeated until nothing changes (each
round dilates only the pixels the previous round added).  The CUDA kernel uses union-find instead.
No cv2 or scipy here: the module must import where neither is installed."""
from __future__ import annotations

import numpy as np

TG22 = 13573  # round(tan(22.5 deg) * 2^15)


def _sobel(ch: np.ndarray):
    p = np.pad(ch.astype(np.int32), 1, mode="edge")
    H, W = ch.shape
    s = lambda dy, dx: p[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]  # noqa: E731
    dx = (s(-1, 1) + 2 * s(0, 1) + s(1, 1)) - (s(-1, -1) + 2 * s(0, -1) + s(1, -1))
    dy = (s(1, -1) + 2 * s(1, 0) + s(1, 1)) - (s(-1, -1) + 2 * s(-1, 0) + s(-1, 1))
    return dx, dy


def gradient(img: np.ndarray):
    """(dx, dy, m) int32 [H, W] after the per-pixel channel selection of rule 2."""
    img = img if img.ndim == 3 else img[:, :, None]
    dx, dy = _sobel(img[:, :, 0])
    m = np.abs(dx) + np.abs(dy)
    for c in range(1, img.shape[2]):
        cdx, cdy = _sobel(img[:, :, c])
        cm = np.abs(cdx) + np.abs(cdy)
        take = cm > m
        dx, dy, m = np.where(take, cdx, dx), np.where(take, cdy, dy), np.where(take, cm, m)
    return dx, dy, m


def thresholds(lo: float, hi: float):
    if lo > hi:
        lo, hi = hi, lo
    return int(np.floor(lo)), int(np.floor(hi))


def candidates(img: np.ndarray, lo: float, hi: float):
    """(candidate, strong) boolean [H, W] maps of rule 4."""
    low, high = thresholds(lo, hi)
    dx, dy, m = gradient(img)
    H, W = m.shape
    mp = np.pad(m, 1)  # m = 0 outside the image
    n = lambda oy, ox: mp[1 + oy:1 + oy + H, 1 + ox:1 + ox + W]  # noqa: E731
    xs, ys = np.abs(dx).astype(np.int64), np.abs(dy).astype(np.int64)
    tg22x = xs * TG22
    y = ys << 15
    tg67x = tg22x + (xs << 16)
    anti = (dx ^ dy) < 0
    keep = np.where(y < tg22x, (m > n(0, -1)) & (m >= n(0, 1)),
           np.where(y > tg67x, (m > n(-1, 0)) & (m >= n(1, 0)),
           np.where(anti, (m > n(-1, 1)) & (m > n(1, -1)),
                          (m > n(-1, -1)) & (m > n(1, 1)))))
    cand = keep & (m > low)
    return cand, cand & (m > high)


def hysteresis(cand: np.ndarray, strong: np.ndarray) -> np.ndarray:
    H, W = cand.shape
    cp = np.zeros((H + 2, W + 2), bool)
    cp[1:-1, 1:-1] = cand
    edge = np.zeros_like(cp)
    edge[1:-1, 1:-1] = strong
    flat_c, flat_e = cp.ravel(), edge.ravel()
    offs = np.array([dy * (W + 2) + dx for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dy or dx])
    front = np.flatnonzero(flat_e)
    while front.size:
        nb = np.unique((front[:, None] + offs[None, :]).ravel())
        nb = nb[flat_c[nb] & ~flat_e[nb]]
        flat_e[nb] = True
        front = nb
    return edge[1:-1, 1:-1]


def canny(img: np.ndarray, lo: float, hi: float) -> np.ndarray:
    """uint8 [H, W] (0 / 255) for a uint8 [H, W] or [H, W, C] image, = cv2.Canny(img, lo, hi)."""
    assert img.dtype == np.uint8 and img.ndim in (2, 3)
    cand, strong = candidates(img, lo, hi)
    return hysteresis(cand, strong).astype(np.uint8) * 255


def pixel_values(img: np.ndarray) -> np.ndarray:
    """process/diffusiondb_canny.py:42-43: float32 [3, H, W] = tensor(img.astype(float32)).permute(2,0,1) / 127.5 - 1,
    each operation rounded to float32."""
    x = img.astype(np.float32).transpose(2, 0, 1)
    return (x / np.float32(127.5)) - np.float32(1)


def guide_values(edges: np.ndarray) -> np.ndarray:
    """process/diffusiondb_canny.py:40,45 (edges.astype(float32) / 127.5 - 1, repeated to 3 channels) and
    apps/gradio_canny2image.py:72-74 (HWC3, [..., ::-1], / 127.5 - 1; the three channels are equal): float32 [3, H, W]."""
    g = (edges.astype(np.float32) / np.float32(127.5)) - np.float32(1)
    return np.repeat(g[None], 3, axis=0)
