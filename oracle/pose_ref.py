"""ORACLE (tests only): the reference's draw_bodypose (annotator/openpose/util.py:37-70) restated in numpy, rule by rule,
and the guide arithmetic of apps/gradio_pose2image.py:70-78 and process/mpii_pose.py:29-44.  Every primitive is pinned
to OpenCV 4.13 by tests/test_pose.py, and the whole function to the reference's own.

    circle        cv2.circle(img, c, 4, colour, thickness=-1): drawing.cpp Circle(), the integer midpoint rasteriser,
                  each row's span clipped to the image
    ellipse2Poly  drawing.cpp ellipse2Poly: points in double from OpenCV's float sine table (pose_sin_table.h),
                  cvRound (half to even), consecutive duplicates dropped, a lone point doubled
    line          drawing.cpp Line() with LINE_8: LineIterator (leftToRight) after clipLine
    fillConvexPoly  drawing.cpp FillConvexPoly, shift 0, LINE_8: every edge stroked with line(), then the 16-bit
                  fixed-point scanline walk of both edge chains from the topmost vertex
    addWeighted   cv2.addWeighted(a, 0.4, b, 0.6, 0) on uint8 = saturate(rint(0.4f * a + 0.6f * b)) in float32
    INTER_NEAREST cv2.resize: source index min(floor(x * (1 / (dst / src))), src - 1) in double
No cv2 here: the module must import where it is not installed."""
from __future__ import annotations

import math
import re
from pathlib import Path

import numpy as np

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
STICKWIDTH = 4
# util.py:39-45; only the first 17 limbs are drawn (util.py:53)
LIMB_SEQ = [[2, 3], [2, 6], [3, 4], [4, 5], [6, 7], [7, 8], [2, 9], [9, 10], [10, 11], [2, 12], [12, 13], [13, 14],
            [2, 1], [1, 15], [15, 17], [1, 16], [16, 18], [3, 17], [6, 18]]
COLORS = [[255, 0, 0], [255, 85, 0], [255, 170, 0], [255, 255, 0], [170, 255, 0], [85, 255, 0], [0, 255, 0],
          [0, 255, 85], [0, 255, 170], [0, 255, 255], [0, 170, 255], [0, 85, 255], [0, 0, 255], [85, 0, 255],
          [170, 0, 255], [255, 0, 255], [255, 0, 170], [255, 0, 85]]

_TABLE = Path(__file__).resolve().parent.parent / "controllora_b200" / "csrc" / "pose_sin_table.h"


def sin_table_q30() -> np.ndarray:
    """int64 [451]: 2^30 * OpenCV's SinTable, read from the header the kernel compiles."""
    text = _TABLE.read_text()
    body = text[text.index("#define CL_POSE_SIN_Q30 {"):]
    vals = [int(v) for v in re.findall(r"-?\d+", body[body.index("{"):body.index("}")])]
    assert len(vals) == 451
    return np.array(vals, np.int64)


SIN = (sin_table_q30().astype(np.float64) / (1 << 30)).astype(np.float32)   # exact: every entry is k / 2^30


def cv_round(v: float) -> int:
    return int(np.rint(v))                     # cvRound: round half to even


# ------------------------------------------------------------------------------------------------------ ellipse2Poly
def ellipse2poly(center, axes, angle: int, arc_start: int = 0, arc_end: int = 360, delta: int = 1) -> np.ndarray:
    """int32 [n, 2] (x, y) points of cv2.ellipse2Poly with an integer centre and axes."""
    while angle < 0:
        angle += 360
    while angle > 360:
        angle -= 360
    if arc_start > arc_end:
        arc_start, arc_end = arc_end, arc_start
    while arc_start < 0:
        arc_start += 360
        arc_end += 360
    while arc_end > 360:
        arc_end -= 360
        arc_start -= 360
    if arc_end - arc_start > 360:
        arc_start, arc_end = 0, 360
    a = angle + (360 if angle < 0 else 0)
    alpha, beta = float(SIN[450 - a]), float(SIN[a])          # cos, sin as float
    cx, cy = float(center[0]), float(center[1])
    out = []
    prev = None
    for i in range(arc_start, arc_end + delta, delta):
        t = min(i, arc_end)
        if t < 0:
            t += 360
        x = float(axes[0]) * float(SIN[450 - t])
        y = float(axes[1]) * float(SIN[t])
        pt = (cv_round(cx + x * alpha - y * beta), cv_round(cy + x * beta + y * alpha))
        if pt != prev:
            out.append(pt)
            prev = pt
    if len(out) == 1:
        out = [(int(center[0]), int(center[1]))] * 2
    return np.array(out, np.int32).reshape(-1, 2)


# ------------------------------------------------------------------------------------------------------------- line
def _trunc(v: float) -> int:
    return int(v)                              # (int64)(double): toward zero


def clip_line(W: int, H: int, x1: int, y1: int, x2: int, y2: int):
    """drawing.cpp clipLine(Size, Point&, Point&): (visible, x1, y1, x2, y2)."""
    if W <= 0 or H <= 0:
        return False, x1, y1, x2, y2
    right, bottom = W - 1, H - 1
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += _trunc(float(a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += _trunc(float(a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += _trunc(float(a - x1) * (y2 - y1) / (x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += _trunc(float(a - x2) * (y2 - y1) / (x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, x1, y1, x2, y2


def line_pixels(W: int, H: int, p1, p2):
    """(xs, ys) of cv2.line(img, p1, p2, c, 1, LINE_8) on a W x H image: LineIterator(img, p1, p2, 8, leftToRight=True)."""
    x1, y1 = int(p1[0]), int(p1[1])
    x2, y2 = int(p2[0]), int(p2[1])
    if not (0 <= x1 < W and 0 <= x2 < W and 0 <= y1 < H and 0 <= y2 < H):
        ok, x1, y1, x2, y2 = clip_line(W, H, x1, y1, x2, y2)
        if not ok:
            return np.zeros(0, np.int64), np.zeros(0, np.int64)
    sx = sy = 1
    dx, dy = x2 - x1, y2 - y1
    if dx < 0:                                 # leftToRight
        dx, dy = -dx, -dy
        x1, y1, x2, y2 = x2, y2, x1, y1
    if dy < 0:
        dy, sy = -dy, -1
    vert = dy > dx
    if vert:
        dx, dy = dy, dx
        sx, sy = sy, sx
    err = dx - (dy + dy)
    plus, minus = dx + dx, -(dy + dy)
    count = dx + 1
    xs, ys = np.empty(count, np.int64), np.empty(count, np.int64)
    x, y = x1, y1
    for k in range(count):
        xs[k], ys[k] = x, y
        neg = err < 0
        err += minus + (plus if neg else 0)
        if vert:                               # minor steps go along x
            y += sx
            x += sy if neg else 0
        else:
            x += sx
            y += sy if neg else 0
    return xs, ys


# ------------------------------------------------------------------------------------------------------ fillConvexPoly
def fill_convex_poly_mask(H: int, W: int, pts: np.ndarray) -> np.ndarray:
    """bool [H, W]: the pixels cv2.fillConvexPoly(img, pts, c) (LINE_8, shift 0) writes."""
    m = np.zeros((H, W), bool)
    v = [(int(x), int(y)) for x, y in np.asarray(pts).reshape(-1, 2)]
    n = len(v)
    if n == 0:
        return m
    p0 = v[-1]
    xmin = xmax = v[0][0]
    ymin = ymax = v[0][1]
    imin = 0
    for i, p in enumerate(v):
        if p[1] < ymin:
            ymin, imin = p[1], i
        ymax, xmax, xmin = max(ymax, p[1]), max(xmax, p[0]), min(xmin, p[0])
        xs, ys = line_pixels(W, H, p0, p)
        m[ys, xs] = True
        p0 = p
    if n < 3 or xmax < 0 or ymax < 0 or xmin >= W or ymin >= H:
        return m
    ymax = min(ymax, H - 1)
    # edge: [idx, di, x, dx, ye]
    edge = [[imin, 1, -XY_ONE, 0, ymin], [imin, n - 1, -XY_ONE, 0, ymin]]
    y = ymin
    edges = n
    half = XY_ONE >> 1
    while True:
        for e in edge:
            if y >= e[4]:
                idx0, di = e[0], e[1]
                idx = idx0 + di
                if idx >= n:
                    idx -= n
                while True:
                    go = edges > 0
                    edges -= 1
                    if not go:
                        break
                    ty = v[idx][1]
                    if ty > y:
                        xs, xe = v[idx0][0] << XY_SHIFT, v[idx][0] << XY_SHIFT
                        num, den = (xe - xs) * 2 + (ty - y), 2 * (ty - y)
                        q = abs(num) // den
                        e[4], e[3], e[2], e[0] = ty, (q if num >= 0 else -q), xs, idx    # C division: toward zero
                        break
                    idx0 = idx
                    idx += di
                    if idx >= n:
                        idx -= n
        if edges < 0:
            break
        if y >= 0:
            l, r = (1, 0) if edge[0][2] > edge[1][2] else (0, 1)
            xx1 = (edge[l][2] + half) >> XY_SHIFT
            xx2 = (edge[r][2] + half) >> XY_SHIFT
            if xx2 >= 0 and xx1 < W:
                m[y, max(xx1, 0):min(xx2, W - 1) + 1] = True
            step = 1
        else:                                  # rows above the image: no edge changes before min(ye, 0)
            step = min(edge[0][4], edge[1][4], 0) - y
        edge[0][2] += edge[0][3] * step
        edge[1][2] += edge[1][3] * step
        y += step
        if y > ymax:
            break
    return m


# ------------------------------------------------------------------------------------------------------------ circle
def circle_spans(radius: int):
    """{dy: half-width} of drawing.cpp Circle(fill=1): the rows center.y + dy hold [center.x - hw, center.x + hw]."""
    err, dx, dy, plus, minus = 0, radius, 0, 1, (radius << 1) - 1
    hw = {}
    while dx >= dy:
        for oy, h in ((dy, dx), (-dy, dx), (dx, dy), (-dx, dy)):
            hw[oy] = max(hw.get(oy, -1), h)
        dy += 1
        err += plus
        plus += 2
        mask = -1 if err > 0 else 0            # (err <= 0) - 1
        err -= minus & mask
        dx += mask
        minus -= mask & 2
    return hw


def circle_mask(H: int, W: int, cx: int, cy: int, radius: int = 4) -> np.ndarray:
    m = np.zeros((H, W), bool)
    for oy, h in circle_spans(radius).items():
        y = cy + oy
        if 0 <= y < H and cx - h < W and cx + h >= 0:
            m[y, max(cx - h, 0):min(cx + h, W - 1) + 1] = True
    return m


# ------------------------------------------------------------------------------------------------------------- blend
def add_weighted(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """cv2.addWeighted(a, 0.4, b, 0.6, 0) on uint8."""
    t = np.float32(0.4) * a.astype(np.float32) + np.float32(0.6) * b.astype(np.float32)
    return np.clip(np.rint(t), 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------- INTER_NEAREST
def nearest_index(src: int, dst: int) -> np.ndarray:
    """Source index of each of dst outputs: cv2.resize(INTER_NEAREST) along one axis of length src."""
    inv = 1.0 / (dst / src)
    return np.minimum(np.floor(np.arange(dst, dtype=np.float64) * inv).astype(np.int64), src - 1)


def resize_nearest(img: np.ndarray, H: int, W: int) -> np.ndarray:
    return img[nearest_index(img.shape[0], H)][:, nearest_index(img.shape[1], W)]


# ------------------------------------------------------------------------------------------------------ draw_bodypose
def limb_params(candidate: np.ndarray, i0: int, i1: int):
    """util.py:59-65 on float64 keypoints, with the reference's own numpy scalar operations: ellipse2Poly's
    (centre x, centre y, half length, angle)."""
    index = np.array([i0, i1])
    Y = candidate[index.astype(int), 0]
    X = candidate[index.astype(int), 1]
    mX = np.mean(X)
    mY = np.mean(Y)
    length = ((X[0] - X[1]) ** 2 + (Y[0] - Y[1]) ** 2) ** 0.5
    angle = math.degrees(math.atan2(X[0] - X[1], Y[0] - Y[1]))
    return int(mY), int(mX), int(length / 2), int(angle)


def limb_mask(H: int, W: int, cx: int, cy: int, half_len: int, angle: int) -> np.ndarray:
    return fill_convex_poly_mask(H, W, ellipse2poly((cx, cy), (half_len, STICKWIDTH), angle, 0, 360, 1))


def draw_bodypose(canvas: np.ndarray, candidate: np.ndarray, subset: np.ndarray) -> np.ndarray:
    """util.py:37-70: uint8 [H, W, 3] canvas with every person's circles, then every limb blended over it."""
    canvas = np.array(canvas, np.uint8, copy=True)
    H, W = canvas.shape[:2]
    candidate = np.asarray(candidate, np.float64)
    subset = np.asarray(subset)
    for i in range(18):
        for n in range(len(subset)):
            index = int(subset[n][i])
            if index == -1:
                continue
            x, y = candidate[index][0:2]
            canvas[circle_mask(H, W, int(x), int(y))] = COLORS[i]
    for i in range(17):
        for n in range(len(subset)):
            index = subset[n][np.array(LIMB_SEQ[i]) - 1]
            if -1 in index:
                continue
            m = limb_mask(H, W, *limb_params(candidate, *index.astype(int)))
            canvas[m] = add_weighted(canvas[m], np.array(COLORS[i], np.uint8)[None, :])
    return canvas


def guide(canvas: np.ndarray, flip: bool = True) -> np.ndarray:
    """fp32 [3, H, W]: apps/gradio_pose2image.py:78 (flip: the canvas' BGR drawing order to RGB) or
    process/mpii_pose.py:40 (no flip), x / 127.5 - 1 with each operation rounded to float32."""
    c = canvas[..., ::-1] if flip else canvas
    return (c.astype(np.float32) / np.float32(127.5) - np.float32(1)).transpose(2, 0, 1).copy()


def window(canvas: np.ndarray, crop=None, out_hw=None) -> np.ndarray:
    """Crop (y0, x0, h, w) of the rendered canvas, then cv2.resize(..., (W, H), INTER_NEAREST)."""
    if crop is not None:
        y0, x0, h, w = crop
        canvas = canvas[y0:y0 + h, x0:x0 + w]
    if out_hw is not None:
        canvas = resize_nearest(canvas, *out_hw)
    return canvas
