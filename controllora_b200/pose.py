"""OpenPose body-skeleton guides on the device: the reference's draw_bodypose (annotator/openpose/util.py:37-70) bit for
bit, and the guide tensors the pose configs train and sample with.  Keypoints in, guide out: the body network that
finds the keypoints is not part of this package.

    draw_bodypose(canvas, candidate, subset)   = util.draw_bodypose: numpy in -> numpy out, CUDA tensor in -> CUDA out
    pose_batch(keypoints, canvas_hw, ...)      = the guides of a training batch, fp32 [B, 3, H, W] in the layout
                                                 Trainer.step_from_pixels and sampler.generate take; per image a canvas
                                                 size, an optional crop (process/mpii_pose.py:29-36 crops the drawn
                                                 guide) and an optional INTER_NEAREST resize
    pose_control(candidate, subset, ...)       = the control tensor of apps/gradio_pose2image.py:70-78

Host work per call: the integer ellipse parameters of every limb (Python floats, the reference's own operations: a
vectorised atan2 may differ from libm in the last bit, and int() of a near-integer angle depends on it), one upload of
the descriptors, and one cl_pose_render call (two launches).  Keypoints are float64 (x, y); coordinates are limited to
|x|, |y| < 2^21.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence, Union

import numpy as np
import torch

from . import ops
from ._lib import CLError, PoseCircle, PoseImage, PoseLimb, require_cuda
from .transforms import resize_image_size

STICKWIDTH = 4
MAX_COORD = float(1 << 21)
MAX_CANVAS = 4096
# util.py:39-45; only the first 17 limbs are drawn (util.py:53)
LIMB_SEQ = [[2, 3], [2, 6], [3, 4], [4, 5], [6, 7], [7, 8], [2, 9], [9, 10], [10, 11], [2, 12], [12, 13], [13, 14],
            [2, 1], [1, 15], [15, 17], [1, 16], [16, 18], [3, 17], [6, 18]]
COLORS = [[255, 0, 0], [255, 85, 0], [255, 170, 0], [255, 255, 0], [170, 255, 0], [85, 255, 0], [0, 255, 0],
          [0, 255, 85], [0, 255, 170], [0, 255, 255], [0, 170, 255], [0, 85, 255], [0, 0, 255], [85, 0, 255],
          [170, 0, 255], [255, 0, 255], [255, 0, 170], [255, 0, 85]]
_PACKED = [c[0] | (c[1] << 8) | (c[2] << 16) for c in COLORS]


def _point(x, y, what: str) -> tuple[float, float]:
    x, y = float(x), float(y)
    if not (abs(x) < MAX_COORD and abs(y) < MAX_COORD):
        raise CLError(f"{what}: keypoint ({x}, {y}) is not finite or outside |x|, |y| < 2^21")
    return x, y


def limb_params(x0: float, y0: float, x1: float, y1: float) -> tuple[int, int, int, int]:
    """util.py:59-65 for a limb from (x0, y0) to (x1, y1): ellipse2Poly's (centre x, centre y, half length, angle).
    The reference names x `Y` and y `X`; np.mean of two float64 values is (a + b) / 2."""
    mX, mY = (y0 + y1) / 2, (x0 + x1) / 2
    length = ((y0 - y1) ** 2 + (x0 - x1) ** 2) ** 0.5
    angle = math.degrees(math.atan2(y0 - y1, x0 - x1))
    return int(mY), int(mX), int(length / 2), int(angle)


def _prims_from_candidate(candidate, subset, what: str):
    """util.py:46-67's loops: circles [(x, y, colour)] and limbs [(cx, cy, half_len, angle, colour)] in draw order."""
    candidate = np.asarray(candidate, np.float64)
    subset = np.asarray(subset, np.float64)
    if subset.size == 0:
        return [], []
    if subset.ndim != 2 or subset.shape[1] < 18 or candidate.ndim != 2 or candidate.shape[1] < 2:
        raise CLError(f"{what}: expected candidate [N, >=2] and subset [P, >=18], got {candidate.shape} and {subset.shape}")
    circles, limbs = [], []
    for i in range(18):
        for n in range(len(subset)):
            index = int(subset[n][i])
            if index == -1:
                continue
            x, y = _point(*candidate[index][0:2], what)
            circles.append((int(x), int(y), _PACKED[i]))
    for i in range(17):
        for n in range(len(subset)):
            index = subset[n][np.array(LIMB_SEQ[i]) - 1]
            if -1 in index:
                continue
            a, b = index.astype(int)
            x0, y0 = _point(*candidate[a][0:2], what)
            x1, y1 = _point(*candidate[b][0:2], what)
            limbs.append(limb_params(x0, y0, x1, y1) + (_PACKED[i],))
    return circles, limbs


def _prims_from_dense(kp: np.ndarray, what: str):
    """kp: [P, 18, 3] (x, y, present): the same primitives as _prims_from_candidate for the present keypoints."""
    present = kp[:, :, 2] > 0
    xy = kp[:, :, :2]
    if not np.all(np.abs(xy[present]) < MAX_COORD):
        raise CLError(f"{what}: keypoints must be finite with |x|, |y| < 2^21")
    circles, limbs = [], []
    P = kp.shape[0]
    for i in range(18):
        for n in range(P):
            if present[n, i]:
                circles.append((int(xy[n, i, 0]), int(xy[n, i, 1]), _PACKED[i]))
    for i in range(17):
        a, b = LIMB_SEQ[i][0] - 1, LIMB_SEQ[i][1] - 1
        for n in range(P):
            if present[n, a] and present[n, b]:
                limbs.append(limb_params(float(xy[n, a, 0]), float(xy[n, a, 1]), float(xy[n, b, 0]), float(xy[n, b, 1]))
                             + (_PACKED[i],))
    return circles, limbs


def _box(cx: int, cy: int, half: int, H: int, W: int):
    """A box that holds every pixel the limb's polygon, its edge lines and its fill can reach, clipped to the canvas:
    the polygon's points lie within half + 4 of the centre before rounding."""
    r = half + STICKWIDTH + 2
    x0, y0 = max(cx - r, 0), max(cy - r, 0)
    x1, y1 = min(cx + r, W - 1), min(cy + r, H - 1)
    if x1 < x0 or y1 < y0:
        return 0, 0, 0, 0
    return x0, y0, x1 - x0 + 1, y1 - y0 + 1


class _Plan:
    """Host side of one cl_pose_render call: the three descriptor arrays, their bytes back to back, the mask size."""

    def __init__(self, prims, canvas_hw, crops, bg_offs, limb_capacity: Optional[int] = None):
        B = len(prims)
        nc = sum(len(c) for c, _ in prims)
        nl = sum(len(l) for _, l in prims)
        cap = nl if limb_capacity is None else limb_capacity
        if nl > cap:
            raise CLError(f"pose: {nl} limbs exceed the buffer's capacity of {cap}")
        self.img, self.circles, self.limbs = (PoseImage * B)(), (PoseCircle * max(nc, 0))(), (PoseLimb * cap)()
        ci = li = 0
        words = 0
        for b, ((circles, limbs), (H, W), (y0, x0, h, w), bg_off) in enumerate(zip(prims, canvas_hw, crops, bg_offs)):
            d = self.img[b]
            d.bg_off, d.Hc, d.Wc, d.y0, d.x0, d.h, d.w = bg_off, H, W, y0, x0, h, w
            d.circle0, d.n_circles, d.limb0, d.n_limbs = ci, len(circles), li, len(limbs)
            for x, y, col in circles:
                c = self.circles[ci]
                c.x, c.y, c.color = x, y, col
                ci += 1
            for cx, cy, half, angle, col in limbs:
                L = self.limbs[li]
                L.image, L.cx, L.cy, L.half_len, L.angle, L.color = b, cx, cy, half, angle, col
                L.bx0, L.by0, L.bw, L.bh = _box(cx, cy, half, H, W)
                L.mask_off = words
                words += L.bh * ((L.bw + 31) // 32)
                li += 1
        for i in range(li, cap):
            self.limbs[i].image = -1
        self.mask_words = words
        self.bytes = np.frombuffer(bytes(self.img) + bytes(self.circles) + bytes(self.limbs), np.uint8)


def _windows(B, canvas_hw, crops, out_hw, what):
    if isinstance(canvas_hw[0], (int, np.integer)):
        canvas_hw = [tuple(canvas_hw)] * B
    canvas_hw = [(int(h), int(w)) for h, w in canvas_hw]
    if len(canvas_hw) != B:
        raise CLError(f"{what}: {len(canvas_hw)} canvas sizes for {B} images")
    for H, W in canvas_hw:
        if not (0 < H <= MAX_CANVAS and 0 < W <= MAX_CANVAS):
            raise CLError(f"{what}: canvas {H} x {W}, expected 1..{MAX_CANVAS} on each side")
    crops = [(0, 0, H, W) for H, W in canvas_hw] if crops is None else [tuple(int(v) for v in c) for c in crops]
    if len(crops) != B:
        raise CLError(f"{what}: {len(crops)} crops for {B} images")
    for (H, W), (y0, x0, h, w) in zip(canvas_hw, crops):
        if y0 < 0 or x0 < 0 or h <= 0 or w <= 0 or y0 + h > H or x0 + w > W:
            raise CLError(f"{what}: crop ({y0}, {x0}) + {h} x {w} outside the {H} x {W} canvas")
    if out_hw is None:
        sizes = {(h, w) for _, _, h, w in crops}
        if len(sizes) != 1:
            raise CLError(f"{what}: windows of different sizes {sorted(sizes)} need out_hw")
        out_hw = sizes.pop()
    out_hw = (int(out_hw[0]), int(out_hw[1]))
    if not (0 < out_hw[0] <= MAX_CANVAS and 0 < out_hw[1] <= MAX_CANVAS):
        raise CLError(f"{what}: output size {out_hw}, expected 1..{MAX_CANVAS} on each side")
    return canvas_hw, crops, out_hw


def _stage(data: np.ndarray, device) -> torch.Tensor:
    staged = torch.empty(max(data.size, 1), dtype=torch.uint8, pin_memory=True)
    staged.numpy()[:data.size] = data
    return staged.to(device, non_blocking=True)


def _render(prims, canvas_hw, crops, out_hw, backgrounds, flip, want_canvas, want_guide, device):
    B = len(prims)
    bg, bg_offs = None, [-1] * B
    if backgrounds is not None:
        if len(backgrounds) != B:
            raise CLError(f"pose: {len(backgrounds)} backgrounds for {B} images")
        parts, off = [], 0
        for b, (x, (H, W)) in enumerate(zip(backgrounds, canvas_hw)):
            if x is None:
                continue
            t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
            if t.dtype != torch.uint8 or tuple(t.shape) != (H, W, 3):
                raise CLError(f"pose: background {b} must be uint8 [{H}, {W}, 3], got {t.dtype} {tuple(t.shape)}")
            parts.append(t.reshape(-1).to(device))
            bg_offs[b] = off
            off += t.numel()
        bg = torch.cat(parts) if parts else None
    plan = _Plan(prims, canvas_hw, crops, bg_offs)
    packed = _stage(plan.bytes, device)
    mask = torch.empty(max(plan.mask_words, 1), dtype=torch.int32, device=device)
    oh, ow = out_hw
    canvas = torch.empty(B, oh, ow, 3, dtype=torch.uint8, device=device) if want_canvas else None
    guide = torch.empty(B, 3, oh, ow, dtype=torch.float32, device=device) if want_guide else None
    ops.pose_render(plan.img, plan.circles, plan.limbs, packed, mask, oh, ow, flip=flip, bg=bg, out_canvas=canvas,
                    out_guide=guide)
    return canvas, guide


def _dense_prims(keypoints, what):
    if isinstance(keypoints, torch.Tensor):
        keypoints = keypoints.detach().cpu().numpy()
    if isinstance(keypoints, np.ndarray):
        kp = np.asarray(keypoints, np.float64)
        if kp.ndim != 4 or kp.shape[2:] != (18, 3):
            raise CLError(f"{what}: expected keypoints [B, P, 18, 3] (x, y, present), got {kp.shape}")
        return [_prims_from_dense(kp[b], what) for b in range(kp.shape[0])]
    return [_prims_from_candidate(c, s, what) for c, s in keypoints]


def draw_bodypose(canvas: Union[np.ndarray, torch.Tensor], candidate, subset):
    """util.py:37-70 on the GPU: canvas uint8 [H, W, 3] (numpy, copied to and from the current CUDA device, or a CUDA
    tensor), candidate [N, 4] (x, y, score, id) and subset [P, 20] as body.py returns them.  Returns the drawn canvas as
    the same kind of object; the input is not modified."""
    as_numpy = isinstance(canvas, np.ndarray)
    if as_numpy:
        x = torch.from_numpy(np.ascontiguousarray(canvas))
        device = torch.device("cuda")
    else:
        require_cuda(canvas.device, "draw_bodypose")
        x, device = canvas, canvas.device
    if x.dtype != torch.uint8 or x.dim() != 3 or x.shape[2] != 3:
        raise CLError(f"draw_bodypose: expected a uint8 [H, W, 3] canvas, got {x.dtype} {tuple(x.shape)}")
    H, W = int(x.shape[0]), int(x.shape[1])
    canvas_hw, crops, out_hw = _windows(1, (H, W), None, None, "draw_bodypose")
    out, _ = _render([_prims_from_candidate(candidate, subset, "draw_bodypose")], canvas_hw, crops, out_hw, [x], True,
                     True, False, device)
    return out[0].cpu().numpy() if as_numpy else out[0]


def pose_batch(keypoints, canvas_hw, crops: Optional[Sequence] = None, out_hw=None, backgrounds=None, flip: bool = True,
               canvas: bool = False, device=None):
    """Pose guides of a batch.  keypoints: [B, P, 18, 3] (x, y, present) as a numpy array or tensor (P padded; a keypoint
    is drawn when present > 0), or a list of B (candidate, subset) pairs as body.py returns them.  canvas_hw: one (H, W)
    for every canvas or one per image.  crops: per image (y0, x0, h, w) of the drawn canvas (default: all of it), then
    a cv2 INTER_NEAREST resize to out_hw (default: the crop size, which must then be the same for every image).
    backgrounds: None (zero canvases, as OpenposeDetector draws) or per image a uint8 [H, W, 3] canvas or None.
    flip: guide channels reversed from the drawing order (the app's [..., ::-1]); flip=False keeps the drawing order.
    Returns the fp32 [B, 3, H, W] guide x / 127.5 - 1 (and, with canvas=True, also the uint8 [B, H, W, 3] window)."""
    device = torch.device(device if device is not None else "cuda")
    require_cuda(device, "pose_batch")
    prims = _dense_prims(keypoints, "pose_batch")
    canvas_hw, crops, out_hw = _windows(len(prims), canvas_hw, crops, out_hw, "pose_batch")
    u8, guide = _render(prims, canvas_hw, crops, out_hw, backgrounds, flip, canvas, True, device)
    return (guide, u8) if canvas else guide


def pose_control(candidate, subset, input_hw, detect_resolution: int = 512, image_resolution: int = 512, device=None):
    """apps/gradio_pose2image.py:70-78: the skeleton drawn on a zero canvas of resize_image(input, detect_resolution)'s
    size (candidate and subset are in that image's pixels), resized with INTER_NEAREST to resize_image(input,
    image_resolution)'s size, channels flipped, / 127.5 - 1: fp32 [1, 3, H, W]."""
    h, w = int(input_hw[0]), int(input_hw[1])
    dh, dw, _ = resize_image_size(h, w, detect_resolution)
    ih, iw, _ = resize_image_size(h, w, image_resolution)
    return pose_batch([(candidate, subset)], (dh, dw), out_hw=(ih, iw), device=device)


class PoseBuffers:
    """Fixed device buffers for repeated pose_batch calls of one shape (B images, up to P persons, dense keypoints, zero
    canvases): every device address stays the same, so a call can be captured in a CUDA graph.  stage() writes new
    keypoints into the pinned staging buffer on the host; the captured call's upload re-reads it on every replay.  The
    caller must not restage while a replay that reads the staging buffer is in flight."""

    def __init__(self, B: int, P: int, canvas_hw, crops=None, out_hw=None, flip: bool = True, device=None):
        self.device = torch.device(device if device is not None else "cuda")
        require_cuda(self.device, "PoseBuffers")
        self.B, self.P, self.flip = B, P, flip
        self.canvas_hw, self.crops, self.out_hw = _windows(B, canvas_hw, crops, out_hw, "PoseBuffers")
        self.limb_capacity = B * P * 17
        # worst case: every limb's box is its whole canvas
        self.mask_words = max(P * 17 * sum(H * ((W + 31) // 32) for H, W in self.canvas_hw), 1)
        self.nbytes = C.sizeof(PoseImage) * B + C.sizeof(PoseCircle) * B * P * 18 + C.sizeof(PoseLimb) * self.limb_capacity
        self.staging = torch.zeros(self.nbytes, dtype=torch.uint8, pin_memory=True)
        self.packed = torch.zeros(self.nbytes, dtype=torch.uint8, device=self.device)
        self.mask = torch.zeros(self.mask_words, dtype=torch.int32, device=self.device)
        self.guide = torch.empty(B, 3, *self.out_hw, dtype=torch.float32, device=self.device)
        self.plan = None

    def stage(self, keypoints) -> None:
        kp = keypoints.detach().cpu().numpy() if isinstance(keypoints, torch.Tensor) else np.asarray(keypoints)
        if kp.shape != (self.B, self.P, 18, 3):
            raise CLError(f"PoseBuffers: expected keypoints {(self.B, self.P, 18, 3)}, got {kp.shape}")
        plan = _Plan(_dense_prims(kp, "PoseBuffers"), self.canvas_hw, self.crops, [-1] * self.B, self.limb_capacity)
        circles = (PoseCircle * (self.B * self.P * 18))()      # the circle array keeps its capacity too
        C.memmove(circles, plan.circles, C.sizeof(plan.circles))
        plan.circles = circles
        if plan.mask_words > self.mask_words:
            raise CLError(f"PoseBuffers: {plan.mask_words} mask words exceed the capacity of {self.mask_words}")
        data = np.frombuffer(bytes(plan.img) + bytes(plan.circles) + bytes(plan.limbs), np.uint8)
        self.staging.numpy()[:] = data
        self.plan = plan

    def launch(self) -> torch.Tensor:
        """Upload the staged descriptors and render into self.guide (fp32 [B, 3, H, W])."""
        if self.plan is None:
            raise CLError("PoseBuffers: stage() keypoints before launch()")
        self.packed.copy_(self.staging, non_blocking=True)
        ops.pose_render(self.plan.img, self.plan.circles, self.plan.limbs, self.packed, self.mask, *self.out_hw,
                        flip=self.flip, out_guide=self.guide)
        return self.guide
