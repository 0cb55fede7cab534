"""Canny annotator on the device (annotator/canny/__init__.py of the reference, cv2.Canny bit for bit) and the batch
transform the canny configs train and sample with.

    CannyDetector()(img, low, high)          = cv2.Canny(img, low, high): numpy in -> numpy out, CUDA tensor in -> CUDA out
    canny_batch(images, thresholds)          = process/diffusiondb_canny.py:35-45 after the crop, for a whole batch:
                                               (pixel_values, guide), fp32 [B, 3, H, W], the layouts Trainer.step_from_pixels
                                               and sampler.generate take
    canny_batch(images, thr, pixel_values=False) = the control tensor of apps/gradio_canny2image.py:71-74

Random crops and threshold draws stay with the caller's data pipeline.  The channels are used in the order given: the
reference's dataset passes RGB, its make-dataset script BGR (cv2.imread), and on a gradient-magnitude tie between channels
the first one wins, so the two orders can give different maps.
"""
from __future__ import annotations

from typing import Union

import numpy as np
import torch

from . import ops
from ._lib import require_cuda


def _threshold_table(thresholds, B: int, device) -> torch.Tensor:
    if isinstance(thresholds, torch.Tensor) and thresholds.dim() == 2:
        return thresholds.to(device=device, dtype=torch.float32).contiguous()
    lo, hi = (float(v) for v in thresholds)
    return torch.tensor([[lo, hi]], dtype=torch.float32, device=device).expand(B, 2).contiguous()


def _as_nhwc(images: torch.Tensor) -> torch.Tensor:
    if images.dim() == 3:           # [B, H, W] grey
        images = images.unsqueeze(-1)
    return images.contiguous()


class CannyDetector:
    """annotator/canny/__init__.py:6 on the GPU."""

    def __call__(self, img: Union[np.ndarray, torch.Tensor], low_threshold: float, high_threshold: float):
        """img: uint8 [H, W] or [H, W, C] (C = 1 or 3), a numpy array (copied to and from the current CUDA device) or a CUDA
        tensor.  Returns the [H, W] uint8 edge map (0 / 255) as the same kind of object."""
        as_numpy = isinstance(img, np.ndarray)
        if as_numpy:
            if img.dtype != np.uint8 or img.ndim not in (2, 3):
                raise ValueError(f"CannyDetector: expected a uint8 [H, W] or [H, W, C] array, got {img.dtype} {img.shape}")
            x = torch.from_numpy(np.ascontiguousarray(img)).to("cuda")
        else:
            require_cuda(img.device, "CannyDetector")
            x = img
        if x.dim() == 2:
            x = x.unsqueeze(-1)
        H, W = x.shape[0], x.shape[1]
        edges = torch.empty(1, H, W, dtype=torch.uint8, device=x.device)
        ops.canny(x.unsqueeze(0).contiguous(), _threshold_table((low_threshold, high_threshold), 1, x.device), edges=edges)
        return edges[0].cpu().numpy() if as_numpy else edges[0]


def canny_batch(images: torch.Tensor, thresholds, pixel_values: bool = True):
    """images: CUDA uint8 [B, H, W, 3] (RGB crops as the dataset reads them; [B, H, W, 1] or [B, H, W] grey when
    pixel_values=False).  thresholds: a [B, 2] (lo, hi) tensor, one pair per image in either order, or one (lo, hi) pair for
    the whole batch.  Pass a contiguous fp32 CUDA table to keep the call free of host copies (CUDA-graph capture).
    Returns (pixel_values, guide), or guide alone: fp32 [B, 3, H, W]; pixel_values = img / 127.5 - 1 and guide =
    canny / 127.5 - 1 (exactly +-1) repeated to 3 channels, bit-identical to the reference's float32 arithmetic."""
    require_cuda(images.device, "canny_batch")
    x = _as_nhwc(images)
    B, H, W = x.shape[0], x.shape[1], x.shape[2]
    thr = _threshold_table(thresholds, B, x.device)
    guide = torch.empty(B, 3, H, W, dtype=torch.float32, device=x.device)
    pix = torch.empty(B, 3, H, W, dtype=torch.float32, device=x.device) if pixel_values else None
    ops.canny(x, thr, guide=guide, pixels=pix)
    return (pix, guide) if pixel_values else guide
