"""controllora_b200 — H100-native (sm_90a) implementation of the ControlLoRA UNet hot path.

Public surface mirrors /root/reference/models.py plus the slice of diffusers' UNet2DConditionModel that the reference
drivers use.  Importing the package does not require a GPU; running any op does (there is no CPU fallback).
"""
from .models import (ControlLoRA, ControlLoRACrossAttnProcessor, ControlLoRACrossAttnProcessorV2, ControlLoRAOutput,
                     LoRACrossAttnProcessor, LoRALinearLayer)
from .unet_module import UNet2DConditionModel
from .vae import AutoencoderKL
from .clip import CLIPTextModel
from .annotator import CannyDetector, canny_batch
from .transforms import HWC3, reference_crops, resize_image, train_transform
from .pose import draw_bodypose, pose_batch, pose_control
from .jpeg import decode_jpeg, dreambooth_crops, dreambooth_transform
from .png import decode_images, decode_png

__all__ = [
    "ControlLoRA", "ControlLoRAOutput", "ControlLoRACrossAttnProcessor", "ControlLoRACrossAttnProcessorV2",
    "LoRACrossAttnProcessor", "LoRALinearLayer", "UNet2DConditionModel", "AutoencoderKL", "CLIPTextModel",
    "CannyDetector", "canny_batch", "HWC3", "reference_crops", "resize_image", "train_transform",
    "draw_bodypose", "pose_batch", "pose_control", "decode_jpeg", "dreambooth_crops", "dreambooth_transform",
    "decode_png", "decode_images",
]
