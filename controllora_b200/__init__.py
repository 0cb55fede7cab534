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

__all__ = [
    "ControlLoRA", "ControlLoRAOutput", "ControlLoRACrossAttnProcessor", "ControlLoRACrossAttnProcessorV2",
    "LoRACrossAttnProcessor", "LoRALinearLayer", "UNet2DConditionModel", "AutoencoderKL", "CLIPTextModel",
    "CannyDetector", "canny_batch",
]
