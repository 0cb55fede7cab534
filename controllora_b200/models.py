"""Drop-in class surface of /root/reference/models.py, backed by the CUDA kernels.

Same class names, constructor kwargs, attribute names and state-dict keys as the reference (models.py:72-835), so the
reference's configs/*.json and the wiring code of train_text_to_image_control_lora.py:469-487 work unchanged:

    control_lora = ControlLoRA.from_config("configs/fill50k.json")
    unet = UNet2DConditionModel.from_state_dict(sd)           # diffusers key names
    ... pop processors from control_lora.lora_layers, unet.set_attn_processor(procs) ...
    control_lora(guide)                                        # injects control states into the processors
    noise_pred = unet(noisy_latents, timesteps, encoder_hidden_states).sample

The processors here are *parameter containers + wiring*: inside this package's UNet the arithmetic of a processor call
(models.py:118-152, 222-287, 357-431) is part of the whole-network program (controllora_b200/lora_runtime.py).  Installed on
a real diffusers UNet they are called per attention module like the reference's (`processor(attn, hidden_states, ...)`), which
runs the same kernels for that one layer through an autograd bridge (controllora_b200/eager_attn.py).  There is no
PyTorch/CPU implementation of the arithmetic in this package.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional, Tuple

import torch
import torch.nn as nn


class LoRALinearLayer(nn.Module):
    """Parameter container with diffusers' LoRALinearLayer layout/initialisation: down ~ N(0, 1/rank), up = 0."""

    def __init__(self, in_features: int, out_features: int, rank: int = 4):
        super().__init__()
        if rank > min(in_features, out_features):
            raise ValueError(f"LoRA rank {rank} must be less or equal than {min(in_features, out_features)}")
        self.down = nn.Linear(in_features, rank, bias=False)
        self.up = nn.Linear(rank, out_features, bias=False)
        nn.init.normal_(self.down.weight, std=1 / rank)
        nn.init.zeros_(self.up.weight)

    def forward(self, x):
        """up(down(x)) on the CUDA kernels (fp32 rank space), differentiable w.r.t. x, down and up."""
        from .eager_attn import lora_linear_forward

        return lora_linear_forward(self, x)


class LoRACrossAttnProcessor(nn.Module):
    """models.py:72-152 (constructor, flags and skip_* helpers)."""

    def __init__(self, hidden_size, cross_attention_dim=None, rank=4, post_add=False, key_states_skipped=False,
                 value_states_skipped=False, output_states_skipped=False):
        super().__init__()
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        self.rank = rank
        self.post_add = post_add
        kv_in = hidden_size if post_add else (cross_attention_dim or hidden_size)
        self.to_q_lora = LoRALinearLayer(hidden_size, hidden_size, rank)
        if not key_states_skipped:
            self.to_k_lora = LoRALinearLayer(kv_in, hidden_size, rank)
        if not value_states_skipped:
            self.to_v_lora = LoRALinearLayer(kv_in, hidden_size, rank)
        if not output_states_skipped:
            self.to_out_lora = LoRALinearLayer(hidden_size, hidden_size, rank)
        self.key_states_skipped: bool = key_states_skipped
        self.value_states_skipped: bool = value_states_skipped
        self.output_states_skipped: bool = output_states_skipped

    def skip_key_states(self, is_skipped: bool = True):
        if not is_skipped:
            assert hasattr(self, "to_k_lora")
        self.key_states_skipped = is_skipped

    def skip_value_states(self, is_skipped: bool = True):
        if not is_skipped:
            assert hasattr(self, "to_q_lora")  # sic: models.py:110
        self.value_states_skipped = is_skipped

    def skip_output_states(self, is_skipped: bool = True):
        if not is_skipped:
            assert hasattr(self, "to_out_lora")
        self.output_states_skipped = is_skipped

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, scale=1.0):
        """The call diffusers' CrossAttention.forward makes (models.py:118-152 / 222-287 / 357-431 for the three processor classes;
        which algebra runs is decided by the class and its pre / post chain): one attention layer on the CUDA kernels, inside
        torch autograd."""
        from .eager_attn import call_processor

        return call_processor(self, attn, hidden_states, encoder_hidden_states, attention_mask, scale)


class ControlLoRACrossAttnProcessor(LoRACrossAttnProcessor):
    """models.py:155-287."""

    def __init__(self, hidden_size, cross_attention_dim=None, rank=4, control_rank=None, post_add=False,
                 concat_hidden=False, control_channels=None, control_self_add=True, key_states_skipped=False,
                 value_states_skipped=False, output_states_skipped=False, **kwargs):
        super().__init__(hidden_size, cross_attention_dim, rank, post_add=post_add, key_states_skipped=key_states_skipped,
                         value_states_skipped=value_states_skipped, output_states_skipped=output_states_skipped)
        control_rank = rank if control_rank is None else control_rank
        control_channels = hidden_size if control_channels is None else control_channels
        self.concat_hidden = concat_hidden
        self.control_self_add = control_self_add if control_channels is None else False   # always False (models.py:182)
        self.control_states: Optional[torch.Tensor] = None
        self.to_control = LoRALinearLayer(control_channels + (hidden_size if concat_hidden else 0), hidden_size, control_rank)
        self.pre_loras: List[LoRACrossAttnProcessor] = []
        self.post_loras: List[LoRACrossAttnProcessor] = []

    def inject_pre_lora(self, lora_layer):
        self.pre_loras.append(lora_layer)

    def inject_post_lora(self, lora_layer):
        self.post_loras.append(lora_layer)

    def inject_control_states(self, control_states):
        self.control_states = control_states


class ControlLoRACrossAttnProcessorV2(LoRACrossAttnProcessor):
    """models.py:292-431."""

    def __init__(self, hidden_size, cross_attention_dim=None, rank=4, control_rank=None, control_channels=None, **kwargs):
        super().__init__(hidden_size, cross_attention_dim, rank, post_add=False, key_states_skipped=True,
                         value_states_skipped=True, output_states_skipped=False)
        control_rank = rank if control_rank is None else control_rank
        control_channels = hidden_size if control_channels is None else control_channels
        self.concat_hidden = True
        self.control_self_add = False
        self.control_states: Optional[torch.Tensor] = None
        self.to_control = LoRALinearLayer(hidden_size + control_channels, hidden_size, control_rank)
        self.to_control_out = LoRALinearLayer(hidden_size + control_channels, hidden_size, control_rank)
        self.pre_loras: List[LoRACrossAttnProcessor] = []
        self.post_loras: List[LoRACrossAttnProcessor] = []

    def inject_pre_lora(self, lora_layer):
        self.pre_loras.append(lora_layer)

    def inject_post_lora(self, lora_layer):
        self.post_loras.append(lora_layer)

    def inject_control_states(self, control_states):
        self.control_states = control_states


# ------------------------------------------------------------------------------------------------ hint encoder modules
class ConvBlock2D(nn.Module):
    """Parameter container for models.py:434-547 as configured by ControlLoRA (no temb, no up/down)."""

    def __init__(self, *, in_channels, out_channels=None, conv_kernel_size=3, groups=32, eps=1e-6, **unused):
        super().__init__()
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.groups, self.eps, self.kernel_size = groups, eps, conv_kernel_size
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps, affine=True)
        self.conv1 = nn.Conv2d(in_channels, out_channels, conv_kernel_size, stride=1, padding=conv_kernel_size // 2)
        self.time_emb_proj = None
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps, affine=True)


class _Downsample(nn.Module):
    """diffusers Downsample2D(use_conv=True, padding=0, name='op'): parameters live under `.conv` (models.py:591-598)."""

    def __init__(self, channels, out_channels, padding):
        super().__init__()
        self.padding = padding
        self.conv = nn.Conv2d(channels, out_channels, 3, stride=2, padding=padding)


class SimpleDownEncoderBlock2D(nn.Module):
    """models.py:550-610."""

    def __init__(self, in_channels, out_channels, num_layers=1, convnet_eps=1e-6, convnet_groups=32, convnet_kernel_size=3,
                 add_downsample=True, downsample_padding=1, **unused):
        super().__init__()
        self.convnets = nn.ModuleList([
            ConvBlock2D(in_channels=in_channels if i == 0 else out_channels, out_channels=out_channels,
                        conv_kernel_size=convnet_kernel_size, groups=convnet_groups, eps=convnet_eps)
            for i in range(num_layers)])
        cin = in_channels if num_layers == 0 else out_channels
        self.downsamplers = nn.ModuleList([_Downsample(cin, out_channels, downsample_padding)]) if add_downsample else None


@dataclass
class ControlLoRAOutput:
    control_states: Tuple[torch.Tensor, ...]


_CONFIG_DEFAULTS = dict(
    in_channels=3,
    down_block_types=("SimpleDownEncoderBlock2D",) * 4,
    block_out_channels=(32, 64, 128, 256),
    layers_per_block=1,
    act_fn="silu",
    norm_num_groups=32,
    lora_pre_down_block_types=(None, "SimpleDownEncoderBlock2D", "SimpleDownEncoderBlock2D", "SimpleDownEncoderBlock2D"),
    lora_pre_down_layers_per_block=1,
    lora_pre_conv_skipped=False,
    lora_pre_conv_types=("SimpleDownEncoderBlock2D",) * 4,
    lora_pre_conv_layers_per_block=1,
    lora_pre_conv_layers_kernel_size=1,
    lora_block_in_channels=(256, 256, 256, 256),
    lora_block_out_channels=(320, 640, 1280, 1280),
    lora_cross_attention_dims=([None, 768] * 5, [None, 768] * 5, [None, 768] * 5, [None, 768]),
    lora_rank=4,
    lora_control_rank=None,
    lora_post_add=False,
    lora_concat_hidden=False,
    lora_control_channels=(None, None, None, None),
    lora_control_self_add=True,
    lora_key_states_skipped=False,
    lora_value_states_skipped=False,
    lora_output_states_skipped=False,
    lora_control_version=1,
)


class ControlLoRA(nn.Module):
    """models.py:618-835.  `forward` runs the hint-encoder kernels (controllora_b200/hint_encoder.py) and injects the
    control states into every processor of `lora_layers` as a side effect, exactly like the reference (models.py:828-829)."""

    config_name = "config.json"

    def __init__(self, **kwargs):
        super().__init__()
        cfg = dict(_CONFIG_DEFAULTS)
        unknown = set(kwargs) - set(cfg)
        if unknown:
            raise TypeError(f"ControlLoRA.__init__() got unexpected config keys {sorted(unknown)}")
        cfg.update(kwargs)
        self._config = dict(cfg)
        c = cfg
        if c["act_fn"] not in ("silu", "swish"):
            raise NotImplementedError("only act_fn='silu' is implemented on the CUDA path")
        proc_cls = ControlLoRACrossAttnProcessorV2 if c["lora_control_version"] == 2 else ControlLoRACrossAttnProcessor
        assert c["lora_block_in_channels"][0] == c["block_out_channels"][-1]
        control_channels = c["lora_control_channels"]
        self_add = c["lora_control_self_add"]
        if c["lora_pre_conv_skipped"]:
            control_channels = c["lora_block_in_channels"]
            self_add = False
        self.layers_per_block = c["layers_per_block"]
        self.lora_pre_down_layers_per_block = c["lora_pre_down_layers_per_block"]
        self.lora_pre_conv_layers_per_block = c["lora_pre_conv_layers_per_block"]
        groups, boc = c["norm_num_groups"], c["block_out_channels"]
        self.conv_in = nn.Conv2d(c["in_channels"], boc[0], kernel_size=3, stride=1, padding=1)
        self.down_blocks = nn.ModuleList([])
        self.pre_lora_layers = nn.ModuleList([])
        self.lora_layers = nn.ModuleList([])

        def pre_conv(i, cin):
            if c["lora_pre_conv_skipped"]:
                return nn.Identity()
            cout = c["lora_block_out_channels"][i] if control_channels[i] is None else control_channels[i]
            return SimpleDownEncoderBlock2D(cin, cout, num_layers=c["lora_pre_conv_layers_per_block"], convnet_groups=groups,
                                            convnet_kernel_size=c["lora_pre_conv_layers_kernel_size"], add_downsample=False,
                                            downsample_padding=0)

        def procs(i):
            return nn.ModuleList([
                proc_cls(c["lora_block_out_channels"][i], cross_attention_dim=xd, rank=c["lora_rank"],
                         control_rank=c["lora_control_rank"], post_add=c["lora_post_add"], concat_hidden=c["lora_concat_hidden"],
                         control_channels=control_channels[i], control_self_add=self_add,
                         key_states_skipped=c["lora_key_states_skipped"], value_states_skipped=c["lora_value_states_skipped"],
                         output_states_skipped=c["lora_output_states_skipped"])
                for xd in c["lora_cross_attention_dims"][i]])

        stack, out_ch = [], boc[0]
        for i in range(len(c["down_block_types"])):
            in_ch, out_ch = out_ch, boc[i]
            stack.append(SimpleDownEncoderBlock2D(in_ch, out_ch, num_layers=self.layers_per_block, convnet_groups=groups,
                                                  add_downsample=i != len(boc) - 1, downsample_padding=0))
        self.down_blocks.append(nn.Sequential(*stack))
        self.pre_lora_layers.append(pre_conv(0, c["lora_block_in_channels"][0]))
        self.lora_layers.append(procs(0))
        out_ch = c["lora_block_in_channels"][0]
        for i in range(1, len(c["lora_pre_down_block_types"])):
            in_ch, out_ch = out_ch, c["lora_block_in_channels"][i]
            self.down_blocks.append(SimpleDownEncoderBlock2D(in_ch, out_ch, num_layers=self.lora_pre_down_layers_per_block,
                                                             convnet_groups=groups, add_downsample=True, downsample_padding=0))
            self.pre_lora_layers.append(pre_conv(i, out_ch))
            self.lora_layers.append(procs(i))
        self._engine = None

    # ---------------------------------------------------------------------------------- ConfigMixin / ModelMixin subset
    @property
    def config(self):
        return dict(self._config)

    @classmethod
    def from_config(cls, config, **kwargs):
        """Accepts a dict, a path to a .json file, or a directory containing config.json (the reference passes a path
        string, train_text_to_image_control_lora.py:427)."""
        if isinstance(config, (str, os.PathLike)):
            p = Path(config)
            if p.is_dir():
                p = p / cls.config_name
            config = json.loads(p.read_text())
        cfg = {k: v for k, v in dict(config).items() if not k.startswith("_")}
        cfg.update(kwargs)
        return cls(**cfg)

    def save_config(self, save_directory):
        os.makedirs(save_directory, exist_ok=True)
        out = {"_class_name": "ControlLoRA", "_diffusers_version": "0.13.0.dev0"}
        out.update({k: (list(v) if isinstance(v, tuple) else v) for k, v in self._config.items()})
        with open(os.path.join(save_directory, self.config_name), "w") as f:
            json.dump(out, f, indent=2, sort_keys=True)

    def save_pretrained(self, save_directory, safe_serialization: bool = False, **unused):
        self.save_config(save_directory)
        sd = {k: v.detach().to("cpu").contiguous() for k, v in self.state_dict().items()}
        if safe_serialization:
            from safetensors.torch import save_file

            save_file(sd, os.path.join(save_directory, "diffusion_pytorch_model.safetensors"))
        else:
            torch.save(sd, os.path.join(save_directory, "diffusion_pytorch_model.bin"))

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder: Optional[str] = None, **unused):
        root = Path(pretrained_model_name_or_path)
        if subfolder:
            root = root / subfolder
        if not root.is_dir():
            raise OSError(f"{root} is not a local directory (no network access: hub ids cannot be resolved here)")
        model = cls.from_config(root)
        st = root / "diffusion_pytorch_model.safetensors"
        if st.exists():
            from safetensors.torch import load_file

            sd = load_file(str(st))
        else:
            sd = torch.load(root / "diffusion_pytorch_model.bin", map_location="cpu")
        model.load_state_dict(sd)
        return model

    # ---------------------------------------------------------------------------------- forward
    def forward(self, x: torch.Tensor, return_dict: bool = True):
        from .hint_encoder import hint_encoder_apply

        states = hint_encoder_apply(self, x)
        for procs, cs in zip(self.lora_layers, states):
            for proc in procs:
                proc.inject_control_states(cs)
        if not return_dict:
            return tuple(states)
        return ControlLoRAOutput(control_states=tuple(states))
