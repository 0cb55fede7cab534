"""Imports the REAL /root/reference/models.py in this container so that the oracle restatement (oracle/models_ref.py) can be pinned
to the reference's own code and golden vectors can be generated from it (tests/golden/make_reference_golden.py).

`models.py` imports ten names from `diffusers` (models.py:7-12), which is not installed and not installable offline.  Everything
the hot path cites - the three processor classes, ConvBlock2D, SimpleDownEncoderBlock2D, ControlLoRA and its wiring - is the
reference's own code and runs unmodified.  Only the diffusers names are stood in for, inside a throw-away module tree that exists
while the file is being imported:
  * two small classes restated from diffusers 0.13 (`LoRALinearLayer`: down / up Linear without bias, N(0, 1/rank) / zeros init,
    fp32 side path; `Downsample2D(use_conv=True)`: 3x3 stride-2 conv, with F.pad(x, (0, 1, 0, 1)) when padding == 0);
  * base classes with no arithmetic (`ModelMixin` = nn.Module, `ConfigMixin`, `register_to_config`, `BaseOutput`);
  * names that the ControlLoRA configs never reach (`get_down_block` for non-"Simple" block types, `Upsample2D`, `upsample_2d`,
    `downsample_2d`, `Mish`), which raise if they ever are;
  * `CrossAttention` (a type annotation in models.py: the attention module is passed INTO a processor call by the caller).
Test infrastructure: used in this container only (the reference tree does not travel to the GPU box)."""
import functools
import importlib.util
import sys
import types
from pathlib import Path

import torch.nn as nn
import torch.nn.functional as F

REFERENCE_ROOT = Path("/root/reference")


def available() -> bool:
    try:
        return (REFERENCE_ROOT / "models.py").is_file()
    except OSError:        # e.g. a parent directory this user may not enter
        return False


class LoRALinearLayer(nn.Module):
    """diffusers 0.13 models/cross_attention.py"""

    def __init__(self, in_features, out_features, rank=4):
        super().__init__()
        if rank > min(in_features, out_features):
            raise ValueError(f"LoRA rank {rank} must be less or equal than {min(in_features, out_features)}")
        self.down = nn.Linear(in_features, rank, bias=False)
        self.up = nn.Linear(rank, out_features, bias=False)
        nn.init.normal_(self.down.weight, std=1 / rank)
        nn.init.zeros_(self.up.weight)

    def forward(self, hidden_states):
        orig_dtype = hidden_states.dtype
        dtype = self.down.weight.dtype
        return self.up(self.down(hidden_states.to(dtype))).to(orig_dtype)


class Downsample2D(nn.Module):
    """diffusers 0.13 models/resnet.py (the use_conv=True branch ControlLoRA uses; name="op" -> attribute `conv`)"""

    def __init__(self, channels, use_conv=False, out_channels=None, padding=1, name="conv"):
        super().__init__()
        if not use_conv:
            raise NotImplementedError("stand-in covers Downsample2D(use_conv=True) only")
        self.channels, self.out_channels, self.use_conv, self.padding, self.name = channels, out_channels or channels, use_conv, padding, name
        self.conv = nn.Conv2d(self.channels, self.out_channels, 3, stride=2, padding=padding)

    def forward(self, hidden_states):
        assert hidden_states.shape[1] == self.channels
        if self.use_conv and self.padding == 0:
            hidden_states = F.pad(hidden_states, (0, 1, 0, 1), mode="constant", value=0)
        return self.conv(hidden_states)


def _unreached(name):
    def f(*a, **k):
        raise NotImplementedError(f"diffusers.{name} is outside the ControlLoRA path and has no stand-in")
    return f


class _Unreached(nn.Module):
    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError("this diffusers class is outside the ControlLoRA path and has no stand-in")


def _register_to_config(init):
    @functools.wraps(init)
    def wrapped(self, *args, **kwargs):
        import inspect

        bound = inspect.signature(init).bind(self, *args, **kwargs)
        bound.apply_defaults()
        cfg = {k: v for k, v in bound.arguments.items() if k != "self"}
        init(self, *args, **kwargs)
        self.config = types.SimpleNamespace(**cfg)
    return wrapped


def _stub_tree():
    mods = {}

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        mods[name] = m
        return m

    mod("diffusers")
    mod("diffusers.utils")
    mod("diffusers.utils.outputs", BaseOutput=type("BaseOutput", (), {}))
    mod("diffusers.configuration_utils", ConfigMixin=type("ConfigMixin", (), {}), register_to_config=_register_to_config)
    mod("diffusers.models")
    mod("diffusers.models.modeling_utils", ModelMixin=type("ModelMixin", (nn.Module,), {}))
    mod("diffusers.models.unet_2d_blocks", get_down_block=_unreached("get_down_block"))
    mod("diffusers.models.resnet", Mish=_Unreached, Upsample2D=_Unreached, Downsample2D=Downsample2D, upsample_2d=_unreached("upsample_2d"),
        downsample_2d=_unreached("downsample_2d"), partial=functools.partial)
    mod("diffusers.models.cross_attention", CrossAttention=type("CrossAttention", (nn.Module,), {}), LoRALinearLayer=LoRALinearLayer)
    return mods


_CACHED = None


def reference_models():
    """The module object of /root/reference/models.py (imported once)."""
    global _CACHED
    if _CACHED is not None:
        return _CACHED
    if not available():
        raise FileNotFoundError("/root/reference/models.py is not present on this machine")
    stubs = _stub_tree()
    saved = {k: sys.modules.get(k) for k in stubs}
    sys.modules.update(stubs)
    try:
        spec = importlib.util.spec_from_file_location("reference_models_py", str(REFERENCE_ROOT / "models.py"))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    _CACHED = m
    return m


def reference_config(name: str) -> dict:
    """kwargs of ControlLoRA(...) from /root/reference/configs/<name>.json (private `_keys` dropped, like ConfigMixin.from_config)."""
    import json

    raw = json.loads((REFERENCE_ROOT / "configs" / f"{name}.json").read_text())
    return {k: v for k, v in raw.items() if not k.startswith("_")}
