"""`UNet2DConditionModel` — the slice of diffusers' UNet surface that the reference drivers touch
(train_text_to_image_control_lora.py:407-487,782; apps/gradio_canny2image.py:36-63; mix_lora_and_control_lora.py:82-151):
`.config.block_out_channels / .cross_attention_dim`, `.attn_processors`, `.set_attn_processor(dict)`, `.requires_grad_`,
`.to`, `.train/.eval`, and `__call__(sample, timestep, encoder_hidden_states).sample` — participating in torch autograd so
`accelerator.backward(loss)` delivers gradients to the ControlLoRA parameters and to the hint encoder.
"""
from __future__ import annotations

from collections import OrderedDict
from types import SimpleNamespace
from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import engine as E
from . import ops
from .engine import Ctx, Tape, Var
from .lora_runtime import LoraRuntime
from .unet import UNetWeights, conv_out_fwd, synthetic_state_dict, unet_forward

BF16 = torch.bfloat16


class GradStore:
    """fp32 gradient accumulators of the trainable parameters.  Default: one lazily allocated buffer per parameter;
    the Trainer swaps in views of its flat gradient arena."""

    def __init__(self):
        self.bufs: Dict[int, torch.Tensor] = {}
        self.params: Dict[int, torch.Tensor] = {}

    def get(self, p: torch.Tensor) -> torch.Tensor:
        b = self.bufs.get(id(p))
        if b is None:
            b = torch.zeros(p.shape, device=p.device, dtype=torch.float32)
            self.bufs[id(p)] = b
            self.params[id(p)] = p
        return b

    def zero(self):
        for b in self.bufs.values():
            b.zero_()


class _DefaultProcessor:
    """Placeholder for attention layers without a LoRA processor (diffusers' plain CrossAttnProcessor)."""


def _control_to_var(cs: torch.Tensor, rg: bool) -> Var:
    """Processor control state (reference layout: NCHW, any float dtype; or already [B, HW, C]) -> NHWC bf16 Var."""
    if cs.dim() == 4:
        n, c, h, w = cs.shape
        if cs.dtype == BF16 and cs.permute(0, 2, 3, 1).is_contiguous():
            data = cs.permute(0, 2, 3, 1).reshape(n, h * w, c)         # channels-last memory: free view
        else:
            x = cs if cs.dtype in (torch.float32, BF16) else cs.float()
            data = ops.nchw_to_nhwc(x.contiguous()).view(n, h * w, c)
    else:
        data = cs if cs.dtype == BF16 else ops.f32_to_bf16(cs.float().contiguous())
    return Var(data, rg=rg)


def _refuse_unbuilt_options(raw: dict) -> None:
    """config.json values that change the UNet's arithmetic and that this package does not build (the SD-2 depth, inpainting and
    upscaler UNets, class-conditioned UNets): refused by name instead of silently ignored."""
    def bad(key, ok):
        if key in raw and not ok(raw[key]):
            raise NotImplementedError(f"UNet2DConditionModel.from_pretrained: config.json {key} = {raw[key]!r} is not implemented")

    bad("class_embed_type", lambda v: v is None)
    bad("num_class_embeds", lambda v: v is None)
    bad("only_cross_attention", lambda v: not (any(v) if isinstance(v, (list, tuple)) else v))
    bad("dual_cross_attention", lambda v: not v)
    bad("resnet_time_scale_shift", lambda v: v == "default")
    bad("in_channels", lambda v: v == 4)


class UNet2DConditionModel(nn.Module):
    def __init__(self, weights: UNetWeights):
        super().__init__()
        self.weights = weights
        self.device_ = weights.conv_out_w.device
        cfg = weights.cfg
        self.config = SimpleNamespace(**cfg)
        self._procs: "OrderedDict[str, object]" = OrderedDict((k, _DefaultProcessor()) for k in weights.attn_layers)
        self._proc_modules = nn.ModuleDict()
        self._runtime: Optional[LoraRuntime] = None
        self.grad_store = GradStore()

    # ------------------------------------------------------------------------------------------------ construction
    @classmethod
    def from_state_dict(cls, sd: Dict[str, torch.Tensor], device="cuda", config: Optional[dict] = None):
        return cls(UNetWeights(sd, torch.device(device), config))

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder: Optional[str] = None, device="cuda", **unused):
        """Load a diffusers-format UNet directory (`<root>[/subfolder]/config.json` +
        `diffusion_pytorch_model.safetensors` or `.bin`), the layout `UNet2DConditionModel.from_pretrained(...,
        subfolder="unet")` reads at train_text_to_image_control_lora.py:407-409.  Local directories only (no hub access)."""
        import json
        import os

        root = os.path.join(pretrained_model_name_or_path, subfolder) if subfolder else str(pretrained_model_name_or_path)
        if not os.path.isdir(root):
            raise FileNotFoundError(f"{root}: not a local directory (hub download is not available)")
        config = None
        cfg_path = os.path.join(root, "config.json")
        if os.path.isfile(cfg_path):
            with open(cfg_path) as f:
                raw = json.load(f)
            _refuse_unbuilt_options(raw)
            keep = ("block_out_channels", "layers_per_block", "cross_attention_dim", "attention_head_dim", "in_channels",
                    "out_channels", "norm_num_groups", "norm_eps")
            config = {k: (tuple(v) if isinstance(v, list) else v) for k, v in raw.items() if k in keep}
            # SD-2.x switches; kept only when set, so an SD-1.5 config.json loads to the same config as without them
            config.update({k: True for k in ("use_linear_projection", "upcast_attention") if raw.get(k)})
        st = os.path.join(root, "diffusion_pytorch_model.safetensors")
        if os.path.isfile(st):
            from safetensors.torch import load_file

            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(root, "diffusion_pytorch_model.bin"), map_location="cpu")
        return cls.from_state_dict(sd, device, config)

    @classmethod
    def synthetic(cls, device="cuda", config: Optional[dict] = None, seed: int = 0):
        return cls.from_state_dict(synthetic_state_dict(config, seed), device, config)

    # ------------------------------------------------------------------------------------------------ processors
    @property
    def attn_processors(self) -> Dict[str, object]:
        return OrderedDict(self._procs)

    def set_attn_processor(self, processor):
        names = list(self.weights.attn_layers.keys())
        if isinstance(processor, dict):
            if len(processor) != len(names):
                raise ValueError(f"A dict of processors was passed, but the number of processors {len(processor)} does not "
                                 f"match the number of attention layers: {len(names)}. Please make sure to pass {len(names)} "
                                 f"processor classes.")
            mapping = processor
        else:
            mapping = {n: processor for n in names}
        for n in names:
            p = mapping[n]
            self._procs[n] = p
            self.weights.attn_layers[n].processor = p if hasattr(p, "to_q_lora") else None
            key = n.replace(".", "_")
            if isinstance(p, nn.Module):
                self._proc_modules[key] = p      # shared ownership with ControlLoRA.lora_layers, like diffusers
            elif key in self._proc_modules:
                del self._proc_modules[key]
        self._runtime = None

    # diffusers' UNet2DConditionLoadersMixin surface used by train_dreambooth_lora.py:944 (`unet.save_attn_procs(output_dir)`) and
    # test_dreambooth_lora.py / apps (`pipe.unet.load_attn_procs(path)`): one state dict "<attn_processors key>.<parameter name>"
    def attn_procs_state_dict(self) -> Dict[str, torch.Tensor]:
        return {f"{k}.{n}": p.detach() for k, proc in self._procs.items() if isinstance(proc, nn.Module) for n, p in proc.named_parameters()}

    def save_attn_procs(self, save_directory, weight_name: str = "pytorch_lora_weights.bin") -> str:
        import os

        os.makedirs(str(save_directory), exist_ok=True)
        path = os.path.join(str(save_directory), weight_name)
        torch.save({k: v.cpu().clone() for k, v in self.attn_procs_state_dict().items()}, path)
        return path

    def load_attn_procs(self, pretrained_model_name_or_path_or_dict, weight_name: str = "pytorch_lora_weights.bin", **unused) -> None:
        """Builds a `LoRACrossAttnProcessor` per attention layer from the file's shapes (rank, cross-attention width) and installs
        them - diffusers' behaviour for a LoRA attention-processor file."""
        import os
        from .models import LoRACrossAttnProcessor

        sd = pretrained_model_name_or_path_or_dict
        if not isinstance(sd, dict):
            f = str(sd) if os.path.isfile(str(sd)) else os.path.join(str(sd), weight_name)
            if f.endswith(".safetensors"):
                from safetensors.torch import load_file

                sd = load_file(f)
            else:
                sd = torch.load(f, map_location="cpu")
        groups: Dict[str, Dict[str, torch.Tensor]] = {}
        for k, v in sd.items():
            key, sub = ".".join(k.split(".")[:-3]), ".".join(k.split(".")[-3:])        # "...attn1.processor" + "to_q_lora.down.weight"
            groups.setdefault(key, {})[sub] = v
        names = list(self.weights.attn_layers.keys())
        if set(groups) != set(names):
            raise ValueError(f"load_attn_procs: file covers {len(groups)} attention processors, this UNet has {len(names)}")
        procs = {}
        for n in names:
            g = groups[n]
            rank, hidden = g["to_q_lora.down.weight"].shape
            has_k = "to_k_lora.down.weight" in g
            xd = g["to_k_lora.down.weight"].shape[1] if has_k else None
            p = LoRACrossAttnProcessor(hidden, None if (xd is None or n.endswith("attn1.processor")) else xd, rank=rank,
                                       key_states_skipped=not has_k, value_states_skipped="to_v_lora.down.weight" not in g,
                                       output_states_skipped="to_out_lora.down.weight" not in g)
            p.load_state_dict(g)
            procs[n] = p.to(self.device_)
        self.set_attn_processor(procs)

    def _get_runtime(self) -> LoraRuntime:
        sig = LoraRuntime.make_signature(self.weights)
        if self._runtime is None or self._runtime.signature != sig:
            self._runtime = LoraRuntime(self.weights, self.device_, self.grad_store.get)
        return self._runtime

    def trainable_parameters(self) -> List[torch.nn.Parameter]:
        seen, out = set(), []
        for p in self._procs.values():
            if isinstance(p, nn.Module):
                chain = [*getattr(p, "pre_loras", []), p, *getattr(p, "post_loras", [])]
                for m in chain:
                    for q in m.parameters():
                        if id(q) not in seen:
                            seen.add(id(q))
                            out.append(q)
        return out

    # ------------------------------------------------------------------------------------------------ engine entry
    def prepare_inference(self, scale: float = 1.0) -> Ctx:
        """Timestep-invariant part of a forward, run ONCE per denoise loop (SURVEY f2): LoRA operand packing, the per-level
        control products u = Ac c, the v1 `t_add` tables, and (filled lazily on the first evaluation) the k / v
        projections of the text states.  The returned Ctx is passed to `run_engine(..., prepared=ctx)` for every step;
        the injected control states and `encoder_hidden_states` must stay the same tensors for its lifetime."""
        rt = self._get_runtime()
        ctx = Ctx(tape=None, scale=scale)
        control, _ = self.collect_control(False)
        rt.begin(ctx, control)
        ctx.stash["kv_cache"] = {}
        return ctx

    def run_engine(self, sample: torch.Tensor, timesteps: torch.Tensor, ehs: torch.Tensor, control: Dict[int, Var],
                   tape: Optional[Tape], scale: float = 1.0, prepared: Optional[Ctx] = None):
        """Low-level entry (also used by the fused Trainer): returns (pred Var [B,4,H,W] fp32, ctx, runtime)."""
        rt = self._get_runtime()
        if prepared is not None:
            assert tape is None, "a prepared (inference) context carries no tape"
            ctx = prepared
        else:
            ctx = Ctx(tape=tape, scale=scale)
            rt.begin(ctx, control)
        if tape is not None:
            # recorded before any UNet op => runs after all of them in the backward sweep
            tape.record(lambda: rt.finish_backward(ctx))
        ehs_var = Var(ehs, rg=False)
        h = unet_forward(ctx, self.weights, sample, timesteps, ehs_var, rt.attn_fn)
        pred = conv_out_fwd(ctx, self.weights, h)
        return pred, ctx, rt

    def collect_control(self, need_grad: bool):
        """Group the processors' injected control states by tensor; returns ({data_ptr: Var}, [tensors])."""
        control: Dict[int, Var] = {}
        tensors: List[torch.Tensor] = []
        for p in self._procs.values():
            # stacked ControlLoRA processors (pre / post LoRAs, models.py:234-236, 366-372) carry their own control states
            for m in [*getattr(p, "pre_loras", []), p, *getattr(p, "post_loras", [])]:
                cs = getattr(m, "control_states", None)
                if cs is None or not torch.is_tensor(cs):
                    continue
                if cs.data_ptr() not in control:
                    control[cs.data_ptr()] = _control_to_var(cs.detach(), rg=need_grad and cs.requires_grad)
                    tensors.append(cs)
        return control, tensors

    @staticmethod
    def _match_control_batch(control: Dict[int, Var], batch: int, need_grad: bool) -> None:
        """Control states injected with a smaller batch than the UNet call (the pipelines run classifier-free guidance with UNet batch
        2 while `control_lora(guide)` saw batch 1: apps/gradio_*2image.py:75-89, mix_lora_and_control_lora.py:163-164).  The reference
        broadcasts them (v1, models.py:236-238: only defined for control batch 1) or repeats each sample b2 // b1 times in place
        (concat_hidden / V2, models.py:209-212, 344-347); both are `repeat_interleave` along the batch, done here once per call as a copy
        at the boundary (inference only - a training step always injects the UNet's own batch)."""
        for key, v in control.items():
            b1 = v.data.shape[0]
            if b1 == batch:
                continue
            if batch % b1 != 0:
                raise ValueError(f"control states with batch {b1} cannot be matched to a UNet batch of {batch}")
            if need_grad and v.rg:
                raise NotImplementedError("differentiating through control states that are repeated along the batch is not supported: "
                                          "inject control states with the UNet's batch size (control_lora(guide) on the same batch)")
            control[key] = Var(v.data.repeat_interleave(batch // b1, dim=0).contiguous(), rg=False)

    @staticmethod
    def _prep_inputs(sample, timestep, encoder_hidden_states):
        dev = sample.device
        from ._lib import require_cuda

        require_cuda(sample.device, "UNet2DConditionModel")
        x = sample.detach()
        if x.dtype != torch.float32:
            x = x.float()
        x = x.contiguous()
        B = x.shape[0]
        t = timestep
        if not torch.is_tensor(t):
            t = torch.tensor([float(t)], device=dev)
        t = t.to(device=dev, dtype=torch.float32).reshape(-1)
        if t.numel() == 1 and B > 1:
            t = t.expand(B)
        t = t.contiguous()
        e = encoder_hidden_states.detach()
        e = (e if e.dtype == BF16 else ops.f32_to_bf16(e.float().contiguous())).contiguous()
        return x, t, e

    def forward(self, sample, timestep, encoder_hidden_states, cross_attention_kwargs=None, return_dict=True, **unused):
        scale = float((cross_attention_kwargs or {}).get("scale", 1.0))
        x, t, e = self._prep_inputs(sample, timestep, encoder_hidden_states)
        params = [p for p in self.trainable_parameters() if p.requires_grad]
        need_grad = torch.is_grad_enabled() and (len(params) > 0)
        control, ctensors = self.collect_control(need_grad)
        self._match_control_batch(control, x.shape[0], need_grad)
        if not need_grad:
            pred, _, _ = self.run_engine(x, t, e, control, tape=None, scale=scale)
            out = pred.data
        else:
            out = _UNetFn.apply(self, x, t, e, control, scale, len(ctensors), *ctensors, *params)
        if not return_dict:
            return (out,)
        return SimpleNamespace(sample=out)


class _UNetFn(torch.autograd.Function):
    """Bridges the tape engine into torch autograd: one node for the whole UNet."""

    @staticmethod
    def forward(fctx, unet: UNet2DConditionModel, x, t, e, control, scale, n_ctrl, *tensors):
        tape = Tape()
        pred, ctx, rt = unet.run_engine(x, t, e, control, tape, scale)
        fctx.unet, fctx.tape, fctx.ctx, fctx.rt, fctx.pred = unet, tape, ctx, rt, pred
        fctx.control = control
        fctx.ctensors = tensors[:n_ctrl]
        fctx.params = tensors[n_ctrl:]
        return pred.data

    @staticmethod
    def backward(fctx, gout):
        unet, rt = fctx.unet, fctx.rt
        store = unet.grad_store
        store.zero()
        fctx.pred.grad = gout.contiguous().float()
        fctx.tape.backward()
        grads = []
        for cs in fctx.ctensors:
            v = fctx.control[cs.data_ptr()]
            if v.grad is None or not cs.requires_grad:
                grads.append(None)
                continue
            if cs.dim() == 4:
                n, c, h, w = cs.shape
                g = ops.nhwc_to_nchw_f32(v.grad.view(n, h, w, c)).to(cs.dtype)
            else:
                g = v.grad.to(cs.dtype)
            grads.append(g)
        for p in fctx.params:
            b = store.bufs.get(id(p))
            grads.append(None if b is None else b.clone())
        return (None, None, None, None, None, None, None, *grads)
