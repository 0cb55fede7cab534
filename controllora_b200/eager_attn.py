"""Calling a processor the way diffusers does: `processor(attn, hidden_states, encoder_hidden_states, attention_mask, scale)`
(/root/reference/models.py:118-152, 222-287, 357-431 are invoked like this by diffusers' `CrossAttention.forward`).

Inside this package's own `UNet2DConditionModel` the processors are executed as part of the whole-network program and this
entry is never used.  It exists for the other way a reference user can hold these objects: installed on a REAL diffusers UNet
(`unet.set_attn_processor(procs)`), where each attention module calls its processor with its own frozen `to_q / to_k / to_v /
to_out` Linear layers.  One call = one single-layer run of the same runtime (`LoraRuntime.attn_fn`: fused projection + LoRA GEMMs,
flash attention, v1 / V2 control algebra, the general chain path) bridged into torch autograd: gradients reach `hidden_states`,
every adapter / control parameter of the chain and the injected control states.  The frozen projection weights are converted to
the kernels' layouts on the first call per attention module (`refresh_bindings()` after changing them).

Not differentiated: `encoder_hidden_states` of a cross-attention call (the text encoder is frozen in every reference driver);
`attention_mask` must be None (SD-1.5 never passes one, models.py:122)."""
from __future__ import annotations

from collections import OrderedDict
from types import SimpleNamespace
from typing import Dict

import torch

from . import ops
from ._lib import require_cuda
from .engine import Ctx, Tape, Var
from .lora_runtime import LoraRuntime
from .unet import AttnLayer
from .unet_module import GradStore, _control_to_var

BF16 = torch.bfloat16


class _Binding:
    """One (processor, attention module) pair: the module's frozen weights in kernel layout + a one-layer runtime."""

    def __init__(self, proc, attn):
        w = attn.to_q.weight
        require_cuda(w.device, "processor call")
        # the SD-1.5 / SD-2.x flavour of diffusers' CrossAttention only (what the reference runs on): no group norm, no added k/v
        # projections, biased output projection.  upcast_attention / upcast_softmax (set by some SD-2.x UNets) ask for QK^T and
        # the softmax in fp32; the attention kernels always compute QK^T from the bf16 operands with fp32 accumulation and the
        # softmax in fp32, so up-cast modules run unchanged.
        for attr, what in (("group_norm", "group-normalised"), ("added_kv_proj_dim", "added-kv")):
            if getattr(attn, attr, None) is not None:
                raise NotImplementedError(f"controllora_b200 processors: {what} attention modules are outside the SD-1.5 path")
        if attn.to_q.bias is not None or attn.to_out[0].bias is None:
            raise NotImplementedError("controllora_b200 processors: expected to_q/to_k/to_v without bias and a biased to_out[0]")
        sd = {"to_q.weight": attn.to_q.weight.detach(), "to_k.weight": attn.to_k.weight.detach(),
              "to_v.weight": attn.to_v.weight.detach(), "to_out.0.weight": attn.to_out[0].weight.detach(),
              "to_out.0.bias": attn.to_out[0].bias.detach()}
        is_cross = attn.to_k.weight.shape[1] != attn.to_q.weight.shape[1] or getattr(proc, "cross_attention_dim", None) is not None
        self.layer = AttnLayer(sd, "", "attn.processor", w.device, int(attn.heads), is_cross)
        self.layer.processor = proc
        self.weights = SimpleNamespace(attn_layers=OrderedDict([(self.layer.name, self.layer)]))
        self.store = GradStore()
        self.device = w.device
        self.rt = None

    def runtime(self) -> LoraRuntime:
        sig = LoraRuntime.make_signature(self.weights)
        if self.rt is None or self.rt.signature != sig:
            self.rt = LoraRuntime(self.weights, self.device, self.store.get)
        return self.rt


def _chain(proc):
    return [*getattr(proc, "pre_loras", []), proc, *getattr(proc, "post_loras", [])]


def _bindings(proc) -> Dict[int, _Binding]:
    b = proc.__dict__.get("_clb_bindings")
    if b is None:
        b = proc.__dict__["_clb_bindings"] = {}
    return b


def refresh_bindings(proc) -> None:
    """Forget the converted frozen weights (call after changing an attention module's to_q / to_k / to_v / to_out)."""
    proc.__dict__.pop("_clb_bindings", None)


def call_processor(proc, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, scale=1.0):
    if attention_mask is not None:
        raise NotImplementedError("controllora_b200 processors: attention_mask is not supported (SD-1.5 passes None, models.py:122)")
    bind = _bindings(proc).get(id(attn))
    if bind is None:
        bind = _bindings(proc)[id(attn)] = _Binding(proc, attn)
    if bind.layer.is_cross and encoder_hidden_states is None:
        raise ValueError("this processor was built for cross-attention (cross_attention_dim is set) but no encoder_hidden_states were passed")
    ctensors, seen = [], set()
    for m in _chain(proc):
        cs = getattr(m, "control_states", None)
        if torch.is_tensor(cs) and cs.data_ptr() not in seen:
            seen.add(cs.data_ptr())
            ctensors.append(cs)
    params, pseen = [], set()
    for m in _chain(proc):
        for p in m.parameters():
            if id(p) not in pseen:
                pseen.add(id(p))
                params.append(p)
    need_grad = torch.is_grad_enabled() and (hidden_states.requires_grad or any(p.requires_grad for p in params)
                                             or any(c.requires_grad for c in ctensors))
    if not need_grad:
        return _run(bind, hidden_states, encoder_hidden_states, float(scale), ctensors, None)[0].to(hidden_states.dtype)
    out = _AttnFn.apply(bind, hidden_states, encoder_hidden_states, float(scale), len(ctensors), *ctensors, *params)
    return out.to(hidden_states.dtype)


def _bf16(x: torch.Tensor) -> torch.Tensor:
    x = x.detach()
    return (x if x.dtype == BF16 else ops.f32_to_bf16(x.float().contiguous())).contiguous()


def _run(bind: _Binding, hs, ehs, scale, ctensors, tape, hs_rg=False, c_rg=()):
    rt = bind.runtime()
    ctx = Ctx(tape=tape, scale=scale)
    control = {}
    for i, cs in enumerate(ctensors):
        control[cs.data_ptr()] = _control_to_var(cs.detach(), rg=bool(tape is not None and i < len(c_rg) and c_rg[i]))
    from .unet_module import UNet2DConditionModel

    UNet2DConditionModel._match_control_batch(control, hs.shape[0], tape is not None)      # CFG pipelines: control batch 1, UNet batch 2
    rt.begin(ctx, control)
    if tape is not None:
        tape.record(lambda: rt.finish_backward(ctx))
    h = Var(_bf16(hs), rg=hs_rg)
    e = None if ehs is None else Var(_bf16(ehs), rg=False)
    out = rt.attn_fn(ctx, bind.layer, h, e, None)
    return out.data, out, h, control


class _AttnFn(torch.autograd.Function):
    """One attention layer of the tape engine as a torch autograd node."""

    @staticmethod
    def forward(fctx, bind, hs, ehs, scale, n_ctrl, *tensors):
        ctensors, params = tensors[:n_ctrl], tensors[n_ctrl:]
        tape = Tape()
        data, out, h, control = _run(bind, hs, ehs, scale, ctensors, tape, hs_rg=hs.requires_grad,
                                     c_rg=[c.requires_grad for c in ctensors])
        fctx.bind, fctx.tape, fctx.out, fctx.h, fctx.control = bind, tape, out, h, control
        fctx.ctensors, fctx.params, fctx.hs_dtype = ctensors, params, hs.dtype
        return data

    @staticmethod
    def backward(fctx, gout):
        bind = fctx.bind
        bind.store.zero()
        fctx.out.grad = _bf16(gout)
        fctx.tape.backward()
        g_hs = None if fctx.h.grad is None else fctx.h.grad.to(fctx.hs_dtype)
        grads = []
        for cs in fctx.ctensors:
            v = fctx.control[cs.data_ptr()]
            if v.grad is None or not cs.requires_grad:
                grads.append(None)
            elif cs.dim() == 4:
                n, c, hh, ww = cs.shape
                grads.append(ops.nhwc_to_nchw_f32(v.grad.view(n, hh, ww, c)).to(cs.dtype))
            else:
                grads.append(v.grad.to(cs.dtype))
        for p in fctx.params:
            b = bind.store.bufs.get(id(p))
            grads.append(None if (b is None or not p.requires_grad) else b.clone())
        return (None, g_hs, None, None, None, *grads)


# ---------------------------------------------------------------------------------------------------- LoRALinearLayer.forward
class _LoraLinearFn(torch.autograd.Function):
    """diffusers' LoRALinearLayer.forward: up(down(x)) in fp32 rank space (hi/lo skinny GEMM + rank-8 update passes)."""

    @staticmethod
    def forward(fctx, layer, x, down, up):
        from .lora_generic import GAdapter

        require_cuda(x.device, "LoRALinearLayer")
        store = GradStore()
        plan = ops.PackPlan(x.device)
        ad = GAdapter(down, up, plan, store.get, x.device)
        plan.run()
        K = x.shape[-1]
        x2 = _bf16(x).view(-1, K)
        t = ad.project(x2)
        y = ad.update(torch.zeros(x2.shape[0], ad.N, device=x.device, dtype=BF16), t, 1.0)
        fctx.ad, fctx.store, fctx.x2, fctx.t, fctx.shape, fctx.dt_in = ad, store, x2, t, x.shape, x.dtype
        fctx.need_x = x.requires_grad
        return y.view(*x.shape[:-1], ad.N).to(x.dtype)

    @staticmethod
    def backward(fctx, gout):
        ad = fctx.ad
        dy2 = _bf16(gout).view(-1, ad.N)
        dt = ad.dt(dy2)
        ad.grads(fctx.t, dt, dy2, fctx.x2, 1.0)
        ops.SKINNY.flush()
        gx = ad.back_input(dt, 1.0).view(fctx.shape).to(fctx.dt_in) if fctx.need_x else None
        return None, gx, fctx.store.get(ad.down_full).clone(), fctx.store.get(ad.up).clone()


def lora_linear_forward(layer, x):
    return _LoraLinearFn.apply(layer, x, layer.down.weight, layer.up.weight)
