"""Execution of the ControlLoRA hint encoder (/root/reference/models.py:810-835: conv_in, the SimpleDownEncoderBlock2D
pyramid, the per-level pre-LoRA 1x1 ConvBlock2D) on the CUDA kernels, forward and backward.  Unlike the UNet these
layers are trainable: the backward also produces dW (wgmma wgrad), dbias, dgamma, dbeta.

Activations are NHWC bf16; parameters stay fp32 nn.Parameters and are re-laid-out to bf16 GEMM operands every step.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import torch

from . import engine as E
from . import ops
from .engine import Ctx, Tape, Var

BF16 = torch.bfloat16


class _ConvP:
    """A trainable conv: fp32 master (nn.Conv2d) + per-step bf16 operands."""

    def __init__(self, conv: torch.nn.Conv2d, grad_of, stride=1, pad_lo=1):
        self.conv = conv
        self.cout, self.cin, self.k, _ = conv.weight.shape
        self.stride, self.pad_lo = stride, pad_lo
        dev = conv.weight.device
        kk = self.k * self.k
        self.wf = torch.empty(self.cout, kk * self.cin, device=dev, dtype=BF16)
        self.wd = torch.empty(self.cin, kk * self.cout, device=dev, dtype=BF16)
        self.gw = grad_of(conv.weight)
        self.gb = grad_of(conv.bias)

    def prep(self):
        ops.conv_weight_prep(self.conv.weight, self.wf, self.wd)


class HintEncoderEngine:
    def __init__(self, model, grad_of: Callable):
        self.model = model
        self.grad_of = grad_of
        cfg = model.config
        self.groups = cfg["norm_num_groups"]
        self.conv_in = model.conv_in
        self.conv_in_w = torch.empty(model.conv_in.weight.shape[0], 9 * model.conv_in.weight.shape[1],
                                     device=model.conv_in.weight.device, dtype=BF16)
        self.convs: List[_ConvP] = []
        self.levels = []          # per level: (list of (block ops)), pre-conv ops
        for down, pre in zip(model.down_blocks, model.pre_lora_layers):
            blocks = list(down) if isinstance(down, torch.nn.Sequential) else [down]
            lvl_ops = []
            for blk in blocks:
                lvl_ops += self._block_ops(blk)
            pre_ops = [] if isinstance(pre, torch.nn.Identity) else self._block_ops(pre)
            self.levels.append((lvl_ops, pre_ops))

    def _block_ops(self, blk):
        out = []
        for cb in blk.convnets:
            c = _ConvP(cb.conv1, self.grad_of, 1, 1)
            self.convs.append(c)
            out.append(("convblock", cb, c))
        if blk.downsamplers is not None:
            for d in blk.downsamplers:
                c = _ConvP(d.conv, self.grad_of, 2, d.padding)
                self.convs.append(c)
                out.append(("down", d, c))
        return out

    # ------------------------------------------------------------------------------------------------ ops
    def _gn(self, ctx: Ctx, x: Var, norm: torch.nn.GroupNorm) -> Var:
        g, b = norm.weight, norm.bias
        y, stats = ops.groupnorm_fwd(x.data, g, b, norm.num_groups, norm.eps, True)
        out = Var(y, rg=True)
        if ctx.tape is not None:
            gg, gb = self.grad_of(g), self.grad_of(b)

            def bwd():
                dy = out.grad
                out.grad = None
                if dy is None:
                    return
                if x.rg:
                    E.give_produce(x, lambda buf, acc: ops.groupnorm_bwd(x.data, dy, g, b, stats, norm.num_groups, True, dx=buf,
                                                                         accumulate=acc, dgamma=gg, dbeta=gb))
                else:
                    scratch = torch.empty_like(x.data)
                    ops.groupnorm_bwd(x.data, dy, g, b, stats, norm.num_groups, True, dx=scratch, dgamma=gg, dbeta=gb)

            ctx.tape.record(bwd)
        return out

    def _conv(self, ctx: Ctx, x: Var, c: _ConvP) -> Var:
        n, H, W, _ = x.data.shape
        if c.k == 3:
            y = ops.gemm(x.data, c.wf, conv_stride=c.stride, pad_lo=c.pad_lo, bias=c.conv.bias)
        else:
            y = ops.gemm(x.data.view(-1, c.cin), c.wf, bias=c.conv.bias).view(n, H, W, c.cout)
        out = Var(y, rg=True)
        if ctx.tape is not None:
            def bwd():
                dy = out.grad
                out.grad = None
                if dy is None:
                    return
                ops.colsum(dy, c.gb)
                ops.conv_wgrad(dy, x.data, c.gw, c.k, c.stride, c.pad_lo)
                if x.rg:
                    if c.k == 3:
                        src = dy if c.stride == 1 else ops.zero_insert2x(dy, 0 if c.pad_lo == 1 else 1)
                        E.give_produce(x, lambda buf, acc: ops.gemm(src, c.wd, conv_stride=1, out=buf, residual=buf if acc else None))
                    else:
                        E.give_produce(x, lambda buf, acc: ops.gemm(dy.view(-1, c.cout), c.wd, out=buf.view(-1, c.cin),
                                                                    residual=buf.view(-1, c.cin) if acc else None))

            ctx.tape.record(bwd)
        return out

    def _run_ops(self, ctx: Ctx, h: Var, oplist) -> Var:
        for kind, mod, c in oplist:
            if kind == "convblock":
                h = self._gn(ctx, h, mod.norm1)
                h = self._conv(ctx, h, c)
                h = self._gn(ctx, h, mod.norm2)
            else:
                h = self._conv(ctx, h, c)
        return h

    # ------------------------------------------------------------------------------------------------ forward
    def forward(self, ctx: Ctx, guide: torch.Tensor) -> List[Var]:
        """guide: NCHW fp32 [B, 3, H, W] -> control states, one NHWC bf16 Var per level."""
        m = self.model
        ci = m.conv_in
        ops.conv_weight_prep(ci.weight, self.conv_in_w, None)
        for c in self.convs:
            c.prep()
        cout = ci.weight.shape[0]
        y = ops.conv_in(guide, self.conv_in_w.view(cout, 3, 3, -1), ci.bias, cout)
        h = Var(y, rg=True)
        if ctx.tape is not None:
            gw, gb = self.grad_of(ci.weight), self.grad_of(ci.bias)
            h_in = h      # `h` is re-bound below; the closure must keep conv_in's own output

            def bwd_in():
                dy = h_in.grad
                h_in.grad = None
                if dy is None:
                    return
                ops.colsum(dy, gb)
                ops.conv_in_wgrad(guide, dy, gw)

            ctx.tape.record(bwd_in)
        states = []
        for lvl_ops, pre_ops in self.levels:
            h = self._run_ops(ctx, h, lvl_ops)
            states.append(self._run_ops(ctx, h, pre_ops) if pre_ops else h)
        return states


class _HintFn(torch.autograd.Function):
    @staticmethod
    def forward(fctx, eng: HintEncoderEngine, store, guide, *params):
        tape = Tape()
        ctx = Ctx(tape=tape)
        states = eng.forward(ctx, guide)
        fctx.tape, fctx.states, fctx.store, fctx.params = tape, states, store, params
        outs = []
        for s in states:
            n, H, W, C = s.data.shape
            outs.append(s.data.permute(0, 3, 1, 2))       # NCHW view of channels-last memory
        return tuple(outs)

    @staticmethod
    def backward(fctx, *gouts):
        for s, g in zip(fctx.states, gouts):
            if g is None:
                continue
            if g.dtype == BF16 and g.permute(0, 2, 3, 1).is_contiguous():
                s.grad = g.permute(0, 2, 3, 1)
            else:
                gx = g if g.dtype in (torch.float32, BF16) else g.float()
                s.grad = ops.nchw_to_nhwc(gx.contiguous())
            s.owned = False
        for p in fctx.params:
            fctx.store.get(p).zero_()
        fctx.tape.backward()
        return (None, None, None, *[fctx.store.get(p).clone() for p in fctx.params])


def hint_encoder_apply(model, x: torch.Tensor):
    """ControlLoRA.forward body: returns the list of control-state tensors (NCHW views, bf16)."""
    from .unet_module import GradStore

    if getattr(model, "_engine", None) is None or model._engine_dev != model.conv_in.weight.device:
        model._store = getattr(model, "_store", None) or GradStore()
        model._engine = HintEncoderEngine(model, model._store.get)
        model._engine_dev = model.conv_in.weight.device
    guide = x.detach()
    if guide.dtype != torch.float32:
        guide = guide.float()
    guide = guide.contiguous()
    params = [p for n, p in model.named_parameters() if not n.startswith("lora_layers.")]
    if torch.is_grad_enabled() and any(p.requires_grad for p in params):
        return list(_HintFn.apply(model._engine, model._store, guide, *params))
    states = model._engine.forward(Ctx(tape=None), guide)
    return [s.data.permute(0, 3, 1, 2) for s in states]
