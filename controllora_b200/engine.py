"""Tape-based execution engine for the UNet hot path.

Every forward op launches sm_90a kernels through the C ABI and (when a tape is active) records a closure that launches
the backward kernels.  Gradients of frozen weights are never computed ("frozen-weight gradient path elided"): the
backward emits only activation gradients (dX), LoRA dA/dB, and gradients w.r.t. the injected control states.

torch is used as the device allocator (torch.empty) and nothing else: no ATen math runs on this path.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Optional

import torch

from . import ops

BF16 = torch.bfloat16


class Var:
    """A device tensor plus its (lazily materialised) gradient."""

    __slots__ = ("data", "grad", "rg", "owned")

    def __init__(self, data: torch.Tensor, rg: bool = False):
        self.data = data
        self.grad: Optional[torch.Tensor] = None
        self.rg = rg
        self.owned = False


def give_tensor(v: Var, g: torch.Tensor) -> None:
    """Accumulate a finished gradient tensor into v (aliasing it when it is the first contribution)."""
    if not v.rg:
        return
    if v.grad is None:
        v.grad, v.owned = g, False
    elif v.owned:
        ops.add(v.grad, g, out=v.grad)
    else:
        v.grad, v.owned = ops.add(v.grad, g), True


def give_produce(v: Var, fn: Callable[[torch.Tensor, bool], None]) -> None:
    """fn(out, accumulate) writes (or adds) this contribution; avoids a separate add kernel where the producer can
    accumulate in its epilogue."""
    if not v.rg:
        return
    if v.grad is None:
        buf = torch.empty_like(v.data)
        fn(buf, False)
        v.grad, v.owned = buf, True
    elif v.owned:
        fn(v.grad, True)
    else:
        buf = torch.empty_like(v.data)
        fn(buf, False)
        v.grad, v.owned = ops.add(v.grad, buf), True


class Tape:
    def __init__(self):
        self.fns: List[Callable[[], None]] = []

    def record(self, fn: Callable[[], None]) -> None:
        self.fns.append(fn)

    def backward(self) -> None:
        while self.fns:
            self.fns.pop()()
        ops.SKINNY.flush()      # batched LoRA dA/dB reductions still queued


# ---------------------------------------------------------------------------------------------------- frozen weights
@dataclass
class LinearW:
    w: torch.Tensor                      # bf16 [N, K]
    bias: Optional[torch.Tensor] = None  # fp32 [N]
    wt: Optional[torch.Tensor] = None    # bf16 [K, N]  (dX operand)

    @staticmethod
    def make(w: torch.Tensor, bias: Optional[torch.Tensor], device, need_dx: bool = True) -> "LinearW":
        w2 = w.reshape(w.shape[0], -1).to(device=device, dtype=BF16).contiguous()
        b = None if bias is None else bias.to(device=device, dtype=BF16).float().contiguous()
        wt = w2.t().contiguous() if need_dx else None
        return LinearW(w2, b, wt)


@dataclass
class ConvW:
    w: torch.Tensor                      # bf16 [Cout, 9*Cin]   k = (ky*3+kx)*Cin + ci
    bias: Optional[torch.Tensor]
    wd: Optional[torch.Tensor] = None    # bf16 [Cin, 9*Cout]   flipped taps, for dX
    cin: int = 0
    cout: int = 0

    @staticmethod
    def make(w: torch.Tensor, bias: Optional[torch.Tensor], device, need_dx: bool = True) -> "ConvW":
        cout, cin = w.shape[0], w.shape[1]
        wb = w.to(device=device, dtype=BF16)
        wf = wb.permute(0, 2, 3, 1).contiguous().view(cout, 9 * cin)
        wd = None
        if need_dx:
            wd = wb.flip(2, 3).permute(1, 2, 3, 0).contiguous().view(cin, 9 * cout)
        b = None if bias is None else bias.to(device=device, dtype=BF16).float().contiguous()
        return ConvW(wf, b, wd, cin, cout)


@dataclass
class NormW:
    gamma: torch.Tensor
    beta: torch.Tensor

    @staticmethod
    def make(g: torch.Tensor, b: torch.Tensor, device) -> "NormW":
        return NormW(g.to(device=device, dtype=BF16).float().contiguous(), b.to(device=device, dtype=BF16).float().contiguous())


# ---------------------------------------------------------------------------------------------------- LoRA slot
@dataclass
class Adapter:
    """One LoRALinearLayer of the chain feeding a projection (models.py:89-97)."""
    down: torch.Tensor            # fp32 parameter [r, K]
    up: torch.Tensor              # fp32 parameter [N, r]
    col: int                      # first column of this adapter inside the slot's rank-rp space
    down_grad: Optional[torch.Tensor] = None   # fp32 accumulators (views into the gradient arena)
    up_grad: Optional[torch.Tensor] = None
    unscaled: bool = False        # the reference adds this adapter's delta WITHOUT `scale` (stacked value adapters,
                                  # models.py:260,265,397,402): its up-table is packed with 1/scale (PackPlan.set_unscaled_mul)


class LoraSlot:
    """All adapters stacked on one frozen projection, packed for the fused GEMM epilogue (fwd) and for the dX GEMM
    (bwd, where `up` plays the role of the rank-r 'down' operand and `down` that of the epilogue table)."""

    def __init__(self, N: int, K: int, device):
        self.N, self.K = N, K
        self.adapters: List[Adapter] = []
        self.rank = 0
        self.device = device
        self.rp = 4
        self.ext = self.up_tab = self.ext_t = self.down_tab = None
        self.post_add = False     # models.py:125,132,135,147: the adapter reads the base projection's OUTPUT (then K == N)

    def add(self, down: torch.Tensor, up: torch.Tensor, unscaled: bool = False) -> Adapter:
        r = down.shape[0]
        # up may cover only the FIRST rows of a fused projection (q of a fused q|k|v weight): the other rows stay zero
        assert down.shape == (r, self.K) and up.shape[1] == r and up.shape[0] <= self.N
        a = Adapter(down, up, self.rank, unscaled=unscaled)
        self.adapters.append(a)
        self.rank += r
        if self.rank > 8:
            raise NotImplementedError("stacked LoRA rank > 8 on one projection is not supported by the fused epilogue")
        return a

    def finalize(self, plan: "ops.PackPlan", need_dx: bool) -> None:
        self.rp = 4 if self.rank <= 4 else 8
        dev = self.device
        self.ext = torch.zeros(16, self.K, device=dev, dtype=BF16)
        self.up_tab = torch.zeros(self.N, self.rp, device=dev, dtype=torch.float32)
        self.ext_t = torch.zeros(16, self.N, device=dev, dtype=BF16)
        self.down_tab = torch.zeros(self.K, self.rp, device=dev, dtype=torch.float32) if need_dx else None
        for a in self.adapters:
            # forward: y += s * t_j (m B_j)^T ; backward: e_j = dy (m B_j), dX += s e_j A_j, dA_j += s e_j^T x, dB_j += s m dy^T t_j
            plan.add_ext(a.down, self.ext, row_off=a.col)
            plan.add_table(a.up, self.up_tab, col_off=a.col, unscaled=a.unscaled)
            plan.add_ext(a.up, self.ext_t, row_off=a.col, transposed=True, unscaled=a.unscaled)
            if need_dx:
                plan.add_table(a.down, self.down_tab, col_off=a.col, transposed=True)


@dataclass
class Ctx:
    tape: Optional[Tape]
    scale: float = 1.0
    stash: dict = field(default_factory=dict)


# ---------------------------------------------------------------------------------------------------- ops
def linear(ctx: Ctx, x: Var, lw: LinearW, *, residual: Optional[Var] = None, slot: Optional[LoraSlot] = None,
           t_add: Optional[torch.Tensor] = None, on_slot_bwd: Optional[Callable] = None, out_shape=None) -> Var:
    """y = x W^T + b (+ residual) (+ scale * (x A^T + t_add) B^T).  x: [..., K] bf16."""
    if slot is not None and slot.rank > 0 and slot.post_add:
        return _linear_post_add(ctx, x, lw, residual, slot, t_add, on_slot_bwd, out_shape)
    K = x.data.shape[-1]
    x2 = x.data.view(-1, K)
    N = lw.w.shape[0]
    t_out = None
    kw = {}
    if slot is not None and slot.rank > 0:
        t_out = torch.empty(x2.shape[0], slot.rp, device=x2.device, dtype=torch.float32)
        kw = dict(ext=slot.ext, lora_up=slot.up_tab, lora_scale=ctx.scale, t_add=t_add, t_out=t_out)
    y = ops.gemm(x2, lw.w, bias=lw.bias, residual=None if residual is None else residual.data.view(-1, N), **kw)
    y = y.view(*(out_shape or (*x.data.shape[:-1], N)))
    trainable = slot is not None and slot.rank > 0
    out = Var(y, rg=x.rg or trainable or (residual is not None and residual.rg))
    if ctx.tape is not None and out.rg:
        scale = ctx.scale
        inv_scale = 1.0 / scale if scale != 0.0 else 0.0

        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            dy2 = dy.view(-1, N)
            if residual is not None:
                give_tensor(residual, dy.view(residual.data.shape))
            e = None
            if x.rg:
                def prod(buf, acc):
                    nonlocal e
                    b2 = buf.view(-1, K)
                    if trainable:
                        e = torch.empty(x2.shape[0], slot.rp, device=x2.device, dtype=torch.float32)
                        ops.gemm(dy2, lw.wt, out=b2, residual=b2 if acc else None, ext=slot.ext_t, lora_up=slot.down_tab,
                                 lora_scale=scale, t_out=e)
                    else:
                        ops.gemm(dy2, lw.wt, out=b2, residual=b2 if acc else None)
                give_produce(x, prod)
            if trainable:
                if e is None:
                    e = ops.rowdot(dy2, slot.up_tab)          # dY * B_up  (no dX GEMM ran)
                for a in slot.adapters:
                    r = a.down.shape[0]
                    # dB[n, j] += s * sum_m dy[m, n] * t[m, j] ; dA[j, k] += s * sum_m e[m, j] * x[m, k]
                    dyu = dy2 if a.up.shape[0] == N else dy2[:, :a.up.shape[0]]     # fused q|k|v weight: the adapter owns the q columns
                    ops.SKINNY.add(t_out[:, a.col:], r, dyu, a.up_grad, 1, r, scale * inv_scale if a.unscaled else scale)
                    ops.SKINNY.add(e[:, a.col:], r, x2, a.down_grad, K, 1, scale)
                if on_slot_bwd is not None:
                    on_slot_bwd(e, t_out, dy2)

        ctx.tape.record(bwd)
    return out


def _linear_post_add(ctx: Ctx, x: Var, lw: LinearW, residual: Optional[Var], slot: LoraSlot, t_add, on_slot_bwd, out_shape) -> Var:
    """post_add LoRA (models.py:125,132,135,147 / :236-238):  y0 = x W^T + b;  t = y0 A^T (+ t_add);  y = y0 + s t B^T (+ res).
    The adapter reads the projection's own output, so its rank-r product needs complete output rows: base GEMM, then the
    same skinny-GEMM + fused rank-4 update kernels as the V2 control injection.  One adapter of rank <= 4 per projection."""
    assert len(slot.adapters) == 1 and slot.rank <= 4 and slot.K == slot.N
    a = slot.adapters[0]
    r = a.down.shape[0]
    K = x.data.shape[-1]
    x2 = x.data.view(-1, K)
    N = lw.w.shape[0]
    scale = ctx.scale
    y0 = ops.gemm(x2, lw.w, bias=lw.bias)                                   # [M, N] bf16
    th16 = ops.gemm(y0, slot.ext, out_fp32=True)                            # hi/lo columns of y0 A^T
    y, t = ops.v2_inject_fwd(y0, th16, t_add, r, slot.up_tab, scale)        # t [M, 8] (cols < r valid), y = y0 + s t B^T
    if residual is not None:
        y = ops.add(y, residual.data.view(-1, N))
    y = y.view(*(out_shape or (*x.data.shape[:-1], N)))
    out = Var(y, rg=True)
    if ctx.tape is not None:
        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            dy2 = dy.contiguous().view(-1, N)
            if residual is not None:
                give_tensor(residual, dy.view(residual.data.shape))
            # dt = dy B (unscaled);  dy0 = dy + s dt A
            dt, dy0 = ops.v2_inject_bwd(dy2, slot.up_tab, slot.down_tab, scale, need_dh=True)
            ops.SKINNY.add(t, r, dy2, a.up_grad, 1, r, scale)               # dB[n, j] += s sum_m dy[m, n] t[m, j]
            ops.SKINNY.add(dt, r, y0, a.down_grad, N, 1, scale)             # dA[j, n] += s sum_m dt[m, j] y0[m, n]
            if x.rg:
                give_produce(x, lambda buf, acc: ops.gemm(dy0, lw.wt, out=buf.view(-1, K), residual=buf.view(-1, K) if acc else None))
            if on_slot_bwd is not None:
                on_slot_bwd(dt, t, dy2)

        ctx.tape.record(bwd)
    return out


def conv3x3(ctx: Ctx, x: Var, cw: ConvW, *, row_bias: Optional[torch.Tensor] = None, residual: Optional[Var] = None,
            stride: int = 1, pad_lo: int = 1) -> Var:
    n, H, W, _ = x.data.shape
    Ho, Wo = H // stride, W // stride
    y = ops.gemm(x.data, cw.w, conv_stride=stride, pad_lo=pad_lo, bias=cw.bias, row_bias=row_bias, rows_per_group=Ho * Wo,
                 residual=None if residual is None else residual.data)
    out = Var(y, rg=x.rg or (residual is not None and residual.rg))
    if ctx.tape is not None and out.rg:
        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            if residual is not None:
                give_tensor(residual, dy)
            if x.rg:
                src = dy if stride == 1 else ops.zero_insert2x(dy, 0 if pad_lo == 1 else 1)
                give_produce(x, lambda buf, acc: ops.gemm(src, cw.wd, conv_stride=1, out=buf, residual=buf if acc else None))

        ctx.tape.record(bwd)
    return out


def groupnorm(ctx: Ctx, x: Var, nw: NormW, groups: int, eps: float, silu: bool) -> Var:
    y, stats = ops.groupnorm_fwd(x.data, nw.gamma, nw.beta, groups, eps, silu)
    out = Var(y, rg=x.rg)
    if ctx.tape is not None and out.rg:
        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            give_produce(x, lambda buf, acc: ops.groupnorm_bwd(x.data, dy, nw.gamma, nw.beta, stats, groups, silu, dx=buf,
                                                               accumulate=acc))

        ctx.tape.record(bwd)
    return out


def layernorm(ctx: Ctx, x: Var, nw: NormW, eps: float = 1e-5) -> Var:
    y, stats = ops.layernorm_fwd(x.data, nw.gamma, nw.beta, eps)
    out = Var(y, rg=x.rg)
    if ctx.tape is not None and out.rg:
        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            give_produce(x, lambda buf, acc: ops.layernorm_bwd(x.data, dy, nw.gamma, stats, dx=buf, accumulate=acc))

        ctx.tape.record(bwd)
    return out


def geglu(ctx: Ctx, p: Var) -> Var:
    y = ops.geglu_fwd(p.data)
    out = Var(y, rg=p.rg)
    if ctx.tape is not None and out.rg:
        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            give_tensor(p, ops.geglu_bwd(p.data, dy))

        ctx.tape.record(bwd)
    return out


def attention(ctx: Ctx, q: Var, k: Var, v: Var, heads: int) -> Var:
    d = q.data.shape[-1] // heads
    scale = d ** -0.5
    need = ctx.tape is not None and (q.rg or k.rg or v.rg)
    o, lse = ops.attention_fwd(q.data, k.data, v.data, heads, scale, need_lse=need)
    out = Var(o, rg=q.rg or k.rg or v.rg)
    if need:
        def bwd():
            do = out.grad
            out.grad = None
            if do is None:
                return
            dq, dk, dv = ops.attention_bwd(q.data, k.data, v.data, o, do, lse, heads, scale, need_dq=q.rg,
                                           need_dkv=(k.rg or v.rg))
            if q.rg:
                give_tensor(q, dq)
            if k.rg:
                give_tensor(k, dk)
            if v.rg:
                give_tensor(v, dv)

        ctx.tape.record(bwd)
    return out


def attention_qkv(ctx: Ctx, qkv: Var, heads: int) -> Var:
    """Self-attention on a fused projection output qkv [B, N, 3C] = [q | k | v] (one GEMM, models.py:231,248,257 as a single
    N = 3C launch): q / k / v are strided views, and the backward writes dq | dk | dv straight into ONE [B, N, 3C] buffer so
    that the projection's dX is one K = 3C GEMM instead of three accumulating ones."""
    B, Nt, C3 = qkv.data.shape
    Cc = C3 // 3
    d = Cc // heads
    scale = d ** -0.5
    q, k, v = qkv.data[..., :Cc], qkv.data[..., Cc:2 * Cc], qkv.data[..., 2 * Cc:]
    need = ctx.tape is not None and qkv.rg
    o, lse = ops.attention_fwd(q, k, v, heads, scale, need_lse=need)
    out = Var(o, rg=qkv.rg)
    if need:
        def bwd():
            do = out.grad
            out.grad = None
            if do is None:
                return
            g = torch.empty_like(qkv.data)
            ops.attention_bwd(q, k, v, o, do, lse, heads, scale, need_dq=True, need_dkv=True,
                              dq=g[..., :Cc], dk=g[..., Cc:2 * Cc], dv=g[..., 2 * Cc:])
            give_tensor(qkv, g)

        ctx.tape.record(bwd)
    return out


def upsample2x(ctx: Ctx, x: Var) -> Var:
    out = Var(ops.upsample2x_fwd(x.data), rg=x.rg)
    if ctx.tape is not None and out.rg:
        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            give_produce(x, lambda buf, acc: ops.upsample2x_bwd(dy, dx=buf, accumulate=acc))

        ctx.tape.record(bwd)
    return out


def concat(ctx: Ctx, a: Var, b: Var) -> Var:
    out = Var(ops.concat_channels(a.data, b.data), rg=a.rg or b.rg)
    if ctx.tape is not None and out.rg:
        Ca, Cb = a.data.shape[-1], b.data.shape[-1]

        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            if a.rg:
                give_produce(a, lambda buf, acc: ops.slice_channels(dy, 0, Ca, dst=buf, accumulate=acc))
            if b.rg:
                give_produce(b, lambda buf, acc: ops.slice_channels(dy, Ca, Cb, dst=buf, accumulate=acc))

        ctx.tape.record(bwd)
    return out
