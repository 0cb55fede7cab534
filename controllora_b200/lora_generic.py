"""General adapter chains: every wiring of /root/reference/models.py:118-431 that the fused one-launch path (lora_runtime.py) does
not cover, executed adapter by adapter in the reference's own order.

The fused path packs a projection and all of its LoRA deltas into ONE wgmma GEMM, which needs every adapter to read the
projection's INPUT and the ranks to sum to <= 8.  The reference allows more (models.py:232-243, 248-265, 275-282, 366-426):

  * `post_add` adapters inside a stacked chain: adapter i reads the running projection output, i.e. the sum of the base
    projection and of all EARLIER deltas (`query if pre_lora.post_add else hidden_states`);
  * any rank (one adapter > 8, or a chain whose ranks sum to > 8), any control rank on a v1 / V2 processor;
  * a ControlLoRA processor stacked as another's pre / post LoRA (its own control states enter ITS q adapter, models.py:234-236 /
    240-242; stacked V2 processors rewrite the hidden states one after the other, models.py:366-372, 412-418);
  * `concat_hidden` control combined with stacked adapters / `post_add` / a q rank > 4.

Here a projection is: base GEMM, then per adapter (in chain order) a skinny hi/lo GEMM `t = in A^T` (N = 16 per 8 ranks: ~fp32 accuracy
like the reference's fp32 LoRALinearLayer) and a rank-8 update pass `y += a t B^T`; the backward walks the chain in reverse with
`dt = dy B`, the two rank-r reductions (dA, dB) and `d in += a dt A`.  These are the kernels the fused path already uses for its own
side products (cl_gemm with the `ext` operand as B, cl_hilo_combine, cl_rank_update, cl_rowdot, cl_skinny_atb_batch, cl_rowmat):
more launches and more passes over the activations than the fused path - it is the compatibility path, chosen per attention layer
only when the fused one cannot express the wiring.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, List, Optional

import torch

from . import engine as E
from . import ops
from .engine import Ctx, Var

BF16 = torch.bfloat16
DENSE_RANK = 16          # control MLPs wider than this run as dense bf16 GEMMs (like the danbooru-sketch path), not as hi/lo blocks


def _is_v1(p) -> bool:
    return type(p).__name__ == "ControlLoRACrossAttnProcessor"


def _is_v2(p) -> bool:
    return type(p).__name__ == "ControlLoRACrossAttnProcessorV2"


class GAdapter:
    """One LoRALinearLayer (models.py:89-97: down [r, K], up [N, r], fp32 masters) packed in blocks of 8 ranks:
    ext [16*nb, K] bf16 (hi / lo rows of `down`), up_tab[b] [N, 8] and down_tab[b] [K, 8] fp32 (zero padded)."""

    def __init__(self, down: torch.Tensor, up: torch.Tensor, plan: "ops.PackPlan", grad_of: Callable, device, col_lo: int = 0,
                 col_hi: Optional[int] = None):
        # [col_lo, col_hi) selects the input columns of `down` this adapter reads (the h / c halves of a concat_hidden layer)
        col_hi = down.shape[1] if col_hi is None else col_hi
        self.down_full, self.up = down, up
        self.col_lo = col_lo
        self.r = r = down.shape[0]
        self.K, self.N = col_hi - col_lo, up.shape[0]
        self.nb = nb = (r + 7) // 8
        self.ext = torch.zeros(16 * nb, self.K, device=device, dtype=BF16)
        self.up_tab = [torch.zeros(self.N, 8, device=device, dtype=torch.float32) for _ in range(nb)]
        self.down_tab = [torch.zeros(self.K, 8, device=device, dtype=torch.float32) for _ in range(nb)]
        dn = down[:, col_lo:col_hi]
        for b in range(nb):
            rb = min(8, r - 8 * b)
            plan.add_ext(dn[8 * b:8 * b + rb], self.ext[16 * b:16 * b + 16])
            plan.add_table(up[:, 8 * b:8 * b + rb], self.up_tab[b])
            plan.add_table(dn[8 * b:8 * b + rb], self.down_tab[b], transposed=True)
        self.down_grad = grad_of(down)      # fp32 [r, K_full] accumulators (views into the gradient arena)
        self.up_grad = grad_of(up)

    def rb(self, b: int) -> int:
        return min(8, self.r - 8 * b)

    def project(self, x2: torch.Tensor) -> torch.Tensor:
        """t [M, 8*nb] fp32 = x2 A^T (columns >= r are zero)."""
        return ops.hilo_combine(ops.gemm(x2, self.ext, out_fp32=True), self.nb)

    def update(self, y: torch.Tensor, t: torch.Tensor, alpha: float) -> torch.Tensor:
        """y + alpha * t B^T (a new tensor: earlier values of y are inputs of other adapters' backward)."""
        for b in range(self.nb):
            y = ops.rank_update(y, t[:, 8 * b:], self.up_tab[b], alpha)
        return y

    def dt(self, dy2: torch.Tensor) -> torch.Tensor:
        """dy B  [M, 8*nb] (unscaled)."""
        if self.nb == 1:
            return ops.rowdot(dy2, self.up_tab[0])
        out = torch.empty(dy2.shape[0], 8 * self.nb, device=dy2.device, dtype=torch.float32)
        eye = _eye8(dy2.device)
        for b in range(self.nb):
            ops.rowmat(ops.rowdot(dy2, self.up_tab[b]), eye, 8, 1, 8, 8, 1.0, out[:, 8 * b:], 8 * self.nb)
        return out

    def grads(self, t: torch.Tensor, dt: torch.Tensor, dy2: torch.Tensor, x2: torch.Tensor, alpha: float) -> None:
        """dB[n, j] += alpha sum_m dy[m, n] t[m, j];  dA[j, k] += alpha sum_m dt[m, j] x[m, k]."""
        Kf = self.down_full.shape[1]
        for b in range(self.nb):
            rb = self.rb(b)
            ops.SKINNY.add(t[:, 8 * b:], rb, dy2, self.up_grad[:, 8 * b:], 1, self.r, alpha)
            ops.SKINNY.add(dt[:, 8 * b:], rb, x2, self.down_grad[8 * b:, self.col_lo:], Kf, 1, alpha)

    def back_input(self, dt: torch.Tensor, alpha: float, base: Optional[torch.Tensor] = None) -> torch.Tensor:
        """(base or 0) + alpha * dt A   (bf16 [M, K], a new tensor: `base` is never written)."""
        cur, ours = base, False
        if cur is None:
            cur, ours = torch.zeros(dt.shape[0], self.K, device=dt.device, dtype=BF16), True
        for b in range(self.nb):
            cur = ops.rank_update(cur, dt[:, 8 * b:], self.down_tab[b], alpha, out=cur if ours else None)
            ours = True
        return cur


_EYE = {}


def _eye8(device) -> torch.Tensor:
    e = _EYE.get(device)
    if e is None:
        e = _EYE[device] = torch.eye(8, device=device, dtype=torch.float32)
    return e


@dataclass
class Entry:
    """One adapter application inside a projection's chain."""
    ad: GAdapter
    post_add: bool                 # reads the running output instead of the projection's input
    alpha: float                   # `scale`, or 1.0 for the reference's unscaled stacked value deltas (models.py:260,265,397,402)
    extra: Optional[Var] = None    # dense control term added to the adapter's input (concat_hidden control processors)
    t_add: Optional[torch.Tensor] = None                       # rank-space control term (v1 without concat_hidden), [M, 8*nb] fp32
    on_bwd: Optional[Callable[[torch.Tensor], None]] = None    # receives dt (unscaled dy B) of this adapter


def chain_linear(ctx: Ctx, x: Var, lw: E.LinearW, entries: List[Entry], residual: Optional[Var] = None) -> Var:
    """y = x W^T + b, then for every entry in order  y <- y + alpha * up(down(in)),  in = (y if post_add else x) (+ extra)
    (models.py:231-243, 248-265, 275-282), finally + residual."""
    if not entries:
        return E.linear(ctx, x, lw, residual=residual)
    K = x.data.shape[-1]
    x2 = x.data.view(-1, K)
    N = lw.w.shape[0]
    any_post = any(e.post_add for e in entries)
    fold_res = residual is not None and not any_post
    y = ops.gemm(x2, lw.w, bias=lw.bias, residual=residual.data.view(-1, N) if fold_res else None)
    recs = []
    for e in entries:
        src = y if e.post_add else x2
        if e.extra is not None:
            src = ops.add(src, e.extra.data.view(src.shape))
        t = e.ad.project(src)
        if e.t_add is not None:
            ops.axpy_matrix(e.t_add, t)
        recs.append((e, src, t))
        y = e.ad.update(y, t, e.alpha)
    if residual is not None and not fold_res:
        y = ops.add(y, residual.data.view(-1, N))
    out = Var(y.view(*x.data.shape[:-1], N), rg=True)
    if ctx.tape is not None:
        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            if residual is not None:
                E.give_tensor(residual, dy.view(residual.data.shape))
            dy_cur = dy.contiguous().view(-1, N)
            dx_extra, dx_owned = None, False
            for e, src, t in reversed(recs):
                dt = e.ad.dt(dy_cur)
                e.ad.grads(t, dt, dy_cur, src, e.alpha)
                if e.on_bwd is not None:
                    e.on_bwd(dt)
                need_in = e.post_add or x.rg or (e.extra is not None and e.extra.rg)
                if not need_in:
                    continue
                g_in = e.ad.back_input(dt, e.alpha)                       # alpha * dt A   [M, K_in]
                if e.extra is not None:
                    E.give_tensor(e.extra, g_in.view(e.extra.data.shape))
                if e.post_add:
                    dy_cur = ops.add(dy_cur, g_in)                        # gradient of the running output seen by earlier adapters
                elif x.rg:
                    # g_in may now be aliased as e.extra's gradient (give_tensor keeps the tensor): never accumulate into a shared buffer
                    shared = e.extra is not None
                    if dx_extra is None:
                        dx_extra, dx_owned = g_in, not shared
                    elif dx_owned:
                        ops.add(dx_extra, g_in, out=dx_extra)
                    else:
                        dx_extra, dx_owned = ops.add(dx_extra, g_in), True
            if x.rg:
                def prod(buf, acc):
                    b2 = buf.view(-1, K)
                    ops.gemm(dy_cur, lw.wt, out=b2, residual=b2 if acc else None)
                    if dx_extra is not None:
                        ops.add(b2, dx_extra, out=b2)
                E.give_produce(x, prod)

        ctx.tape.record(bwd)
    return out


class ControlMLP:
    """`scale * to_control([h ; c])` of a concat_hidden processor (models.py:207-220 / 342-355) - or `to_control(c)` when the layer
    takes the control states alone - as a term that is either added to the hidden states (V2: h' = h + term) or handed out on its
    own.  Ranks <= DENSE_RANK: hi/lo skinny GEMMs + rank-8 updates (fp32-accurate rank space, like the fused V2 kernels); wider
    control MLPs (danbooru-sketch's rank 256): dense bf16 GEMMs with wgmma weight gradients, like lora_runtime._v1cat_q."""

    def __init__(self, layer, C: int, plan, grad_of, device, concat_hidden: bool):
        down, up = layer.down.weight, layer.up.weight
        self.down, self.up, self.C = down, up, C
        self.R = down.shape[0]
        self.concat = concat_hidden
        self.Cc = down.shape[1] - (C if concat_hidden else 0)
        self.grad_of = grad_of
        self.device = device
        self.dense = self.R > DENSE_RANK
        if not self.dense:
            self.ad_h = GAdapter(down, up, plan, grad_of, device, 0, C) if concat_hidden else None
            self.ad_c = GAdapter(down, up, plan, grad_of, device, C if concat_hidden else 0, None)

    def apply(self, ctx: Ctx, h: Var, c: Var, add_to_h: bool) -> Var:
        """returns  (h if add_to_h else 0) + scale * up(down([h ; c]))   as a Var shaped like h."""
        return self._dense(ctx, h, c, add_to_h) if self.dense else self._blocks(ctx, h, c, add_to_h)

    # -------------------------------------------------------------------------------- hi/lo blocks
    def _blocks(self, ctx, h, c, add_to_h):
        s = ctx.scale
        C, Cc = self.C, self.Cc
        T = h.data.numel() // C
        h2, c2 = h.data.view(T, C), c.data.view(T, Cc)
        t = self.ad_c.project(c2)
        if self.concat:
            ops.axpy_matrix(self.ad_h.project(h2), t)
        base = h2 if add_to_h else torch.zeros(T, C, device=h2.device, dtype=BF16)
        out = Var(self.ad_c.update(base, t, s).view(h.data.shape), rg=True)
        if ctx.tape is not None:
            def bwd():
                dy = out.grad
                out.grad = None
                if dy is None:
                    return
                dy2 = dy.contiguous().view(T, C)
                dt = self.ad_c.dt(dy2)
                # the two halves of `down` share `up`: dB once, dA per half
                Kf = self.down.shape[1]
                for b in range(self.ad_c.nb):
                    rb = self.ad_c.rb(b)
                    ops.SKINNY.add(t[:, 8 * b:], rb, dy2, self.ad_c.up_grad[:, 8 * b:], 1, self.R, s)
                    ops.SKINNY.add(dt[:, 8 * b:], rb, c2, self.ad_c.down_grad[8 * b:, self.ad_c.col_lo:], Kf, 1, s)
                    if self.concat:
                        ops.SKINNY.add(dt[:, 8 * b:], rb, h2, self.ad_h.down_grad[8 * b:, 0:], Kf, 1, s)
                if c.rg:
                    E.give_tensor(c, self.ad_c.back_input(dt, s).view(c.data.shape))
                if h.rg:
                    if self.concat:
                        g = self.ad_h.back_input(dt, s, base=dy2 if add_to_h else None)
                        E.give_tensor(h, g.view(h.data.shape))
                    elif add_to_h:
                        E.give_tensor(h, dy)

            ctx.tape.record(bwd)
        return out

    # -------------------------------------------------------------------------------- dense bf16 GEMMs
    def _dense(self, ctx, h, c, add_to_h):
        s = ctx.scale
        C, Cc, R = self.C, self.Cc, self.R
        Ac, Bc = self.down, self.up
        ldA = Ac.stride(0)
        T = h.data.numel() // C
        h2, c2 = h.data.view(T, C), c.data.view(T, Cc)
        off = C if self.concat else 0
        Ac_c = ops.cast_matrix(Ac[:, off:], R, Cc, ldA, 1)
        Bc_s = ops.cast_matrix(Bc, C, R, Bc.stride(0), 1, alpha=s)
        if self.concat:
            u = ops.gemm(h2, ops.cast_matrix(Ac, R, C, ldA, 1))
            ops.gemm(c2, Ac_c, residual=u, out=u)
        else:
            u = ops.gemm(c2, Ac_c)
        out = Var(ops.gemm(u, Bc_s, residual=h2 if add_to_h else None).view(h.data.shape), rg=True)
        if ctx.tape is not None:
            def bwd():
                dy = out.grad
                out.grad = None
                if dy is None:
                    return
                dy2 = dy.contiguous().view(T, C)
                du = ops.gemm(dy2, ops.cast_matrix(Bc, R, C, 1, Bc.stride(0), alpha=s))                # [T, R] = dy (s Bc)
                ops.conv_wgrad(dy2.view(1, 1, T, C), u.view(1, 1, T, R), self.grad_of(Bc).view(C, R, 1, 1), 1, 1, 0, s)
                gAc = self.grad_of(Ac)
                tmp_c = torch.zeros(R, Cc, 1, 1, device=self.device, dtype=torch.float32)
                ops.conv_wgrad(du.view(1, 1, T, R), c2.view(1, 1, T, Cc), tmp_c, 1, 1, 0, 1.0)
                ops.axpy_matrix(tmp_c.view(R, Cc), gAc[:, off:])
                if self.concat:
                    tmp_h = torch.zeros(R, C, 1, 1, device=self.device, dtype=torch.float32)
                    ops.conv_wgrad(du.view(1, 1, T, R), h2.view(1, 1, T, C), tmp_h, 1, 1, 0, 1.0)
                    ops.axpy_matrix(tmp_h.view(R, C), gAc[:, :C])
                if c.rg:
                    E.give_produce(c, lambda buf, acc: ops.gemm(du, ops.cast_matrix(Ac[:, off:], Cc, R, 1, ldA), out=buf.view(T, Cc),
                                                                residual=buf.view(T, Cc) if acc else None))
                if h.rg:
                    if self.concat:
                        def prod(buf, acc):
                            b2 = buf.view(T, C)
                            res = b2 if acc else (dy2 if add_to_h else None)
                            ops.gemm(du, ops.cast_matrix(Ac, C, R, 1, ldA), out=b2, residual=res)
                            if acc and add_to_h:
                                ops.add(b2, dy2, out=b2)
                        E.give_produce(h, prod)
                    elif add_to_h:
                        E.give_tensor(h, dy)

            ctx.tape.record(bwd)
        return out


class V1RankControl:
    """Control term of a v1 processor WITHOUT concat_hidden, kept in rank space (models.py:237-238):
        to_q_lora(in + s Bc Ac c) = A in + s (A Bc)(Ac c)        ->  t_add = s u Mx^T,  u = Ac c,  Mx = A Bc  [r, rc]
    for any rank r / control rank rc (blocks of 8)."""

    def __init__(self, proc, q_ad: GAdapter, plan, grad_of, device):
        self.proc, self.q = proc, q_ad
        layer = proc.to_control
        self.Ac, self.Bc = layer.down.weight, layer.up.weight          # [rc, Cc], [C, rc]
        self.rc = self.Ac.shape[0]
        self.ad_c = GAdapter(self.Ac, self.Bc, plan, grad_of, device)
        self.grad_of = grad_of
        self.device = device

    def prepare(self, ctx: Ctx, c: Var, entry: Entry) -> None:
        s = ctx.scale
        Aq, Bc, rc, r = self.q.down_full, self.Bc, self.rc, self.q.r
        C = Aq.shape[1]
        T = c.data.numel() // c.data.shape[-1]
        c2 = c.data.view(T, -1)
        Mx = torch.empty(r, rc, device=self.device, dtype=torch.float32)
        ops.small_matmul(Aq, C, 1, Bc, rc, 1, Mx, rc, 1, r, C, rc)                       # Mx = Aq Bc
        u = self.ad_c.project(c2)                                                        # [T, 8*nbc]
        ldt = 8 * self.q.nb
        t_add = torch.zeros(T, ldt, device=self.device, dtype=torch.float32)
        for ib in range(self.q.nb):
            ri = self.q.rb(ib)
            for jb in range(self.ad_c.nb):
                rj = self.ad_c.rb(jb)
                # t_add[:, 8ib + i] += s * sum_j u[:, 8jb + j] * Mx[8ib + i, 8jb + j]
                ops.rowmat(u[:, 8 * jb:], Mx[8 * ib:, 8 * jb:], rc, 1, ri, rj, s, t_add[:, 8 * ib:], ldt, accumulate=jb > 0)
        entry.t_add = t_add
        if ctx.tape is None:
            return

        def on_bwd(e):
            """e = dy Bq (unscaled) [T, 8*nbq];  dL/dt_add = s e."""
            G = torch.zeros(r, rc, device=self.device, dtype=torch.float32)              # G = e^T u
            for ib in range(self.q.nb):
                for jb in range(self.ad_c.nb):
                    ri, rj = self.q.rb(ib), self.ad_c.rb(jb)
                    if self.q.nb == 1 and self.ad_c.nb == 1:
                        ops.skinny_small(e, ri, u, rj, G, 1.0)
                        continue
                    g8 = torch.zeros(64, device=self.device, dtype=torch.float32)        # dense [ri, rj] block, row stride rj
                    ops.skinny_small(e[:, 8 * ib:], ri, u[:, 8 * jb:], rj, g8, 1.0)
                    ops.small_matmul(g8, rj, 1, _eye8(self.device), 8, 1, G[8 * ib:, 8 * jb:], rc, 1, ri, rj, rj)
            ops.small_matmul(G, rc, 1, Bc, 1, rc, self.q.down_grad, C, 1, r, rc, C, alpha=s * s, accumulate=True)          # dAq += s^2 G Bc^T
            ops.small_matmul(Aq, 1, C, G, rc, 1, self.grad_of(Bc), rc, 1, C, r, rc, alpha=s * s, accumulate=True)          # dBc += s^2 Aq^T G
            ldu = 8 * self.ad_c.nb
            du = torch.zeros(T, ldu, device=self.device, dtype=torch.float32)                                              # du = s^2 e Mx
            for jb in range(self.ad_c.nb):
                for ib in range(self.q.nb):
                    ops.rowmat(e[:, 8 * ib:], Mx[8 * ib:, 8 * jb:], 1, rc, self.ad_c.rb(jb), self.q.rb(ib), s * s, du[:, 8 * jb:], ldu,
                               accumulate=ib > 0)
            gAc = self.grad_of(self.Ac)
            Cc = self.Ac.shape[1]
            for jb in range(self.ad_c.nb):
                ops.SKINNY.add(du[:, 8 * jb:], self.ad_c.rb(jb), c2, gAc[8 * jb:], Cc, 1, 1.0)                              # dAc += du^T c
            if c.rg:
                E.give_tensor(c, self.ad_c.back_input(du, 1.0).view(c.data.shape))                                          # dc += du Ac

        entry.on_bwd = on_bwd


class GenericLayer:
    """The adapter chain [pre_loras..., processor, post_loras...] of one attention layer in general form."""

    def __init__(self, rt, L, proc, chain):
        self.rt, self.L, self.p, self.chain = rt, L, proc, chain
        dev, plan, grad_of = rt.device, rt.plan, rt.grad_of
        C = L.to_q.w.shape[0]
        self.C = C
        mk = lambda layer: GAdapter(layer.down.weight, layer.up.weight, plan, grad_of, dev)
        self.q = [mk(a.to_q_lora) for a in chain]
        self.k = [(a, mk(a.to_k_lora)) for a in chain if not a.key_states_skipped]
        self.v = [(a, mk(a.to_v_lora)) for a in chain if not a.value_states_skipped]
        # quirk kept (models.py:279, 423): the processor's own to_out_lora is applied even when its skip flag is set
        self.o = [(a, mk(a.to_out_lora)) for a in chain if a is proc or not a.output_states_skipped]
        self.v1_main, self.v2_main = _is_v1(proc), _is_v2(proc)
        self.q_ctrl = {}
        if self.v1_main:
            # models.py:234-236, 240-242: inside a v1 processor every *v1* chain member adds its control term to its q-adapter input
            for a, qa in zip(chain, self.q):
                if _is_v1(a):
                    if a.concat_hidden:
                        self.q_ctrl[id(a)] = ControlMLP(a.to_control, C, plan, grad_of, dev, concat_hidden=True)
                    else:
                        self.q_ctrl[id(a)] = V1RankControl(a, qa, plan, grad_of, dev)
        self.v2 = []
        if self.v2_main:
            # models.py:366-372, 412-418: every *V2* chain member rewrites the hidden states, in chain order
            for a in chain:
                if _is_v2(a):
                    self.v2.append((a, ControlMLP(a.to_control, C, plan, grad_of, dev, True), ControlMLP(a.to_control_out, C, plan, grad_of, dev, True)))

    @staticmethod
    def _cvar(ctx: Ctx, a) -> Var:
        cs = a.control_states
        assert cs is not None, "inject_control_states() must run before the UNet forward (models.py:227, 362)"
        cv = ctx.stash["control_vars"]
        v = cv.get(cs.data_ptr())
        if v is None:
            # control states the caller did not register (e.g. a frozen second ControlLoRA next to the Trainer's own): constants
            from .unet_module import _control_to_var

            v = cv[cs.data_ptr()] = _control_to_var(cs.detach(), rg=False)
        return v

    def run(self, ctx: Ctx, hs: Var, ehs: Optional[Var], residual: Var) -> Var:
        L, p, s = self.L, self.p, ctx.scale
        for a, mlp_in, _ in self.v2:
            hs = mlp_in.apply(ctx, hs, self._cvar(ctx, a), add_to_h=True)
        q_entries = []
        for a, qa in zip(self.chain, self.q):
            e = Entry(qa, bool(a.post_add), s)
            ctl = self.q_ctrl.get(id(a))
            if isinstance(ctl, V1RankControl):
                ctl.prepare(ctx, self._cvar(ctx, a), e)
            elif ctl is not None:
                e.extra = ctl.apply(ctx, hs, self._cvar(ctx, a), add_to_h=False)
            q_entries.append(e)
        q = chain_linear(ctx, hs, L.to_q, q_entries)
        kv_in = hs if ehs is None else ehs
        k = chain_linear(ctx, kv_in, L.to_k, [Entry(ad, bool(a.post_add), s) for a, ad in self.k])
        # quirk kept (models.py:260,265,397,402): stacked adapters' VALUE deltas are added without `scale`
        v = chain_linear(ctx, kv_in, L.to_v, [Entry(ad, bool(a.post_add), s if a is p else 1.0) for a, ad in self.v])
        o = E.attention(ctx, q, k, v, L.heads)
        for a, _, mlp_out in self.v2:
            o = mlp_out.apply(ctx, o, self._cvar(ctx, a), add_to_h=True)
        return chain_linear(ctx, o, L.to_out, [Entry(ad, bool(a.post_add), s) for a, ad in self.o], residual=residual)
