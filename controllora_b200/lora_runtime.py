"""Maps the reference's attention-processor objects (LoRACrossAttnProcessor / ControlLoRACrossAttnProcessor[V2],
/root/reference/models.py:72-431) onto fused kernel launches.

For every attention layer the adapter chain [pre_loras..., processor, post_loras...] (models.py:232-243 etc.) is packed
into one rank<=8 `LoraSlot` per projection, so a projection and all of its LoRA deltas are ONE wgmma GEMM launch.

v1 control (models.py:237-238):  q = Wq h + s Bq Aq (h + s Bc Ac c)
        = Wq h + s Bq ( Aq h  +  s (Aq Bc) (Ac c) )               -> `t_add` of the fused GEMM epilogue,
  with u = Ac c computed for all processors of a UNet level by one GEMM over the level's control state.
v1 control with `concat_hidden` (models.py:208-214; configs/danbooru-sketch.json, control_rank 256):
        ctrl = s Bc Ac [h ; c]  is a real two-layer MLP, so it runs as dense wgmma GEMMs (Ac_h, Ac_c, Bc are trainable: their
        weight gradients are dense GEMMs too), followed by the rank-4 `to_q_lora` on h + ctrl.
V2 control (models.py:369, 415):  h' = h + s Bc Ac [h ; c]  is a rank-r update of the hidden states (before q/k/v and
  again before to_out), done by one skinny GEMM + one rank-update kernel.
"""
from __future__ import annotations

import os
from types import SimpleNamespace
from typing import Callable, Dict, List, Optional

import torch

from . import engine as E
from . import ops
from .engine import Ctx, LoraSlot, Var

BF16 = torch.bfloat16


def _is_v1(p) -> bool:
    return type(p).__name__ == "ControlLoRACrossAttnProcessor"


def _is_v2(p) -> bool:
    return type(p).__name__ == "ControlLoRACrossAttnProcessorV2"


class _LevelCtx:
    """Per control-state tensor (== per UNet resolution level): the stacked `to_control.down` operands of every
    processor fed by that tensor, and the per-forward products."""

    def __init__(self):
        self.procs: List = []           # (processor, LayerPlan)
        self.cc = 0                     # control channels
        self.stack = None               # bf16 [16*nb, Cc]   (hi/lo rows of the control-down matrices)
        self.stack_t = None             # bf16 [Cc, 16*nb]   (transposed, hi duplicated) for the d-control GEMM
        self.nb = 0
        # per-forward products (c Var [B, HW, Cc] bf16, u fp32 [T, 8*nb], du bf16 [T, 16*nb]) live in Ctx.stash


class LayerPlan:
    def __init__(self):
        self.kind = "none"
        self.proc = None
        self.chain: List = []
        self.q = self.k = self.v = self.out = None   # LoraSlot
        self.level: Optional[_LevelCtx] = None
        self.col = 0           # first column of this processor's block inside level.u
        self.ctrl_adapter = None        # engine.Adapter of the processor's own to_q_lora (v1)
        self.v_chain = None             # [(is the processor's own adapter, GAdapter)] when the value projection carries unscaled adapters
        # V2 helper tables (fp32): Bc [C, rp] etc. are read directly from the parameters


class LoraRuntime:
    """Built once per (UNet, processor wiring); `begin()` runs at the start of every UNet forward."""

    def __init__(self, weights, device, grad_of: Callable[[torch.nn.Parameter], torch.Tensor]):
        self.W = weights
        self.device = device
        self.grad_of = grad_of
        self.plan = ops.PackPlan(device)        # slot operands (ext / tables of every projection)
        self.v2_plan = ops.PackPlan(device)     # V2 hidden-state-update operands
        self.level_plan = ops.PackPlan(device)  # stacked control-down operands per level (rebuilt when levels change)
        self.layers: Dict[str, LayerPlan] = {}
        self.level_list: List[_LevelCtx] = []
        self.signature = None
        self._build()

    # ------------------------------------------------------------------------------------------------ build
    @staticmethod
    def make_signature(weights) -> tuple:
        sig = []
        for name, L in weights.attn_layers.items():
            p = L.processor
            if p is None or not hasattr(p, "to_q_lora"):
                sig.append(None)
                continue
            chain = [*getattr(p, "pre_loras", []), p, *getattr(p, "post_loras", [])]
            sig.append(tuple((id(a), a.key_states_skipped, a.value_states_skipped, a.output_states_skipped) for a in chain))
        return tuple(sig)

    @staticmethod
    def _needs_generic(p, chain, post_add, cat) -> Optional[str]:
        """None when the fused one-launch path covers this layer's adapter chain, else the reason it does not."""
        if os.environ.get("CLB_GENERIC_CHAIN", "0") == "1":      # tests: run EVERY layer through lora_generic
            return "CLB_GENERIC_CHAIN=1"
        if any(post_add) and (len(chain) > 1 or _is_v2(p)):
            return "post_add inside a stacked chain"
        if any(a is not p and (_is_v1(a) or _is_v2(a)) for a in chain):
            return "a ControlLoRA processor stacked as pre / post LoRA"
        if cat and (len(chain) > 1 or any(post_add) or p.to_q_lora.down.weight.shape[0] > 4):
            return "concat_hidden control combined with stacked adapters / post_add / q rank > 4"
        if not cat and (_is_v1(p) or _is_v2(p)):
            ctrl = [p.to_control] + ([p.to_control_out] if _is_v2(p) else [])
            if any(c.down.weight.shape[0] > 4 for c in ctrl):
                return "control rank > 4"

        def total(name, skip):
            return sum(getattr(a, name).down.weight.shape[0] for a in chain if not skip(a))

        ranks = [total("to_q_lora", lambda a: False), total("to_k_lora", lambda a: a.key_states_skipped),
                 total("to_v_lora", lambda a: a.value_states_skipped),
                 total("to_out_lora", lambda a: a is not p and a.output_states_skipped)]
        if max(ranks) > 8:
            return "adapter ranks on one projection sum to more than 8"
        if any(post_add) and max(ranks) > 4:
            return "post_add adapter of rank > 4"
        return None

    def _adapter(self, slot: LoraSlot, layer, unscaled: bool = False) -> E.Adapter:
        a = slot.add(layer.down.weight, layer.up.weight, unscaled=unscaled)
        a.down_grad = self.grad_of(layer.down.weight)
        a.up_grad = self.grad_of(layer.up.weight)
        return a

    def _build(self):
        dev = self.device
        for name, L in self.W.attn_layers.items():
            lp = LayerPlan()
            self.layers[name] = lp
            p = L.processor
            if p is None or not hasattr(p, "to_q_lora"):
                continue
            lp.proc = p
            chain = [*getattr(p, "pre_loras", []), p, *getattr(p, "post_loras", [])]
            lp.chain = chain
            post_add = [bool(getattr(a, "post_add", False)) for a in chain]
            cat = _is_v1(p) and getattr(p, "concat_hidden", False)
            lp.kind = "v1cat" if cat else ("v1" if _is_v1(p) else ("v2" if _is_v2(p) else "plain"))
            why = self._needs_generic(p, chain, post_add, cat)
            if why is not None:
                # a wiring the one-launch path cannot express (see lora_generic.py): this layer runs adapter by adapter
                from .lora_generic import GenericLayer

                lp.kind, lp.generic_reason = "generic", why
                lp.generic = GenericLayer(self, L, p, chain)
                continue
            C = L.to_q.w.shape[0]
            kv_in = L.to_k.w.shape[1]
            lp.post_add = any(post_add)
            # V2 self-attention: k / v carry no LoRA (models.py:306-307) and read the same h' as q -> ONE fused q|k|v projection
            # (N = 3C, the q adapter owns the first C output rows)
            lp.fuse_qkv = bool(_is_v2(p) and not L.is_cross and len(chain) == 1 and not any(post_add))
            lp.q = LoraSlot(3 * C if lp.fuse_qkv else C, C, dev)
            # post_add adapters read the projection's output: their `down` has C input features even for the text k / v
            lp.k = LoraSlot(C, C if lp.post_add else kv_in, dev)
            lp.v = LoraSlot(C, C if lp.post_add else kv_in, dev)
            lp.out = LoraSlot(C, C, dev)
            for sl in (lp.q, lp.k, lp.v, lp.out):
                sl.post_add = lp.post_add
            for a in chain:
                if lp.kind == "v1cat":
                    ad = None                                   # the q adapter reads h + ctrl: handled by _v1cat_q
                else:
                    ad = self._adapter(lp.q, a.to_q_lora)
                if a is p:
                    lp.ctrl_adapter = ad
                if not a.key_states_skipped:
                    self._adapter(lp.k, a.to_k_lora)
                if not a.value_states_skipped:
                    # quirk kept from the reference: stacked adapters' VALUE deltas carry no `scale` (models.py:260,265,397,402)
                    self._adapter(lp.v, a.to_v_lora, unscaled=a is not p)
                if a is p or not a.output_states_skipped:
                    self._adapter(lp.out, a.to_out_lora)
            # value projections with unscaled (stacked) adapters keep an adapter-by-adapter form as well: begin() selects it for a
            # forward whose `scale` differs from the one the shared tables are packed for while another forward is still in flight
            lp.v_chain = None
            if any(ad.unscaled for ad in lp.v.adapters):
                from .lora_generic import GAdapter

                lp.v_chain = [(a is p, GAdapter(a.to_v_lora.down.weight, a.to_v_lora.up.weight, self.plan, self.grad_of, dev))
                              for a in chain if not a.value_states_skipped]
            lp.q.finalize(self.plan, need_dx=True)
            lp.k.finalize(self.plan, need_dx=lp.post_add or not L.is_cross)     # post_add: down_tab = A^T feeds dy0 = dy + s dt A
            lp.v.finalize(self.plan, need_dx=lp.post_add or not L.is_cross)
            lp.out.finalize(self.plan, need_dx=True)
            if lp.kind == "v2":
                self._v2_tables(lp)
            if lp.kind == "v1cat":
                ql = p.to_q_lora
                lp.cat_ext = torch.zeros(16, C, device=dev, dtype=BF16)                       # hi/lo rows of Aq
                lp.cat_up = torch.zeros(C, 4, device=dev, dtype=torch.float32)                # Bq
                lp.cat_down = torch.zeros(C, 4, device=dev, dtype=torch.float32)              # Aq^T
                self.plan.add_ext(ql.down.weight, lp.cat_ext)
                self.plan.add_table(ql.up.weight, lp.cat_up)
                self.plan.add_table(ql.down.weight, lp.cat_down, transposed=True)
        self.signature = self.make_signature(self.W)

    # ------------------------------------------------------------------------------------------------ per forward
    def begin(self, ctx: Ctx, control_vars: Dict[int, Var]):
        """control_vars: data_ptr of each processor's control-state tensor -> Var [B, HW, Cc] (NHWC bf16)."""
        # (re)group control processors by the tensor that was injected into them
        groups: Dict[int, List[LayerPlan]] = {}
        for lp in self.layers.values():
            if lp.kind in ("v1", "v2", "v1cat"):
                cs = lp.proc.control_states
                assert cs is not None, "inject_control_states() must run before the UNet forward (models.py:227)"
                groups.setdefault(cs.data_ptr(), []).append(lp)
        # level structure = which processors share a control tensor (pointer values change every step, membership not)
        key = tuple(tuple(id(lp) for lp in v) for v in groups.values())
        if getattr(self, "_level_key", None) != key:
            self._build_levels(groups, control_vars)
            self._level_key = key
        ctx.stash["control_vars"] = control_vars          # generic layers look their processors' control states up themselves
        s = ctx.scale
        if self.plan._unscaled:
            # The fused epilogue has ONE scale per projection, so the unscaled stacked value deltas (models.py:260,265,397,402) are
            # packed with 1/scale into tables that every forward of this runtime shares.  They may only be re-packed for another
            # scale when no earlier forward still needs them for its backward (two UNet calls with different `scale` before one
            # backward): such a forward - and scale == 0, where 1/scale does not exist - takes the adapter-by-adapter value
            # projection instead, which applies each adapter's own factor.
            inflight = getattr(self, "_inflight", 0)
            packed = 1.0 / self.plan._unscaled_mul
            if s == 0.0 or (inflight > 0 and abs(packed - s) > 1e-12 * max(1.0, abs(s))):
                ctx.stash["v_chain"] = True
            else:
                self.plan.set_unscaled_mul(1.0 / s)
            if ctx.tape is not None:
                self._inflight = inflight + 1
                ctx.stash["counts_inflight"] = True
        self.plan.run()
        self.v2_plan.run()
        self.level_plan.run()
        # per-forward products live in ctx.stash (keyed by level / layer plan), never on the shared runtime objects: two
        # forwards may be in flight before the first backward (gradient accumulation, several UNet calls per loss)
        for (k, lps), lv in zip(groups.items(), self.level_list):
            c = control_vars[k]
            st = self._fs(ctx, lv)
            st.c, st.u, st.du = c, None, None
            T = c.data.shape[0] * c.data.shape[1]
            assert c.data.shape[-1] == lv.cc
            if lv.nb == 0:                       # concat_hidden levels: every processor runs its own dense control MLP
                continue
            c2 = c.data.view(T, lv.cc)
            u16 = ops.gemm(c2, lv.stack, out_fp32=True)
            st.u = ops.hilo_combine(u16, lv.nb)
            if ctx.tape is not None and c.rg:
                st.du = torch.zeros(T, 16 * lv.nb, device=self.device, dtype=BF16)
        for lp in self.layers.values():
            if lp.kind == "v1":
                self._v1_prepare(ctx, lp)

    @staticmethod
    def _fs(ctx: Ctx, obj) -> SimpleNamespace:
        """Per-forward state of a level / layer plan inside this forward's Ctx."""
        st = ctx.stash.get(id(obj))
        if st is None:
            st = ctx.stash[id(obj)] = SimpleNamespace(c=None, u=None, du=None, t_add=None, M=None)
        return st

    def _build_levels(self, groups, control_vars):
        self.level_list = []
        plan = ops.PackPlan(self.device)
        for key, lps in groups.items():
            lv = _LevelCtx()
            cvar = control_vars[key]
            lv.cc = cvar.data.shape[-1]
            if lps[0].kind == "v1cat":
                for lp in lps:
                    lp.level = lv
                self.level_list.append(lv)
                continue
            v2 = lps[0].kind == "v2"
            lv.nb = len(lps) if v2 else (len(lps) + 1) // 2
            lv.stack = torch.zeros(16 * lv.nb, lv.cc, device=self.device, dtype=BF16)
            lv.stack_t = torch.zeros(lv.cc, 16 * lv.nb, device=self.device, dtype=BF16)
            for i, lp in enumerate(lps):
                lp.level = lv
                p = lp.proc
                C = p.hidden_size
                if v2:
                    lp.col = 8 * i
                    downs = [(p.to_control.down.weight[:, C:], 0), (p.to_control_out.down.weight[:, C:], 4)]
                    blk = i
                else:
                    lp.col = 4 * i
                    downs = [(p.to_control.down.weight, 4 * (i % 2))]
                    blk = i // 2
                for dn, off in downs:
                    assert dn.shape[1] == lv.cc, "control-state channels do not match to_control.down"
                    plan.add_ext(dn, lv.stack[16 * blk:16 * blk + 16], row_off=off)
                    r = dn.shape[0]
                    # kind 2: stack_t[k, 16*blk + off + j] and [.. + 8 ..] <- bf16(dn[j, k])
                    plan.add(dn, lv.stack_t[:, 16 * blk:], 2, r, lv.cc, dn.stride(0), dn.stride(1), lv.stack_t.stride(0), off)
            self.level_list.append(lv)
        self.level_plan = plan

    # ------------------------------------------------------------------------------------------------ v1
    def _v1_prepare(self, ctx: Ctx, lp: LayerPlan):
        p, lv, ad = lp.proc, lp.level, lp.ctrl_adapter
        s = ctx.scale
        r = ad.down.shape[0]
        Aq = ad.down                      # [r, C]
        Bc = p.to_control.up.weight       # [C, rc]
        rc = Bc.shape[1]
        C = Aq.shape[1]
        M = torch.empty(r, rc, device=self.device, dtype=torch.float32)
        ops.small_matmul(Aq, C, 1, Bc, rc, 1, M, rc, 1, r, C, rc)                  # M = Aq Bc
        lvs = self._fs(ctx, lv)
        T = lvs.u.shape[0]
        rp = lp.q.rp
        t_add = torch.zeros(T, rp, device=self.device, dtype=torch.float32) if lp.q.rank != r else \
            torch.empty(T, rp, device=self.device, dtype=torch.float32)
        u = lvs.u[:, lp.col:]
        # t_add[:, col_a + i] = s * sum_j u[:, j] * M[i, j]
        ops.rowmat(u, M, rc, 1, r, rc, s, t_add[:, ad.col:], rp)
        st = self._fs(ctx, lp)
        st.t_add, st.M = t_add, M

    def _v1_q_bwd(self, ctx: Ctx, lp: LayerPlan, e, t_out, dy2):
        """Gradients of the control branch of a v1 q-projection (see module docstring)."""
        p, lv, ad = lp.proc, lp.level, lp.ctrl_adapter
        s = ctx.scale
        r = ad.down.shape[0]
        Aq, Bc, Ac = ad.down, p.to_control.up.weight, p.to_control.down.weight
        rc = Bc.shape[1]
        C = Aq.shape[1]
        lvs, lps = self._fs(ctx, lv), self._fs(ctx, lp)
        u = lvs.u[:, lp.col:]
        ea = e[:, ad.col:]
        G = torch.zeros(r, rc, device=self.device, dtype=torch.float32)
        ops.skinny_small(ea, r, u, rc, G, 1.0)                                     # G = e^T u
        ops.small_matmul(G, rc, 1, Bc, 1, rc, ad.down_grad, C, 1, r, rc, C, alpha=s * s, accumulate=True)   # dAq += s^2 G Bc^T
        ops.small_matmul(Aq, 1, C, G, rc, 1, self.grad_of(Bc), rc, 1, C, r, rc, alpha=s * s, accumulate=True)  # dBc += s^2 Aq^T G
        T = u.shape[0]
        du = torch.empty(T, rc, device=self.device, dtype=torch.float32)
        ops.rowmat(ea, lps.M, 1, rc, rc, r, s * s, du, rc)                          # du = s^2 e M
        ops.SKINNY.add(du, rc, lvs.c.data.view(T, lv.cc), self.grad_of(Ac), lv.cc, 1, 1.0)   # dAc += du^T c
        if lvs.du is not None:
            i = lp.col // 4
            ops.rowmat(ea, lps.M, 1, rc, rc, r, s * s, lvs.du, 16 * lv.nb, out_mode=1, col_off=16 * (i // 2) + 4 * (i % 2), lo_off=8)

    # ------------------------------------------------------------------------------------------------ v1 + concat_hidden
    def _v1cat_q(self, ctx: Ctx, lp: LayerPlan, L, hs: Var) -> Var:
        """q = Wq h + s Bq Aq (h + ctrl),  ctrl = s Bc Ac [h ; c]   (models.py:208-218, 237-238 with concat_hidden)."""
        p, lv = lp.proc, lp.level
        s = ctx.scale
        C = p.hidden_size
        Ac, Bc = p.to_control.down.weight, p.to_control.up.weight          # [R, C + Cc], [C, R]  (fp32 masters)
        ql = p.to_q_lora
        r = ql.down.weight.shape[0]
        c = self._fs(ctx, lv).c
        T = hs.data.shape[0] * hs.data.shape[1]
        h2, c2 = hs.data.view(T, C), c.data.view(T, lv.cc)
        # bf16 operands of the trainable dense layers (and their transposes for the backward), re-derived from the fp32 masters
        # every step by strided cast kernels: Ac = [Ac_h | Ac_c] is [R, C + Cc] row-major, Bc is [C, R]
        R, ldA = Ac.shape[0], Ac.stride(0)
        Ac_h = ops.cast_matrix(Ac, R, C, ldA, 1)                           # [R, C]
        Ac_c = ops.cast_matrix(Ac[:, C:], R, lv.cc, ldA, 1)                # [R, Cc]
        Bc_s = ops.cast_matrix(Bc, C, R, Bc.stride(0), 1, alpha=s)         # [C, R]   (scale folded)
        u = ops.gemm(h2, Ac_h)
        ops.gemm(c2, Ac_c, residual=u, out=u)                              # u = Ac [h ; c]          [T, R]
        xp = ops.gemm(u, Bc_s, residual=h2)                                # x' = h + s Bc u         [T, C]
        th16 = ops.gemm(xp, lp.cat_ext, out_fp32=True)                     # hi/lo columns of x' Aq^T
        q0 = ops.gemm(h2, L.to_q.w, bias=L.to_q.bias)
        qd, t = ops.v2_inject_fwd(q0, th16, None, r, lp.cat_up, s)         # q = q0 + s t Bq^T,  t = Aq x'
        out = Var(qd.view(*hs.data.shape[:-1], C), rg=True)
        if ctx.tape is not None:
            def bwd():
                dq = out.grad
                out.grad = None
                if dq is None:
                    return
                dq2 = dq.contiguous().view(T, C)
                dt, _ = ops.v2_inject_bwd(dq2, lp.cat_up, None, s, need_dh=False)           # dt = dq Bq  (unscaled)
                ops.SKINNY.add(t, r, dq2, self.grad_of(ql.up.weight), 1, r, s)             # dBq
                ops.SKINNY.add(dt, r, xp, self.grad_of(ql.down.weight), C, 1, s)           # dAq += s dt^T x'
                zero = torch.empty_like(xp)
                zero.zero_()                                                                # allocator-level memset
                dxp = ops.rank_update(zero, dt, lp.cat_down, s, out=zero)                   # dL/dx' = s dt Aq   [T, C]
                # control MLP:  x' = h + (s Bc) u,  u = Ac_h h + Ac_c c
                Bc_st = ops.cast_matrix(Bc, R, C, 1, Bc.stride(0), alpha=s)                 # (s Bc)^T  [R, C]
                du = ops.gemm(dxp, Bc_st)                                                   # [T, R] = dx' (s Bc)
                ops.conv_wgrad(dxp.view(1, 1, T, C), u.view(1, 1, T, R), self.grad_of(Bc).view(C, R, 1, 1), 1, 1, 0, s)   # dBc += s dx'^T u
                gAc = self.grad_of(Ac)
                tmp_h = torch.zeros(R, C, 1, 1, device=self.device, dtype=torch.float32)
                tmp_c = torch.zeros(R, lv.cc, 1, 1, device=self.device, dtype=torch.float32)
                ops.conv_wgrad(du.view(1, 1, T, R), h2.view(1, 1, T, C), tmp_h, 1, 1, 0, 1.0)                         # dAc_h = du^T h
                ops.conv_wgrad(du.view(1, 1, T, R), c2.view(1, 1, T, lv.cc), tmp_c, 1, 1, 0, 1.0)                     # dAc_c = du^T c
                ops.axpy_matrix(tmp_h.view(R, C), gAc[:, :C])
                ops.axpy_matrix(tmp_c.view(R, lv.cc), gAc[:, C:])
                if hs.rg:
                    def prod(buf, acc):
                        b2 = buf.view(T, C)
                        ops.gemm(dq2, L.to_q.wt, out=b2, residual=b2 if acc else None)      # dq Wq
                        ops.add(b2, dxp, out=b2)                                            # + dL/dx'
                        ops.gemm(du, ops.cast_matrix(Ac, C, R, 1, ldA), out=b2, residual=b2)  # + du Ac_h   (operand = Ac_h^T [C, R])
                    E.give_produce(hs, prod)
                if c.rg:
                    E.give_produce(c, lambda buf, acc: ops.gemm(du, ops.cast_matrix(Ac[:, C:], lv.cc, R, 1, ldA), out=buf.view(T, lv.cc),
                                                                residual=buf.view(T, lv.cc) if acc else None))

            ctx.tape.record(bwd)
        return out

    # ------------------------------------------------------------------------------------------------ V2
    def _v2_inject(self, ctx: Ctx, lp: LayerPlan, h: Var, which: int) -> Var:
        """h' = h + s * Bc ( Ac_h h + Ac_c c )   (which = 0: to_control before q/k/v, 1: to_control_out before to_out)."""
        p, lv = lp.proc, lp.level
        layer = p.to_control if which == 0 else p.to_control_out
        s = ctx.scale
        C = p.hidden_size
        down, up = layer.down.weight, layer.up.weight      # [rc, C + Cc], [C, rc]
        rc = down.shape[0]
        T = h.data.shape[0] * h.data.shape[1]
        h2 = h.data.view(T, C)
        lvs = self._fs(ctx, lv)
        uc = lvs.u[:, lp.col + 4 * which:]
        # one pass over h: t = h Ac_h^T + u_c (fp32 row dots), h' = h + s * t Bc^T   (t [T, 4] kept for the backward)
        out_data, t = ops.rank4_project_update(h.data, lp.v2_down_tab[which], lp.v2_up[which], uc, rc, s)
        out = Var(out_data, rg=True)
        if ctx.tape is not None:
            def bwd():
                dy = out.grad
                out.grad = None
                if dy is None:
                    return
                dy2 = dy.view(T, C)
                # one pass over dy: dt = dy Bc (unscaled, [T, 4]) and dh = dy + s * dt Ac_h
                dt, dh = ops.v2_inject_bwd(dy, lp.v2_up[which], lp.v2_down_tab[which], s, need_dh=h.rg)
                # dBc[c, j] += s * sum_m dy[m, c] t[m, j]
                ops.SKINNY.add(t, rc, dy2, self.grad_of(up), 1, rc, s)
                # dAc_h[j, k] += s * sum_m dt[m, j] h[m, k] ; dAc_c likewise with c
                gdown = self.grad_of(down)
                ops.SKINNY.add(dt, rc, h2, gdown, C + lv.cc, 1, s)
                ops.SKINNY.add(dt, rc, lvs.c.data.view(T, lv.cc), gdown[:, C:], C + lv.cc, 1, s)
                # dh = dy + s * dt Ac_h
                if h.rg:
                    E.give_tensor(h, dh)
                if lvs.du is not None:
                    i = lp.col // 8
                    ops.rowmat(dt, lp.v2_eye, 4, 1, rc, rc, s, lvs.du, 16 * lv.nb, out_mode=1, col_off=16 * i + 4 * which, lo_off=8)

            ctx.tape.record(bwd)
        return out

    def _v2_tables(self, lp: LayerPlan):
        """Per-processor fp32 tables of the V2 hidden-state update (built once, re-packed from the parameters every step):
        v2_down_tab[w][c, j] = Ac_h[j, c] (projection h -> t, and dt -> dh in the backward), v2_up[w][c, j] = Bc[c, j]."""
        if getattr(lp, "v2_up", None) is not None:
            return
        p = lp.proc
        C = p.hidden_size
        dev = self.device
        lp.v2_up, lp.v2_down_tab = [], []
        for layer in (p.to_control, p.to_control_out):
            down, up = layer.down.weight, layer.up.weight
            upt = torch.zeros(C, 4, device=dev, dtype=torch.float32)
            dnt = torch.zeros(C, 4, device=dev, dtype=torch.float32)
            self.v2_plan.add_table(up, upt)
            self.v2_plan.add_table(down[:, :C], dnt, transposed=True)
            lp.v2_up.append(upt); lp.v2_down_tab.append(dnt)
        lp.v2_eye = torch.eye(4, device=dev, dtype=torch.float32)

    # ------------------------------------------------------------------------------------------------ attention layer
    def attn_fn(self, ctx: Ctx, L, hs: Var, ehs: Optional[Var], residual: Var) -> Var:
        lp = self.layers[L.name]
        if lp.kind == "generic":
            return lp.generic.run(ctx, hs, ehs, residual)
        if lp.kind == "v2":
            hs = self._v2_inject(ctx, lp, hs, 0)
        kv_in = hs if ehs is None else ehs
        on_q = None
        if lp.kind == "v1":
            on_q = lambda e, t_out, dy2: self._v1_q_bwd(ctx, lp, e, t_out, dy2)
        if lp.kind == "v2" and ehs is None and lp.fuse_qkv:
            # q | k | v of V2 self-attention as ONE GEMM over h' and ONE attention op on the fused buffer
            if getattr(L, "w_qkv", None) is None:
                w = torch.cat([L.to_q.w, L.to_k.w, L.to_v.w], 0).contiguous()                  # [3C, C]
                L.w_qkv = E.LinearW(w, None, w.t().contiguous())
            qkv = E.linear(ctx, hs, L.w_qkv, slot=lp.q)
            o = E.attention_qkv(ctx, qkv, L.heads)
            o = self._v2_inject(ctx, lp, o, 1)
            return E.linear(ctx, o, L.to_out, slot=lp.out, residual=residual)
        if lp.kind == "v1cat":
            q = self._v1cat_q(ctx, lp, L, hs)
        else:
            q = E.linear(ctx, hs, L.to_q, slot=lp.q, t_add=self._fs(ctx, lp).t_add, on_slot_bwd=on_q)
        kvc = ctx.stash.get("kv_cache") if (ehs is not None and ctx.tape is None) else None
        if kvc is not None and L.name in kvc:
            k, v = kvc[L.name]                # text-state projections are timestep-invariant inside a denoise loop
        elif ehs is not None and (lp.k is None or lp.k.rank == 0) and (lp.v is None or lp.v.rank == 0) and not kv_in.rg:
            # no adapters on k / v (V2, or plain attention) and nothing to differentiate: k | v of the text states as ONE GEMM
            if getattr(L, "w_kv", None) is None:
                L.w_kv = E.LinearW(torch.cat([L.to_k.w, L.to_v.w], 0).contiguous(), None, None)
            kv = E.linear(ctx, kv_in, L.w_kv)
            Cc = L.to_k.w.shape[0]
            k, v = Var(kv.data[..., :Cc]), Var(kv.data[..., Cc:])
            if kvc is not None:
                kvc[L.name] = (k, v)
        else:
            k = E.linear(ctx, kv_in, L.to_k, slot=lp.k)
            if lp.v_chain is not None and ctx.stash.get("v_chain"):
                from .lora_generic import Entry, chain_linear

                v = chain_linear(ctx, kv_in, L.to_v, [Entry(ad, False, ctx.scale if own else 1.0) for own, ad in lp.v_chain])
            else:
                v = E.linear(ctx, kv_in, L.to_v, slot=lp.v)
            if kvc is not None:
                kvc[L.name] = (k, v)
        o = E.attention(ctx, q, k, v, L.heads)
        if lp.kind == "v2":
            o = self._v2_inject(ctx, lp, o, 1)
        return E.linear(ctx, o, L.to_out, slot=lp.out, residual=residual)

    def finish_backward(self, ctx: Ctx):
        """After the tape ran: one GEMM per level turns the collected du blocks into d(control state)."""
        if ctx.stash.pop("counts_inflight", False):
            self._inflight = max(0, getattr(self, "_inflight", 0) - 1)
        for lv in getattr(self, "level_list", []):
            st = self._fs(ctx, lv)
            if st.du is None or st.c is None or not st.c.rg:
                continue
            T = st.du.shape[0]
            E.give_produce(st.c, lambda buf, acc, lv=lv, st=st, T=T: ops.gemm(st.du, lv.stack_t, out=buf.view(T, lv.cc),
                                                                             residual=buf.view(T, lv.cc) if acc else None))
            st.du = None
