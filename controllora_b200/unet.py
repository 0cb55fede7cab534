"""H100-native SD-1.5 UNet (the frozen network that /root/reference/train_text_to_image_control_lora.py:782 calls as
`unet(noisy_latents, timesteps, encoder_hidden_states).sample`), built on the tape engine.

Topology / parameter names follow diffusers 0.13 `UNet2DConditionModel` (state-dict compatible), the compute is ours:
channels-last bf16 activations, every conv / linear on the wgmma GEMM, fused attention, fused norm kernels, and a
backward pass that only produces what ControlLoRA training needs (dX, LoRA dA/dB, d control-states).
"""
from __future__ import annotations

import math
from collections import OrderedDict
from types import SimpleNamespace
from typing import Dict, List, Optional

import torch

from . import engine as E
from . import ops
from .engine import ConvW, Ctx, LinearW, NormW, Var

BF16 = torch.bfloat16

SD15_CONFIG = dict(
    in_channels=4,
    out_channels=4,
    block_out_channels=(320, 640, 1280, 1280),
    down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
    up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
    layers_per_block=2,
    attention_head_dim=8,
    cross_attention_dim=768,
    norm_num_groups=32,
    norm_eps=1e-5,
)


class _Resnet:
    def __init__(self, sd, prefix, dev, need_dx):
        g = lambda k: sd[prefix + k]
        self.norm1 = NormW.make(g("norm1.weight"), g("norm1.bias"), dev)
        self.conv1 = ConvW.make(g("conv1.weight"), g("conv1.bias"), dev, need_dx)
        self.temb = LinearW.make(g("time_emb_proj.weight"), g("time_emb_proj.bias"), dev, need_dx=False)
        self.norm2 = NormW.make(g("norm2.weight"), g("norm2.bias"), dev)
        self.conv2 = ConvW.make(g("conv2.weight"), g("conv2.bias"), dev, need_dx)
        self.shortcut = None
        if prefix + "conv_shortcut.weight" in sd:
            self.shortcut = LinearW.make(g("conv_shortcut.weight"), g("conv_shortcut.bias"), dev, need_dx)
        self.row_bias = None  # filled per forward


class AttnLayer:
    """One diffusers CrossAttention module: frozen projections + (optional) LoRA processor wiring."""

    def __init__(self, sd, prefix, name, dev, heads, is_cross):
        g = lambda k: sd[prefix + k]
        self.name = name
        self.heads = heads
        self.is_cross = is_cross
        self.to_q = LinearW.make(g("to_q.weight"), None, dev)
        self.to_k = LinearW.make(g("to_k.weight"), None, dev, need_dx=not is_cross)
        self.to_v = LinearW.make(g("to_v.weight"), None, dev, need_dx=not is_cross)
        self.to_out = LinearW.make(g("to_out.0.weight"), g("to_out.0.bias"), dev)
        self.processor = None
        self.plan = None   # built by UNet._prepare


class _Transformer:
    def __init__(self, sd, prefix, name_prefix, dev, heads, need_dx_in):
        g = lambda k: sd[prefix + k]
        self.norm = NormW.make(g("norm.weight"), g("norm.bias"), dev)
        self.proj_in = LinearW.make(g("proj_in.weight"), g("proj_in.bias"), dev, need_dx_in)
        b = prefix + "transformer_blocks.0."
        self.ln1 = NormW.make(sd[b + "norm1.weight"], sd[b + "norm1.bias"], dev)
        self.ln2 = NormW.make(sd[b + "norm2.weight"], sd[b + "norm2.bias"], dev)
        self.ln3 = NormW.make(sd[b + "norm3.weight"], sd[b + "norm3.bias"], dev)
        self.attn1 = AttnLayer(sd, b + "attn1.", name_prefix + "transformer_blocks.0.attn1.processor", dev, heads, False)
        self.attn2 = AttnLayer(sd, b + "attn2.", name_prefix + "transformer_blocks.0.attn2.processor", dev, heads, True)
        self.ff1 = LinearW.make(sd[b + "ff.net.0.proj.weight"], sd[b + "ff.net.0.proj.bias"], dev)
        self.ff2 = LinearW.make(sd[b + "ff.net.2.weight"], sd[b + "ff.net.2.bias"], dev)
        self.proj_out = LinearW.make(g("proj_out.weight"), g("proj_out.bias"), dev)


class UNetWeights:
    """Frozen SD-1.5 UNet weights converted once to the kernels' layouts (bf16, [out, ky, kx, in], transposed copies for
    the dX GEMMs).  `sd` uses diffusers' key names (e.g. the tensors of unet/diffusion_pytorch_model.safetensors)."""

    def __init__(self, sd: Dict[str, torch.Tensor], device, config: Optional[dict] = None):
        cfg = dict(SD15_CONFIG)
        cfg.update(config or {})
        self.cfg = cfg
        dev = device
        ch = list(cfg["block_out_channels"])
        layers = cfg["layers_per_block"]
        heads = cfg["attention_head_dim"]
        self.conv_in = ConvW.make(sd["conv_in.weight"], sd["conv_in.bias"], dev, need_dx=False)
        self.time1 = LinearW.make(sd["time_embedding.linear_1.weight"], sd["time_embedding.linear_1.bias"], dev, False)
        self.time2 = LinearW.make(sd["time_embedding.linear_2.weight"], sd["time_embedding.linear_2.bias"], dev, False)
        self.down = []
        self.attn_layers: "OrderedDict[str, AttnLayer]" = OrderedDict()
        first = True
        for i, typ in enumerate(cfg["down_block_types"]):
            blk = SimpleNamespace(resnets=[], attns=[], down=None)
            for j in range(layers):
                # nothing trainable sits upstream of the very first resnet: its dX is never needed
                blk.resnets.append(_Resnet(sd, f"down_blocks.{i}.resnets.{j}.", dev, need_dx=not first))
                if typ == "CrossAttnDownBlock2D":
                    blk.attns.append(_Transformer(sd, f"down_blocks.{i}.attentions.{j}.", f"down_blocks.{i}.attentions.{j}.",
                                                  dev, heads, need_dx_in=not first))
                first = False
            if i != len(ch) - 1:
                blk.down = ConvW.make(sd[f"down_blocks.{i}.downsamplers.0.conv.weight"],
                                      sd[f"down_blocks.{i}.downsamplers.0.conv.bias"], dev)
            self.down.append(blk)
        self.up = []
        for i, typ in enumerate(cfg["up_block_types"]):
            blk = SimpleNamespace(resnets=[], attns=[], up=None)
            for j in range(layers + 1):
                blk.resnets.append(_Resnet(sd, f"up_blocks.{i}.resnets.{j}.", dev, True))
                if typ == "CrossAttnUpBlock2D":
                    blk.attns.append(_Transformer(sd, f"up_blocks.{i}.attentions.{j}.", f"up_blocks.{i}.attentions.{j}.",
                                                  dev, heads, True))
            if i != len(ch) - 1:
                blk.up = ConvW.make(sd[f"up_blocks.{i}.upsamplers.0.conv.weight"], sd[f"up_blocks.{i}.upsamplers.0.conv.bias"], dev)
            self.up.append(blk)
        self.mid = SimpleNamespace(
            resnets=[_Resnet(sd, "mid_block.resnets.0.", dev, True), _Resnet(sd, "mid_block.resnets.1.", dev, True)],
            attn=_Transformer(sd, "mid_block.attentions.0.", "mid_block.attentions.0.", dev, heads, True))
        self.temb_cat = None
        self.norm_out = NormW.make(sd["conv_norm_out.weight"], sd["conv_norm_out.bias"], dev)
        self.conv_out_w = sd["conv_out.weight"].to(device=dev, dtype=BF16).permute(0, 2, 3, 1).contiguous()
        self.conv_out_b = sd["conv_out.bias"].to(device=dev, dtype=BF16).float().contiguous()
        # attn_processors key order = diffusers module registration order: down_blocks, up_blocks, mid_block
        for blk in self.down:
            for t in blk.attns:
                self.attn_layers[t.attn1.name] = t.attn1
                self.attn_layers[t.attn2.name] = t.attn2
        for blk in self.up:
            for t in blk.attns:
                self.attn_layers[t.attn1.name] = t.attn1
                self.attn_layers[t.attn2.name] = t.attn2
        self.attn_layers[self.mid.attn.attn1.name] = self.mid.attn.attn1
        self.attn_layers[self.mid.attn.attn2.name] = self.mid.attn.attn2

    def all_resnets(self) -> List[_Resnet]:
        out = []
        for blk in self.down:
            out += blk.resnets
        out += self.mid.resnets
        for blk in self.up:
            out += blk.resnets
        return out


# ---------------------------------------------------------------------------------------------------- forward program
def resnet_fwd(ctx: Ctx, W: UNetWeights, r: _Resnet, x: Var) -> Var:
    G, eps = W.cfg["norm_num_groups"], W.cfg["norm_eps"]
    n, H, Wd, Cin = x.data.shape
    h = E.groupnorm(ctx, x, r.norm1, G, eps, True)
    h = E.conv3x3(ctx, h, r.conv1, row_bias=r.row_bias)
    h = E.groupnorm(ctx, h, r.norm2, G, eps, True)
    if r.shortcut is not None:
        cout = r.shortcut.w.shape[0]
        xs = E.linear(ctx, x, r.shortcut, out_shape=(n, H, Wd, cout))
    else:
        xs = x
    return E.conv3x3(ctx, h, r.conv2, residual=xs)


def transformer_fwd(ctx: Ctx, W: UNetWeights, t: _Transformer, x: Var, ehs: Var, attn_fn) -> Var:
    G = W.cfg["norm_num_groups"]
    n, H, Wd, Cc = x.data.shape
    h = E.groupnorm(ctx, x, t.norm, G, 1e-6, False)
    h = E.linear(ctx, h, t.proj_in, out_shape=(n, H * Wd, Cc))
    # BasicTransformerBlock
    a = attn_fn(ctx, t.attn1, E.layernorm(ctx, h, t.ln1), None, h)
    a = attn_fn(ctx, t.attn2, E.layernorm(ctx, a, t.ln2), ehs, a)
    f = E.linear(ctx, E.layernorm(ctx, a, t.ln3), t.ff1)
    f = E.geglu(ctx, f)
    a = E.linear(ctx, f, t.ff2, residual=a)
    return E.linear(ctx, a, t.proj_out, residual=x, out_shape=(n, H, Wd, Cc))


def unet_forward(ctx: Ctx, W: UNetWeights, sample: torch.Tensor, timesteps: torch.Tensor, ehs: Var, attn_fn) -> Var:
    """sample: NCHW fp32 [B, 4, H, W]; returns Var of the NHWC bf16 activation feeding conv_out (post GN+SiLU)."""
    cfg = W.cfg
    B = sample.shape[0]
    ch0 = cfg["block_out_channels"][0]
    temb = ops.timestep_embedding(timesteps, ch0)
    temb = ops.small_linear(temb, W.time1.w, W.time1.bias, silu_out=True)
    temb = ops.small_linear(temb, W.time2.w, W.time2.bias)
    # every ResnetBlock2D.time_emb_proj in ONE launch: the stacked [sum(Cout), 1280] matrix is built once; each resnet's conv1
    # epilogue then reads its slice of the [B, sum(Cout)] result (row pitch = sum(Cout))
    if W.temb_cat is None:
        rs = W.all_resnets()
        W.temb_cat = (torch.cat([r.temb.w for r in rs], 0).contiguous(), torch.cat([r.temb.bias for r in rs], 0).contiguous())
        off = 0
        for r in rs:
            r.temb_off, off = off, off + r.temb.w.shape[0]
    tall = ops.small_linear(temb, W.temb_cat[0], W.temb_cat[1], silu_in=True)
    for r in W.all_resnets():
        r.row_bias = tall[:, r.temb_off:r.temb_off + r.temb.w.shape[0]]
    h = Var(ops.conv_in(sample, W.conv_in.w.view(ch0, 3, 3, -1), W.conv_in.bias, ch0), rg=False)
    skips = [h]
    for blk in W.down:
        for j, r in enumerate(blk.resnets):
            h = resnet_fwd(ctx, W, r, h)
            if blk.attns:
                h = transformer_fwd(ctx, W, blk.attns[j], h, ehs, attn_fn)
            skips.append(h)
        if blk.down is not None:
            h = E.conv3x3(ctx, h, blk.down, stride=2, pad_lo=1)
            skips.append(h)
    h = resnet_fwd(ctx, W, W.mid.resnets[0], h)
    h = transformer_fwd(ctx, W, W.mid.attn, h, ehs, attn_fn)
    h = resnet_fwd(ctx, W, W.mid.resnets[1], h)
    for blk in W.up:
        for j, r in enumerate(blk.resnets):
            h = resnet_fwd(ctx, W, r, E.concat(ctx, h, skips.pop()))
            if blk.attns:
                h = transformer_fwd(ctx, W, blk.attns[j], h, ehs, attn_fn)
        if blk.up is not None:
            h = E.conv3x3(ctx, E.upsample2x(ctx, h), blk.up)
    return E.groupnorm(ctx, h, W.norm_out, cfg["norm_num_groups"], cfg["norm_eps"], True)


def conv_out_fwd(ctx: Ctx, W: UNetWeights, h: Var) -> Var:
    """NHWC bf16 -> NCHW fp32 noise prediction (the tensor `.sample` of the reference UNet)."""
    y = ops.conv_out(h.data, W.conv_out_w, W.conv_out_b)
    out = Var(y, rg=h.rg)
    if ctx.tape is not None and out.rg:
        def bwd():
            dy = out.grad
            out.grad = None
            if dy is None:
                return
            E.give_tensor(h, ops.conv_out_bwd(dy, W.conv_out_w, h.data.shape[-1]))

        ctx.tape.record(bwd)
    return out


def synthetic_state_dict(config: Optional[dict] = None, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Random-init weights with diffusers' key names / shapes (no SD-1.5 checkpoint is reachable offline).
    Distribution: W ~ N(0, 1/fan_in), biases 0.02 N, norm gamma 1 + 0.1 N, beta 0.1 N.  Used by bench.py; the parity
    tests instead copy the oracle's state dict."""
    cfg = dict(SD15_CONFIG)
    cfg.update(config or {})
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    ch = list(cfg["block_out_channels"])
    temb = ch[0] * 4
    xd = cfg["cross_attention_dim"]

    def lin(name, n, k, bias=True):
        sd[name + ".weight"] = torch.randn(n, k, generator=g) / math.sqrt(k)
        if bias:
            sd[name + ".bias"] = 0.02 * torch.randn(n, generator=g)

    def conv(name, co, ci, ks):
        sd[name + ".weight"] = torch.randn(co, ci, ks, ks, generator=g) / math.sqrt(ci * ks * ks)
        sd[name + ".bias"] = 0.02 * torch.randn(co, generator=g)

    def norm(name, c):
        sd[name + ".weight"] = 1 + 0.1 * torch.randn(c, generator=g)
        sd[name + ".bias"] = 0.1 * torch.randn(c, generator=g)

    def resnet(p, ci, co):
        norm(p + "norm1", ci); conv(p + "conv1", co, ci, 3); lin(p + "time_emb_proj", co, temb)
        norm(p + "norm2", co); conv(p + "conv2", co, co, 3)
        if ci != co:
            conv(p + "conv_shortcut", co, ci, 1)

    def transformer(p, c):
        norm(p + "norm", c); conv(p + "proj_in", c, c, 1)
        b = p + "transformer_blocks.0."
        for n_ in ("norm1", "norm2", "norm3"):
            norm(b + n_, c)
        for a, kv in (("attn1", c), ("attn2", xd)):
            lin(b + a + ".to_q", c, c, False); lin(b + a + ".to_k", c, kv, False); lin(b + a + ".to_v", c, kv, False)
            lin(b + a + ".to_out.0", c, c)
        lin(b + "ff.net.0.proj", 8 * c, c); lin(b + "ff.net.2", c, 4 * c)
        conv(p + "proj_out", c, c, 1)

    conv("conv_in", ch[0], cfg["in_channels"], 3)
    lin("time_embedding.linear_1", temb, ch[0]); lin("time_embedding.linear_2", temb, temb)
    out = ch[0]
    L = cfg["layers_per_block"]
    for i, typ in enumerate(cfg["down_block_types"]):
        inp, out = out, ch[i]
        for j in range(L):
            resnet(f"down_blocks.{i}.resnets.{j}.", inp if j == 0 else out, out)
            if typ == "CrossAttnDownBlock2D":
                transformer(f"down_blocks.{i}.attentions.{j}.", out)
        if i != len(ch) - 1:
            conv(f"down_blocks.{i}.downsamplers.0.conv", out, out, 3)
    resnet("mid_block.resnets.0.", ch[-1], ch[-1]); transformer("mid_block.attentions.0.", ch[-1]); resnet("mid_block.resnets.1.", ch[-1], ch[-1])
    rev = list(reversed(ch))
    out = rev[0]
    for i, typ in enumerate(cfg["up_block_types"]):
        prev, out = out, rev[i]
        inp = rev[min(i + 1, len(ch) - 1)]
        for j in range(L + 1):
            skip = inp if j == L else out
            rin = prev if j == 0 else out
            resnet(f"up_blocks.{i}.resnets.{j}.", rin + skip, out)
            if typ == "CrossAttnUpBlock2D":
                transformer(f"up_blocks.{i}.attentions.{j}.", out)
        if i != len(ch) - 1:
            conv(f"up_blocks.{i}.upsamplers.0.conv", out, out, 3)
    norm("conv_norm_out", ch[0]); conv("conv_out", cfg["out_channels"], ch[0], 3)
    return sd
