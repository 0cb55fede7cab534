"""`AutoencoderKL` — the frozen SD-1.5 VAE either side of the hot path, on the same sm_90a kernels (SURVEY.md 8f rank 3):

  latents = vae.encode(pixel_values).latent_dist.sample() * vae.config.scaling_factor      train_text_to_image_control_lora.py:753-754
  image   = vae.decode(latents / vae.config.scaling_factor).sample                          StableDiffusionPipeline (…:829-843, apps/*)

Forward only (the reference freezes the VAE, train_…:430).  Every conv runs on the wgmma implicit-GEMM kernel, the norms on
the GroupNorm kernels; the mid-block `AttentionBlock` has ONE head of width 512 (beyond the flash kernels' head-dim range), so
it runs as GEMMs around a row-softmax kernel (scores in fp32).  The 1x1 `quant_conv` is folded into `encoder.conv_out`, the
1x1 `post_quant_conv` into `decoder.conv_in` (exact: weight products; its bias becomes a per-channel shift of the latents).
State-dict keys = diffusers' `vae/diffusion_pytorch_model.safetensors` (0.13 names; the later `to_q / to_k / to_v / to_out.0`
attention names are accepted as well).
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn as nn

from . import engine as E
from . import ops
from .engine import ConvW, Ctx, LinearW, NormW, Var

BF16 = torch.bfloat16

SD15_VAE_CONFIG = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=(128, 256, 512, 512),
                       layers_per_block=2, norm_num_groups=32, scaling_factor=0.18215)


def synthetic_vae_state_dict(config: Optional[dict] = None, seed: int = 0) -> Dict[str, torch.Tensor]:
    """State dict of a diffusers-0.13 AutoencoderKL with this config (exact key names and shapes of the published SD-1.5 `vae/`
    checkpoint for the default config: 83 653 863 parameters), filled with seeded random values."""
    cfg = dict(SD15_VAE_CONFIG)
    cfg.update(config or {})
    ch, L, lat = list(cfg["block_out_channels"]), cfg["layers_per_block"], cfg["latent_channels"]
    g = torch.Generator().manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}

    def conv(name, cout, cin, k):
        sd[name + ".weight"] = torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)
        sd[name + ".bias"] = 0.02 * torch.randn(cout, generator=g)

    def lin(name, cout, cin):
        sd[name + ".weight"] = torch.randn(cout, cin, generator=g) / math.sqrt(cin)
        sd[name + ".bias"] = 0.02 * torch.randn(cout, generator=g)

    def norm(name, c):
        sd[name + ".weight"] = 1.0 + 0.1 * torch.randn(c, generator=g)
        sd[name + ".bias"] = 0.1 * torch.randn(c, generator=g)

    def resnet(p, cin, cout):
        norm(p + "norm1", cin); conv(p + "conv1", cout, cin, 3); norm(p + "norm2", cout); conv(p + "conv2", cout, cout, 3)
        if cin != cout:
            conv(p + "conv_shortcut", cout, cin, 1)

    def mid(p, c):
        norm(p + "attentions.0.group_norm", c)
        for k in ("query", "key", "value", "proj_attn"):
            lin(p + "attentions.0." + k, c, c)
        resnet(p + "resnets.0.", c, c); resnet(p + "resnets.1.", c, c)

    conv("encoder.conv_in", ch[0], cfg["in_channels"], 3)
    cin = ch[0]
    for i, c in enumerate(ch):
        for j in range(L):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}.", cin, c)
            cin = c
        if i != len(ch) - 1:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", c, c, 3)
    mid("encoder.mid_block.", ch[-1])
    norm("encoder.conv_norm_out", ch[-1]); conv("encoder.conv_out", 2 * lat, ch[-1], 3)
    conv("decoder.conv_in", ch[-1], lat, 3)
    mid("decoder.mid_block.", ch[-1])
    rev = ch[::-1]
    cin = rev[0]
    for i, c in enumerate(rev):
        for j in range(L + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}.", cin, c)
            cin = c
        if i != len(rev) - 1:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", c, c, 3)
    norm("decoder.conv_norm_out", rev[-1]); conv("decoder.conv_out", cfg["out_channels"], rev[-1], 3)
    conv("quant_conv", 2 * lat, 2 * lat, 1); conv("post_quant_conv", lat, lat, 1)
    # near-identity 1x1 quant convs keep the latent statistics of the encoder (and post_quant_conv well conditioned: it is inverted)
    sd["quant_conv.weight"] = torch.eye(2 * lat).view(2 * lat, 2 * lat, 1, 1) + 0.05 * sd["quant_conv.weight"]
    sd["post_quant_conv.weight"] = torch.eye(lat).view(lat, lat, 1, 1) + 0.05 * sd["post_quant_conv.weight"]
    return sd


class DiagonalGaussianDistribution:
    """diffusers' DiagonalGaussianDistribution over NCHW fp32 moments (logvar clamped to [-30, 20])."""

    def __init__(self, mean: torch.Tensor, logvar: torch.Tensor):
        self.mean = mean
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        eps = torch.randn(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype)
        return self.mean + self.std * eps

    def mode(self) -> torch.Tensor:
        return self.mean


class _Resnet:
    def __init__(self, sd, p, dev):
        g = lambda k: sd[p + k]
        self.norm1 = NormW.make(g("norm1.weight"), g("norm1.bias"), dev)
        self.conv1 = ConvW.make(g("conv1.weight"), g("conv1.bias"), dev, need_dx=False)
        self.norm2 = NormW.make(g("norm2.weight"), g("norm2.bias"), dev)
        self.conv2 = ConvW.make(g("conv2.weight"), g("conv2.bias"), dev, need_dx=False)
        self.shortcut = None
        if p + "conv_shortcut.weight" in sd:
            self.shortcut = LinearW.make(g("conv_shortcut.weight"), g("conv_shortcut.bias"), dev, need_dx=False)


class _Attn:
    def __init__(self, sd, p, dev):
        def pick(*names):
            for nm in names:
                if p + nm + ".weight" in sd:
                    return sd[p + nm + ".weight"], sd[p + nm + ".bias"]
            raise KeyError(p + names[0])

        gw, gb = pick("group_norm")
        self.norm = NormW.make(gw, gb, dev)
        self.q = LinearW.make(*pick("query", "to_q"), dev, need_dx=False)
        self.k = LinearW.make(*pick("key", "to_k"), dev, need_dx=False)
        self.v = LinearW.make(*pick("value", "to_v"), dev, need_dx=False)
        self.proj = LinearW.make(*pick("proj_attn", "to_out.0"), dev, need_dx=False)


class AutoencoderKL(nn.Module):
    def __init__(self, sd: Dict[str, torch.Tensor], device="cuda", config: Optional[dict] = None):
        super().__init__()
        cfg = dict(SD15_VAE_CONFIG)
        cfg.update(config or {})
        self.config = SimpleNamespace(**cfg)
        dev = torch.device(device)
        self.device_ = dev
        ch, L, lat = list(cfg["block_out_channels"]), cfg["layers_per_block"], cfg["latent_channels"]
        self.G = cfg["norm_num_groups"]
        f32 = lambda t: t.detach().to(torch.float32).cpu()
        # ---------------- encoder
        self.enc_conv_in_w = sd["encoder.conv_in.weight"].to(device=dev, dtype=BF16).permute(0, 2, 3, 1).contiguous()
        self.enc_conv_in_b = sd["encoder.conv_in.bias"].to(device=dev, dtype=BF16).float().contiguous()
        self.enc_down = []
        for i in range(len(ch)):
            blk = SimpleNamespace(resnets=[_Resnet(sd, f"encoder.down_blocks.{i}.resnets.{j}.", dev) for j in range(L)], down=None)
            k = f"encoder.down_blocks.{i}.downsamplers.0.conv.weight"
            if k in sd:
                blk.down = ConvW.make(sd[k], sd[k[:-6] + "bias"], dev, need_dx=False)
            self.enc_down.append(blk)
        self.enc_mid = SimpleNamespace(res=[_Resnet(sd, "encoder.mid_block.resnets.0.", dev), _Resnet(sd, "encoder.mid_block.resnets.1.", dev)],
                                       attn=_Attn(sd, "encoder.mid_block.attentions.0.", dev))
        self.enc_norm_out = NormW.make(sd["encoder.conv_norm_out.weight"], sd["encoder.conv_norm_out.bias"], dev)
        # quant_conv (1x1, 2*lat -> 2*lat) folded into conv_out:  W' = Wq Wc,  b' = Wq bc + bq
        wq, bq = f32(sd["quant_conv.weight"]).view(2 * lat, 2 * lat), f32(sd["quant_conv.bias"])
        wc, bc = f32(sd["encoder.conv_out.weight"]), f32(sd["encoder.conv_out.bias"])
        self.enc_conv_out = ConvW.make(torch.einsum("om,mikl->oikl", wq, wc), wq @ bc + bq, dev, need_dx=False)
        # ---------------- decoder
        # post_quant_conv folded into conv_in: conv_in(Wp z + bp) = conv_in'(z + Wp^-1 bp) with conv_in' = conv_in o Wp (exact; the
        # shift is applied to the latents before the zero-padded conv, which a folded bias could not reproduce at the borders)
        wp, bp = f32(sd["post_quant_conv.weight"]).view(lat, lat), f32(sd["post_quant_conv.bias"])
        wci = f32(sd["decoder.conv_in.weight"])
        self.dec_conv_in_w = torch.einsum("omkl,mc->ockl", wci, wp).to(device=dev, dtype=BF16).permute(0, 2, 3, 1).contiguous()
        self.dec_conv_in_b = sd["decoder.conv_in.bias"].to(device=dev, dtype=BF16).float().contiguous()
        self.dec_shift = torch.linalg.solve(wp.double(), bp.double()).float().to(dev).contiguous()       # Wp^-1 bp
        self.dec_mid = SimpleNamespace(res=[_Resnet(sd, "decoder.mid_block.resnets.0.", dev), _Resnet(sd, "decoder.mid_block.resnets.1.", dev)],
                                       attn=_Attn(sd, "decoder.mid_block.attentions.0.", dev))
        self.dec_up = []
        for i in range(len(ch)):
            blk = SimpleNamespace(resnets=[_Resnet(sd, f"decoder.up_blocks.{i}.resnets.{j}.", dev) for j in range(L + 1)], up=None)
            k = f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"
            if k in sd:
                blk.up = ConvW.make(sd[k], sd[k[:-6] + "bias"], dev, need_dx=False)
            self.dec_up.append(blk)
        self.dec_norm_out = NormW.make(sd["decoder.conv_norm_out.weight"], sd["decoder.conv_norm_out.bias"], dev)
        # conv_out has 3 output channels: padded to 4 (the GEMM wants N % 4 == 0), the extra plane is dropped
        wo, bo = f32(sd["decoder.conv_out.weight"]), f32(sd["decoder.conv_out.bias"])
        self.out_channels = wo.shape[0]
        pad = (-wo.shape[0]) % 4
        if pad:
            wo = torch.cat([wo, torch.zeros(pad, *wo.shape[1:])], 0)
            bo = torch.cat([bo, torch.zeros(pad)], 0)
        self.dec_conv_out = ConvW.make(wo, bo, dev, need_dx=False)

    # ------------------------------------------------------------------------------------------------ construction
    @classmethod
    def from_state_dict(cls, sd, device="cuda", config: Optional[dict] = None):
        return cls(sd, device, config)

    @classmethod
    def synthetic(cls, device="cuda", config: Optional[dict] = None, seed: int = 0):
        """Seeded random weights of the architecture (diffusers key names; W ~ N(0, 1/fan_in), norm gamma ~ 1): benchmarks and smoke runs
        on machines without the published checkpoint."""
        return cls(synthetic_vae_state_dict(config, seed), device, config)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder: Optional[str] = None, device="cuda", **unused):
        """Local diffusers-format directory (`<root>[/subfolder]/config.json` + `diffusion_pytorch_model.safetensors|.bin`), the
        layout `AutoencoderKL.from_pretrained(..., subfolder="vae")` reads at train_text_to_image_control_lora.py:404-406."""
        import json
        import os

        root = os.path.join(pretrained_model_name_or_path, subfolder) if subfolder else str(pretrained_model_name_or_path)
        if not os.path.isdir(root):
            raise FileNotFoundError(f"{root}: not a local directory (hub download is not available)")
        config = None
        if os.path.isfile(os.path.join(root, "config.json")):
            with open(os.path.join(root, "config.json")) as f:
                raw = json.load(f)
            config = {k: (tuple(v) if isinstance(v, list) else v) for k, v in raw.items() if k in SD15_VAE_CONFIG}
        st = os.path.join(root, "diffusion_pytorch_model.safetensors")
        if os.path.isfile(st):
            from safetensors.torch import load_file

            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(root, "diffusion_pytorch_model.bin"), map_location="cpu")
        return cls(sd, device, config)

    # ------------------------------------------------------------------------------------------------ building blocks
    def _resnet(self, ctx: Ctx, r: _Resnet, x: Var) -> Var:
        n, H, W, _ = x.data.shape
        h = E.groupnorm(ctx, x, r.norm1, self.G, 1e-6, True)
        h = E.conv3x3(ctx, h, r.conv1)
        h = E.groupnorm(ctx, h, r.norm2, self.G, 1e-6, True)
        xs = x if r.shortcut is None else E.linear(ctx, x, r.shortcut, out_shape=(n, H, W, r.shortcut.w.shape[0]))
        return E.conv3x3(ctx, h, r.conv2, residual=xs)

    def _attention(self, ctx: Ctx, a: _Attn, x: Var) -> Var:
        """AttentionBlock with one head: softmax(q k^T / sqrt(C)) v per image as GEMMs around a row-softmax (fp32 scores)."""
        n, H, W, C = x.data.shape
        HW = H * W
        hn = E.groupnorm(ctx, x, a.norm, self.G, 1e-6, False).data.view(n * HW, C)
        q = ops.gemm(hn, a.q.w, bias=a.q.bias)
        k = ops.gemm(hn, a.k.w, bias=a.k.bias)
        o = torch.empty(n * HW, C, device=x.data.device, dtype=BF16)
        scale = 1.0 / math.sqrt(C)
        for i in range(n):
            sl = slice(i * HW, (i + 1) * HW)
            s = ops.gemm(q[sl], k[sl], out_fp32=True)                         # [HW, HW] = q k^T
            p = ops.softmax_rows(s, scale)                                    # bf16
            vt = ops.gemm(a.v.w, hn[sl])                                      # [C, HW] = Wv h^T = V^T without its bias
            ops.gemm(p, vt, bias=a.v.bias, out=o[sl])                         # P V + bv  (rows of P sum to 1)
        y = ops.gemm(o, a.proj.w, bias=a.proj.bias, residual=x.data.view(n * HW, C))
        return Var(y.view(n, H, W, C))

    # ------------------------------------------------------------------------------------------------ public API
    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """x [n, 3, H, W] in [-1, 1] (any float dtype) -> object with `.latent_dist` (DiagonalGaussianDistribution, fp32 NCHW)."""
        from ._lib import require_cuda

        require_cuda(x.device, "AutoencoderKL")
        ctx = Ctx(tape=None)
        cin = self.enc_conv_in_w.shape[-1]
        h = Var(ops.conv_in(x.detach().float().contiguous(), self.enc_conv_in_w.view(self.enc_conv_in_w.shape[0], 3, 3, cin),
                            self.enc_conv_in_b, self.enc_conv_in_w.shape[0]))
        for blk in self.enc_down:
            for r in blk.resnets:
                h = self._resnet(ctx, r, h)
            if blk.down is not None:
                h = E.conv3x3(ctx, h, blk.down, stride=2, pad_lo=0)              # F.pad(x, (0,1,0,1)) + stride-2 conv
        h = self._resnet(ctx, self.enc_mid.res[0], h)
        h = self._attention(ctx, self.enc_mid.attn, h)
        h = self._resnet(ctx, self.enc_mid.res[1], h)
        h = E.groupnorm(ctx, h, self.enc_norm_out, self.G, 1e-6, True)
        m = E.conv3x3(ctx, h, self.enc_conv_out)                                 # [n, h, w, 2*lat]  (quant_conv folded in)
        mom = ops.nhwc_to_nchw_f32(m.data)
        lat = self.config.latent_channels
        dist = DiagonalGaussianDistribution(mom[:, :lat].contiguous(), mom[:, lat:].contiguous())
        return SimpleNamespace(latent_dist=dist) if return_dict else (dist,)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True):
        """z [n, 4, h, w] (already divided by scaling_factor, like the reference's call) -> `.sample` [n, 3, 8h, 8w] fp32."""
        from ._lib import require_cuda

        require_cuda(z.device, "AutoencoderKL")
        ctx = Ctx(tape=None)
        zs = ops.channel_affine_nchw(z.detach().float().contiguous(), 1.0, self.dec_shift)
        c0 = self.dec_conv_in_w.shape[0]
        h = Var(ops.conv_in(zs, self.dec_conv_in_w.view(c0, 3, 3, -1), self.dec_conv_in_b, c0))
        h = self._resnet(ctx, self.dec_mid.res[0], h)
        h = self._attention(ctx, self.dec_mid.attn, h)
        h = self._resnet(ctx, self.dec_mid.res[1], h)
        for blk in self.dec_up:
            for r in blk.resnets:
                h = self._resnet(ctx, r, h)
            if blk.up is not None:
                h = E.conv3x3(ctx, E.upsample2x(ctx, h), blk.up)
        h = E.groupnorm(ctx, h, self.dec_norm_out, self.G, 1e-6, True)
        y = E.conv3x3(ctx, h, self.dec_conv_out)
        img = ops.nhwc_to_nchw_f32(y.data)[:, :self.out_channels].contiguous()
        return SimpleNamespace(sample=img) if return_dict else (img,)
