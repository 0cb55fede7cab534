"""`CLIPTextModel` — the frozen text encoder in front of the hot path (SURVEY.md 8f rank 3), on the same sm_90a kernels:

  encoder_hidden_states = text_encoder(batch["input_ids"])[0]                  train_text_to_image_control_lora.py:768
  (and the prompt embeddings of the pipelines, train_…:829-843, apps/gradio_*2image.py, mix_lora_and_control_lora.py)

Forward only (the reference freezes it, train_…:431).  SD-1.5 `text_encoder/config.json` = CLIP ViT-L/14 text tower: 12 pre-LN
transformer layers of width 768, 12 heads of 64, MLP 3072 with `quick_gelu`, 77 learned positions, vocabulary 49408, causal
self-attention, final LayerNorm; `[0]` of the output = `last_hidden_state` [B, 77, 768].  Per layer: LayerNorm kernel -> ONE
fused q|k|v projection (N = 2304, bias in the GEMM epilogue) -> causal attention of the 77-token sequence (one CTA per
(batch, head), fp32 online softmax) -> out-projection with bias + residual in the epilogue -> LayerNorm -> fc1 (+bias) ->
quick_gelu -> fc2 (+bias, +residual).  State-dict keys = transformers' `CLIPTextModel` (`text_model.embeddings.…`,
`text_model.encoder.layers.{i}.…`, `text_model.final_layer_norm.…`).  Tokenisation stays with `transformers.CLIPTokenizer`
(host-side string processing, not part of this path).
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn as nn

from . import ops

BF16 = torch.bfloat16

SD15_TEXT_CONFIG = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                        max_position_embeddings=77, layer_norm_eps=1e-5, hidden_act="quick_gelu")


class _Layer:
    def __init__(self, sd, p, dev):
        f32 = lambda k: sd[p + k].detach().to(dev, torch.float32).contiguous()
        w16 = lambda k: sd[p + k].detach().to(dev, BF16).contiguous()
        self.ln1 = (f32("layer_norm1.weight"), f32("layer_norm1.bias"))
        self.ln2 = (f32("layer_norm2.weight"), f32("layer_norm2.bias"))
        self.w_qkv = torch.cat([w16("self_attn.q_proj.weight"), w16("self_attn.k_proj.weight"), w16("self_attn.v_proj.weight")], 0).contiguous()
        self.b_qkv = torch.cat([f32("self_attn.q_proj.bias"), f32("self_attn.k_proj.bias"), f32("self_attn.v_proj.bias")], 0).contiguous()
        self.w_o, self.b_o = w16("self_attn.out_proj.weight"), f32("self_attn.out_proj.bias")
        self.w_fc1, self.b_fc1 = w16("mlp.fc1.weight"), f32("mlp.fc1.bias")
        self.w_fc2, self.b_fc2 = w16("mlp.fc2.weight"), f32("mlp.fc2.bias")


class CLIPTextModel(nn.Module):
    """Drop-in for the one call the reference makes: `text_encoder(input_ids)[0]` / `.last_hidden_state` (bf16 [B, T, 768])."""

    def __init__(self, sd: Dict[str, torch.Tensor], device="cuda", config: Optional[dict] = None):
        super().__init__()
        cfg = dict(SD15_TEXT_CONFIG)
        cfg.update(config or {})
        if cfg["hidden_act"] != "quick_gelu":
            raise NotImplementedError("CLIPTextModel: only the quick_gelu MLP of SD-1.5's text encoder is implemented")
        self.config = SimpleNamespace(**cfg)
        dev = torch.device(device)
        from ._lib import require_cuda

        require_cuda(dev, "CLIPTextModel")
        self.device_ = dev
        pre = "text_model." if any(k.startswith("text_model.") for k in sd) else ""
        self.tok = sd[pre + "embeddings.token_embedding.weight"].detach().to(dev, BF16).contiguous()
        self.pos = sd[pre + "embeddings.position_embedding.weight"].detach().to(dev, BF16).contiguous()
        self.layers = [_Layer(sd, f"{pre}encoder.layers.{i}.", dev) for i in range(cfg["num_hidden_layers"])]
        self.ln_f = (sd[pre + "final_layer_norm.weight"].detach().to(dev, torch.float32).contiguous(),
                     sd[pre + "final_layer_norm.bias"].detach().to(dev, torch.float32).contiguous())
        self.heads = cfg["num_attention_heads"]
        if cfg["hidden_size"] % self.heads or cfg["hidden_size"] // self.heads > 64:
            raise NotImplementedError("CLIPTextModel: head dim must divide the width and be <= 64")

    @classmethod
    def from_state_dict(cls, sd, device="cuda", config: Optional[dict] = None):
        return cls(sd, device, config)

    @classmethod
    def synthetic(cls, device="cuda", config: Optional[dict] = None, seed: int = 0):
        """Seeded random weights with transformers' key names (123 060 480 parameters for the SD-1.5 text tower): benchmarks / smoke
        runs on machines without the published checkpoint."""
        cfg = dict(SD15_TEXT_CONFIG)
        cfg.update(config or {})
        g = torch.Generator().manual_seed(seed)
        Cw, Fi = cfg["hidden_size"], cfg["intermediate_size"]
        sd = {"text_model.embeddings.token_embedding.weight": 0.02 * torch.randn(cfg["vocab_size"], Cw, generator=g),
              "text_model.embeddings.position_embedding.weight": 0.01 * torch.randn(cfg["max_position_embeddings"], Cw, generator=g)}
        for i in range(cfg["num_hidden_layers"]):
            p = f"text_model.encoder.layers.{i}."
            for name, (o, n) in {"self_attn.q_proj": (Cw, Cw), "self_attn.k_proj": (Cw, Cw), "self_attn.v_proj": (Cw, Cw),
                                 "self_attn.out_proj": (Cw, Cw), "mlp.fc1": (Fi, Cw), "mlp.fc2": (Cw, Fi)}.items():
                sd[p + name + ".weight"] = torch.randn(o, n, generator=g) / math.sqrt(n)
                sd[p + name + ".bias"] = 0.02 * torch.randn(o, generator=g)
            for ln in ("layer_norm1", "layer_norm2"):
                sd[p + ln + ".weight"] = 1.0 + 0.1 * torch.randn(Cw, generator=g)
                sd[p + ln + ".bias"] = 0.1 * torch.randn(Cw, generator=g)
        sd["text_model.final_layer_norm.weight"] = 1.0 + 0.1 * torch.randn(Cw, generator=g)
        sd["text_model.final_layer_norm.bias"] = 0.1 * torch.randn(Cw, generator=g)
        return cls(sd, device, cfg)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder: Optional[str] = None, device="cuda", **unused):
        """Local transformers-format directory (`<root>[/subfolder]/config.json` + `model.safetensors | pytorch_model.bin`), the
        layout `CLIPTextModel.from_pretrained(..., subfolder="text_encoder")` reads at train_text_to_image_control_lora.py:401-403."""
        import json
        import os

        root = os.path.join(pretrained_model_name_or_path, subfolder) if subfolder else str(pretrained_model_name_or_path)
        if not os.path.isdir(root):
            raise FileNotFoundError(f"{root}: not a local directory (hub download is not available)")
        config = None
        if os.path.isfile(os.path.join(root, "config.json")):
            with open(os.path.join(root, "config.json")) as f:
                raw = json.load(f)
            raw = raw.get("text_config", raw)
            config = {k: raw[k] for k in SD15_TEXT_CONFIG if k in raw}
        st = os.path.join(root, "model.safetensors")
        if os.path.isfile(st):
            from safetensors.torch import load_file

            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(root, "pytorch_model.bin"), map_location="cpu")
        return cls(sd, device, config)

    def requires_grad_(self, flag: bool = False):      # train_…:431 `text_encoder.requires_grad_(False)`: nothing is trainable here
        return self

    def to(self, *args, **kwargs):                      # train_…:445 `.to(accelerator.device, dtype=weight_dtype)`: already resident, bf16
        return self

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask=None, return_dict: bool = True):
        if attention_mask is not None:
            raise NotImplementedError("CLIPTextModel: the reference never passes an attention_mask (padded prompts attend causally)")
        if input_ids.device != self.device_:
            input_ids = input_ids.to(self.device_)
        ids = input_ids.to(torch.int64).contiguous()
        B, T = ids.shape
        cfg = self.config
        if T > cfg.max_position_embeddings:
            raise ValueError(f"sequence length {T} > max_position_embeddings {cfg.max_position_embeddings}")
        Cw = cfg.hidden_size
        x = ops.clip_embed(ids, self.tok, self.pos).view(B * T, Cw)
        scale = 1.0 / math.sqrt(Cw // self.heads)
        for L in self.layers:
            h, _ = ops.layernorm_fwd(x, L.ln1[0], L.ln1[1], cfg.layer_norm_eps)
            qkv = ops.gemm(h, L.w_qkv, bias=L.b_qkv)
            a = ops.causal_attention_small(qkv, B, T, self.heads, scale)
            x = ops.gemm(a, L.w_o, bias=L.b_o, residual=x)
            h, _ = ops.layernorm_fwd(x, L.ln2[0], L.ln2[1], cfg.layer_norm_eps)
            f = ops.quick_gelu_(ops.gemm(h, L.w_fc1, bias=L.b_fc1))
            x = ops.gemm(f, L.w_fc2, bias=L.b_fc2, residual=x)
        y, _ = ops.layernorm_fwd(x, self.ln_f[0], self.ln_f[1], cfg.layer_norm_eps)
        y = y.view(B, T, Cw)
        if not return_dict:
            return (y,)
        return _Output(last_hidden_state=y)


class _Output(dict):
    """`out[0]`, `out.last_hidden_state` and `out["last_hidden_state"]` like transformers' ModelOutput."""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.__dict__.update(kw)

    def __getitem__(self, k):
        if isinstance(k, int):
            return list(self.values())[k]
        return super().__getitem__(k)
