"""ORACLE (tests only): the SD-2.x options on top of the SD-1.5 oracles of oracle/, restated from diffusers 0.13.

* UNet: `attention_head_dim` per block (the number of heads: down block i takes list[i], up block i reversed(list)[i], the mid
  block list[-1]; the projection widths do not depend on it, so the oracle is built with one head and each CrossAttention is
  given its block's head count and 1/sqrt(head dim) scale), `use_linear_projection` ([C, C] proj_in / proj_out linears on the
  [B, HW, C] tokens: the same arithmetic as the 1x1 convs, so a linear-projection state dict is loaded by viewing those weights
  as [C, C, 1, 1]), `cross_attention_dim` (already a parameter of the SD-1.5 oracle), `upcast_attention` (fp32 throughout here).
* Schedulers with prediction_type "v_prediction" (diffusers 0.13):
    DDIMScheduler.step              x0 = sqrt(a_t) x - sqrt(1 - a_t) v;  eps = sqrt(a_t) v + sqrt(1 - a_t) x
    DPMSolverMultistepScheduler     convert_model_output (dpmsolver++): x0 = alpha_t x - sigma_t v
    PNDMScheduler._get_prev_sample  model_output = sqrt(a_t) model_output + sqrt(1 - a_t) sample, with a_t = alphas_cumprod of the
                                    `timestep` argument (t + ratio on the restart call), after the PLMS combination
* Text encoder: `clip_text_forward`, transformers' CLIPTextModel.forward with either MLP activation (`quick_gelu` of SD-1.5,
  the exact erf `gelu` of SD-2's OpenCLIP-H tower); pinned to transformers.CLIPTextModel at SD21_TEXT_CONFIG and to
  oracle/clip_ref.py at the SD-1.5 activation (tests/test_sd2.py)."""
import torch

from oracle import sampler_ref as SR
from oracle import unet_ref as UR
from tests.test_pndm import PNDMPLMS


def block_heads(cfg):
    h = cfg["attention_head_dim"]
    n = len(cfg["down_block_types"])
    h = [h] * n if isinstance(h, int) else list(h)
    return h, h[::-1], h[-1]


def unet(cfg) -> UR.UNet2DConditionModel:
    """The oracle UNet of an SD-2-style config (per-block heads; keys of a conv-projection state dict)."""
    base = {k: v for k, v in cfg.items() if k not in ("use_linear_projection", "upcast_attention")}
    base["attention_head_dim"] = 1
    m = UR.UNet2DConditionModel(**base)
    m.config.attention_head_dim = cfg["attention_head_dim"]
    down, up, mid = block_heads(dict(UR.SD15_CONFIG, **cfg))

    def set_heads(blocks, heads):
        for blk, h in zip(blocks, heads):
            for t in getattr(blk, "attentions", None) or []:
                for a in (t.transformer_blocks[0].attn1, t.transformer_blocks[0].attn2):
                    a.heads = h
                    a.scale = (a.to_q.weight.shape[0] // h) ** -0.5

    set_heads(m.down_blocks, down)
    set_heads(m.up_blocks, up)
    set_heads([m.mid_block], [mid])
    return m


def to_linear_projection(sd):
    """A conv-projection state dict as a use_linear_projection checkpoint stores it: proj_in / proj_out weights [C, C]."""
    return {k: (v.reshape(v.shape[0], v.shape[1]) if k.endswith(("proj_in.weight", "proj_out.weight")) else v) for k, v in sd.items()}


def cfg_ddim_step_v(v_uncond, v_cond, x, t, num_inference_steps, guidance, ac=None):
    ac = SR.alphas_cumprod() if ac is None else ac
    v = v_uncond + guidance * (v_cond - v_uncond)
    prev = int(t) - 1000 // num_inference_steps
    a_t = ac[int(t)]
    a_p = ac[prev] if prev >= 0 else ac[0]
    x0 = a_t.sqrt() * x - (1 - a_t).sqrt() * v
    eps = a_t.sqrt() * v + (1 - a_t).sqrt() * x
    return (a_p.sqrt() * x0 + (1 - a_p).sqrt() * eps).to(x.dtype)


class DPMSolverPP2MV(SR.DPMSolverPP2M):
    """DPMSolverPP2M with prediction_type "v_prediction": only the data prediction differs."""

    def step(self, v, timestep, x):
        i = self.timesteps.index(int(timestep))
        n = len(self.timesteps)
        prev = 0 if i == n - 1 else self.timesteps[i + 1]
        final = (i == n - 1) and self.lower_order_final and n < 15
        xd, vd = x.double(), v.double()
        x0 = self.alpha_t[timestep] * xd - self.sigma_t[timestep] * vd
        self.model_outputs = [self.model_outputs[1], x0]
        if self.lower_order_nums < 1 or final:
            out = self._first_order(x0, int(timestep), prev, xd)
        else:
            out = self._second_order(x0, self.model_outputs[0], self.timesteps[i - 1], int(timestep), prev, xd)
        if self.lower_order_nums < 2:
            self.lower_order_nums += 1
        return out.to(x.dtype)


class PNDMPLMSV(PNDMPLMS):
    """PNDMPLMS with prediction_type "v_prediction": the history holds v, converted to eps in _get_prev_sample."""

    def _get_prev_sample(self, sample, timestep, prev_timestep, model_output):
        a_t = self.alphas_cumprod[timestep]
        model_output = a_t ** 0.5 * model_output + (1 - a_t) ** 0.5 * sample
        return super()._get_prev_sample(sample, timestep, prev_timestep, model_output)


# ------------------------------------------------------------------------------------------------ restatements of the v kernels
def solver_v_step_restated(v2, latents, x0_prev, coef, step_ctr, guidance, kind):
    """torch restatement of cl_cfg_solver_step_v_dev (same operation order), in the dtype of `latents`."""
    c = [float(v) for v in coef[int(step_ctr)]]
    u, cc = v2.reshape(2, -1)
    v = (u + guidance * (cc - u)).view_as(latents)
    x0 = c[0] * latents - c[1] * v
    if kind == 0:
        latents.copy_(c[2] * x0 + c[3] * (c[0] * v + c[1] * latents))
    else:
        latents.copy_(c[2] * latents + c[3] * x0 + c[4] * x0_prev)
        x0_prev.copy_(x0)
    step_ctr += 1


def plms_v_step_restated(v2, latents, ring, saved, rows, step_ctr, guidance):
    """torch restatement of cl_cfg_plms_step_v_dev (same operation order), in the dtype of `latents`."""
    r = [float(x) for x in rows[int(step_ctr)]]
    u, c = v2.reshape(2, -1)
    v = (u + guidance * (c - u)).view_as(latents)
    flags = int(r[7])
    vp = r[3] * v + r[4] * ring[0] + r[5] * ring[1] + r[6] * ring[2]
    s = saved.clone() if flags & 4 else latents.clone()
    if flags & 2:
        saved.copy_(s)
    latents.copy_(r[1] * s + r[2] * (r[8] * vp + r[9] * s))
    if flags & 1:
        ring[2].copy_(ring[1])
        ring[1].copy_(ring[0])
        ring[0].copy_(v)
    step_ctr += 1


def gelu_restated(x):
    xf = x.float()
    x.copy_(torch.nn.functional.gelu(xf).to(torch.bfloat16))
    return x


def clip_text_forward(sd, ids, cfg):
    """last_hidden_state of CLIPTextModel with state dict `sd` (transformers key names), fp32, for hidden_act quick_gelu or gelu:
    pre-LN layers x + attn(LN1(x)), x + mlp(LN2(x)); q/k/v/out with bias, causal softmax at scale d^-0.5; final LayerNorm."""
    import torch.nn.functional as F

    pre = "text_model." if any(k.startswith("text_model.") for k in sd) else ""
    g = lambda k: sd[pre + k].float()
    B, T = ids.shape
    H, Cw, eps = cfg["num_attention_heads"], cfg["hidden_size"], cfg["layer_norm_eps"]
    d = Cw // H
    act = {"gelu": F.gelu, "quick_gelu": lambda f: f * torch.sigmoid(1.702 * f)}[cfg["hidden_act"]]
    x = g("embeddings.token_embedding.weight")[ids] + g("embeddings.position_embedding.weight")[:T][None]
    mask = torch.full((T, T), float("-inf"), device=x.device).triu(1)
    for i in range(cfg["num_hidden_layers"]):
        m = f"encoder.layers.{i}."
        h = F.layer_norm(x, (Cw,), g(m + "layer_norm1.weight"), g(m + "layer_norm1.bias"), eps)
        q, k, v = (F.linear(h, g(m + f"self_attn.{n}_proj.weight"), g(m + f"self_attn.{n}_proj.bias")).reshape(B, T, H, d).transpose(1, 2)
                   for n in "qkv")
        a = torch.softmax((q * d ** -0.5) @ k.transpose(-1, -2) + mask, -1) @ v
        x = x + F.linear(a.transpose(1, 2).reshape(B, T, Cw), g(m + "self_attn.out_proj.weight"), g(m + "self_attn.out_proj.bias"))
        h = F.layer_norm(x, (Cw,), g(m + "layer_norm2.weight"), g(m + "layer_norm2.bias"), eps)
        x = x + F.linear(act(F.linear(h, g(m + "mlp.fc1.weight"), g(m + "mlp.fc1.bias"))), g(m + "mlp.fc2.weight"), g(m + "mlp.fc2.bias"))
    return F.layer_norm(x, (Cw,), g("final_layer_norm.weight"), g("final_layer_norm.bias"), eps)
