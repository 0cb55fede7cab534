"""Denoise loop on the CUDA UNet: classifier-free guidance + DDIM (eta = 0) or DPM-Solver++(2M), the inference call
pattern of the reference (`StableDiffusionPipeline.__call__` as used at train_text_to_image_control_lora.py:829-843 and
apps/gradio_canny2image.py:81-89; BASELINE config 3 = 50-step DDIM at batch 8 -> UNet batch 16; the reference swaps in
`DPMSolverMultistepScheduler` for validation / the apps: train_text_to_image_control_lora.py:817-823,
mix_lora_and_control_lora.py:80).

The control states do not depend on the timestep: `control_lora(guide)` runs once per image batch, every UNet evaluation
of the loop re-uses the injected states.  The guide must be tiled to the CFG batch 2B (SURVEY.md §3.3)."""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from . import ops


def sd15_alphas_cumprod(num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012) -> List[float]:
    """SD-1.5 scheduler constants: scaled-linear betas (diffusers `scaled_linear`), cumulative product of 1 - beta."""
    import math

    out, acc = [], 1.0
    s0, s1 = math.sqrt(beta_start), math.sqrt(beta_end)
    for i in range(num_train_timesteps):
        b = (s0 + (s1 - s0) * i / (num_train_timesteps - 1)) ** 2
        acc *= 1.0 - b
        out.append(acc)
    return out


def ddim_timesteps(num_inference_steps: int, num_train_timesteps: int = 1000, steps_offset: int = 1) -> List[int]:
    ratio = num_train_timesteps // num_inference_steps
    return [i * ratio + steps_offset for i in range(num_inference_steps)][::-1]


def ddim_coeffs(t: int, num_inference_steps: int, ac: List[float], num_train_timesteps: int = 1000) -> Tuple[float, float]:
    """(alpha_prod_t, alpha_prod_prev) of diffusers' DDIMScheduler.step with set_alpha_to_one=False."""
    prev = t - num_train_timesteps // num_inference_steps
    return ac[t], (ac[prev] if prev >= 0 else ac[0])


@torch.no_grad()
def ddim_sample(unet, control_lora, guide: torch.Tensor, cond: torch.Tensor, uncond: torch.Tensor, num_inference_steps: int = 50,
                guidance_scale: float = 7.5, latents: Optional[torch.Tensor] = None, seed: int = 0) -> torch.Tensor:
    """guide [B,3,H,W] in [-1,1]; cond / uncond text states [B,77,D] bf16.  Returns the final latents [B,4,H/8,W/8] fp32."""
    B = guide.shape[0]
    dev = guide.device
    h, w = guide.shape[2] // 8, guide.shape[3] // 8
    if latents is None:
        g = torch.Generator(device="cpu").manual_seed(seed)
        latents = torch.randn(B, 4, h, w, generator=g).to(dev)
    latents = latents.float().contiguous().clone()
    control_lora(torch.cat([guide, guide], 0))                     # inject once, for [uncond | cond]
    ehs = torch.cat([uncond, cond], 0).to(torch.bfloat16).contiguous()
    ac = sd15_alphas_cumprod()
    for t in ddim_timesteps(num_inference_steps):
        x2 = torch.cat([latents, latents], 0)
        tt = torch.full((2 * B,), float(t), device=dev)
        eps2 = unet(x2, tt, ehs).sample
        a_t, a_prev = ddim_coeffs(t, num_inference_steps, ac)
        ops.cfg_ddim_step(eps2, latents, guidance_scale, a_t, a_prev)
    return latents


# ---------------------------------------------------------------------------------------------- DPM-Solver++ (2M)
def dpm_timesteps(num_inference_steps: int, num_train_timesteps: int = 1000) -> List[int]:
    """diffusers-0.13 DPMSolverMultistepScheduler.set_timesteps: linspace(0, T-1, N+1).round()[::-1][:-1]."""
    # reproduces numpy bit for bit: linspace = arange(N + 1) * step (step = (T-1)/N in double, last element = T-1 exactly),
    # np.round = Python round = half to even  (e.g. N = 30: 15 * 33.3 = 499.49999999999994 -> 499, not 500)
    step = (num_train_timesteps - 1) / num_inference_steps
    out = [int(round(i * step)) for i in range(num_inference_steps)] + [num_train_timesteps - 1]
    return out[::-1][:-1]


def dpmpp_2m_coeffs(i: int, timesteps: List[int], ac: List[float], lower_order_final: bool = True):
    """Scalars of step i of the multistep solver (epsilon prediction, midpoint, order 2; first step and - for < 15 steps -
    the last step are first order):  x0 = (x - sigma_s eps) / alpha_s;  x <- c_x x + c_m0 x0 + c_m1 x0_prev.
    Returns (alpha_s, sigma_s, c_x, c_m0, c_m1)."""
    import math

    def asl(t):
        a, s = math.sqrt(ac[t]), math.sqrt(1.0 - ac[t])
        return a, s, math.log(a) - math.log(s)

    n = len(timesteps)
    s0 = timesteps[i]
    t = 0 if i == n - 1 else timesteps[i + 1]
    a_t, sg_t, l_t = asl(t)
    a_s, sg_s, l_s = asl(s0)
    h = l_t - l_s
    c = a_t * (math.exp(-h) - 1.0)
    first = i == 0 or (i == n - 1 and lower_order_final and n < 15)
    if first:
        return a_s, sg_s, sg_t / sg_s, -c, 0.0
    _, _, l_s1 = asl(timesteps[i - 1])
    r0 = (l_s - l_s1) / h
    return a_s, sg_s, sg_t / sg_s, -c * (1.0 + 0.5 / r0), 0.5 * c / r0


@torch.no_grad()
def dpmpp_sample(unet, control_lora, guide: torch.Tensor, cond: torch.Tensor, uncond: torch.Tensor, num_inference_steps: int = 30,
                 guidance_scale: float = 7.5, latents: Optional[torch.Tensor] = None, seed: int = 0) -> torch.Tensor:
    """Same contract as ddim_sample with the DPM-Solver++(2M) update; one fused CFG + solver kernel per step."""
    B = guide.shape[0]
    dev = guide.device
    h, w = guide.shape[2] // 8, guide.shape[3] // 8
    if latents is None:
        g = torch.Generator(device="cpu").manual_seed(seed)
        latents = torch.randn(B, 4, h, w, generator=g).to(dev)
    latents = latents.float().contiguous().clone()
    x0_prev = torch.zeros_like(latents)
    control_lora(torch.cat([guide, guide], 0))                     # inject once, for [uncond | cond]
    ehs = torch.cat([uncond, cond], 0).to(torch.bfloat16).contiguous()
    ac = sd15_alphas_cumprod()
    ts = dpm_timesteps(num_inference_steps)
    for i, t in enumerate(ts):
        x2 = torch.cat([latents, latents], 0)
        tt = torch.full((2 * B,), float(t), device=dev)
        eps2 = unet(x2, tt, ehs).sample
        a_s, sg_s, c_x, c_m0, c_m1 = dpmpp_2m_coeffs(i, ts, ac)
        ops.cfg_dpmpp_step(eps2, latents, x0_prev, guidance_scale, a_s, sg_s, c_x, c_m0, c_m1)
    return latents


# ---------------------------------------------------------------------------------------------- whole loop as one replayed graph
class GraphedSampler:
    """The denoise loop of the reference's pipelines (train_text_to_image_control_lora.py:829-843, apps/gradio_canny2image.py:
    81-89, mix_lora_and_control_lora.py:153-164) as ONE captured CUDA graph that is replayed once per step:

        prep (x2 = [latents | latents], timestep from a device table)  ->  UNet on the CFG batch 2B
        ->  fused CFG + solver update (coefficients from a device table)  ->  device step counter + 1

    Everything that does not depend on the timestep runs once per image batch, outside the graph (SURVEY f2): the hint
    encoder, LoRA operand packing, the per-level control products `u = Ac c` / v1 `t_add` tables, and the k / v projections
    of the text states.  scheduler: "ddim" (eta = 0, config C3) or "dpmpp" (DPM-Solver++(2M), the reference's validation /
    app scheduler, config C5)."""

    def __init__(self, unet, control_lora, batch: int, height: int = 512, width: int = 512, scheduler: str = "ddim",
                 num_inference_steps: int = 50, guidance_scale: float = 7.5, scale: float = 1.0, text_dim: Optional[int] = None):
        if scheduler not in ("ddim", "dpmpp"):
            raise ValueError(f"unknown scheduler {scheduler}")
        self.unet, self.cl = unet, control_lora
        self.B, self.h, self.w = batch, height // 8, width // 8
        self.kind = 0 if scheduler == "ddim" else 1
        self.steps, self.guidance, self.scale = int(num_inference_steps), float(guidance_scale), float(scale)
        dev = unet.device_
        ac = sd15_alphas_cumprod()
        if self.kind == 0:
            ts = ddim_timesteps(self.steps)
            rows = []
            for t in ts:
                a_t, a_p = ddim_coeffs(t, self.steps, ac)
                rows.append([a_t ** 0.5, (1 - a_t) ** 0.5, a_p ** 0.5, (1 - a_p) ** 0.5, 0, 0, 0, 0])
        else:
            ts = dpm_timesteps(self.steps)
            rows = [list(dpmpp_2m_coeffs(i, ts, ac)) + [0, 0, 0] for i in range(self.steps)]
        self.timesteps = ts
        self.ts_table = torch.tensor([float(t) for t in ts], dtype=torch.float32, device=dev)
        self.coef = torch.tensor(rows, dtype=torch.float32, device=dev).contiguous()
        B2 = 2 * batch
        td = text_dim if text_dim is not None else unet.config.cross_attention_dim
        self.latents = torch.zeros(batch, 4, self.h, self.w, device=dev, dtype=torch.float32)
        self.x0_prev = torch.zeros_like(self.latents)
        self.x2 = torch.zeros(B2, 4, self.h, self.w, device=dev, dtype=torch.float32)
        self.tt = torch.zeros(B2, device=dev, dtype=torch.float32)
        self.ehs = torch.zeros(B2, 77, td, device=dev, dtype=torch.bfloat16)
        self.guide2 = torch.zeros(B2, 3, height, width, device=dev, dtype=torch.float32)
        self.step_ctr = torch.zeros(1, device=dev, dtype=torch.int64)
        self._graph = None
        self._ctx = None
        self.launches_per_step = None

    def _one_step(self):
        ops.sampler_prep(self.latents, self.x2, self.tt, self.ts_table, self.step_ctr)
        ctx = self._ctx
        pred, _, _ = self.unet.run_engine(self.x2, self.tt, self.ehs, {}, tape=None, scale=self.scale, prepared=ctx)
        ops.cfg_solver_step_dev(pred.data, self.latents, self.x0_prev, self.coef, self.step_ctr, self.guidance, self.kind)

    @torch.no_grad()
    def __call__(self, guide: torch.Tensor, cond: torch.Tensor, uncond: torch.Tensor, latents: Optional[torch.Tensor] = None,
                 seed: int = 0, use_graph: bool = True) -> torch.Tensor:
        """guide [B,3,H,W] in [-1,1]; cond / uncond [B,77,D].  Returns the final latents [B,4,H/8,W/8] fp32 (a view of the
        sampler's static buffer: clone it before the next call)."""
        from . import _lib

        B = self.B
        assert guide.shape[0] == B
        if latents is None:
            g = torch.Generator(device="cpu").manual_seed(seed)
            latents = torch.randn(B, 4, self.h, self.w, generator=g)
        self.latents.copy_(latents.to(self.latents.device, torch.float32))
        self.x0_prev.zero_()
        self.step_ctr.zero_()
        self.guide2[:B].copy_(guide)
        self.guide2[B:].copy_(guide)
        self.ehs[:B].copy_(uncond.to(torch.bfloat16))
        self.ehs[B:].copy_(cond.to(torch.bfloat16))
        # once per image batch: hint encoder (control states into static memory), packing, u = Ac c, t_add tables
        self.cl(self.guide2)
        if self._graph is None or not use_graph:
            self._ctx = self.unet.prepare_inference(self.scale)
        else:
            # the captured kernels read the addresses held by the prepared context: refresh its contents in place
            self._refresh_prepared()
        if not use_graph:
            for _ in range(self.steps):
                self._one_step()
            return self.latents
        first = 0
        if self._graph is None:
            self._one_step()                      # eager warm-up step (fills the text k / v cache, allocator warm-up)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                self._one_step()
            self.launches_per_step = int(_lib.launch_count() - n0)
            self._graph = graph
            # the capture itself does not execute: state is after ONE eager step
            first = 1
        for _ in range(first, self.steps):
            self._graph.replay()
        return self.latents

    def _refresh_prepared(self):
        """A later call with a new guide / prompt: recompute the timestep-invariant products INTO the buffers the captured
        graph reads (control states, u, t_add, cached text k / v)."""
        old = self._ctx
        new = self.unet.prepare_inference(self.scale)
        # first evaluation with the new context fills its k / v cache; then copy every product into the old buffers
        ops.sampler_prep(self.latents, self.x2, self.tt, self.ts_table, self.step_ctr)
        self.unet.run_engine(self.x2, self.tt, self.ehs, {}, tape=None, scale=self.scale, prepared=new)
        for key, st_old in old.stash.items():
            st_new = new.stash.get(key)
            if key == "kv_cache":
                for name, (k_old, v_old) in st_old.items():
                    k_new, v_new = st_new[name]
                    k_old.data.copy_(k_new.data)
                    v_old.data.copy_(v_new.data)
                continue
            for f in ("u", "t_add", "M"):
                a, b = getattr(st_old, f, None), getattr(st_new, f, None)
                if a is not None and b is not None:
                    a.copy_(b)
            if getattr(st_old, "c", None) is not None and getattr(st_new, "c", None) is not None:
                if st_old.c.data.data_ptr() != st_new.c.data.data_ptr():
                    st_old.c.data.copy_(st_new.c.data)


@torch.no_grad()
def generate(unet, control_lora, vae, text_encoder, guide: torch.Tensor, input_ids: torch.Tensor, uncond_input_ids: torch.Tensor,
             num_inference_steps: int = 50, guidance_scale: float = 7.5, scheduler: str = "ddim", latents: Optional[torch.Tensor] = None,
             seed: int = 0, sampler: Optional["GraphedSampler"] = None) -> torch.Tensor:
    """What the reference's validation loop and apps ask of `StableDiffusionPipeline` after `control_lora(guide)`
    (train_text_to_image_control_lora.py:824-843, apps/gradio_*2image.py:75-89, mix_lora_and_control_lora.py:153-164), on this
    package's frozen encoders: prompt / negative-prompt token ids -> text states (`text_encoder(ids)[0]`), the CFG denoise loop
    (`scheduler` = "ddim" or "dpmpp"; pass a `GraphedSampler` to replay the captured step instead of launching from Python), then
    `vae.decode(latents / scaling_factor).sample` mapped from [-1, 1] to [0, 1] like the pipeline's `(image / 2 + 0.5).clamp(0, 1)`.
    guide [B,3,H,W] in [-1,1]; ids [B,77] (tokenisation stays with the caller: the tokenizer is data-pipeline code).  Returns images
    [B,3,H,W] fp32 in [0,1]."""
    cond = text_encoder(input_ids)[0]
    uncond = text_encoder(uncond_input_ids)[0]
    if sampler is not None:
        lat = sampler(guide, cond, uncond, latents=latents, seed=seed).clone()
    else:
        fn = {"ddim": ddim_sample, "dpmpp": dpmpp_sample}[scheduler]
        lat = fn(unet, control_lora, guide, cond, uncond, num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                 latents=latents, seed=seed)
    img = vae.decode(lat / float(vae.config.scaling_factor)).sample
    return ops.channel_affine_nchw(img.contiguous(), 0.5, torch.full((img.shape[1],), 0.5, device=img.device, dtype=torch.float32)).clamp_(0.0, 1.0)
