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


def _check_control(control_lora, guide) -> None:
    if (control_lora is None) != (guide is None):
        raise ValueError("pass control_lora and guide together, or neither of them (sampling without a ControlLoRA)")


PREDICTION_TYPES = ("epsilon", "v_prediction")


def _check_prediction_type(prediction_type: str) -> None:
    if prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"unknown prediction_type {prediction_type!r}: expected one of {PREDICTION_TYPES}")


def scheduler_prediction_type(pretrained_model_name_or_path, subfolder: str = "scheduler") -> str:
    """`prediction_type` of a local diffusers checkpoint's `<root>/<subfolder>/scheduler_config.json` ("epsilon" when the key is
    absent, diffusers' default) - what train_text_to_image_control_lora.py:774-779 reads from `noise_scheduler.config`.  SD-1.5 and
    SD-2-base give "epsilon", SD-2.1 (768) gives "v_prediction".  Nothing else of the file is read."""
    import json
    import os

    path = os.path.join(str(pretrained_model_name_or_path), subfolder, "scheduler_config.json")
    with open(path) as f:
        value = json.load(f).get("prediction_type", "epsilon")
    _check_prediction_type(value)
    return value


def _begin_loop(control_lora, guide, cond, uncond, latents, seed, height, width):
    """Start of every eager loop: initial latents (seeded CPU draw unless given), `control_lora(guide)` tiled to the CFG batch
    when there is a ControlLoRA, and the [uncond | cond] text states.  Without a ControlLoRA (control_lora = guide = None) the
    UNet runs with whatever attention processors are installed, and the latent size comes from `latents` or height / width."""
    _check_control(control_lora, guide)
    ref = cond if guide is None else guide
    B, dev = ref.shape[0], ref.device
    if guide is not None:
        h, w = guide.shape[2] // 8, guide.shape[3] // 8
    elif latents is not None:
        h, w = latents.shape[2], latents.shape[3]
    else:
        h, w = height // 8, width // 8
    if latents is None:
        g = torch.Generator(device="cpu").manual_seed(seed)
        latents = torch.randn(B, 4, h, w, generator=g).to(dev)
    latents = latents.float().contiguous().clone()
    if control_lora is not None:
        control_lora(torch.cat([guide, guide], 0))                 # inject once, for [uncond | cond]
    ehs = torch.cat([uncond, cond], 0).to(torch.bfloat16).contiguous()
    return B, dev, latents, ehs


@torch.no_grad()
def ddim_sample(unet, control_lora, guide: Optional[torch.Tensor], cond: torch.Tensor, uncond: torch.Tensor, num_inference_steps: int = 50,
                guidance_scale: float = 7.5, latents: Optional[torch.Tensor] = None, seed: int = 0, height: int = 512,
                width: int = 512, prediction_type: str = "epsilon") -> torch.Tensor:
    """guide [B,3,H,W] in [-1,1]; cond / uncond text states [B,77,D] bf16.  Returns the final latents [B,4,H/8,W/8] fp32.
    control_lora = guide = None samples without a ControlLoRA (height / width then give the image size unless latents do).
    prediction_type "v_prediction" reads the UNet output as v (SD-2.1 768), with the step scalars from a device table."""
    _check_prediction_type(prediction_type)
    B, dev, latents, ehs = _begin_loop(control_lora, guide, cond, uncond, latents, seed, height, width)
    if prediction_type == "v_prediction":
        return _v_solver_loop(unet, 0, num_inference_steps, guidance_scale, latents, ehs)
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
def dpmpp_sample(unet, control_lora, guide: Optional[torch.Tensor], cond: torch.Tensor, uncond: torch.Tensor, num_inference_steps: int = 30,
                 guidance_scale: float = 7.5, latents: Optional[torch.Tensor] = None, seed: int = 0, height: int = 512,
                 width: int = 512, prediction_type: str = "epsilon") -> torch.Tensor:
    """Same contract as ddim_sample with the DPM-Solver++(2M) update; one fused CFG + solver kernel per step."""
    _check_prediction_type(prediction_type)
    B, dev, latents, ehs = _begin_loop(control_lora, guide, cond, uncond, latents, seed, height, width)
    if prediction_type == "v_prediction":
        return _v_solver_loop(unet, 1, num_inference_steps, guidance_scale, latents, ehs)
    x0_prev = torch.zeros_like(latents)
    ac = sd15_alphas_cumprod()
    ts = dpm_timesteps(num_inference_steps)
    for i, t in enumerate(ts):
        x2 = torch.cat([latents, latents], 0)
        tt = torch.full((2 * B,), float(t), device=dev)
        eps2 = unet(x2, tt, ehs).sample
        a_s, sg_s, c_x, c_m0, c_m1 = dpmpp_2m_coeffs(i, ts, ac)
        ops.cfg_dpmpp_step(eps2, latents, x0_prev, guidance_scale, a_s, sg_s, c_x, c_m0, c_m1)
    return latents


def solver_table(kind: int, num_inference_steps: int) -> Tuple[List[int], List[List[float]]]:
    """(UNet timesteps, coef rows [steps][8]) of the device-table step: kind 0 = DDIM (sqrt_at, sqrt_1m_at, sqrt_aprev,
    sqrt_1m_aprev), kind 1 = DPM-Solver++(2M) (dpmpp_2m_coeffs).  The rows serve both prediction types."""
    ac = sd15_alphas_cumprod()
    if kind == 0:
        ts = ddim_timesteps(num_inference_steps)
        rows = []
        for t in ts:
            a_t, a_p = ddim_coeffs(t, num_inference_steps, ac)
            rows.append([a_t ** 0.5, (1 - a_t) ** 0.5, a_p ** 0.5, (1 - a_p) ** 0.5, 0, 0, 0, 0])
    else:
        ts = dpm_timesteps(num_inference_steps)
        rows = [list(dpmpp_2m_coeffs(i, ts, ac)) + [0, 0, 0] for i in range(num_inference_steps)]
    return ts, rows


def _v_solver_loop(unet, kind, num_inference_steps, guidance_scale, latents, ehs):
    """Eager DDIM (kind 0) / DPM-Solver++(2M) (kind 1) loop of a v-prediction UNet: one fused CFG + v-step kernel per step,
    reading its scalars from the device table through the device step counter."""
    B, dev = latents.shape[0], latents.device
    ts, rows = solver_table(kind, num_inference_steps)
    coef = torch.tensor(rows, dtype=torch.float32, device=dev)
    ctr = torch.zeros(1, device=dev, dtype=torch.int64)
    x0_prev = torch.zeros_like(latents)
    for t in ts:
        x2 = torch.cat([latents, latents], 0)
        tt = torch.full((2 * B,), float(t), device=dev)
        v2 = unet(x2, tt, ehs).sample
        ops.cfg_solver_step_v_dev(v2, latents, x0_prev, coef, ctr, guidance_scale, kind)
    return latents


# ---------------------------------------------------------------------------------------------- PNDM (PLMS)
PLMS_PUSH, PLMS_SAVE, PLMS_RESTART = 1, 2, 4          # flag bits of a pndm_rows row (column 7)
_PLMS_WEIGHTS = {1: (1.0,), 2: (3 / 2, -1 / 2), 3: (23 / 12, -16 / 12, 5 / 12), 4: (55 / 24, -59 / 24, 37 / 24, -9 / 24)}


def pndm_timesteps(num_inference_steps: int, num_train_timesteps: int = 1000, steps_offset: int = 1) -> List[int]:
    """UNet timesteps of diffusers' PNDMScheduler with skip_prk_steps (the SD-1.5 scheduler config): the DDIM grid with its
    second timestep repeated, concat(t[:-1], t[-2:-1], t[-1:])[::-1] - N + 1 model calls (981, 961, 961, 941, ..., 1 at
    N = 50), a single call at N = 1."""
    ratio = num_train_timesteps // num_inference_steps
    t = [i * ratio + steps_offset for i in range(num_inference_steps)]
    return (t[:-1] + t[-2:-1] + t[-1:])[::-1]


def pndm_rows(num_inference_steps: int, ac: List[float], num_train_timesteps: int = 1000,
              prediction_type: str = "epsilon") -> List[List[float]]:
    """One row per model call of PNDMScheduler.step_plms, the program of cl_cfg_plms_step_dev:
    [UNet timestep, sample_coeff, eps_coeff, w_new, w_1, w_2, w_3, flags].  The update is
    x <- sample_coeff * s + eps_coeff * (w_new eps + w_1 r1 + w_2 r2 + w_3 r3), with r1..r3 the most recent pushed eps and s the
    current sample (or the sample saved at call 0, on the restart at call 1).  Call 1 re-runs the transfer of call 0
    (t + ratio -> t) from the saved sample with the mean of the two eps and does not push; every other call pushes its eps
    and uses the Adams-Bashforth weights of the history length (at most 4).
    prediction_type "v_prediction" gives the 10-column rows of cl_cfg_plms_step_v_dev: two more columns, sqrt(a) and sqrt(1 - a)
    at the transfer's source timestep, where PNDMScheduler._get_prev_sample converts the combined v to eps."""
    _check_prediction_type(prediction_type)
    ratio = num_train_timesteps // num_inference_steps
    rows, n_ets = [], 0
    for c, t in enumerate(pndm_timesteps(num_inference_steps, num_train_timesteps)):
        flags = 0
        if c != 1:
            n_ets = min(n_ets + 1, 4)
            flags |= PLMS_PUSH
            t_from, t_to = t, t - ratio
        else:
            t_from, t_to = t + ratio, t
        if c == 0:
            w, flags = (1.0,), flags | PLMS_SAVE
        elif c == 1:
            w, flags = (0.5, 0.5), flags | PLMS_RESTART
        else:
            w = _PLMS_WEIGHTS[n_ets]
        if t_from >= len(ac):          # N = 1000: the grid 1 .. 1000 leaves the table (diffusers' own index fails there too)
            raise ValueError(f"PNDM with {num_inference_steps} steps reaches timestep {t_from}, outside the {len(ac)} training steps")
        a_t = ac[t_from]
        a_p = ac[t_to] if t_to >= 0 else ac[0]
        denom = a_t * (1.0 - a_p) ** 0.5 + (a_t * (1.0 - a_t) * a_p) ** 0.5
        row = [float(t), (a_p / a_t) ** 0.5, -(a_p - a_t) / denom, *(list(w) + [0.0] * (4 - len(w))), float(flags)]
        if prediction_type == "v_prediction":
            row += [a_t ** 0.5, (1.0 - a_t) ** 0.5]
        rows.append(row)
    return rows


@torch.no_grad()
def pndm_sample(unet, control_lora, guide: Optional[torch.Tensor], cond: torch.Tensor, uncond: torch.Tensor, num_inference_steps: int = 50,
                guidance_scale: float = 7.5, latents: Optional[torch.Tensor] = None, seed: int = 0, height: int = 512,
                width: int = 512, prediction_type: str = "epsilon") -> torch.Tensor:
    """Same contract as ddim_sample with diffusers' PNDMScheduler (skip_prk_steps, the default scheduler of an SD-1.5
    pipeline): N + 1 UNet calls, one fused CFG + PLMS kernel per call reading its row of `pndm_rows` through a device counter."""
    _check_prediction_type(prediction_type)
    B, dev, latents, ehs = _begin_loop(control_lora, guide, cond, uncond, latents, seed, height, width)
    rows = torch.tensor(pndm_rows(num_inference_steps, sd15_alphas_cumprod(), prediction_type=prediction_type), dtype=torch.float32,
                        device=dev)
    step = ops.cfg_plms_step_v_dev if prediction_type == "v_prediction" else ops.cfg_plms_step_dev
    ring = torch.zeros((3,) + tuple(latents.shape), device=dev, dtype=torch.float32)
    saved = torch.zeros_like(latents)
    ctr = torch.zeros(1, device=dev, dtype=torch.int64)
    for t in pndm_timesteps(num_inference_steps):
        x2 = torch.cat([latents, latents], 0)
        tt = torch.full((2 * B,), float(t), device=dev)
        eps2 = unet(x2, tt, ehs).sample
        step(eps2, latents, ring, saved, rows, ctr, guidance_scale)
    return latents


# ---------------------------------------------------------------------------------------------- whole loop as one replayed graph
class GraphedSampler:
    """The denoise loop of the reference's pipelines (train_text_to_image_control_lora.py:829-843, apps/gradio_canny2image.py:
    81-89, mix_lora_and_control_lora.py:153-164) as ONE captured CUDA graph that is replayed once per step:

        prep (x2 = [latents | latents], timestep from a device table)  ->  UNet on the CFG batch 2B
        ->  fused CFG + solver update (coefficients from a device table)  ->  device step counter + 1

    Everything that does not depend on the timestep runs once per image batch, outside the graph (SURVEY f2): the hint
    encoder, LoRA operand packing, the per-level control products `u = Ac c` / v1 `t_add` tables, and the k / v projections
    of the text states.  scheduler: "ddim" (eta = 0, config C3), "dpmpp" (DPM-Solver++(2M), the reference's validation /
    app scheduler, config C5) or "pndm" (PNDMScheduler with skip_prk_steps, the default scheduler of an SD-1.5 pipeline: N + 1
    replays, with the eps history and the saved sample of its restart step in device buffers).

    control_lora = None samples without a ControlLoRA: the UNet runs with whatever processors are installed (DreamBooth LoRA
    processors, or none for the base model), there is no hint encoder and no control product, and `guide` is None.

    prediction_type "v_prediction" (SD-2.1 768) reads the UNet output as v: the step kernel is the v form of the same fused
    CFG + update (cl_cfg_solver_step_v_dev / cl_cfg_plms_step_v_dev), with the same tables (PNDM: two more columns per row)."""

    def __init__(self, unet, control_lora, batch: int, height: int = 512, width: int = 512, scheduler: str = "ddim",
                 num_inference_steps: int = 50, guidance_scale: float = 7.5, scale: float = 1.0, text_dim: Optional[int] = None,
                 prediction_type: str = "epsilon"):
        if scheduler not in ("ddim", "dpmpp", "pndm"):
            raise ValueError(f"unknown scheduler {scheduler}")
        _check_prediction_type(prediction_type)
        self.unet, self.cl = unet, control_lora
        self.B, self.h, self.w = batch, height // 8, width // 8
        self.kind = {"ddim": 0, "dpmpp": 1, "pndm": 2}[scheduler]
        self.prediction_type = prediction_type
        self.steps, self.guidance, self.scale = int(num_inference_steps), float(guidance_scale), float(scale)
        dev = unet.device_
        if self.kind == 2:
            ts = pndm_timesteps(self.steps)
            rows = pndm_rows(self.steps, sd15_alphas_cumprod(), prediction_type=prediction_type)
        else:
            ts, rows = solver_table(self.kind, self.steps)
        self.timesteps = ts
        self.calls = len(ts)                     # UNet calls per image batch: N, or N + 1 for PNDM
        self.ts_table = torch.tensor([float(t) for t in ts], dtype=torch.float32, device=dev)
        self.coef = torch.tensor(rows, dtype=torch.float32, device=dev).contiguous()
        B2 = 2 * batch
        td = text_dim if text_dim is not None else unet.config.cross_attention_dim
        self.latents = torch.zeros(batch, 4, self.h, self.w, device=dev, dtype=torch.float32)
        self.x0_prev = torch.zeros_like(self.latents)
        if self.kind == 2:
            self.ring = torch.zeros((3,) + tuple(self.latents.shape), device=dev, dtype=torch.float32)
            self.saved = torch.zeros_like(self.latents)
        self.x2 = torch.zeros(B2, 4, self.h, self.w, device=dev, dtype=torch.float32)
        self.tt = torch.zeros(B2, device=dev, dtype=torch.float32)
        self.ehs = torch.zeros(B2, 77, td, device=dev, dtype=torch.bfloat16)
        self.guide2 = None if control_lora is None else torch.zeros(B2, 3, height, width, device=dev, dtype=torch.float32)
        self.step_ctr = torch.zeros(1, device=dev, dtype=torch.int64)
        self._graph = None
        self._ctx = None
        self.launches_per_step = None

    def _one_step(self):
        ops.sampler_prep(self.latents, self.x2, self.tt, self.ts_table, self.step_ctr)
        ctx = self._ctx
        pred, _, _ = self.unet.run_engine(self.x2, self.tt, self.ehs, {}, tape=None, scale=self.scale, prepared=ctx)
        v = self.prediction_type == "v_prediction"
        if self.kind == 2:
            step = ops.cfg_plms_step_v_dev if v else ops.cfg_plms_step_dev
            step(pred.data, self.latents, self.ring, self.saved, self.coef, self.step_ctr, self.guidance)
        else:
            step = ops.cfg_solver_step_v_dev if v else ops.cfg_solver_step_dev
            step(pred.data, self.latents, self.x0_prev, self.coef, self.step_ctr, self.guidance, self.kind)

    @torch.no_grad()
    def __call__(self, guide: Optional[torch.Tensor], cond: torch.Tensor, uncond: torch.Tensor, latents: Optional[torch.Tensor] = None,
                 seed: int = 0, use_graph: bool = True) -> torch.Tensor:
        """guide [B,3,H,W] in [-1,1] (None without a ControlLoRA); cond / uncond [B,77,D].  Returns the final latents
        [B,4,H/8,W/8] fp32 (a view of the sampler's static buffer: clone it before the next call)."""
        from . import _lib

        B = self.B
        _check_control(self.cl, guide)
        assert (guide if guide is not None else cond).shape[0] == B
        if latents is None:
            g = torch.Generator(device="cpu").manual_seed(seed)
            latents = torch.randn(B, 4, self.h, self.w, generator=g)
        self.latents.copy_(latents.to(self.latents.device, torch.float32))
        self.x0_prev.zero_()
        if self.kind == 2:
            self.ring.zero_()
            self.saved.zero_()
        self.step_ctr.zero_()
        self.ehs[:B].copy_(uncond.to(torch.bfloat16))
        self.ehs[B:].copy_(cond.to(torch.bfloat16))
        if self.cl is not None:
            self.guide2[:B].copy_(guide)
            self.guide2[B:].copy_(guide)
            # once per image batch: hint encoder (control states into static memory), packing, u = Ac c, t_add tables
            self.cl(self.guide2)
        if self._graph is None or not use_graph:
            self._ctx = self.unet.prepare_inference(self.scale)
        else:
            # the captured kernels read the addresses held by the prepared context: refresh its contents in place
            self._refresh_prepared()
        if not use_graph:
            for _ in range(self.calls):
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
        for _ in range(first, self.calls):
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
def generate(unet, control_lora, vae, text_encoder, guide: Optional[torch.Tensor], input_ids: torch.Tensor, uncond_input_ids: torch.Tensor,
             num_inference_steps: int = 50, guidance_scale: float = 7.5, scheduler: str = "ddim", latents: Optional[torch.Tensor] = None,
             seed: int = 0, sampler: Optional["GraphedSampler"] = None, height: int = 512, width: int = 512,
             use_graph: bool = True, prediction_type: str = "epsilon") -> torch.Tensor:
    """What the reference's validation loop and apps ask of `StableDiffusionPipeline` after `control_lora(guide)`
    (train_text_to_image_control_lora.py:824-843, apps/gradio_*2image.py:75-89, mix_lora_and_control_lora.py:153-164), on this
    package's frozen encoders: prompt / negative-prompt token ids -> text states (`text_encoder(ids)[0]`), the CFG denoise loop
    (`scheduler` = "ddim", "dpmpp" or "pndm"; pass a `GraphedSampler` to replay the captured step instead of launching from
    Python), then `vae.decode(latents / scaling_factor).sample` mapped from [-1, 1] to [0, 1] like the pipeline's
    `(image / 2 + 0.5).clamp(0, 1)`.  guide [B,3,H,W] in [-1,1]; ids [B,77] (tokenisation stays with the caller: the tokenizer is
    data-pipeline code).  control_lora = guide = None is the pipeline without a ControlLoRA (DreamBooth validation images with
    LoRA processors installed, train_dreambooth_lora.py:947-963; the base model's class images, :594-614); height / width then
    give the image size unless `latents` does.  use_graph = False runs a sampler's step program without capturing it.
    prediction_type is the checkpoint scheduler's (scheduler_prediction_type); a given sampler must have been built with the
    same one.  Returns images [B,3,H,W] fp32 in [0,1]."""
    _check_prediction_type(prediction_type)
    if sampler is not None and sampler.prediction_type != prediction_type:
        raise ValueError(f"generate(prediction_type={prediction_type!r}) with a GraphedSampler built for {sampler.prediction_type!r}")
    cond = text_encoder(input_ids)[0]
    uncond = text_encoder(uncond_input_ids)[0]
    if sampler is not None:
        lat = sampler(guide, cond, uncond, latents=latents, seed=seed, use_graph=use_graph).clone()
    else:
        fn = {"ddim": ddim_sample, "dpmpp": dpmpp_sample, "pndm": pndm_sample}[scheduler]
        lat = fn(unet, control_lora, guide, cond, uncond, num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                 latents=latents, seed=seed, height=height, width=width, prediction_type=prediction_type)
    img = vae.decode(lat / float(vae.config.scaling_factor)).sample
    return ops.channel_affine_nchw(img.contiguous(), 0.5, torch.full((img.shape[1],), 0.5, device=img.device, dtype=torch.float32)).clamp_(0.0, 1.0)


@torch.no_grad()
def sample_class_images(unet, vae, text_encoder, class_ids: torch.Tensor, uncond_ids: torch.Tensor, num_images: int, out_dir,
                        sample_batch_size: int = 4, num_inference_steps: int = 50, guidance_scale: float = 7.5, height: int = 512,
                        width: int = 512, seed: int = 0, sampler: Optional["GraphedSampler"] = None,
                        use_graph: bool = True, prediction_type: str = "epsilon") -> List[str]:
    """The prior-preservation class images of train_dreambooth_lora.py:580-620: `out_dir` is topped up to `num_images` entries
    (the entries already there are counted, only the missing images are generated), in batches of `sample_batch_size`, by the
    plain SD-1.5 pipeline - no ControlLoRA, the UNet with whatever processors are installed (none, for the base model), the
    checkpoint's own scheduler (PNDM, 50 steps, guidance 7.5) - replayed as one captured step on a GraphedSampler.  Images
    are converted like the pipeline's numpy_to_pil, `(x * 255).round()` to uint8, and saved through Pillow as
    `<index + existing>-<sha1 of the image bytes>.jpg`.  class_ids / uncond_ids: token ids [77] or [1, 77] of the class prompt
    and of the empty prompt (tokenisation stays with the caller).  The latents of a batch are drawn from `seed` plus the index
    of its first new image.  prediction_type is the checkpoint scheduler's ("v_prediction" for SD-2.1 768).  Returns the paths
    written."""
    import hashlib
    from pathlib import Path

    from PIL import Image

    out = Path(out_dir)
    out.mkdir(parents=True, exist_ok=True)
    cur = len(list(out.iterdir()))
    todo = int(num_images) - cur
    if todo <= 0:
        return []
    bs = int(sample_batch_size)
    if sampler is None:
        sampler = GraphedSampler(unet, None, bs, height, width, scheduler="pndm", num_inference_steps=num_inference_steps,
                                 guidance_scale=guidance_scale, prediction_type=prediction_type)
    elif sampler.cl is not None or sampler.B != bs:
        raise ValueError("sample_class_images needs a GraphedSampler without a ControlLoRA, of batch sample_batch_size")
    ids = class_ids.reshape(1, -1).expand(bs, -1).contiguous()
    neg = uncond_ids.reshape(1, -1).expand(bs, -1).contiguous()
    written = []
    for start in range(0, todo, bs):
        n = min(bs, todo - start)                  # the last batch runs full and keeps its first n images
        img = generate(unet, None, vae, text_encoder, None, ids, neg, sampler=sampler, seed=seed + start, use_graph=use_graph,
                       prediction_type=prediction_type)
        arr = (img[:n].permute(0, 2, 3, 1) * 255.0).round().to(torch.uint8).cpu().numpy()
        for i in range(n):
            image = Image.fromarray(arr[i])
            name = out / f"{start + i + cur}-{hashlib.sha1(image.tobytes()).hexdigest()}.jpg"
            image.save(name)
            written.append(str(name))
    return written
