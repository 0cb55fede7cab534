"""Fused ControlLoRA training step (the body of train_text_to_image_control_lora.py:751-796 after the VAE / text
encoder): hint encoder -> UNet -> MSE -> backward -> (NCCL all-reduce) -> clip_grad_norm -> AdamW -> zero_grad, all as
kernel launches on one stream with no host synchronisation.

All trainable parameters are re-homed into ONE flat fp32 arena (and their gradients into another), so the data-parallel
gradient exchange is a single ncclAllReduce and the optimizer a single kernel.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import engine as E
from . import ops
from .engine import Ctx, Tape, Var
from .arena import ParamArena
from .hint_encoder import HintEncoderEngine

BF16 = torch.bfloat16


def lr_lambda_for(name: str, warmup: int = 0, total: Optional[int] = None):
    """The multiplier schedules of diffusers.optimization.get_scheduler (the six names `--lr_scheduler` accepts, train_...:221-228) as
    functions of the number of completed optimizer steps; None for "constant"."""
    import math

    if name == "constant":
        return None
    if name == "constant_with_warmup":
        return lambda s: min(1.0, s / max(1.0, warmup))
    if total is None:
        raise ValueError(f"lr_scheduler={name!r} needs max_train_steps")
    ramp = lambda s: s / max(1, warmup)
    if name == "linear":
        return lambda s: ramp(s) if s < warmup else max(0.0, (total - s) / max(1, total - warmup))
    if name == "cosine":
        return lambda s: ramp(s) if s < warmup else max(0.0, 0.5 * (1.0 + math.cos(math.pi * 0.5 * 2.0 * (s - warmup) / max(1, total - warmup))))
    if name == "cosine_with_restarts":          # num_cycles = 1 (get_scheduler's default)
        def f(s):
            if s < warmup:
                return ramp(s)
            pr = (s - warmup) / max(1, total - warmup)
            return 0.0 if pr >= 1.0 else max(0.0, 0.5 * (1.0 + math.cos(math.pi * ((1.0 * pr) % 1.0))))
        return f
    if name == "polynomial":                    # power 1.0, lr_end 1e-7: needs the base lr, resolved by the caller as a ratio
        raise NotImplementedError("polynomial decays to an absolute lr_end (1e-7): not expressible as a pure multiplier here")
    raise ValueError(f"unknown lr_scheduler {name!r}")


class Trainer:
    def __init__(self, unet, control_lora, lr: float = 1e-4, betas=(0.9, 0.999), weight_decay: float = 1e-2, eps: float = 1e-8,
                 max_grad_norm: float = 1.0, process_group=None, cuda_graph: bool = False, graph_warmup: int = 2,
                 noise_seed: int = 0, prediction_type: str = "epsilon", num_train_timesteps: int = 1000,
                 prior_loss_weight: Optional[float] = None, lr_scheduler: str = "constant", lr_warmup_steps: int = 0,
                 max_train_steps: Optional[int] = None):
        """control_lora=None trains the adapters installed on the UNet alone (plain `LoRACrossAttnProcessor`s on every attention
        layer): the step of train_dreambooth_lora.py:880-918.  prior_loss_weight (DreamBooth's prior preservation, :898-910): the
        batch is [instance images | class images] and loss = mse(first half) + prior_loss_weight * mse(second half)."""
        self.unet, self.cl = unet, control_lora
        self.prior_loss_weight = None if prior_loss_weight is None else float(prior_loss_weight)
        # `get_scheduler(args.lr_scheduler, num_warmup_steps, num_training_steps)` (train_...:675-681).  "constant" (the reference's
        # default) is the only schedule a captured step graph can hold - the learning rate is a launch scalar - the others apply to
        # per-kernel (cuda_graph=False) stepping.
        self.lr_lambda = lr_lambda_for(lr_scheduler, lr_warmup_steps, max_train_steps)
        self.lr_scheduler_name = lr_scheduler
        if self.lr_lambda is not None and cuda_graph:
            raise NotImplementedError(f"lr_scheduler={lr_scheduler!r} needs cuda_graph=False: a captured step graph holds one constant learning rate")
        self.lr, self.betas, self.wd, self.eps, self.max_norm = lr, betas, weight_decay, eps, max_grad_norm
        self.pg = process_group
        dev = unet.device_
        params: List[torch.nn.Parameter] = [] if control_lora is None else [p for p in control_lora.parameters() if p.requires_grad]
        seen = {id(p) for p in params}
        for p in unet.trainable_parameters():          # e.g. stacked pre_loras that are not part of control_lora
            if id(p) not in seen and p.requires_grad:
                params.append(p)
                seen.add(id(p))
        self.params = params
        self.arena = ParamArena(params, dev, process_group)
        self.world = self.arena.world
        self.flat_p, self.flat_g, self.flat_m, self.flat_v = self.arena.flat_p, self.arena.flat_g, self.arena.flat_m, self.arena.flat_v
        self.numel = self.arena.numel
        store = unet.grad_store
        store.bufs.clear()
        for p in params:
            store.bufs[id(p)] = self.arena.grad_of(p)
            store.params[id(p)] = p
        unet._runtime = None                          # rebuild the LoRA runtime against the arena views
        self.hint = None if control_lora is None else HintEncoderEngine(control_lora, store.get)
        if not params:
            raise ValueError("Trainer: nothing to train (no ControlLoRA and no adapter processors installed on the UNet)")
        self.gnorm_sq = torch.zeros(1, device=dev, dtype=torch.float32)
        self.step_idx = 0
        self.step_dev = torch.zeros(1, device=dev, dtype=torch.int64)     # device copy of step_idx (bias corrections inside the graph)
        # data parallel: ONE all-reduce of the whole gradient arena after the backward.  With world > 1 it stays outside the
        # captured graph (the graph holds forward + backward; the all-reduce and the optimizer launches follow each replay).
        self._tail_in_graph = self.world == 1
        self.levels = None
        # CUDA-graph mode: the forward/backward (~1800 launches) is captured once and replayed, so the step costs the
        # host one graph launch instead of ~40 ms of Python/ctypes work and cannot become launch-bound.
        self.cuda_graph = bool(cuda_graph)
        self.graph_warmup = int(graph_warmup)
        self._graph = None
        self._static = None          # static input buffers the captured kernels read
        self._static_loss = None
        self._eager_calls = 0
        self.launches_per_step = None    # kernel launches of one step (counted while capturing / running eagerly)
        # device-side step glue (train_text_to_image_control_lora.py:757-765,774-779): Philox noise, timesteps, add_noise, target
        if prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(f"Unknown prediction type {prediction_type}")        # train_...:779
        self.prediction_type = prediction_type
        self.noise_seed = int(noise_seed)
        from .sampler import sd15_alphas_cumprod
        ac = torch.tensor(sd15_alphas_cumprod(num_train_timesteps), dtype=torch.float64)
        self.sqrt_ac = ac.sqrt().float().to(dev)
        self.sqrt_1mac = (1.0 - ac).sqrt().float().to(dev)
        rank = torch.distributed.get_rank(process_group) if self.world > 1 else 0
        # every rank draws its own noise / timesteps: the rank is folded into the Philox key, the step counter is shared
        self.rng_counter = torch.zeros(1, device=dev, dtype=torch.int64)
        self._rank_seed = (self.noise_seed + 0x9E3779B97F4A7C15 * rank) & (2**64 - 1)
        self._mode = None                # "noised" (step) or "latents" (step_from_latents): one captured graph per Trainer
        self._micro = 0                  # micro-batches accumulated since the last optimizer step (accumulate())

    def step(self, noisy_latents: torch.Tensor, timesteps: torch.Tensor, ehs: torch.Tensor, guide: torch.Tensor,
             target: torch.Tensor, eager: bool = False) -> torch.Tensor:
        """One optimizer step on device tensors: noisy_latents/target NCHW fp32, timesteps fp32 [B], ehs bf16 [B,77,768],
        guide NCHW fp32 [B,3,512,512].  Returns the (device) loss tensor; nothing is synchronised.

        With cuda_graph=True the first `graph_warmup` calls run eagerly, the next call captures the forward/backward
        into a CUDA graph (inputs are copied into static buffers first) and every later call replays it.  The graph holds
        the forward and backward, and at world 1 also clip + AdamW with a device-side step counter; with world > 1 the gradient
        all-reduce, clip and AdamW run after each replay.  eager=True forces the uncaptured path."""
        return self._run("noised", self._forward_backward, (noisy_latents, timesteps, ehs, guide, target), eager)

    def step_from_latents(self, latents: torch.Tensor, ehs: torch.Tensor, guide: torch.Tensor, eager: bool = False) -> torch.Tensor:
        """The whole body of train_text_to_image_control_lora.py:757-796 after the VAE / text encoder: draws the noise and
        one timestep per image on the device (`cl_add_noise`, counter-based Philox: fresh numbers on every CUDA-graph
        replay), forms noisy latents and the epsilon / v-prediction target, then runs the fused step.  latents: the scaled
        VAE latents [B,4,h,w] fp32."""
        return self._run("latents", self._forward_backward_latents, (latents, ehs, guide), eager)

    def step_from_pixels(self, vae, text_encoder, pixel_values: torch.Tensor, input_ids: torch.Tensor, guide: torch.Tensor,
                         latent_noise: Optional[torch.Tensor] = None, generator: Optional[torch.Generator] = None,
                         eager: bool = False) -> torch.Tensor:
        """The COMPLETE loop body of train_text_to_image_control_lora.py:751-796 from the batch as the dataloader hands it over:
        `vae.encode(pixel_values).latent_dist.sample() * scaling_factor` (:753-754) and `text_encoder(input_ids)[0]` (:768) on the frozen
        `controllora_b200.AutoencoderKL` / `CLIPTextModel`, then step_from_latents (noise, timesteps, add_noise, control injection,
        UNet, loss, backward, clip, AdamW).  The two frozen encoders run in front of the (captured) step; `latent_noise` replaces the
        standard-normal draw of `latent_dist.sample()` (tests)."""
        with torch.no_grad():
            dist = vae.encode(pixel_values).latent_dist
            lat = dist.sample(generator) if latent_noise is None else dist.mean + dist.std * latent_noise.to(dist.mean.device, dist.mean.dtype)
            lat = (lat * float(vae.config.scaling_factor)).contiguous()
            ehs = text_encoder(input_ids)[0]
        self.last_latents = lat
        return self.step_from_latents(lat, ehs, guide, eager=eager)

    def _forward_backward_latents(self, latents, ehs, guide) -> torch.Tensor:
        noisy, target, ts = ops.add_noise(latents, self.sqrt_ac, self.sqrt_1mac, self.rng_counter, self._rank_seed,
                                          v_prediction=self.prediction_type == "v_prediction")
        self.last_noise_draw = (noisy, target, ts)       # kept for inspection / tests (graph mode: static buffers)
        return self._forward_backward(noisy, ts, ehs, guide, target)

    def _run(self, mode: str, fb, args, eager: bool) -> torch.Tensor:
        from . import _lib

        self.step_idx += 1
        if not self.cuda_graph or eager:
            n0 = _lib.launch_count()
            loss = fb(*args)
            self._optimizer_tail()
            self.launches_per_step = int(_lib.launch_count() - n0)
            return loss
        if self._mode is None:
            self._mode = mode
        elif self._mode != mode:
            raise ValueError("Trainer(cuda_graph=True): step() and step_from_latents() cannot be mixed on one Trainer")
        if self._static is None:
            self._static = [None if a_ is None else torch.empty_like(a_).copy_(a_) for a_ in args]
        else:
            for st, a_ in zip(self._static, args):
                if st is None and a_ is None:
                    continue
                if st.shape != a_.shape or st.dtype != a_.dtype:
                    raise ValueError("Trainer(cuda_graph=True): input shapes/dtypes must not change between steps")
                if st.data_ptr() != a_.data_ptr():
                    st.copy_(a_, non_blocking=True)
        if self._graph is None and self._eager_calls < self.graph_warmup:
            self._eager_calls += 1
            loss = fb(*self._static)
            self._optimizer_tail()
            return loss
        if self._graph is None:
            import sys

            n0 = _lib.launch_count()
            graph = torch.cuda.CUDAGraph()
            try:
                with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                    self._static_loss = fb(*self._static)
                    if self._tail_in_graph:
                        self._optimizer_tail()       # world 1: clip and AdamW inside the graph too
            except Exception as ex:
                torch.cuda.synchronize()
                self._static_loss = None
                # capture is an optimisation of the launch path only: say so and keep training eagerly
                print(f"controllora_b200.Trainer: CUDA-graph capture failed ({type(ex).__name__}: {ex}); "
                      f"continuing with per-kernel launches", file=sys.stderr, flush=True)
                self.cuda_graph = False
                loss = fb(*self._static)
                self._optimizer_tail()
                return loss
            self.launches_per_step = int(_lib.launch_count() - n0) + (0 if self._tail_in_graph else 3)
            self._graph = graph
            # capture executes nothing: the first replay below is this call's step
        self._graph.replay()
        if not self._tail_in_graph:
            self._optimizer_tail()
        return self._static_loss

    def _forward_backward(self, noisy_latents, timesteps, ehs, guide, target) -> torch.Tensor:
        tape = Tape()
        hctx = Ctx(tape=tape)
        states = [] if self.cl is None else self.hint.forward(hctx, guide)
        control = {}
        for procs, s in zip([] if self.cl is None else self.cl.lora_layers, states):
            n, H, W, C = s.data.shape
            c = Var(s.data.view(n, H * W, C), rg=True)       # token-matrix view of the same memory for the UNet side
            for proc in procs:
                proc.control_states = c.data
            control[c.data.data_ptr()] = c

            def bridge(s=s, c=c, shape=(n, H, W, C)):
                if c.grad is not None:
                    E.give_tensor(s, c.grad.view(shape))
                    c.grad = None

            tape.record(bridge)      # runs after every UNet backward op (incl. the per-level d-control GEMMs)
        pred, ctx, rt = self.unet.run_engine(noisy_latents, timesteps, ehs, control, tape)
        loss, dpred = self._loss(pred.data, target)
        pred.grad = dpred
        tape.backward()
        return loss

    def _loss(self, pred: torch.Tensor, target: torch.Tensor):
        """MSE (train_text_to_image_control_lora.py:783), or DreamBooth's prior-preservation sum (train_dreambooth_lora.py:898-910):
        mse(instance half) + w * mse(class half) - two launches of the fused loss + gradient kernel on the two halves."""
        if self.prior_loss_weight is None:
            return ops.mse_loss(pred, target)
        B = pred.shape[0]
        if B % 2:
            raise ValueError("prior preservation needs an even batch: [instance images | class images]")
        h = B // 2
        dpred = torch.empty_like(pred)
        loss, _ = ops.mse_loss(pred[:h], target[:h], out=dpred[:h])
        prior, _ = ops.mse_loss(pred[h:], target[h:], gscale=self.prior_loss_weight, out=dpred[h:])
        ops.axpy_matrix(prior.view(1, 1), loss.view(1, 1), self.prior_loss_weight)
        return loss, dpred

    def _optimizer_tail(self) -> None:
        """all-reduce(sum) of the gradient arena (nothing at world 1), then clip_grad_norm_ + AdamW + zero_grad
        (train_...:791-796) as three launches; the step count lives on the device, so at world 1 the tail can sit inside the
        captured graph."""
        self.arena.all_reduce()
        ops.step_begin(self.gnorm_sq, self.step_dev)
        ops.sumsq(self.flat_g, self.gnorm_sq)
        # LambdaLR semantics: the k-th optimizer step (k = 1, 2, ...) runs with base_lr * lambda(k - 1)
        lr = self.lr if self.lr_lambda is None else self.lr * self.lr_lambda(max(self.step_idx - 1, 0))
        self.last_lr = lr
        ops.adamw_dev(self.flat_p, self.flat_g, self.flat_m, self.flat_v, lr, self.betas[0], self.betas[1], self.eps, self.wd,
                      self.step_dev, gnorm_sq=self.gnorm_sq, max_norm=self.max_norm,
                      grad_scale=self.arena.grad_scale / (1 + self._micro), zero_grad=True)
        self._micro = 0

    def accumulate(self, noisy_latents, timesteps, ehs, guide, target) -> torch.Tensor:
        """A micro-batch WITHOUT an optimizer step (`with accelerator.accumulate(control_lora)`, train_...:751, when
        `--gradient_accumulation_steps` > 1): forward + backward only, gradients add up in the arena (every gradient kernel
        accumulates; AdamW zeroes them).  The next step() closes the window: its clip + AdamW see the MEAN over the micro-batches,
        like accelerate's 1/N loss scaling.  Not available on a Trainer that replays a captured step graph."""
        if self.cuda_graph:
            raise NotImplementedError("Trainer(cuda_graph=True) replays one captured whole step: gradient accumulation needs cuda_graph=False")
        loss = self._forward_backward(noisy_latents, timesteps, ehs, guide, target)
        self._micro += 1
        return loss

    # ------------------------------------------------------------------------------------------------ checkpoints
    # The reference checkpoints through accelerate: `accelerator.save_state(output_dir/checkpoint-{global_step})` every
    # `checkpointing_steps` (train_text_to_image_control_lora.py:805-809) and resumes from the highest `checkpoint-N`
    # (:713-735).  Same directory convention here: the ControlLoRA weights in the reference's own format
    # (config.json + diffusion_pytorch_model.safetensors, the files of :927-929) plus the optimizer state of the flat arenas.
    def _named_arena_params(self):
        """(name, parameter) of every tensor in the arena: ControlLoRA parameters under their state-dict names, parameters
        that live outside control_lora (e.g. stacked pre_loras from unet.trainable_parameters()) as `extra.<index>`."""
        if self.cl is None:
            # diffusers' AttnProcsLayers naming (train_dreambooth_lora.py:723): "<attn_processors key>.<parameter name>"
            names = {id(p): f"{k}.{n}" for k, proc in self.unet.attn_processors.items() if isinstance(proc, torch.nn.Module)
                     for n, p in proc.named_parameters()}
        else:
            names = {id(p): n for n, p in self.cl.named_parameters()}
        out, k = [], 0
        for p in self.params:
            if id(p) in names:
                out.append((names[id(p)], p))
            else:
                out.append((f"extra.{k}", p))
                k += 1
        return out

    def _param_slices(self):
        """(name, parameter, arena offset) in arena order."""
        out, off = [], 0
        for n, p in self._named_arena_params():
            out.append((n, p, off))
            off += p.numel()
        return out

    def optimizer_state_dict(self) -> dict:
        """The AdamW state as `torch.optim.AdamW(control_lora.parameters(), ...).state_dict()` would hold it (what
        `accelerator.save_state` pickles into optimizer.bin, train_text_to_image_control_lora.py:512-518, 805-809): per-parameter
        `step` / `exp_avg` / `exp_avg_sq` in parameter order + one param group.  `torch.optim.AdamW.load_state_dict` accepts it."""
        sl = self._param_slices()
        proto = torch.optim.AdamW([torch.nn.Parameter(torch.zeros(1))], lr=self.lr, betas=tuple(self.betas), eps=self.eps,
                                  weight_decay=self.wd).state_dict()["param_groups"][0]
        group = dict(proto)
        group["params"] = list(range(len(sl)))
        state = {}
        if self.step_idx > 0:
            m, v = self.flat_m.detach().cpu(), self.flat_v.detach().cpu()
            for i, (_, p, off) in enumerate(sl):
                k = p.numel()
                state[i] = {"step": torch.tensor(float(self.step_idx)), "exp_avg": m[off:off + k].view(p.shape).clone(),
                            "exp_avg_sq": v[off:off + k].view(p.shape).clone()}
        return {"state": state, "param_groups": [group]}

    def load_optimizer_state_dict(self, sd: dict) -> None:
        """Inverse of optimizer_state_dict(); also reads an optimizer.bin written by accelerate for the reference's AdamW."""
        sl = self._param_slices()
        g = sd["param_groups"][0]
        if len(sd["param_groups"]) != 1 or len(g["params"]) != len(sl):
            raise ValueError("optimizer state does not match this Trainer's parameter list")
        steps = set()
        with torch.no_grad():
            self.flat_m.zero_()
            self.flat_v.zero_()
            for i, (n, p, off) in zip(g["params"], sl):
                st = sd["state"].get(i)
                if st is None:
                    continue
                if tuple(st["exp_avg"].shape) != tuple(p.shape):
                    raise ValueError(f"optimizer state of parameter {i} ({n}) has shape {tuple(st['exp_avg'].shape)}, expected {tuple(p.shape)}")
                k = p.numel()
                self.flat_m[off:off + k].copy_(st["exp_avg"].reshape(-1).to(self.flat_m.device, torch.float32))
                self.flat_v[off:off + k].copy_(st["exp_avg_sq"].reshape(-1).to(self.flat_v.device, torch.float32))
                steps.add(int(float(st["step"])))
        if len(steps) > 1:
            raise ValueError(f"per-parameter AdamW step counts differ ({sorted(steps)}): the fused optimizer keeps one step counter")
        self.step_idx = steps.pop() if steps else 0
        self.step_dev.fill_(self.step_idx)
        self.lr, self.betas, self.eps, self.wd = float(g["lr"]), tuple(g["betas"]), float(g["eps"]), float(g["weight_decay"])

    def save_checkpoint(self, output_dir, global_step: Optional[int] = None) -> str:
        """`checkpoint-N/` with the files `accelerator.save_state` writes (train_text_to_image_control_lora.py:805-809) - so the
        reference's `accelerator.load_state` can resume from it, and `load_checkpoint` reads one written by the reference:
          pytorch_model.bin          control_lora.state_dict()                                  (accelerate's model file)
          optimizer.bin              torch.optim.AdamW state_dict layout (optimizer_state_dict()) + a private `controllora_b200` entry
                                     (arena parameter names, clip norm, parameters that live outside control_lora)
          scheduler.bin              LambdaLR state_dict keys of the reference's default `constant` schedule
          random_states_<rank>.pkl   accelerate's keys (python / numpy / torch / CUDA RNG) + the device Philox (seed, step counter)
        plus the ControlLoRA in the reference's save_pretrained format (config.json + diffusion_pytorch_model.safetensors, :927-929)."""
        import os
        import pickle
        import random

        step = self.step_idx if global_step is None else int(global_step)
        path = os.path.join(str(output_dir), f"checkpoint-{step}")
        os.makedirs(path, exist_ok=True)
        rank = torch.distributed.get_rank(self.pg) if self.world > 1 else 0
        named = self._named_arena_params()
        if rank == 0:
            if self.cl is None:      # the model accelerate would have saved is AttnProcsLayers(unet.attn_processors)
                torch.save({n: p.detach().cpu().clone() for n, p in named if not n.startswith("extra.")}, os.path.join(path, "pytorch_model.bin"))
            else:
                self.cl.save_config(path)
                self.cl.save_pretrained(path, safe_serialization=True)
                torch.save({k: v.detach().cpu().clone() for k, v in self.cl.state_dict().items()}, os.path.join(path, "pytorch_model.bin"))
            opt = self.optimizer_state_dict()
            opt["controllora_b200"] = {"step_idx": self.step_idx, "global_step": step, "numel": self.numel, "max_grad_norm": self.max_norm,
                                       "param_names": [n for n, _ in named], "param_numels": [p.numel() for _, p in named],
                                       "extra_params": {n: p.detach().cpu().clone() for n, p in named if n.startswith("extra.")}}
            torch.save(opt, os.path.join(path, "optimizer.bin"))
            cur = self.lr if self.lr_lambda is None else self.lr * self.lr_lambda(self.step_idx)
            torch.save({"base_lrs": [self.lr], "last_epoch": self.step_idx, "_step_count": self.step_idx + 1, "verbose": False,
                        "_get_lr_called_within_step": False, "_last_lr": [cur], "lr_lambdas": [None], "schedule": self.lr_scheduler_name},
                       os.path.join(path, "scheduler.bin"))
        try:
            import numpy as np
            np_state = np.random.get_state()
        except Exception:
            np_state = None
        cuda_all = torch.cuda.get_rng_state_all() if self.flat_p.is_cuda else None
        with open(os.path.join(path, f"random_states_{rank}.pkl"), "wb") as f:
            pickle.dump({"step": step, "random_state": random.getstate(), "numpy_random_seed": np_state,
                         "torch_manual_seed": torch.get_rng_state(), "torch_cuda_manual_seed": cuda_all,
                         "noise_seed": self.noise_seed, "rank_seed": self._rank_seed, "rng_counter": int(self.rng_counter.item())}, f)
        return path

    @staticmethod
    def latest_checkpoint(output_dir) -> Optional[str]:
        """Highest `checkpoint-N` under output_dir (train_text_to_image_control_lora.py:713-721), or None."""
        import os

        if not os.path.isdir(str(output_dir)):
            return None
        best, best_n = None, -1
        for d in os.listdir(str(output_dir)):
            if d.startswith("checkpoint-") and d[len("checkpoint-"):].isdigit() and int(d[len("checkpoint-"):]) > best_n:
                best, best_n = d, int(d[len("checkpoint-"):])
        return None if best is None else os.path.join(str(output_dir), best)

    def load_checkpoint(self, path) -> int:
        """Restore parameters (into the flat arena the kernels read), AdamW moments, the step count and the RNG state from a
        `checkpoint-N` directory written by save_checkpoint() OR by the reference's `accelerator.save_state` (pytorch_model.bin /
        model.safetensors, torch-format optimizer.bin, scheduler.bin, random_states_<rank>.pkl); returns the global step.  A captured
        CUDA graph stays valid: it reads the same arena / counter addresses."""
        import os
        import pickle
        import random

        path = str(path)
        sd = None
        for fn in ("diffusion_pytorch_model.safetensors", "model.safetensors", "pytorch_model.bin", "diffusion_pytorch_model.bin"):
            f = os.path.join(path, fn)
            if os.path.isfile(f):
                if fn.endswith(".safetensors"):
                    from safetensors.torch import load_file

                    sd = load_file(f)
                else:
                    sd = torch.load(f, map_location="cpu")
                break
        if sd is None:
            raise FileNotFoundError(f"{path}: no model file (pytorch_model.bin / model.safetensors / diffusion_pytorch_model.*)")
        opt = torch.load(os.path.join(path, "optimizer.bin"), map_location="cpu", weights_only=False)
        named = self._named_arena_params()
        priv = opt.get("controllora_b200", {})
        if "param_names" in priv and (list(priv["param_names"]) != [n for n, _ in named]
                                      or list(priv["param_numels"]) != [p.numel() for _, p in named]):
            raise ValueError("checkpoint parameter order / names do not match this Trainer's arena (different wiring or config)")
        extra = priv.get("extra_params", {})
        missing = [n for n, _ in named if (n not in sd and n not in extra)]
        if missing:
            raise KeyError(f"checkpoint {path} lacks parameters: {missing[:4]}...")
        with torch.no_grad():
            for n, p in named:
                src = sd[n] if n in sd else extra[n]
                p.data.copy_(src.to(p.data.device, p.data.dtype))      # p.data is a view into flat_p
            self.flat_g.zero_()
        if "state" in opt:
            self.load_optimizer_state_dict(opt)
        else:                                                          # round-1/2 layout of this framework: flat moments
            if int(opt["numel"]) != self.numel:
                raise ValueError("optimizer state does not match this Trainer's parameter count")
            with torch.no_grad():
                self.flat_m[:self.numel].copy_(opt["exp_avg"].to(self.flat_m.device))
                self.flat_v[:self.numel].copy_(opt["exp_avg_sq"].to(self.flat_v.device))
            self.step_idx = int(opt["step_idx"])
            self.step_dev.fill_(self.step_idx)
            priv = opt
        if "max_grad_norm" in priv:
            self.max_norm = float(priv["max_grad_norm"])
        rank = torch.distributed.get_rank(self.pg) if self.world > 1 else 0
        rs = os.path.join(path, f"random_states_{rank}.pkl")
        if os.path.isfile(rs):
            with open(rs, "rb") as f:
                r = pickle.load(f)
            if "noise_seed" in r:                                       # absent in a checkpoint written by accelerate
                self.noise_seed, self._rank_seed = int(r["noise_seed"]), int(r["rank_seed"])
                self.rng_counter.fill_(int(r["rng_counter"]))
            cpu_state = r.get("torch_manual_seed", r.get("torch_cpu"))
            if cpu_state is not None:
                torch.set_rng_state(cpu_state)
            cuda_state = r.get("torch_cuda_manual_seed", r.get("torch_cuda"))
            if cuda_state is not None and self.flat_p.is_cuda:
                if isinstance(cuda_state, (list, tuple)):
                    if len(cuda_state) == torch.cuda.device_count():
                        torch.cuda.set_rng_state_all(cuda_state)
                else:
                    torch.cuda.set_rng_state(cuda_state, self.flat_p.device)
            np_state = r.get("numpy_random_seed", r.get("numpy"))
            if np_state is not None:
                import numpy as np
                np.random.set_state(np_state)
            py_state = r.get("random_state", r.get("python"))
            if py_state is not None:
                random.setstate(py_state)
        gs = priv.get("global_step")
        if gs is None:
            tail = os.path.basename(os.path.normpath(path))
            gs = int(tail.split("-")[1]) if tail.startswith("checkpoint-") and tail.split("-")[1].isdigit() else self.step_idx
        return int(gs)
