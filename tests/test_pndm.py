"""PNDM sampling (diffusers' PNDMScheduler with skip_prk_steps, the default scheduler of an SD-1.5 pipeline) and sampling
without a ControlLoRA (the DreamBooth-LoRA script's class images and validation images, train_dreambooth_lora.py:586-620,
947-963).

CPU: the host tables against the restated diffusers formulas and the stateful oracle (PNDMPLMS below), the
point-mass property pin, the launcher's argument checks, and - in host-logic mode, in a subprocess running this file with
CLB_EMU=1 and `cfg_plms_step_dev` replaced by the restatement below - the sampler program against the oracle chain.
GPU (-m gpu): the kernel per table row, the loops, graph replay and no-control sampling on the tiny UNets.

usage: python tests/test_pndm.py [case ...]      (host-logic mode; prints one `RESULT <case> OK|FAIL` line per case)"""
import math
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from controllora_b200 import sampler as S  # noqa: E402
from oracle import sampler_ref as SR  # noqa: E402


# ------------------------------------------------------------------------------------------------ oracle: PNDM (PLMS, skip_prk_steps)
class PNDMPLMS:
    """ORACLE (tests only; kept with its tests, beside oracle/sampler_ref.py's DDIM and DPM-Solver++).  Stateful restatement of
    diffusers-0.13 `schedulers/scheduling_pndm.py` with the SD-1.5 scheduler config
    (scaled_linear betas 0.00085 -> 0.012, 1000 steps, skip_prk_steps True, steps_offset 1, set_alpha_to_one False,
    epsilon prediction) - the scheduler of a plain `DiffusionPipeline.from_pretrained(SD-1.5)`, which the reference's
    class-image loop runs (train_dreambooth_lora.py:594-614).  fp32 torch, like the original:
      PNDMScheduler.__init__     betas = linspace(sqrt(b0), sqrt(b1), n, float32) ** 2, alphas_cumprod = cumprod(1 - betas),
                                 final_alpha_cumprod = alphas_cumprod[0] (set_alpha_to_one False), ets = [], counter = 0
      PNDMScheduler.set_timesteps  _timesteps = arange(N) * (n // N) + steps_offset;
                                 plms_timesteps = concat(_t[:-1], _t[-2:-1], _t[-1:])[::-1]; ets = [], counter = 0
      PNDMScheduler.step_plms    prev_t = t - n // N; counter != 1: ets = ets[-3:] + [eps]; counter == 1: prev_t = t,
                                 t += n // N; then by (len(ets), counter): (1, 0) save cur_sample; (1, 1) eps = (eps + ets[-1]) / 2,
                                 sample = cur_sample; 2: (3 e1 - e2) / 2; 3: (23 e1 - 16 e2 + 5 e3) / 12;
                                 4: (55 e1 - 59 e2 + 37 e3 - 9 e4) / 24; counter += 1
      PNDMScheduler._get_prev_sample  a_prev = alphas_cumprod[prev_t] if prev_t >= 0 else final_alpha_cumprod;
                                 sample_coeff = (a_prev / a_t) ** 0.5; denom = a_t (1 - a_prev) ** 0.5 + (a_t (1 - a_t) a_prev) ** 0.5;
                                 prev = sample_coeff * sample - (a_prev - a_t) * eps / denom
    `ac` replaces the fp32 alphas_cumprod (e.g. by the fp64 table to compare with a host-built step table)."""

    def __init__(self, num_inference_steps, n=1000, b0=0.00085, b1=0.012, ac=None):
        if ac is None:
            betas = torch.linspace(b0 ** 0.5, b1 ** 0.5, n, dtype=torch.float32) ** 2
            ac = torch.cumprod(1.0 - betas, 0)
        self.alphas_cumprod = ac
        self.final_alpha_cumprod = ac[0]
        self.n = n
        self.num_inference_steps = num_inference_steps
        ratio = n // num_inference_steps
        t = [i * ratio + 1 for i in range(num_inference_steps)]
        self.timesteps = (t[:-1] + t[-2:-1] + t[-1:])[::-1]
        self.ets = []
        self.counter = 0
        self.cur_sample = None

    def step(self, model_output, timestep, sample):
        timestep = int(timestep)
        prev_timestep = timestep - self.n // self.num_inference_steps
        if self.counter != 1:
            self.ets = self.ets[-3:]
            self.ets.append(model_output)
        else:
            prev_timestep = timestep
            timestep = timestep + self.n // self.num_inference_steps
        if len(self.ets) == 1 and self.counter == 0:
            self.cur_sample = sample
        elif len(self.ets) == 1 and self.counter == 1:
            model_output = (model_output + self.ets[-1]) / 2
            sample = self.cur_sample
            self.cur_sample = None
        elif len(self.ets) == 2:
            model_output = (3 * self.ets[-1] - self.ets[-2]) / 2
        elif len(self.ets) == 3:
            model_output = (23 * self.ets[-1] - 16 * self.ets[-2] + 5 * self.ets[-3]) / 12
        else:
            model_output = (1 / 24) * (55 * self.ets[-1] - 59 * self.ets[-2] + 37 * self.ets[-3] - 9 * self.ets[-4])
        prev_sample = self._get_prev_sample(sample, timestep, prev_timestep, model_output)
        self.counter += 1
        return prev_sample

    def _get_prev_sample(self, sample, timestep, prev_timestep, model_output):
        a_t = self.alphas_cumprod[timestep]
        a_prev = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        b_t, b_prev = 1 - a_t, 1 - a_prev
        sample_coeff = (a_prev / a_t) ** 0.5
        denom = a_t * b_prev ** 0.5 + (a_t * b_t * a_prev) ** 0.5
        return sample_coeff * sample - (a_prev - a_t) * model_output / denom


# ------------------------------------------------------------------------------------------------ restatement of the kernel
def plms_step_restated(eps2, latents, ring, saved, rows, step_ctr, guidance):
    """torch restatement of cl_cfg_plms_step_dev (same operation order), in the dtype of `latents`."""
    r = [float(v) for v in rows[int(step_ctr)]]
    u, c = eps2.reshape(2, -1)
    e = (u + guidance * (c - u)).view_as(latents)
    flags = int(r[7])
    ep = r[3] * e + r[4] * ring[0] + r[5] * ring[1] + r[6] * ring[2]
    s = saved.clone() if flags & S.PLMS_RESTART else latents.clone()
    if flags & S.PLMS_SAVE:
        saved.copy_(s)
    latents.copy_(r[1] * s + r[2] * ep)
    if flags & S.PLMS_PUSH:
        ring[2].copy_(ring[1])
        ring[1].copy_(ring[0])
        ring[0].copy_(e)
    step_ctr += 1


def run_table_program(n_steps, x, eps_seq, guidance=7.5, dtype=torch.float64):
    """The host rows of `pndm_rows` executed by the restated kernel: yields the latents after every call."""
    rows = torch.tensor(S.pndm_rows(n_steps, S.sd15_alphas_cumprod()), dtype=dtype)
    x = x.to(dtype).clone()
    ring = torch.zeros((3,) + tuple(x.shape), dtype=dtype)
    saved = torch.zeros_like(x)
    ctr = torch.zeros(1, dtype=torch.int64)
    for eps2 in eps_seq:
        plms_step_restated(eps2.to(dtype), x, ring, saved, rows, ctr, guidance)
        yield x


# ------------------------------------------------------------------------------------------------ CPU: tables and oracle
@pytest.mark.parametrize("n", [1, 2, 3, 4, 20, 50, 1000])
def test_pndm_timesteps_match_the_diffusers_formula(n):
    import numpy as np

    ratio = 1000 // n
    t = (np.arange(0, n) * ratio).round() + 1                                       # PNDMScheduler.set_timesteps
    want = np.concatenate([t[:-1], t[-2:-1], t[-1:]])[::-1].astype(np.int64).tolist()
    assert S.pndm_timesteps(n) == want == PNDMPLMS(n).timesteps
    assert len(want) == (1 if n == 1 else n + 1)
    if n == 1000:                                        # the grid reaches t = 1000, past alphas_cumprod: no step table
        with pytest.raises(ValueError):
            S.pndm_rows(n, S.sd15_alphas_cumprod())
        return
    rows = S.pndm_rows(n, S.sd15_alphas_cumprod())
    assert [int(r[0]) for r in rows] == want
    if n == 1:                                           # one call, 1 -> -999: a_prev is alphas_cumprod[0] (set_alpha_to_one False)
        ac = S.sd15_alphas_cumprod()
        assert rows[0][1] == pytest.approx(math.sqrt(ac[0] / ac[1]), rel=1e-15)
        assert rows[0][7] == S.PLMS_PUSH | S.PLMS_SAVE
    else:
        assert rows[1][7] == S.PLMS_RESTART and rows[0][1:3] == rows[1][1:3]     # the restart repeats the first transfer
        assert all(abs(sum(r[3:7]) - 1.0) < 1e-15 for r in rows)                  # every weight set sums to 1


@pytest.mark.parametrize("n", [1, 2, 3, 5, 10, 50])
def test_table_program_equals_the_oracle_step_by_step(n):
    """Host rows + restated kernel == PNDMPLMS.step on random noise predictions after every call, the repeated-timestep restart
    included (fp64 on both sides, the same alphas_cumprod: only the table logic is compared)."""
    g = torch.Generator().manual_seed(n)
    x0 = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    seq = [torch.randn(4, 4, 8, 8, generator=g, dtype=torch.float64) for _ in S.pndm_timesteps(n)]
    sched = PNDMPLMS(n, ac=SR.alphas_cumprod())
    x = x0.clone()
    for k, (t, eps2, got) in enumerate(zip(sched.timesteps, seq, run_table_program(n, x0, seq))):
        x = sched.step(SR.cfg_combine(eps2[:2], eps2[2:], 7.5), t, x)
        err = float((got - x).abs().max() / x.abs().max())
        assert err < 1e-12, (n, k, t, err)


def test_fp32_oracle_is_diffusers_alphas_cumprod():
    """The default PNDMPLMS table is diffusers' fp32 scaled_linear schedule; it agrees with the fp64 table to fp32 rounding."""
    o = PNDMPLMS(50)
    assert o.alphas_cumprod.dtype == torch.float32 and float(o.final_alpha_cumprod) == float(o.alphas_cumprod[0])
    assert torch.allclose(o.alphas_cumprod.double(), SR.alphas_cumprod(), rtol=2e-6, atol=0)


@pytest.mark.parametrize("n", [1, 2, 5, 20, 50])
def test_pndm_is_exact_on_the_point_mass_ode(n):
    """Property pin: for data on one point x*, eps(x, t) = (x - sqrt(a_t) x*) / sqrt(1 - a_t) is constant (= eps0) along the
    exact trajectory x_t = sqrt(a_t) x* + sqrt(1 - a_t) eps0.  Every PLMS weight set sums to 1 and PNDM's transfer equals
    DDIM's, so the oracle and the table program must land on that trajectory at the final alpha_bar = alphas_cumprod[0] (not on
    x*: set_alpha_to_one is False), to the precision of the arithmetic."""
    g = torch.Generator().manual_seed(0)
    xs, e0 = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64), torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    for dtype, ac, tol in ((torch.float64, SR.alphas_cumprod(), 1e-10), (torch.float32, PNDMPLMS(n).alphas_cumprod, 2e-5)):
        a = ac.double()
        xs_, e0_ = xs.to(dtype), e0.to(dtype)
        eps = lambda x, t: (x - a[t].sqrt().to(dtype) * xs_) / (1 - a[t]).sqrt().to(dtype)
        want = a[0].sqrt() * xs + (1 - a[0]).sqrt() * e0
        sched = PNDMPLMS(n, ac=ac)
        T = sched.timesteps[0]
        x = (a[T].sqrt() * xs + (1 - a[T]).sqrt() * e0).to(dtype)
        for t in sched.timesteps:
            e = eps(x, t)
            x = sched.step(SR.cfg_combine(e, e, 7.5), t, x)
        assert float((x.double() - want).abs().max()) < tol, ("oracle", dtype, n)
        # the table program, fed the same closed-form eps at each call's UNet timestep
        x = (a[T].sqrt() * xs + (1 - a[T]).sqrt() * e0).to(dtype)
        rows = torch.tensor(S.pndm_rows(n, S.sd15_alphas_cumprod()), dtype=dtype)
        ring, saved, ctr = torch.zeros((3,) + tuple(x.shape), dtype=dtype), torch.zeros_like(x), torch.zeros(1, dtype=torch.int64)
        for t in S.pndm_timesteps(n):
            e = eps(x, t)
            plms_step_restated(torch.cat([e, e]), x, ring, saved, rows, ctr, 7.5)
        assert float((x.double() - want).abs().max()) < tol, ("table", dtype, n)


# ------------------------------------------------------------------------------------------------ CPU: the C launcher
def test_plms_launcher_rejects_bad_arguments_without_a_gpu(built_lib):
    """cl_cfg_plms_step_dev is exported and validates its arguments before any CUDA call: status < 0 and a message."""
    import ctypes

    from controllora_b200 import _lib

    lib = _lib.lib()
    assert hasattr(ctypes.CDLL(str(built_lib)), "cl_cfg_plms_step_dev")
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ctr = ctypes.c_uint64(0)
    pc = ctypes.cast(ctypes.byref(ctr), ctypes.c_void_p)
    f = lib.cl_cfg_plms_step_dev
    for i in range(6):                                        # each pointer null in turn
        args = [p] * 5 + [pc]
        args[i] = None
        assert f(*args, 8, 7.5, None) == -1, i
        assert b"null" in lib.cl_last_error()
    assert f(p, p, p, p, p, pc, 0, 7.5, None) == -1
    assert b"n_half" in lib.cl_last_error()
    assert f(p, p, p, p, p, pc, -4, 7.5, None) == -1


def test_plms_wrapper_refuses_cpu_tensors(monkeypatch):
    from controllora_b200 import _lib, ops

    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    monkeypatch.delenv("CLB_DRYRUN", raising=False)
    x = torch.zeros(2, 4, 8, 8)
    with pytest.raises(_lib.CLError):
        ops.cfg_plms_step_dev(torch.zeros(4, 4, 8, 8), x, torch.zeros(3, 2, 4, 8, 8), torch.zeros_like(x), torch.zeros(3, 8),
                              torch.zeros(1, dtype=torch.int64), 7.5)


def test_control_lora_and_guide_go_together():
    with pytest.raises(ValueError):
        S._check_control(object(), None)
    with pytest.raises(ValueError):
        S._check_control(None, torch.zeros(1))
    S._check_control(None, None)


# ------------------------------------------------------------------------------------------------ cases (host-logic mode and GPU)
def _dev():
    from tests._device import DEV

    return DEV


def _sync():
    from tests._device import sync

    sync()


def _inputs(seed, B=2, HW=16, with_guide=True):
    g = torch.Generator().manual_seed(seed)
    guide = (torch.rand(B, 3, HW * 8, HW * 8, generator=g) * 2 - 1).to(torch.bfloat16).float() if with_guide else None
    cond = torch.randn(B, 77, 64, generator=g).to(torch.bfloat16).float()
    unc = torch.randn(B, 77, 64, generator=g).to(torch.bfloat16).float()
    lat0 = torch.randn(B, 4, HW, HW, generator=g)
    return guide, cond, unc, lat0


def _oracle_chain(ounet, ocl, guide, cond, unc, lat0, scheduler, steps, guidance=7.5):
    B = lat0.shape[0]
    with torch.no_grad():
        if ocl is not None:
            ocl(torch.cat([guide, guide], 0))
        x = lat0.clone()
        if scheduler == "ddim":
            for t in SR.timesteps(steps):
                eps = ounet(torch.cat([x, x], 0), torch.full((2 * B,), int(t)), torch.cat([unc, cond], 0)).sample
                x = SR.cfg_ddim_step(eps[:B], eps[B:], x, t, steps, guidance)
        else:
            sched = PNDMPLMS(steps)
            for t in sched.timesteps:
                eps = ounet(torch.cat([x, x], 0), torch.full((2 * B,), int(t)), torch.cat([unc, cond], 0)).sample
                x = sched.step(SR.cfg_combine(eps[:B], eps[B:], guidance), t, x)
    return x


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / b.norm())


def case_pndm_loop(variant):
    """pndm_sample (control injected once, 4 steps = 5 UNet calls) against the oracle UNet driven by PNDMPLMS."""
    from tests import check_unet

    dev = _dev()
    ounet, munet, ocl, mcl = check_unet.build_pair(variant)
    guide, cond, unc, lat0 = _inputs(31)
    want = _oracle_chain(ounet, ocl, guide, cond, unc, lat0, "pndm", 4)
    got = S.pndm_sample(munet, mcl, guide.to(dev), cond.to(dev).to(torch.bfloat16), unc.to(dev).to(torch.bfloat16),
                        num_inference_steps=4, guidance_scale=7.5, latents=lat0.to(dev))
    _sync()
    err = _rel(got, want)
    print(f"[pndm loop {variant}] 5-call latent rel err {err:.3e}")
    return err < 8e-2


def case_graphed_pndm():
    """GraphedSampler("pndm")'s step program (uncaptured) against the oracle chain, and against pndm_sample (bit for bit in
    host-logic mode)."""
    from tests import check_unet

    dev = _dev()
    ounet, munet, ocl, mcl = check_unet.build_pair("v1")
    guide, cond, unc, lat0 = _inputs(33)
    want = _oracle_chain(ounet, ocl, guide, cond, unc, lat0, "pndm", 4)
    gs = S.GraphedSampler(munet, mcl, 2, 128, 128, scheduler="pndm", num_inference_steps=4, guidance_scale=7.5)
    a = gs(guide.to(dev), cond.to(dev).to(torch.bfloat16), unc.to(dev).to(torch.bfloat16), latents=lat0.to(dev), use_graph=False).clone()
    b = S.pndm_sample(munet, mcl, guide.to(dev), cond.to(dev).to(torch.bfloat16), unc.to(dev).to(torch.bfloat16),
                      num_inference_steps=4, guidance_scale=7.5, latents=lat0.to(dev))
    _sync()
    e_or, e_loop = _rel(a, want), _rel(a, b)
    print(f"[graphed pndm] program vs oracle {e_or:.3e}, vs pndm_sample {e_loop:.3e}, calls {gs.calls}")
    return gs.calls == 5 and e_or < 8e-2 and e_loop <= (0.0 if dev == "cpu" else 2e-2)


def case_nocontrol(variant, scheduler="ddim", graphed=False):
    """No ControlLoRA: variant "plain" = DreamBooth LoRACrossAttnProcessors on every attention layer, "none" = the base UNet."""
    from tests import check_unet

    dev = _dev()
    ounet, munet, _, _ = check_unet.build_pair(variant)
    _, cond, unc, lat0 = _inputs(35, with_guide=False)
    steps = 3 if scheduler == "ddim" else 4
    want = _oracle_chain(ounet, None, None, cond, unc, lat0, scheduler, steps)
    c, u = cond.to(dev).to(torch.bfloat16), unc.to(dev).to(torch.bfloat16)
    if graphed:
        gs = S.GraphedSampler(munet, None, 2, 128, 128, scheduler=scheduler, num_inference_steps=steps, guidance_scale=7.5)
        got = gs(None, c, u, latents=lat0.to(dev), use_graph=dev == "cuda").clone()
    else:
        fn = {"ddim": S.ddim_sample, "pndm": S.pndm_sample}[scheduler]
        got = fn(munet, None, None, c, u, num_inference_steps=steps, guidance_scale=7.5, latents=lat0.to(dev))
    _sync()
    err = _rel(got, want)
    print(f"[no control {variant} {scheduler} graphed={graphed}] latent rel err {err:.3e}")
    return err < (6e-2 if scheduler == "ddim" else 8e-2)


def _tiny_vae_clip():
    import controllora_b200 as cb
    from oracle import clip_ref as CR
    from oracle import vae_ref as VR

    dev = _dev()
    vcfg = dict(block_out_channels=(32, 64, 64, 64), layers_per_block=1)          # 4 levels: 16x16 latents -> 128x128 pixels
    ovae = VR.AutoencoderKL(**vcfg)
    VR.init_synthetic_(ovae, seed=4)
    mvae = cb.AutoencoderKL.from_state_dict({k: v.detach().clone() for k, v in ovae.state_dict().items()}, dev, vcfg)
    ccfg = dict(CR.SD15_TEXT_CONFIG)
    ccfg.update(num_hidden_layers=2, vocab_size=1000, hidden_size=64, intermediate_size=256, num_attention_heads=4)
    csd = CR.synthetic_state_dict(ccfg, seed=0)
    mclip = cb.CLIPTextModel.from_state_dict(csd, dev, ccfg)
    return ovae, mvae, csd, ccfg, mclip


def case_generate_nocontrol(variant="plain"):
    """generate(control_lora=None, guide=None, scheduler="pndm"): ids -> CLIP -> PNDM loop on the LoRA-processor / base UNet ->
    VAE decode, against the oracle chain."""
    from oracle import clip_ref as CR
    from tests import check_unet

    dev = _dev()
    ounet, munet, _, _ = check_unet.build_pair(variant)
    ovae, mvae, csd, ccfg, mclip = _tiny_vae_clip()
    g = torch.Generator().manual_seed(37)
    ids = torch.randint(0, ccfg["vocab_size"], (2, 77), generator=g)
    neg = torch.randint(0, ccfg["vocab_size"], (2, 77), generator=g)
    lat0 = torch.randn(2, 4, 16, 16, generator=g)
    with torch.no_grad():
        cond, unc = CR.clip_text_forward(csd, ids, ccfg), CR.clip_text_forward(csd, neg, ccfg)
        x = _oracle_chain(ounet, None, None, cond, unc, lat0, "pndm", 4)
        want = (ovae.decode(x) / 2 + 0.5).clamp(0, 1)
    got = S.generate(munet, None, mvae, mclip, None, ids.to(dev), neg.to(dev), num_inference_steps=4, scheduler="pndm",
                     latents=lat0.to(dev))
    _sync()
    err = _rel(got, want)
    print(f"[generate no control {variant}] image rel err {err:.3e}, shape {tuple(got.shape)}")
    return err < 5e-2 and tuple(got.shape) == (2, 3, 128, 128)


def case_class_images():
    """sample_class_images tops a directory up to num_images: 5 new images in batches of 2 (the last one partial) named
    `<index>-<sha1 of the uint8 image>.jpg`, equal to generate() on the same sampler and seeds; a second call with a larger
    target generates only the missing images, continuing the indices."""
    import hashlib
    import tempfile

    from tests import check_unet

    dev = _dev()
    _, munet, _, _ = check_unet.build_pair("none")
    _, mvae, _, ccfg, mclip = _tiny_vae_clip()
    g = torch.Generator().manual_seed(39)
    cls_ids = torch.randint(0, ccfg["vocab_size"], (77,), generator=g).to(dev)
    un_ids = torch.randint(0, ccfg["vocab_size"], (1, 77), generator=g).to(dev)
    graph = dev == "cuda"
    ok = True
    with tempfile.TemporaryDirectory() as d:
        Path(d, "existing.jpg").write_bytes(b"")                  # entries already present count, as in the reference
        gs = S.GraphedSampler(munet, None, 2, 128, 128, scheduler="pndm", num_inference_steps=3, guidance_scale=7.5)
        paths = S.sample_class_images(munet, mvae, mclip, cls_ids, un_ids, 6, d, sample_batch_size=2, seed=5, sampler=gs,
                                      use_graph=graph)
        names = sorted(Path(p).name for p in paths)
        want = []
        ids2, neg2 = cls_ids.reshape(1, -1).expand(2, -1), un_ids.expand(2, -1)
        for start in (0, 2, 4):
            img = S.generate(munet, None, mvae, mclip, None, ids2, neg2, sampler=gs, seed=5 + start, use_graph=graph)
            arr = (img.permute(0, 2, 3, 1) * 255.0).round().to(torch.uint8).cpu().numpy()
            for i in range(min(2, 5 - start)):
                want.append(f"{start + i + 1}-{hashlib.sha1(arr[i].tobytes()).hexdigest()}.jpg")
        ok = ok and names == sorted(want) and len(list(Path(d).iterdir())) == 6
        print(f"[class images] first call wrote {names}")
        again = S.sample_class_images(munet, mvae, mclip, cls_ids, un_ids, 6, d, sample_batch_size=2, sampler=gs, use_graph=graph)
        more = S.sample_class_images(munet, mvae, mclip, cls_ids, un_ids, 7, d, sample_batch_size=2, sampler=gs, use_graph=graph)
        ok = ok and again == [] and len(more) == 1 and Path(more[0]).name.startswith("6-") and len(list(Path(d).iterdir())) == 7
        print(f"[class images] second call wrote {again}, third call wrote {[Path(p).name for p in more]}")
    return ok


CASES = {
    "pndm_loop_v1": lambda: case_pndm_loop("v1"),
    "graphed_pndm": case_graphed_pndm,
    "nocontrol_ddim_lora": lambda: case_nocontrol("plain", "ddim"),
    "nocontrol_graphed_pndm_base": lambda: case_nocontrol("none", "pndm", graphed=True),
    "generate_nocontrol_lora": case_generate_nocontrol,
    "class_images": case_class_images,
}


@pytest.fixture(scope="module")
def emulated_results():
    env = dict(os.environ, CLB_EMU="1")
    r = subprocess.run([sys.executable, str(Path(__file__).resolve()), *CASES], capture_output=True, text=True, timeout=1500,
                       cwd=str(ROOT), env=env)
    res = {}
    for line in r.stdout.splitlines():
        if line.startswith("RESULT "):
            _, name, verdict = line.split()[:3]
            res[name] = verdict == "OK"
    return res, r.stdout[-6000:] + r.stderr[-3000:]


@pytest.mark.parametrize("case", list(CASES))
def test_host_logic_matches_oracle(emulated_results, case):
    res, log = emulated_results
    assert case in res, f"{case} did not run:\n{log}"
    assert res[case], f"{case} deviates from the oracle:\n{log}"


# ------------------------------------------------------------------------------------------------ GPU
gpu = pytest.mark.gpu


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@gpu
@pytest.mark.parametrize("n", [1, 2, 50])
def test_plms_kernel_matches_the_oracle_on_every_row(n):
    """cl_cfg_plms_step_dev, one launch per row, from the oracle's own state (sample, eps history, saved sample, step counter):
    the new sample within 6 fp32 ulp of the oracle's scale, the pushed eps and the saved sample equal, the counter + 1."""
    from controllora_b200 import ops

    _need_gpu()
    ac = SR.alphas_cumprod()
    rows = torch.tensor(S.pndm_rows(n, S.sd15_alphas_cumprod()), dtype=torch.float32, device="cuda")
    sched = PNDMPLMS(n, ac=ac)
    g = torch.Generator().manual_seed(100 + n)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ulp = 2.0 ** -23
    for k, t in enumerate(sched.timesteps):
        eps2 = torch.randn(4, 4, 16, 16, generator=g)
        ring = torch.zeros(3, 2, 4, 16, 16)
        hist = sched.ets[-3:][::-1]                       # most recent first
        for j, e in enumerate(hist):
            ring[j] = e
        saved = sched.cur_sample.clone() if sched.cur_sample is not None else torch.zeros_like(x)
        xm, rm, sm = x.cuda(), ring.cuda(), saved.cuda()
        ctr = torch.full((1,), k, dtype=torch.int64, device="cuda")
        ops.cfg_plms_step_dev(eps2.cuda(), xm, rm, sm, rows, ctr, 7.5)
        x = sched.step(SR.cfg_combine(eps2[:2], eps2[2:], 7.5), t, x)
        torch.cuda.synchronize()
        assert int(ctr) == k + 1, k
        d = float((xm.cpu() - x).abs().max())
        assert d <= 6 * ulp * float(x.abs().max()), (n, k, t, d)
        if k != 1:
            assert torch.allclose(rm[0].cpu(), sched.ets[-1], rtol=2 * ulp, atol=2 * ulp * float(sched.ets[-1].abs().max())), k
        if k == 0:
            assert torch.equal(sm.cpu(), sched.cur_sample), k


@gpu
@pytest.mark.parametrize("variant", ["v1", "v2"])
def test_pndm_loop_tracks_oracle_on_tiny_unet(variant):
    _need_gpu()
    assert case_pndm_loop(variant)


@gpu
def test_graphed_pndm_replay_equals_its_eager_program_and_a_fresh_sampler():
    """GraphedSampler("pndm"): N + 1 = 7 replays of the captured step equal the same step program run eagerly, bit for bit; a
    second call with a new guide and prompt (ring, saved sample and counter reset, products refreshed in place) equals a
    fresh sampler's first call, bit for bit."""
    from tests import check_unet

    _need_gpu()
    _, munet, _, mcl = check_unet.build_pair("v1")
    mk = lambda: S.GraphedSampler(munet, mcl, 2, 128, 128, scheduler="pndm", num_inference_steps=6, guidance_scale=7.5, text_dim=64)
    gs = mk()
    outs = []
    for call in range(2):
        guide, cond, unc, lat0 = (v.cuda() if v is not None else None for v in _inputs(40 + call))
        cond, unc = cond.to(torch.bfloat16), unc.to(torch.bfloat16)
        eager = mk()(guide, cond, unc, latents=lat0, use_graph=False).clone()
        graphed = gs(guide, cond, unc, latents=lat0).clone()
        torch.cuda.synchronize()
        print(f"graphed pndm call {call}: max |graph - eager| {float((graphed - eager).abs().max()):.3e}, calls {gs.calls}, "
              f"launches/step {gs.launches_per_step}")
        assert torch.equal(graphed, eager), call
        outs.append((graphed, guide, cond, unc, lat0))
    fresh = mk()(*outs[1][1:4], latents=outs[1][4]).clone()
    torch.cuda.synchronize()
    assert torch.equal(outs[1][0], fresh)
    assert gs._graph is not None and gs.calls == 7


@gpu
@pytest.mark.parametrize("variant,scheduler,graphed", [("plain", "ddim", False), ("plain", "ddim", True), ("plain", "pndm", True),
                                                       ("none", "pndm", True), ("none", "pndm", False)])
def test_nocontrol_sampling_matches_oracle(variant, scheduler, graphed):
    _need_gpu()
    assert case_nocontrol(variant, scheduler, graphed)


@gpu
@pytest.mark.parametrize("variant", ["plain", "none"])
def test_generate_without_control_matches_oracle(variant):
    _need_gpu()
    assert case_generate_nocontrol(variant)


@gpu
def test_sample_class_images_end_to_end():
    _need_gpu()
    assert case_class_images()


# ------------------------------------------------------------------------------------------------ host-logic runner
def _main():
    import contextlib
    import io
    import time
    import traceback

    os.environ["CLB_EMU"] = "1"
    from controllora_b200 import ops
    from tests import _device, emu_ops

    assert _device.DEV == "cpu"
    ops.cfg_plms_step_dev = torch.no_grad()(emu_ops._shadow("cfg_plms_step_dev", ops.cfg_plms_step_dev, plms_step_restated))
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    bad = 0
    for name in sys.argv[1:] or list(CASES):
        t0 = time.time()
        buf = io.StringIO()
        try:
            with contextlib.redirect_stdout(buf):
                ok = bool(CASES[name]())
        except Exception:
            ok = False
            buf.write(traceback.format_exc())
        bad += not ok
        print(buf.getvalue(), flush=True)
        print(f"RESULT {name} {'OK' if ok else 'FAIL'} {time.time() - t0:.1f}", flush=True)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    _main()
