"""Stable Diffusion 2.x: per-block attention heads, linear projections and cross dim 1024 in the UNet, the GELU text tower,
and v-prediction sampling.

CPU: the SD-2 config / key set / parameter counts, config.json loading and the refused options, the CLIP restatement against
transformers at SD21_TEXT_CONFIG, the launchers' argument checks, the v tables and kernel restatements against the stateful
scheduler oracles (tests/sd2_ref.py), the point-mass property, and - in host-logic mode, in a subprocess running this file with
CLB_EMU=1 and the new wrappers replaced by their restatements - the samplers, generate and a tiny SD-2 UNet against the oracle.
GPU (-m gpu): the kernels against fp64 / their fp32 restatement, graph replay, the tiny SD-2 UNet fwd + bwd, the full-width
text tower, and v sampling at 768².  A real-weights case runs when CLB_SD21_DIR names a local SD-2.x diffusers checkpoint.

usage: python tests/test_sd2.py [case ...]      (host-logic mode; prints one `RESULT <case> OK|FAIL` line per case)"""
import json
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
from controllora_b200 import unet as U  # noqa: E402
from oracle import sampler_ref as SR  # noqa: E402
from tests import sd2_ref as R  # noqa: E402

# tiny SD-2-style UNet: heads per block (head dims 32, 32, 16; up blocks reversed), linear projections, cross dim 1024
TINY2 = dict(block_out_channels=(64, 128, 128, 128), layers_per_block=1, cross_attention_dim=1024, attention_head_dim=(2, 4, 4, 8),
             use_linear_projection=True, upcast_attention=True)
TINY2_LORA = dict(lora_block_out_channels=(64, 128, 128, 128),
                  lora_cross_attention_dims=([None, 1024] * 3, [None, 1024] * 3, [None, 1024] * 3, [None, 1024]))


# ------------------------------------------------------------------------------------------------ CPU: UNet config
def _count(sd):
    return sum(v.numel() for v in sd.values())


def test_sd21_config_keys_shapes_and_heads():
    sd = U.synthetic_state_dict(U.SD21_CONFIG)
    p = "down_blocks.1.attentions.0."
    assert sd[p + "proj_in.weight"].shape == (640, 640) and sd[p + "proj_out.weight"].shape == (640, 640)
    assert sd[p + "transformer_blocks.0.attn2.to_k.weight"].shape == (640, 1024)
    assert sd[p + "transformer_blocks.0.attn2.to_v.weight"].shape == (640, 1024)
    sd15 = U.synthetic_state_dict()
    assert set(sd) == set(sd15)                                  # same diffusers key set; only shapes differ
    assert sd15[p + "proj_in.weight"].shape == (640, 640, 1, 1)
    # diffusers' parameter counts of the two UNets (linear and 1x1-conv projections hold the same parameters)
    assert _count(sd15) == 859_520_964 and _count(sd) == 865_910_724
    down, up, mid = U.block_heads(U.SD21_CONFIG)
    assert (down, up, mid) == ([5, 10, 20, 20], [20, 20, 10, 5], 20)
    ch = U.SD21_CONFIG["block_out_channels"]
    assert [c // h for c, h in zip(ch, down)] == [64] * 4 and [c // h for c, h in zip(ch[::-1], up)] == [64] * 4
    assert U.block_heads(U.SD15_CONFIG) == ([8] * 4, [8] * 4, 8)
    with pytest.raises(ValueError):
        U.block_heads(dict(U.SD15_CONFIG, attention_head_dim=(5, 10)))


def test_oracle_unet_keys_match_ours():
    o = R.unet(TINY2)
    ours = U.synthetic_state_dict(TINY2)
    lin = R.to_linear_projection(o.state_dict())
    assert {k: tuple(v.shape) for k, v in lin.items()} == {k: tuple(v.shape) for k, v in ours.items()}
    heads = [(n, m.heads) for n, m in o._attn_modules().items()]
    assert dict(heads)["down_blocks.0.attentions.0.transformer_blocks.0.attn1.processor"] == 2
    assert dict(heads)["up_blocks.3.attentions.0.transformer_blocks.0.attn2.processor"] == 2
    assert dict(heads)["up_blocks.1.attentions.0.transformer_blocks.0.attn1.processor"] == 4
    assert dict(heads)["mid_block.attentions.0.transformer_blocks.0.attn1.processor"] == 8


def _load_config(tmp_path, raw, monkeypatch):
    from controllora_b200.unet_module import UNet2DConditionModel

    (tmp_path / "unet").mkdir(exist_ok=True)
    (tmp_path / "unet" / "config.json").write_text(json.dumps(raw))
    torch.save({}, tmp_path / "unet" / "diffusion_pytorch_model.bin")
    seen = {}
    monkeypatch.setattr(UNet2DConditionModel, "from_state_dict",
                        classmethod(lambda cls, sd, device="cuda", config=None: seen.setdefault("config", config)))
    UNet2DConditionModel.from_pretrained(str(tmp_path), subfolder="unet")
    return seen["config"]


SD15_JSON = {"_class_name": "UNet2DConditionModel", "act_fn": "silu", "attention_head_dim": 8,
             "block_out_channels": [320, 640, 1280, 1280], "center_input_sample": False, "cross_attention_dim": 768,
             "down_block_types": ["CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"],
             "downsample_padding": 1, "flip_sin_to_cos": True, "freq_shift": 0, "in_channels": 4, "layers_per_block": 2,
             "mid_block_scale_factor": 1, "norm_eps": 1e-05, "norm_num_groups": 32, "out_channels": 4, "sample_size": 64,
             "up_block_types": ["UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"]}
SD21_JSON = dict(SD15_JSON, attention_head_dim=[5, 10, 20, 20], cross_attention_dim=1024, dual_cross_attention=False,
                 use_linear_projection=True, upcast_attention=True, only_cross_attention=False, class_embed_type=None,
                 num_class_embeds=None, resnet_time_scale_shift="default", sample_size=96)


def test_from_pretrained_reads_sd2_and_sd15_configs(tmp_path, monkeypatch):
    cfg = _load_config(tmp_path, SD21_JSON, monkeypatch)
    assert cfg == dict(attention_head_dim=(5, 10, 20, 20), block_out_channels=(320, 640, 1280, 1280), cross_attention_dim=1024,
                       in_channels=4, layers_per_block=2, norm_eps=1e-5, norm_num_groups=32, out_channels=4,
                       use_linear_projection=True, upcast_attention=True)
    # an SD-1.5 config.json (with or without the SD-2 switches at their defaults) gives exactly the keys it gave before
    want15 = dict(attention_head_dim=8, block_out_channels=(320, 640, 1280, 1280), cross_attention_dim=768, in_channels=4,
                  layers_per_block=2, norm_eps=1e-5, norm_num_groups=32, out_channels=4)
    assert _load_config(tmp_path, SD15_JSON, monkeypatch) == want15
    assert _load_config(tmp_path, dict(SD15_JSON, use_linear_projection=False, upcast_attention=False, class_embed_type=None,
                                       resnet_time_scale_shift="default"), monkeypatch) == want15


@pytest.mark.parametrize("key,value", [("class_embed_type", "timestep"), ("num_class_embeds", 1000), ("only_cross_attention", True),
                                       ("only_cross_attention", [False, True, False, False]), ("dual_cross_attention", True),
                                       ("resnet_time_scale_shift", "scale_shift"), ("in_channels", 5), ("in_channels", 9)])
def test_from_pretrained_refuses_unbuilt_options(tmp_path, monkeypatch, key, value):
    with pytest.raises(NotImplementedError, match=key):
        _load_config(tmp_path, dict(SD21_JSON, **{key: value}), monkeypatch)


def test_scheduler_prediction_type(tmp_path):
    (tmp_path / "scheduler").mkdir()
    f = tmp_path / "scheduler" / "scheduler_config.json"
    f.write_text(json.dumps({"_class_name": "DDIMScheduler", "prediction_type": "v_prediction", "beta_start": 0.00085}))
    assert S.scheduler_prediction_type(tmp_path) == "v_prediction"
    f.write_text(json.dumps({"_class_name": "PNDMScheduler"}))
    assert S.scheduler_prediction_type(tmp_path) == "epsilon"
    f.write_text(json.dumps({"prediction_type": "sample"}))
    with pytest.raises(ValueError):
        S.scheduler_prediction_type(tmp_path)


# ------------------------------------------------------------------------------------------------ CPU: text encoder
def test_clip_oracle_equals_transformers_at_sd21_width():
    """The SD-2 text-tower oracle (tests/sd2_ref.py clip_text_forward, the fp32 reference of every CLIPTextModel test here)
    equals transformers.CLIPTextModel at SD21_TEXT_CONFIG, whose parameter count is SD-2's text encoder's; with
    hidden_act quick_gelu it equals the SD-1.5 oracle (oracle/clip_ref.py)."""
    import transformers

    from controllora_b200.clip import SD21_TEXT_CONFIG as C2
    from oracle import clip_ref as CR

    hf_cfg = transformers.CLIPTextConfig(vocab_size=C2["vocab_size"], hidden_size=C2["hidden_size"],
                                         intermediate_size=C2["intermediate_size"], num_hidden_layers=C2["num_hidden_layers"],
                                         num_attention_heads=C2["num_attention_heads"],
                                         max_position_embeddings=C2["max_position_embeddings"], hidden_act=C2["hidden_act"],
                                         layer_norm_eps=C2["layer_norm_eps"])
    torch.manual_seed(0)
    m = transformers.CLIPTextModel(hf_cfg).eval()
    assert sum(p.numel() for p in m.parameters()) == 340_387_840
    sd = {k: v for k, v in m.state_dict().items() if "position_ids" not in k}
    ids = torch.randint(0, C2["vocab_size"], (2, 77), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = m(ids)[0]
        got = R.clip_text_forward(sd, ids, C2)
    assert float((got - want).abs().max()) < 1e-4
    c15 = dict(CR.SD15_TEXT_CONFIG, num_hidden_layers=2, vocab_size=1000)
    sd15 = CR.synthetic_state_dict(c15, seed=0)
    ids15 = torch.randint(0, 1000, (2, 77), generator=torch.Generator().manual_seed(2))
    assert float((R.clip_text_forward(sd15, ids15, c15) - CR.clip_text_forward(sd15, ids15, c15)).abs().max()) < 1e-4


def test_clip_refuses_other_activations():
    from controllora_b200.clip import CLIPTextModel

    with pytest.raises(NotImplementedError, match="relu"):
        CLIPTextModel({}, "cuda", dict(hidden_act="relu"))


# ------------------------------------------------------------------------------------------------ CPU: launchers
def test_new_launchers_reject_bad_arguments_without_a_gpu(built_lib):
    import ctypes

    from controllora_b200 import _lib

    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ctr = ctypes.c_uint64(0)
    pc = ctypes.cast(ctypes.byref(ctr), ctypes.c_void_p)
    for n in (0, -8, 12):
        assert lib.cl_gelu(p, ctypes.c_int64(n), None) == -1
        assert b"cl_gelu" in lib.cl_last_error()
    assert lib.cl_gelu(None, ctypes.c_int64(8), None) == -1
    f = lib.cl_cfg_solver_step_v_dev
    g = ctypes.c_float(7.5)
    for i in (0, 1, 3, 4):                                        # every required pointer null in turn
        args = [p, p, p, p, pc]
        args[i] = None
        assert f(*args, ctypes.c_int64(8), g, 0, None) == -1, i
        assert b"null" in lib.cl_last_error()
    assert f(p, p, None, p, pc, ctypes.c_int64(8), g, 1, None) == -1 and b"x0_prev" in lib.cl_last_error()
    assert f(p, p, p, p, pc, ctypes.c_int64(8), g, 2, None) == -1 and b"kind" in lib.cl_last_error()
    assert f(p, p, p, p, pc, ctypes.c_int64(0), g, 0, None) == -1 and b"n_half" in lib.cl_last_error()
    f = lib.cl_cfg_plms_step_v_dev
    for i in range(6):
        args = [p] * 5 + [pc]
        args[i] = None
        assert f(*args, 8, 7.5, None) == -1, i
        assert b"null" in lib.cl_last_error()
    assert f(p, p, p, p, p, pc, 0, 7.5, None) == -1 and b"n_half" in lib.cl_last_error()


def test_prediction_type_is_checked():
    with pytest.raises(ValueError):
        S.pndm_rows(5, S.sd15_alphas_cumprod(), prediction_type="sample")
    with pytest.raises(ValueError):
        S.GraphedSampler(None, None, 1, prediction_type="v")


# ------------------------------------------------------------------------------------------------ CPU: v tables vs the oracles
def _pm(xs, e0, a, t):
    return a[t].sqrt() * xs + (1 - a[t]).sqrt() * e0


@pytest.mark.parametrize("n", [1, 2, 3, 5, 10, 50])
def test_pndm_v_rows_equal_the_oracle_step_by_step(n):
    """10-column rows + restated kernel == PNDMPLMSV.step after every call, the restart included (fp64 both sides); the
    epsilon columns are the epsilon rows."""
    rows = S.pndm_rows(n, S.sd15_alphas_cumprod(), prediction_type="v_prediction")
    assert [r[:8] for r in rows] == S.pndm_rows(n, S.sd15_alphas_cumprod()) and all(len(r) == 10 for r in rows)
    g = torch.Generator().manual_seed(n)
    x = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    sched = R.PNDMPLMSV(n, ac=SR.alphas_cumprod())
    rt = torch.tensor(rows, dtype=torch.float64)
    xm, ring, saved, ctr = x.clone(), torch.zeros((3,) + tuple(x.shape), dtype=torch.float64), torch.zeros_like(x), torch.zeros(1, dtype=torch.int64)
    for k, t in enumerate(sched.timesteps):
        v2 = torch.randn(4, 4, 8, 8, generator=g, dtype=torch.float64)
        x = sched.step(SR.cfg_combine(v2[:2], v2[2:], 7.5), t, x)
        R.plms_v_step_restated(v2, xm, ring, saved, rt, ctr, 7.5)
        assert float((xm - x).abs().max() / x.abs().max()) < 1e-12, (n, k, t)


@pytest.mark.parametrize("kind,n", [(0, 1), (0, 2), (0, 50), (1, 1), (1, 2), (1, 10), (1, 25)])
def test_solver_v_table_equals_the_oracle_step_by_step(kind, n):
    ts, rows = S.solver_table(kind, n)
    coef = torch.tensor(rows, dtype=torch.float64)
    g = torch.Generator().manual_seed(10 * n + kind)
    x = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    xm, x0p, ctr = x.clone(), torch.zeros_like(x), torch.zeros(1, dtype=torch.int64)
    sched = R.DPMSolverPP2MV(n) if kind == 1 else None
    for k, t in enumerate(ts):
        v2 = torch.randn(4, 4, 8, 8, generator=g, dtype=torch.float64)
        if kind == 0:
            x = R.cfg_ddim_step_v(v2[:2], v2[2:], x, t, n, 7.5)
        else:
            x = sched.step(SR.cfg_combine(v2[:2], v2[2:], 7.5), t, x)
        R.solver_v_step_restated(v2, xm, x0p, coef, ctr, 7.5, kind)
        assert float((xm - x).abs().max() / x.abs().max()) < 1e-12, (kind, n, k, t)


@pytest.mark.parametrize("scheduler,n", [("ddim", 1), ("ddim", 20), ("dpmpp", 2), ("dpmpp", 25), ("pndm", 1), ("pndm", 2), ("pndm", 5), ("pndm", 50)])
def test_v_samplers_on_the_point_mass_ode(scheduler, n):
    """Property pin: for data on one point x*, the exact v along x_t = sqrt(a_t) x* + sqrt(1 - a_t) eps0 is
    v = sqrt(a_t) eps0 - sqrt(1 - a_t) x*.  DDIM and DPM-Solver++ convert each v at its own timestep, so the oracles and the
    table programs land on sqrt(a_0) x* + sqrt(1 - a_0) eps0 exactly.  PNDM combines v from several timesteps before it converts
    (diffusers' order), and v is not constant along the trajectory: only its single-call loop is exact.  For longer PNDM loops no
    error bound is derived; what is pinned there is the table program == the oracle (1e-12)."""
    g = torch.Generator().manual_seed(0)
    xs, e0 = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64), torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64)
    a = SR.alphas_cumprod()
    vel = lambda x, t: a[t].sqrt() * (x - a[t].sqrt() * xs) / (1 - a[t]).sqrt() - (1 - a[t]).sqrt() * xs
    final = _pm(xs, e0, a, 0)
    if scheduler == "pndm":
        sched = R.PNDMPLMSV(n, ac=a)
        ts, step = sched.timesteps, lambda v, t, x: sched.step(v, t, x)
        rows = torch.tensor(S.pndm_rows(n, S.sd15_alphas_cumprod(), prediction_type="v_prediction"), dtype=torch.float64)
    else:
        kind = 0 if scheduler == "ddim" else 1
        ts, rows = S.solver_table(kind, n)
        rows = torch.tensor(rows, dtype=torch.float64)
        sched = R.DPMSolverPP2MV(n) if kind else None
        step = (lambda v, t, x: sched.step(v, t, x)) if kind else (lambda v, t, x: R.cfg_ddim_step_v(v, v, x, t, n, 7.5))
    x = _pm(xs, e0, a, ts[0])
    for t in ts:
        x = step(vel(x, t), t, x)
    if scheduler != "pndm" or n == 1:
        assert float((x - final).abs().max()) < 1e-9, ("oracle", scheduler, n)
    x_oracle = x
    x = _pm(xs, e0, a, ts[0])
    ring, saved, x0p, ctr = torch.zeros((3,) + tuple(x.shape), dtype=torch.float64), torch.zeros_like(x), torch.zeros_like(x), torch.zeros(1, dtype=torch.int64)
    for t in ts:
        v = vel(x, t)
        if scheduler == "pndm":
            R.plms_v_step_restated(torch.cat([v, v]), x, ring, saved, rows, ctr, 7.5)
        else:
            R.solver_v_step_restated(torch.cat([v, v]), x, x0p, rows, ctr, 7.5, 0 if scheduler == "ddim" else 1)
    assert float((x - x_oracle).abs().max()) < 1e-12, ("table", scheduler, n)


# ------------------------------------------------------------------------------------------------ cases (host-logic mode and GPU)
def _dev():
    from tests._device import DEV

    return DEV


def _sync():
    from tests._device import sync

    sync()


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def build_pair(variant, seed=0):
    """Oracle and package UNet of TINY2 with the same bf16-rounded weights (ours loaded from a linear-projection state dict),
    and the processors of `variant`: "none", "plain" (DreamBooth LoRACrossAttnProcessor(cross_attention_dim=1024) on every
    layer), "v1" or "v2" (a ControlLoRA at cross dim 1024, fused path), "v1_stacked" (v1 + a pre-LoRA: the generic chain path)."""
    from oracle import models_ref as MR
    from oracle import unet_ref as UR
    import controllora_b200 as cb

    dev = _dev()
    torch.manual_seed(seed)
    ounet = R.unet(TINY2)
    UR.init_synthetic_(ounet, seed=1)
    with torch.no_grad():
        for p in ounet.parameters():
            p.copy_(p.to(torch.bfloat16).float())
    sd = R.to_linear_projection({k: v.detach().clone() for k, v in ounet.state_dict().items()})
    munet = cb.UNet2DConditionModel.from_state_dict(sd, dev, TINY2)
    ocl = mcl = None
    if variant == "plain":
        oprocs, mprocs = {}, {}
        g = torch.Generator().manual_seed(7)
        for name, oa in ounet._attn_modules().items():
            C = oa.to_q.weight.shape[0]
            xd = None if name.endswith("attn1.processor") else 1024
            op = MR.LoRACrossAttnProcessor(C, xd, rank=4)
            for n_, p_ in op.named_parameters():
                if n_.endswith("up.weight"):
                    with torch.no_grad():
                        p_.copy_(0.05 * torch.randn(p_.shape, generator=g))
            mp = cb.LoRACrossAttnProcessor(C, xd, rank=4)
            mp.load_state_dict(op.state_dict())
            oprocs[name], mprocs[name] = op, mp.to(dev)
        ounet.set_attn_processor(oprocs)
        munet.set_attn_processor(mprocs)
    elif variant != "none":
        kw = dict(TINY2_LORA)
        if variant == "v2":
            kw.update(lora_control_version=2, lora_pre_conv_skipped=True)
        ocl, mcl = MR.ControlLoRA(**kw), cb.ControlLoRA(**kw)
        MR.randomize_lora_up_(ocl, seed=3, std=0.05)
        mcl.load_state_dict(ocl.state_dict())
        mcl.to(dev)
        oprocs, mprocs = MR.wire_processors(ounet, ocl), MR.wire_processors(munet, mcl)
        if variant == "v1_stacked":
            g = torch.Generator().manual_seed(11)
            for name in oprocs:
                op = MR.LoRACrossAttnProcessor(oprocs[name].hidden_size, oprocs[name].cross_attention_dim, rank=4)
                for n_, p_ in op.named_parameters():
                    if n_.endswith("up.weight"):
                        with torch.no_grad():
                            p_.copy_(0.05 * torch.randn(p_.shape, generator=g))
                mp = cb.LoRACrossAttnProcessor(oprocs[name].hidden_size, oprocs[name].cross_attention_dim, rank=4).to(dev)
                mp.load_state_dict(op.state_dict())
                oprocs[name].inject_pre_lora(op)
                mprocs[name].inject_pre_lora(mp)
                oprocs[name]._extra, mprocs[name]._extra = op, mp
    return ounet, munet, ocl, mcl


def case_unet(variant):
    """Forward + backward of the tiny SD-2 UNet against the fp32 oracle, check_unet's tolerances (noise prediction <= 2e-2, worst
    LoRA gradient tensor <= 8e-2), with a v-prediction target sqrt(a) eps - sqrt(1 - a) x0 (the SD-2.1 training loss)."""
    dev = _dev()
    B, HW = 2, 16
    ounet, munet, ocl, mcl = build_pair(variant)
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(B, 4, HW, HW, generator=g)
    noise = torch.randn(B, 4, HW, HW, generator=g)
    t = torch.tensor([17, 801])
    sample = SR.add_noise(x0.double(), noise.double(), t).float().to(torch.bfloat16).float()
    target = SR.get_velocity(x0.double(), noise.double(), t).float()
    ehs = torch.randn(B, 77, 1024, generator=g).to(torch.bfloat16).float()
    ctrl_o, ctrl_m = [], []
    if ocl is not None:
        cc = [256] * 4 if variant == "v2" else list(TINY2["block_out_channels"])
        for lvl in range(4):
            s = HW >> lvl
            c = (0.5 * torch.randn(B, cc[lvl], s, s, generator=g)).to(torch.bfloat16).float()
            co, cm = c.clone().requires_grad_(True), c.clone().to(dev).requires_grad_(True)
            ctrl_o.append(co)
            ctrl_m.append(cm)
            for p in ocl.lora_layers[lvl]:
                p.inject_control_states(co)
            for p in mcl.lora_layers[lvl]:
                p.inject_control_states(cm)
    po = ounet(sample, t, ehs).sample
    lo = torch.nn.functional.mse_loss(po, target)
    pm = munet(sample.to(dev), t.to(dev), ehs.to(dev).to(torch.bfloat16)).sample
    lm = torch.nn.functional.mse_loss(pm, target.to(dev))
    worst = 0.0
    if variant != "none":
        lo.backward()
        lm.backward()
        _sync()
        for name in ounet.attn_processors:
            op, mp = ounet.attn_processors[name], munet.attn_processors[name]
            pairs = [(op, mp)] + ([(op._extra, mp._extra)] if hasattr(op, "_extra") else [])
            for o_, m_ in pairs:
                for (n1, p1), (n2, p2) in zip(o_.named_parameters(), m_.named_parameters()):
                    if p1.grad is not None:
                        assert p2.grad is not None, (name, n2)
                        worst = max(worst, _rel(p2.grad, p1.grad))
        for co, cm in zip(ctrl_o, ctrl_m):
            worst = max(worst, _rel(cm.grad, co.grad))
    _sync()
    e = _rel(pm, po)
    print(f"[unet {variant}] noise-pred rel {e:.3e}, worst gradient rel {worst:.3e}")
    return e < 2e-2 and worst < 8e-2


def _inputs(seed, B=2, HW=16, with_guide=True):
    g = torch.Generator().manual_seed(seed)
    guide = (torch.rand(B, 3, HW * 8, HW * 8, generator=g) * 2 - 1).to(torch.bfloat16).float() if with_guide else None
    cond = torch.randn(B, 77, 1024, generator=g).to(torch.bfloat16).float()
    unc = torch.randn(B, 77, 1024, generator=g).to(torch.bfloat16).float()
    return guide, cond, unc, torch.randn(B, 4, HW, HW, generator=g)


def _oracle_chain(ounet, ocl, guide, cond, unc, lat0, scheduler, steps, guidance=7.5):
    B = lat0.shape[0]
    with torch.no_grad():
        if ocl is not None:
            ocl(torch.cat([guide, guide], 0))
        x = lat0.clone()
        run = lambda x, t: ounet(torch.cat([x, x], 0), torch.full((2 * B,), int(t)), torch.cat([unc, cond], 0)).sample
        if scheduler == "ddim":
            for t in SR.timesteps(steps):
                v = run(x, t)
                x = R.cfg_ddim_step_v(v[:B], v[B:], x, t, steps, guidance)
        elif scheduler == "dpmpp":
            sched = R.DPMSolverPP2MV(steps)
            for t in sched.timesteps:
                v = run(x, t)
                x = sched.step(SR.cfg_combine(v[:B], v[B:], guidance), t, x)
        else:
            sched = R.PNDMPLMSV(steps)
            for t in sched.timesteps:
                v = run(x, t)
                x = sched.step(SR.cfg_combine(v[:B], v[B:], guidance), t, x)
    return x


def case_sampler(scheduler, variant="v1", graphed=True):
    """v-prediction sampling on the tiny SD-2 UNet against the oracle chain: GraphedSampler's step program, and the eager loop
    (bit for bit equal to it in host-logic mode)."""
    dev = _dev()
    ounet, munet, ocl, mcl = build_pair(variant)
    guide, cond, unc, lat0 = _inputs(31, with_guide=mcl is not None)
    steps = {"ddim": 3, "dpmpp": 3, "pndm": 4}[scheduler]
    want = _oracle_chain(ounet, ocl, guide, cond, unc, lat0, scheduler, steps)
    gd = None if guide is None else guide.to(dev)
    c, u = cond.to(dev).to(torch.bfloat16), unc.to(dev).to(torch.bfloat16)
    gs = S.GraphedSampler(munet, mcl, 2, 128, 128, scheduler=scheduler, num_inference_steps=steps, prediction_type="v_prediction")
    a = gs(gd, c, u, latents=lat0.to(dev), use_graph=graphed and dev == "cuda").clone()
    fn = {"ddim": S.ddim_sample, "dpmpp": S.dpmpp_sample, "pndm": S.pndm_sample}[scheduler]
    b = fn(munet, mcl, gd, c, u, num_inference_steps=steps, latents=lat0.to(dev), prediction_type="v_prediction")
    _sync()
    e_or, e_loop = _rel(a, want), _rel(a, b)
    print(f"[v sampler {scheduler} {variant}] graphed vs oracle {e_or:.3e}, vs eager loop {e_loop:.3e}")
    # the v loops of this random-weight UNet double the latents' norm, and x0 = sqrt(a) x - sqrt(1 - a) v passes the bf16 UNet
    # error on at full weight at high t: the latent error is about twice the epsilon loops' (whose bound is 8e-2).  Driven by
    # the fp32 oracle UNet, the same loops agree with the oracle chain to 1e-5.
    return e_or < 1.5e-1 and e_loop <= (0.0 if dev == "cpu" else 2e-2)


def _tiny_vae_clip():
    """Tiny VAE and a two-layer gelu text tower at SD-2's width (1024, 16 heads of 64), bf16-rounded weights."""
    import controllora_b200 as cb
    from controllora_b200.clip import SD21_TEXT_CONFIG
    from oracle import clip_ref as CR
    from oracle import vae_ref as VR

    dev = _dev()
    vcfg = dict(block_out_channels=(32, 64, 64, 64), layers_per_block=1)
    ovae = VR.AutoencoderKL(**vcfg)
    VR.init_synthetic_(ovae, seed=4)
    mvae = cb.AutoencoderKL.from_state_dict({k: v.detach().clone() for k, v in ovae.state_dict().items()}, dev, vcfg)
    ccfg = dict(SD21_TEXT_CONFIG, num_hidden_layers=2, vocab_size=1000, intermediate_size=512)
    csd = {k: v.to(torch.bfloat16).float() for k, v in CR.synthetic_state_dict(ccfg, seed=3).items()}
    mclip = cb.CLIPTextModel.from_state_dict(csd, dev, ccfg)
    return ovae, mvae, csd, ccfg, mclip


def case_clip():
    """CLIPTextModel's program at SD-2 width with the gelu MLP (cl_gelu), 3 layers, against the text-tower oracle."""
    import controllora_b200 as cb
    from controllora_b200.clip import SD21_TEXT_CONFIG
    from oracle import clip_ref as CR

    dev = _dev()
    cfg = dict(SD21_TEXT_CONFIG, num_hidden_layers=3)
    sd = {k: v.to(torch.bfloat16).float() for k, v in CR.synthetic_state_dict(cfg, seed=5).items()}
    ids = torch.randint(0, cfg["vocab_size"], (2, 77), generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        want = R.clip_text_forward(sd, ids, cfg)
    got = cb.CLIPTextModel.from_state_dict(sd, dev, cfg)(ids.to(dev))[0]
    _sync()
    err = _rel(got, want)
    print(f"[clip sd2 width] last_hidden_state rel err {err:.3e}")
    return tuple(got.shape) == (2, 77, 1024) and err < 2e-2


def case_generate(variant="v1", scheduler="dpmpp"):
    """generate(prediction_type="v_prediction"): ids -> gelu text tower -> v loop on the tiny SD-2 UNet -> VAE decode."""
    dev = _dev()
    ounet, munet, ocl, mcl = build_pair(variant)
    ovae, mvae, csd, ccfg, mclip = _tiny_vae_clip()
    g = torch.Generator().manual_seed(37)
    ids = torch.randint(0, 1000, (2, 77), generator=g)
    neg = torch.randint(0, 1000, (2, 77), generator=g)
    lat0 = torch.randn(2, 4, 16, 16, generator=g)
    guide = (torch.rand(2, 3, 128, 128, generator=g) * 2 - 1).to(torch.bfloat16).float() if mcl is not None else None
    with torch.no_grad():
        cond, unc = R.clip_text_forward(csd, ids, ccfg), R.clip_text_forward(csd, neg, ccfg)
        x = _oracle_chain(ounet, ocl, guide, cond, unc, lat0, scheduler, 3)
        want = (ovae.decode(x) / 2 + 0.5).clamp(0, 1)
    got = S.generate(munet, mcl, mvae, mclip, None if guide is None else guide.to(dev), ids.to(dev), neg.to(dev),
                     num_inference_steps=3, scheduler=scheduler, latents=lat0.to(dev), prediction_type="v_prediction")
    _sync()
    err = _rel(got, want)
    print(f"[generate v {variant} {scheduler}] image rel err {err:.3e}")
    return err < 5e-2 and tuple(got.shape) == (2, 3, 128, 128)


def case_train(variant):
    """One fused Trainer step on the tiny SD-2 UNet (prediction_type "v_prediction", the v target built on the host): the gradient
    arena against the oracle's autograd gradients, check_hint.train_case's gradient tolerance (<= 5e-2 on the concatenated
    gradient, provably-zero-gradient biases excluded).  variant "plain" is the DreamBooth step: Trainer(unet, None) over the
    LoRACrossAttnProcessor(cross_attention_dim=1024) adapters installed on the UNet, no ControlLoRA."""
    from controllora_b200.trainer import Trainer
    from tests.check_hint import _zero_grad_biases

    dev = _dev()
    B, HW = 2, 16
    ounet, munet, ocl, mcl = build_pair(variant)
    for n, p in ounet.named_parameters():                           # frozen UNet; the wired processors stay trainable
        if ".processor." not in n:
            p.requires_grad_(False)
    tr = Trainer(munet, mcl, lr=1e-4, prediction_type="v_prediction")
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(B, 4, HW, HW, generator=g)
    noise = torch.randn(B, 4, HW, HW, generator=g)
    t = torch.randint(0, 1000, (B,), generator=g)
    x = SR.add_noise(x0.double(), noise.double(), t).float().to(torch.bfloat16).float()
    tgt = SR.get_velocity(x0.double(), noise.double(), t).float()
    e = torch.randn(B, 77, 1024, generator=g).to(torch.bfloat16).float()
    guide = (torch.rand(B, 3, HW * 8, HW * 8, generator=g) * 2 - 1).to(torch.bfloat16).float()
    if ocl is None:
        oparams = [p for op in ounet.attn_processors.values() for p in op.parameters()]
        torch.nn.functional.mse_loss(ounet(x, t, e).sample, tgt).backward()
        lm = tr._forward_backward(x.to(dev), t.to(dev).float(), e.to(dev).to(torch.bfloat16), None, tgt.to(dev))
        _sync()
        if tr.numel != sum(p.numel() for p in oparams):
            return False
        err = _rel(tr.flat_g[:tr.numel].detach().float().cpu(), torch.cat([p.grad.flatten() for p in oparams]))
        print(f"[train {variant}] loss {float(lm):.5f}, gradient arena rel {err:.3e}")
        return err < 5e-2
    ocl(guide)
    torch.nn.functional.mse_loss(ounet(x, t, e).sample, tgt).backward()
    lm = tr._forward_backward(x.to(dev), t.to(dev).float(), e.to(dev).to(torch.bfloat16), guide.to(dev), tgt.to(dev))
    _sync()
    zero_b = _zero_grad_biases(ocl)
    pairs = [(n, po, pm) for (n, po), (_, pm) in zip(ocl.named_parameters(), mcl.named_parameters()) if n not in zero_b]
    unused = [pm for _, po, pm in pairs if po.grad is None]          # adapters the wiring leaves idle: no gradient either side
    if any(float(tr.arena.grad_of(pm).abs().max()) != 0.0 for pm in unused):
        return False
    sel = [x for x in pairs if x[1].grad is not None]
    err = _rel(torch.cat([tr.arena.grad_of(pm).detach().float().cpu().flatten() for _, _, pm in sel]),
               torch.cat([po.grad.flatten() for _, po, _ in sel]))
    print(f"[train {variant}] loss {float(lm):.5f}, gradient arena rel {err:.3e}")
    return err < 5e-2


CASES = {
    "unet_none": lambda: case_unet("none"),
    "unet_plain_lora_1024": lambda: case_unet("plain"),
    "unet_v1": lambda: case_unet("v1"),
    "unet_v2": lambda: case_unet("v2"),
    "unet_v1_stacked_generic": lambda: case_unet("v1_stacked"),
    "sampler_ddim_v1": lambda: case_sampler("ddim"),
    "sampler_dpmpp_v2": lambda: case_sampler("dpmpp", "v2"),
    "sampler_pndm_plain": lambda: case_sampler("pndm", "plain"),
    "generate_v1_dpmpp": case_generate,
    "generate_nocontrol_pndm": lambda: case_generate("none", "pndm"),
    "train_v1": lambda: case_train("v1"),
    "train_v2": lambda: case_train("v2"),
    "train_lora_only_1024": lambda: case_train("plain"),
    "clip_sd2_width": case_clip,
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
@pytest.mark.parametrize("numel", [8, 8 * 4097, 4 * 77 * 4096])
def test_gelu_kernel_against_fp64(numel):
    """cl_gelu on a view inside a sentinel canvas: every output within one bf16 rounding of the fp64 GELU of the bf16 input plus
    the fp32 evaluation error (erff <= 2 ulp and the products: <= 8 fp32 ulp of |x|), sentinels untouched; inputs span the bf16
    range (tiny, denormal, +-large, zero)."""
    from controllora_b200 import ops

    _need_gpu()
    g = torch.Generator(device="cuda").manual_seed(numel)
    edge = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 3e38, -3e38, 6.0, -6.0, 1e-3, -3.0, 0.5, -0.5, 10.0, -10.0, 100.0, -100.0],
                        device="cuda")
    body = torch.randn(max(numel - 16, 0), generator=g, device="cuda") * 4.0
    x0 = torch.cat([edge, body])[:numel].to(torch.bfloat16)
    pad = 64
    canvas = torch.full((numel + 2 * pad,), -7.0, device="cuda").to(torch.bfloat16)
    canvas[pad:pad + numel] = x0
    view = canvas[pad:pad + numel]
    ops.gelu_(view)
    torch.cuda.synchronize()
    assert torch.all(canvas[:pad] == -7.0) and torch.all(canvas[pad + numel:] == -7.0), "sentinel overwritten"
    x64 = x0.double()
    ref = 0.5 * x64 * (1 + torch.erf(x64 / math.sqrt(2.0)))
    got = view.double()
    ulp_bf16 = torch.where(ref == 0, torch.zeros_like(ref), 2.0 ** (torch.floor(torch.log2(ref.abs().clamp_min(1e-38))) - 7))
    bound = 0.5 * ulp_bf16 + 8 * 2.0 ** -23 * x64.abs() + 1e-38
    err = (got - ref).abs()
    assert torch.all(err <= bound + 0.5 * ulp_bf16), float((err - bound).max())
    # against the torch restatement (fp32 erf, one bf16 rounding): at most one bf16 step apart, element by element
    restated = R.gelu_restated(x0.clone()).double()
    step = torch.where(restated == 0, torch.full_like(restated, 2.0 ** -133),
                       2.0 ** (torch.floor(torch.log2(restated.abs().clamp_min(2.0 ** -133))) - 7))
    assert torch.all((got - restated).abs() <= step), float(((got - restated).abs() - step).max())


def _v_kernel_run(kind, n, step_fn, rows, restated):
    """Each row from the restatement's state: the kernel's new sample within 6 fp32 ulp of the restated one's scale, the pushed
    v / x0 and the saved sample equal, the counter + 1."""
    g = torch.Generator().manual_seed(100 + n + 7 * kind)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ring, saved, x0p = torch.zeros(3, 2, 4, 16, 16), torch.zeros_like(x), torch.zeros_like(x)
    ulp = 2.0 ** -23
    rows_d = torch.tensor(rows, dtype=torch.float32, device="cuda")
    rows_h = torch.tensor(rows, dtype=torch.float32)
    for k in range(len(rows)):
        v2 = torch.randn(4, 4, 16, 16, generator=g)
        xm, rm, sm, pm = x.cuda(), ring.cuda(), saved.cuda(), x0p.cuda()
        ctr = torch.full((1,), k, dtype=torch.int64, device="cuda")
        ch = torch.full((1,), k, dtype=torch.int64)
        if kind == 2:
            step_fn(v2.cuda(), xm, rm, sm, rows_d, ctr, 7.5)
            restated(v2, x, ring, saved, rows_h, ch, 7.5)
        else:
            step_fn(v2.cuda(), xm, pm, rows_d, ctr, 7.5, kind)
            restated(v2, x, x0p, rows_h, ch, 7.5, kind)
        torch.cuda.synchronize()
        assert int(ctr) == k + 1, k
        d = float((xm.cpu() - x).abs().max())
        assert d <= 6 * ulp * float(x.abs().max()), (kind, n, k, d)
        if kind == 2:
            assert float((rm.cpu() - ring).abs().max()) <= 2 * ulp * float(ring.abs().max() + 1e-30), k
            assert torch.equal(sm.cpu(), saved), k
        elif kind == 1:
            assert float((pm.cpu() - x0p).abs().max()) <= 6 * ulp * float(x0p.abs().max()), k
        # continue from the kernel's own state
        x = xm.cpu()
        if kind == 2:
            ring, saved = rm.cpu(), sm.cpu()
        else:
            x0p = pm.cpu()


@gpu
@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("n", [1, 2, 50])
def test_v_step_kernels_match_their_restatement_on_every_row(kind, n):
    from controllora_b200 import ops

    _need_gpu()
    if kind == 2:
        _v_kernel_run(2, n, ops.cfg_plms_step_v_dev, S.pndm_rows(n, S.sd15_alphas_cumprod(), prediction_type="v_prediction"),
                      R.plms_v_step_restated)
    else:
        _v_kernel_run(kind, n, ops.cfg_solver_step_v_dev, S.solver_table(kind, n)[1], R.solver_v_step_restated)


@gpu
@pytest.mark.parametrize("scheduler", ["ddim", "dpmpp", "pndm"])
def test_graphed_v_sampler_replay_equals_eager(scheduler):
    _need_gpu()
    _, munet, _, mcl = build_pair("v1")
    mk = lambda: S.GraphedSampler(munet, mcl, 2, 128, 128, scheduler=scheduler, num_inference_steps=5, prediction_type="v_prediction")
    guide, cond, unc, lat0 = (v.cuda() for v in _inputs(40))
    cond, unc = cond.to(torch.bfloat16), unc.to(torch.bfloat16)
    eager = mk()(guide, cond, unc, latents=lat0, use_graph=False).clone()
    graphed = mk()(guide, cond, unc, latents=lat0).clone()
    torch.cuda.synchronize()
    assert torch.equal(graphed, eager)


@gpu
@pytest.mark.parametrize("variant", ["none", "plain", "v1", "v2", "v1_stacked"])
def test_tiny_sd2_unet_matches_oracle(variant):
    _need_gpu()
    assert case_unet(variant)


@gpu
@pytest.mark.parametrize("scheduler,variant", [("ddim", "v1"), ("dpmpp", "v2"), ("pndm", "plain")])
def test_v_sampling_matches_oracle(scheduler, variant):
    _need_gpu()
    assert case_sampler(scheduler, variant)


@gpu
@pytest.mark.parametrize("variant", ["v1", "v2", "plain"])
def test_train_step_v_target_matches_oracle(variant):
    _need_gpu()
    assert case_train(variant)


@gpu
def test_generate_v_matches_oracle():
    _need_gpu()
    assert case_generate()


@gpu
def test_sd21_text_tower_matches_transformers():
    """Full SD-2 text tower width (23 layers, 1024, 16 heads of 64, MLP 4096, gelu; the fused q|k|v GEMM has N = 3072) against
    transformers.CLIPTextModel in fp32 on the same bf16-rounded weights: relative L2 of last_hidden_state <= 2e-2 (the SD-1.5
    text tower's cap in tests/check_clip.py is 3e-2)."""
    import transformers

    import controllora_b200 as cb
    from controllora_b200.clip import SD21_TEXT_CONFIG as C2

    _need_gpu()
    torch.manual_seed(0)
    hf = transformers.CLIPTextModel(transformers.CLIPTextConfig(
        vocab_size=C2["vocab_size"], hidden_size=1024, intermediate_size=4096, num_hidden_layers=23, num_attention_heads=16,
        max_position_embeddings=77, hidden_act="gelu", layer_norm_eps=1e-5)).eval()
    with torch.no_grad():
        for p in hf.parameters():
            p.copy_(p.to(torch.bfloat16).float())
    sd = {k: v for k, v in hf.state_dict().items() if "position_ids" not in k}
    m = cb.CLIPTextModel.from_state_dict(sd, "cuda", C2)
    ids = torch.randint(0, C2["vocab_size"], (2, 77), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = hf.cuda()(ids.cuda())[0].float()
        oracle = R.clip_text_forward({k: v.cuda() for k, v in sd.items()}, ids.cuda(), C2).float()
    got = m(ids.cuda())[0].float()
    torch.cuda.synchronize()
    err, err_o = float((got - want).norm() / want.norm()), float((got - oracle).norm() / oracle.norm())
    print(f"SD-2 text tower rel err vs transformers {err:.3e}, vs the oracle {err_o:.3e}")
    assert got.shape == (2, 77, 1024) and err < 2e-2 and err_o < 2e-2


@gpu
@pytest.mark.parametrize("control", [False, True])
def test_v_sampling_at_768(control, tmp_path):
    """SD-2.1 shape end to end on synthetic weights: generate (DPM++ 3 steps, with and without a canny-v2 ControlLoRA at cross
    dim 1024) and sample_class_images (PNDM), prediction_type "v_prediction", 768² images."""
    import controllora_b200 as cb
    from controllora_b200.clip import SD21_TEXT_CONFIG
    from controllora_b200.configs import NAMED, wire_processors

    _need_gpu()
    unet = cb.UNet2DConditionModel.synthetic("cuda", U.SD21_CONFIG)
    vae = cb.AutoencoderKL.synthetic("cuda")
    clip = cb.CLIPTextModel.synthetic("cuda", dict(SD21_TEXT_CONFIG, num_hidden_layers=2))
    ids = torch.randint(0, 49408, (1, 77), device="cuda")
    neg = torch.zeros(1, 77, dtype=torch.int64, device="cuda")
    cl, guide = None, None
    if control:
        cfg = dict(NAMED["diffusiondb-canny-v2"])
        cfg["lora_cross_attention_dims"] = ([None, 1024] * 5, [None, 1024] * 5, [None, 1024] * 5, [None, 1024])
        cl = cb.ControlLoRA(**cfg).to("cuda")
        wire_processors(unet, cl)
        guide = (torch.rand(1, 3, 768, 768, device="cuda") > 0.92).float() * 2 - 1
    img = S.generate(unet, cl, vae, clip, guide, ids, neg, num_inference_steps=3, scheduler="dpmpp", height=768, width=768,
                     prediction_type="v_prediction")
    torch.cuda.synchronize()
    assert img.shape == (1, 3, 768, 768) and bool(torch.isfinite(img).all())
    if not control:
        paths = S.sample_class_images(unet, vae, clip, ids[0], neg, 1, tmp_path, sample_batch_size=1, num_inference_steps=2,
                                      height=768, width=768, prediction_type="v_prediction")
        assert len(paths) == 1 and Path(paths[0]).stat().st_size > 0


class _Tracked(dict):
    """A checkpoint state dict that records which tensors a loader reads."""

    def __init__(self, *a):
        super().__init__(*a)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)

    def get(self, k, default=None):
        self.read.add(k)
        return super().get(k, default)


# parameter counts of the published SD-2 / SD-2.1 diffusers checkpoints (the two share these three networks)
SD2_COUNTS = {"unet": 865_910_724, "vae": 83_653_863, "text_encoder": 340_387_840}


@gpu
def test_real_sd21_checkpoint(monkeypatch):
    """A published SD-2.x diffusers checkpoint (local directory in CLB_SD21_DIR): UNet, VAE and text encoder load through
    from_pretrained; every tensor of each weight file is read by its loader (position_ids buffers aside), and the tensors read
    hold SD-2's parameter count; then one DDIM step with the scheduler config's prediction type runs end to end."""
    root = os.environ.get("CLB_SD21_DIR")
    if not root:
        pytest.skip("CLB_SD21_DIR is not set (a local SD-2.x diffusers checkpoint directory)")
    import safetensors.torch as st

    import controllora_b200 as cb

    _need_gpu()
    loaded = {}

    def track(fn):
        def load(f, *a, **k):
            sd = _Tracked(fn(f, *a, **k))
            loaded[Path(str(f)).parent.name] = sd
            return sd

        return load

    monkeypatch.setattr(st, "load_file", track(st.load_file))
    monkeypatch.setattr(torch, "load", track(torch.load))
    pt = S.scheduler_prediction_type(root)
    unet = cb.UNet2DConditionModel.from_pretrained(root, subfolder="unet")
    vae = cb.AutoencoderKL.from_pretrained(root, subfolder="vae")
    clip = cb.CLIPTextModel.from_pretrained(root, subfolder="text_encoder")
    for sub, want in SD2_COUNTS.items():
        sd = loaded[sub]
        keys = {k for k in dict.keys(sd) if "position_ids" not in k}
        assert keys <= sd.read, (sub, sorted(keys - sd.read)[:5])
        assert sum(dict.__getitem__(sd, k).numel() for k in keys) == want, sub
    assert unet.config.cross_attention_dim == 1024 and clip.config.hidden_act == "gelu"
    ids = torch.randint(0, 49408, (1, 77), device="cuda")
    img = S.generate(unet, None, vae, clip, None, ids, torch.zeros_like(ids), num_inference_steps=1, scheduler="ddim",
                     height=512, width=512, prediction_type=pt)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(img).all())


@gpu
@pytest.mark.parametrize("config", ["diffusiondb-canny-v2", "diffusiondb-canny"])
def test_fullsize_sd2_base_precision_contract(config):
    """SD-2-base shapes (64x64 latents, 512x512 guide, 77x1024 text), v target: ours vs the fp32 oracle <= eager bf16 vs the
    same oracle for the noise prediction and every trainable gradient (tests/check_fullsize_sd2.py)."""
    from tests import check_fullsize_sd2

    _need_gpu()
    assert check_fullsize_sd2.run(config, 1)


# ------------------------------------------------------------------------------------------------ host-logic runner
def _main():
    import contextlib
    import io
    import time
    import traceback

    os.environ["CLB_EMU"] = "1"
    from controllora_b200 import ops
    from tests import _device, emu_ops
    from tests.test_pndm import plms_step_restated

    assert _device.DEV == "cpu"
    ng = torch.no_grad()
    for name, emu in (("cfg_plms_step_dev", plms_step_restated), ("cfg_plms_step_v_dev", R.plms_v_step_restated),
                      ("cfg_solver_step_v_dev", R.solver_v_step_restated), ("gelu_", R.gelu_restated)):
        setattr(ops, name, ng(emu_ops._shadow(name, getattr(ops, name), emu)))
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
