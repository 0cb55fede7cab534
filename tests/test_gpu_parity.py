"""GPU parity tests (pytest -m gpu): every kernel family and the assembled hot path against torch-fp32 references /
the CPU oracle, through the C ABI.  Tolerances: bf16 storage => ~2e-3 relative per op; end-to-end tolerances below."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


# ------------------------------------------------------------------------------------------------ K1 / K4: GEMM + conv
from tests import check_hint, check_unet  # noqa: E402  (the two checkers that execute the oracle live with the tests)
from tools import check_gemm, check_ops, check_ops2  # noqa: E402


@pytest.mark.parametrize("case", ["plain_1tile", "plain_k320", "plain_bn64", "plain_bn160_tail", "plain_bn256", "plain_big",
                                  "epilogue_all", "lora_r4", "lora_r4_tadd", "lora_r8_cross", "conv_s1_64", "conv_s1_small",
                                  "conv_s2", "conv_96", "split_k", "plain_bn320", "conv_bn320", "resident_short_k"])
def test_gemm(case):
    check_gemm.CASES[case]()


def test_conv_32_channels_uses_bk32_path():
    """hint-encoder shapes: 32-channel convs (64-byte swizzle / BLOCK_K = 32 variant of the kernel)."""
    check_gemm._conv_case(2, 64, 64, 32, 32, 1, 1, True)
    check_gemm._conv_case(2, 64, 64, 32, 64, 1, 1, False)
    check_gemm._conv_case(2, 64, 64, 32, 32, 2, 0, False)
    # enough tiles for the resident-weights mode of the 32-channel variant (3 k-blocks per stage, per-lane store epilogue)
    check_gemm._conv_case(1, 256, 256, 32, 32, 1, 1, True)
    check_gemm._conv_case(1, 256, 256, 32, 32, 1, 1, False)
    check_gemm._conv_case(1, 512, 256, 32, 32, 2, 0, False)


# ------------------------------------------------------------------------------------------------ K2: attention
@pytest.mark.parametrize("case", ["attn_d64_one_block", "attn_d40", "attn_cross77", "attn_d80_d160", "attn_small_d", "attn_paired"])
def test_attention_fwd(case):
    check_ops.CASES[case]()


@pytest.mark.parametrize("case", ["attn_bwd_one_block", "attn_bwd_d40", "attn_bwd_d80_d160", "attn_bwd_small_d"])
def test_attention_bwd(case):
    check_ops2.CASES[case]()


def test_attention_full_size_properties():
    """BASELINE-size self-attention (8 x 8 heads x 4096 tokens x d=40): rows of P sum to 1 => attention of constant V is
    constant; permuting the keys/values leaves the output unchanged."""
    from controllora_b200 import ops

    B, H, N, d = 2, 8, 4096, 40
    q = torch.randn(B, N, H * d, device="cuda").to(torch.bfloat16)
    k = torch.randn(B, N, H * d, device="cuda").to(torch.bfloat16)
    v = torch.ones(B, N, H * d, device="cuda", dtype=torch.bfloat16) * 0.5
    o, lse = ops.attention_fwd(q, k, v, H, d ** -0.5)
    assert (o.float() - 0.5).abs().max() < 4e-3
    v2 = torch.randn(B, N, H * d, device="cuda").to(torch.bfloat16)
    o1, _ = ops.attention_fwd(q, k, v2, H, d ** -0.5)
    perm = torch.randperm(N, device="cuda")
    o2, _ = ops.attention_fwd(q, k[:, perm].contiguous(), v2[:, perm].contiguous(), H, d ** -0.5)
    assert (o1.float() - o2.float()).abs().max() < 2e-2


# ------------------------------------------------------------------------------------------------ K5 / glue / edges / LoRA / optimizer
@pytest.mark.parametrize("case", ["groupnorm", "layernorm", "elementwise", "edges", "conv_dgrad"])
def test_norm_elementwise_edges(case):
    check_ops.CASES[case]()


@pytest.mark.parametrize("case", ["lora_kernels", "optimizer"])
def test_lora_and_optimizer(case):
    check_ops2.CASES[case]()


# ------------------------------------------------------------------------------------------------ assembled hot path
@pytest.mark.parametrize("variant", ["none", "plain", "v1", "v1_stacked", "v2", "v1_post_add", "v1_concat",
                                     "v1_stacked@0.5", "v2@0.5", "plain@2.0"])
def test_unet_fwd_bwd_matches_oracle(variant):
    """Noise prediction and every LoRA / control-state gradient vs the fp32 oracle (tiny SD-style config).
    Tolerance: bf16 activations through ~40 layers => <= 2e-2 relative on the prediction, <= 8e-2 on single gradients."""
    assert check_unet.run(variant)


# ------------------------------------------------------------------------------------------------ BASELINE configs, real shapes
@pytest.mark.parametrize("config,batch", [("diffusiondb-canny-v2", 1), ("diffusiondb-canny", 1), ("danbooru-sketch", 1)])
def test_fullsize_parity_and_precision_contract(config, batch):
    """BASELINE C4 (`diffusiondb-canny-v2`, V2 processors), C2 (`diffusiondb-canny`, v1 + pre-convs) and the dense-control
    variant `danbooru-sketch` (concat_hidden, control rank 256: only expressible at the real channel counts) on the real SD-1.5
    shapes through the drop-in classes: noise prediction, loss and every ControlLoRA / hint-encoder gradient against the
    fp32 CPU oracle, and the precision contract ours-vs-fp32 <= (eager bf16 autocast)-vs-fp32 (tests/check_fullsize.py
    states the tolerances)."""
    from tests import check_fullsize

    log = None
    try:
        check_fullsize.LOG_DIR.mkdir(exist_ok=True)
        log = open(check_fullsize.LOG_DIR / f"parity_fullsize_{config}_b{batch}.log", "w")
    except OSError:
        pass
    try:
        assert check_fullsize.run(config, batch, log)
    finally:
        if log is not None:
            log.close()


@pytest.mark.parametrize("case", ["hint_v1", "hint_v2"])
def test_hint_encoder_matches_oracle(case):
    assert check_hint.CASES[case]()


@pytest.mark.parametrize("case", ["train_v1", "train_v2"])
def test_fused_train_step_matches_oracle(case):
    assert check_hint.CASES[case]()


def test_cuda_graph_train_step_matches_eager():
    """Trainer(cuda_graph=True): warm-up, capture and replays give the same losses / parameters as the eager step."""
    assert check_hint.CASES["graph_v2"]()


def test_lora_zero_up_is_exact_noop_on_gpu():
    """With diffusers' default init (up = 0) the fused epilogue must contribute exactly nothing."""
    import controllora_b200 as cb
    from controllora_b200.configs import wire_processors
    from controllora_b200.unet import synthetic_state_dict

    TINY, TINY_LORA = check_unet.TINY, check_unet.TINY_LORA
    sd = synthetic_state_dict(TINY, 0)
    u0 = cb.UNet2DConditionModel.from_state_dict(sd, "cuda", TINY)
    u1 = cb.UNet2DConditionModel.from_state_dict(sd, "cuda", TINY)
    cl = cb.ControlLoRA(**TINY_LORA).cuda()
    wire_processors(u1, cl)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 16, 16, generator=g).cuda()
    t = torch.tensor([3.0, 900.0]).cuda()
    e = torch.randn(2, 77, 64, generator=g).cuda().to(torch.bfloat16)
    guide = (torch.rand(2, 3, 128, 128, generator=g) * 2 - 1).cuda()
    with torch.no_grad():
        cl(guide)
        a = u0(x, t, e).sample
        b = u1(x, t, e).sample
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ denoise loop (CFG + DDIM)
def test_cfg_ddim_step_matches_oracle():
    from controllora_b200 import ops
    from controllora_b200.sampler import ddim_coeffs, ddim_timesteps, sd15_alphas_cumprod
    from oracle import sampler_ref as SR

    g = torch.Generator().manual_seed(0)
    eps2 = torch.randn(4, 4, 16, 16, generator=g)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ac = sd15_alphas_cumprod()
    for t in ddim_timesteps(50)[:3] + ddim_timesteps(50)[-2:]:
        xm = x.clone().cuda()
        a_t, a_p = ddim_coeffs(t, 50, ac)
        ops.cfg_ddim_step(eps2.cuda(), xm, 7.5, a_t, a_p)
        ref = SR.cfg_ddim_step(eps2[:2], eps2[2:], x, t, 50, 7.5)
        assert torch.allclose(xm.cpu(), ref, atol=1e-4, rtol=1e-4), t


def test_cfg_dpmpp_step_matches_oracle():
    """Fused CFG + DPM-Solver++(2M) kernel against the stateful oracle scheduler over a whole 12-step trajectory
    (first-order first and last steps, second-order in between)."""
    from controllora_b200 import ops
    from controllora_b200.sampler import dpm_timesteps, dpmpp_2m_coeffs, sd15_alphas_cumprod
    from oracle import sampler_ref as SR

    steps = 12
    sched = SR.DPMSolverPP2M(steps)
    ts = dpm_timesteps(steps)
    ac = sd15_alphas_cumprod()
    g = torch.Generator().manual_seed(0)
    x_ref = torch.randn(2, 4, 16, 16, generator=g)
    xm = x_ref.clone().cuda()
    x0p = torch.zeros_like(xm)
    for i, t in enumerate(ts):
        eps2 = torch.randn(4, 4, 16, 16, generator=g)
        x_ref = sched.step(SR.cfg_combine(eps2[:2], eps2[2:], 7.5), t, x_ref)
        ops.cfg_dpmpp_step(eps2.cuda(), xm, x0p, 7.5, *dpmpp_2m_coeffs(i, ts, ac))
        assert torch.allclose(xm.cpu(), x_ref, atol=2e-4, rtol=2e-4), (i, t)


def test_dpmpp_loop_tracks_oracle_on_tiny_unet():
    """4 CFG + DPM-Solver++(2M) steps (UNet batch 2B, control injected once) against the oracle UNet + oracle scheduler."""
    from controllora_b200.sampler import dpmpp_sample
    from oracle import sampler_ref as SR

    ounet, munet, ocl, mcl = check_unet.build_pair("v2")
    g = torch.Generator().manual_seed(11)
    B, HW = 2, 16
    guide = (torch.rand(B, 3, HW * 8, HW * 8, generator=g) * 2 - 1).to(torch.bfloat16).float()
    cond = torch.randn(B, 77, 64, generator=g).to(torch.bfloat16).float()
    unc = torch.randn(B, 77, 64, generator=g).to(torch.bfloat16).float()
    lat0 = torch.randn(B, 4, HW, HW, generator=g)
    steps = 4
    sched = SR.DPMSolverPP2M(steps)
    with torch.no_grad():
        ocl(torch.cat([guide, guide], 0))
        x = lat0.clone()
        for t in sched.timesteps:
            eps = ounet(torch.cat([x, x], 0), torch.full((2 * B,), int(t)), torch.cat([unc, cond], 0)).sample
            x = sched.step(SR.cfg_combine(eps[:B], eps[B:], 7.5), t, x)
    out = dpmpp_sample(munet, mcl, guide.cuda(), cond.cuda().to(torch.bfloat16), unc.cuda().to(torch.bfloat16),
                       num_inference_steps=steps, guidance_scale=7.5, latents=lat0.cuda())
    err = float((out.cpu() - x).norm() / x.norm())
    print("dpm-solver++ 4-step latent rel err", err)
    assert err < 8e-2


def test_ddim_loop_tracks_oracle_on_tiny_unet():
    """3 CFG+DDIM steps (UNet batch 2B, control injected once) against the oracle UNet driven by the oracle scheduler."""
    import controllora_b200 as cb
    from controllora_b200.sampler import ddim_sample
    from oracle import models_ref as MR
    from oracle import sampler_ref as SR

    ounet, munet, ocl, mcl = check_unet.build_pair("v1")
    g = torch.Generator().manual_seed(9)
    B, HW = 2, 16
    guide = (torch.rand(B, 3, HW * 8, HW * 8, generator=g) * 2 - 1).to(torch.bfloat16).float()
    cond = torch.randn(B, 77, 64, generator=g).to(torch.bfloat16).float()
    unc = torch.randn(B, 77, 64, generator=g).to(torch.bfloat16).float()
    lat0 = torch.randn(B, 4, HW, HW, generator=g)
    steps = 3
    with torch.no_grad():
        ocl(torch.cat([guide, guide], 0))
        x = lat0.clone()
        for t in SR.timesteps(steps):
            eps = ounet(torch.cat([x, x], 0), torch.full((2 * B,), int(t)), torch.cat([unc, cond], 0)).sample
            x = SR.cfg_ddim_step(eps[:B], eps[B:], x, t, steps, 7.5)
    out = ddim_sample(munet, mcl, guide.cuda(), cond.cuda().to(torch.bfloat16), unc.cuda().to(torch.bfloat16),
                      num_inference_steps=steps, guidance_scale=7.5, latents=lat0.cuda())
    err = float((out.cpu() - x).norm() / x.norm())
    print("ddim 3-step latent rel err", err)
    assert err < 6e-2


# ------------------------------------------------------------------------------------------------ step glue (noise, timesteps, add_noise)
def test_add_noise_matches_oracle_restatement():
    """cl_add_noise against the numpy restatement of its Philox4x32-10 counter layout (oracle/sampler_ref.device_noise,
    itself pinned by Random123's known-answer vectors in tests/test_oracle.py) and the restated DDPMScheduler.add_noise /
    get_velocity: timesteps bit-exact, normals to fp32 libm precision, fresh draws per call, epsilon and v-prediction."""
    import numpy as np
    from controllora_b200 import ops
    from controllora_b200.sampler import sd15_alphas_cumprod
    from oracle import sampler_ref as SR

    B, per = 8, 4 * 64 * 64
    ac = torch.tensor(sd15_alphas_cumprod(), dtype=torch.float64)
    sa, sb = ac.sqrt().float().cuda(), (1 - ac).sqrt().float().cuda()
    x0 = torch.randn(B, 4, 64, 64, generator=torch.Generator().manual_seed(0))
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    seed = 0x1234_5678_9ABC_DEF0
    prev_ts = None
    for step, vpred in ((0, False), (1, True), (2, False)):
        noisy, target, ts = ops.add_noise(x0.cuda(), sa, sb, ctr, seed, v_prediction=vpred)
        torch.cuda.synchronize()
        assert int(ctr) == step + 1                                   # the counter advanced on the stream
        n_ref, t_ref = SR.device_noise(seed, step, B, per)
        assert np.array_equal(ts.cpu().numpy().astype(np.int64), t_ref)
        n_ref = torch.from_numpy(n_ref).view(B, 4, 64, 64)
        t_t = torch.from_numpy(t_ref)
        ref_noisy = SR.add_noise(x0, n_ref, t_t)
        ref_target = SR.get_velocity(x0, n_ref, t_t) if vpred else n_ref
        assert torch.allclose(noisy.cpu(), ref_noisy, atol=2e-5, rtol=1e-5)
        assert torch.allclose(target.cpu(), ref_target, atol=2e-5, rtol=1e-5)
        if prev_ts is not None:
            assert not torch.equal(prev_ts, ts.cpu())
        prev_ts = ts.cpu()
    # distribution sanity at full size
    noisy, target, ts = ops.add_noise(torch.zeros(64, 4, 64, 64, device="cuda"), sa, sb, ctr, seed)
    assert abs(float(target.mean())) < 5e-3 and abs(float(target.std()) - 1.0) < 5e-3
    assert 0 <= float(ts.min()) and float(ts.max()) <= 999


def test_train_step_from_latents_graph_draws_fresh_noise():
    """Trainer.step_from_latents under CUDA-graph replay: every replay draws new timesteps / noise (device step counter)
    and the loss stays finite; the draw of step k equals the oracle restatement for counter k."""
    import numpy as np
    import controllora_b200 as cb
    from controllora_b200.configs import wire_processors
    from controllora_b200.trainer import Trainer
    from controllora_b200.unet import synthetic_state_dict
    from oracle import sampler_ref as SR

    TINY, TINY_LORA = check_unet.TINY, check_unet.TINY_LORA
    unet = cb.UNet2DConditionModel.from_state_dict(synthetic_state_dict(TINY, 0), "cuda", TINY)
    cl = cb.ControlLoRA(**TINY_LORA).cuda()
    wire_processors(unet, cl)
    tr = Trainer(unet, cl, lr=1e-4, cuda_graph=True, noise_seed=77)
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(2, 4, 16, 16, generator=g).cuda()
    e = torch.randn(2, 77, 64, generator=g).cuda().to(torch.bfloat16)
    guide = (torch.rand(2, 3, 128, 128, generator=g) * 2 - 1).cuda()
    seen = []
    for k in range(5):
        loss = tr.step_from_latents(lat, e, guide)
        torch.cuda.synchronize()
        assert torch.isfinite(loss).all()
        _, target, ts = tr.last_noise_draw
        n_ref, t_ref = SR.device_noise(77, k, 2, 4 * 16 * 16)
        assert np.array_equal(ts.cpu().numpy().astype(np.int64), t_ref), k
        assert torch.allclose(target.cpu().view(2, -1), torch.from_numpy(n_ref), atol=2e-5, rtol=1e-5)
        seen.append(tuple(t_ref.tolist()))
    assert tr._graph is not None and len(set(seen)) == 5


@pytest.mark.parametrize("scheduler,variant", [("ddim", "v1"), ("dpmpp", "v2")])
def test_graphed_sampler_matches_eager_loop(scheduler, variant):
    """GraphedSampler (one captured step replayed, timestep-invariant products hoisted, text k/v cached) must reproduce the
    plain per-step loop (ddim_sample / dpmpp_sample, already checked against the oracle schedulers above) - on a first call
    (eager warm-up + capture + replays) and on a second call with a different guide / prompt (in-place refresh of the
    products the captured graph reads)."""
    from controllora_b200.sampler import GraphedSampler, ddim_sample, dpmpp_sample

    _, munet, _, mcl = check_unet.build_pair(variant)
    B, HW, steps = 2, 16, 6
    gs = GraphedSampler(munet, mcl, B, HW * 8, HW * 8, scheduler=scheduler, num_inference_steps=steps, guidance_scale=7.5, text_dim=64)
    loop = ddim_sample if scheduler == "ddim" else dpmpp_sample
    for call in range(2):
        g = torch.Generator().manual_seed(20 + call)
        guide = (torch.rand(B, 3, HW * 8, HW * 8, generator=g) * 2 - 1).cuda()
        cond = torch.randn(B, 77, 64, generator=g).cuda().to(torch.bfloat16)
        unc = torch.randn(B, 77, 64, generator=g).cuda().to(torch.bfloat16)
        lat0 = torch.randn(B, 4, HW, HW, generator=g).cuda()
        ref = loop(munet, mcl, guide, cond, unc, num_inference_steps=steps, guidance_scale=7.5, latents=lat0)
        out = gs(guide, cond, unc, latents=lat0).clone()
        torch.cuda.synchronize()
        err = float((out - ref).norm() / ref.norm())
        print(f"graphed {scheduler}/{variant} call {call}: rel diff vs per-step loop {err:.3e}; launches/step {gs.launches_per_step}")
        assert err < 2e-3, (call, err)
    assert gs._graph is not None


# ------------------------------------------------------------------------------------------------ CLIP text encoder in front of the step
@pytest.mark.parametrize("which", ["tiny", "full"])
def test_clip_text_encoder_matches_oracle(which):
    """`text_encoder(input_ids)[0]` (train_...:768) against the fp32 oracle restatement of transformers' CLIPTextModel (pinned
    to transformers itself in tests/test_oracle.py): a 2-layer config and the SD-1.5 text tower (12 x 768, 12 heads, 77 tokens)
    at batch 8; <= 3e-2 relative and no worse than 1.25x the same math in eager bf16 PyTorch."""
    from tests import check_clip

    assert check_clip.run(which)


# ------------------------------------------------------------------------------------------------ VAE either side of the step
@pytest.mark.parametrize("which", ["tiny", "full"])
def test_vae_encode_decode_matches_oracle(which):
    """`vae.encode(x).latent_dist` moments / sample and `vae.decode(z).sample` (train_...:753-754, pipeline decode) against the
    fp32 oracle restatement of diffusers' AutoencoderKL: a small config and the SD-1.5 VAE shapes (128/256/512/512 channels,
    one-head 512-wide mid attention) at 256x256.  bf16 activations through ~25 conv / norm layers: <= 2e-2 relative."""
    from tests import check_vae

    assert check_vae.run(which)
