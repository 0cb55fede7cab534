"""GPU tests of step-level features and the general adapter chains (the same cases pass in host-logic mode on the CPU, tests/test_host_emulated.py, where
every launch also goes through the real launchers' argument validation).  Ordered from the paths built on kernels / call patterns that earlier
GPU runs already exercised to the newest code, so that `pytest -x` reports as much as possible:
  1. the CUDA path against golden vectors computed by the reference's own models.py (fused path, tests/check_reference_golden.py)
  2. step-level features on the fused path: resume equivalence, accumulation windows, the LoRA-only (DreamBooth) step, the loop body from
     pixels, the generate pipeline
  3. the two per-row rank-r kernels at both template widths (direct kernel checks)
  4. the general adapter-chain path (controllora_b200/lora_generic.py: wirings beyond the fused path, and the standard wirings forced through it)
  5. processors called the way diffusers calls them (controllora_b200/eager_attn.py)"""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from tests import check_eager, check_hint, check_reference_golden, check_sampler, check_variants  # noqa: E402

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ 1
@pytest.mark.parametrize("case", check_reference_golden.CASE_NAMES)
def test_cuda_path_matches_golden_vectors_computed_by_the_reference_code(case):
    """Expected values come from /root/reference/models.py itself (imported unmodified when the fixture was generated,
    tests/golden/make_reference_golden.py), not from the oracle restatement."""
    assert check_reference_golden.CASES[case]()


# ------------------------------------------------------------------------------------------------ 2
def test_checkpoint_resume_equivalence_on_gpu():
    """3 steps == 2 steps + save_checkpoint + fresh Trainer + load_checkpoint + 1 step (counters and the next noise draw exactly, tensors to
    the run-to-run tolerance of the atomically reduced weight gradients), incl. the device Philox counter
    (train_text_to_image_control_lora.py:713-735, 805-809)."""
    assert check_hint.CASES["resume"]()


def test_gradient_accumulation_window_matches_oracle():
    """Trainer.accumulate() x2 + step(): `--gradient_accumulation_steps 3` (train_text_to_image_control_lora.py:751)."""
    assert check_hint.CASES["accumulate"]()


def test_lora_only_train_step_with_prior_preservation_matches_oracle():
    """Trainer(control_lora=None, prior_loss_weight=w): the DreamBooth-LoRA step (train_dreambooth_lora.py:880-918)."""
    assert check_hint.CASES["train_lora_only"]()


def test_whole_loop_body_from_pixels_matches_oracle_chain():
    """Trainer.step_from_pixels: VAE encode + sample, CLIP text tower, device noise glue, hint encoder, UNet, loss (train_...:751-796)."""
    assert check_sampler.CASES["step_from_pixels"]()


def test_generate_pipeline_matches_oracle_chain():
    """sampler.generate: token ids -> text states -> CFG + DDIM loop -> VAE decode -> [0, 1] images (train_...:824-843, apps/*)."""
    assert check_sampler.CASES["generate"]()


# ------------------------------------------------------------------------------------------------ 3
@pytest.mark.parametrize("rp", [4, 8])
def test_rank_update_and_rowdot_kernels(rp):
    """The two per-row rank-r kernels the general chain path leans on, at both template widths, against torch:
    out = x + alpha * t[:, :rp] tab^T (t a strided view, in place and out of place) and e = a u."""
    import torch
    from controllora_b200 import ops

    g = torch.Generator().manual_seed(rp)
    M, C = 1000, 1280
    x = torch.randn(M, C, generator=g).to(torch.bfloat16).cuda()
    t_full = torch.randn(M, 16, generator=g).cuda()
    tab = (0.1 * torch.randn(C, rp, generator=g)).cuda()
    t = t_full[:, 8:] if rp == 8 else t_full[:, 4:]           # a view with row stride 16 and a non-zero column offset (block b of t)
    want = (x.float() + 0.7 * (t[:, :rp] @ tab.t())).to(torch.bfloat16)
    got = ops.rank_update(x, t, tab, 0.7)
    buf = x.clone()
    ops.rank_update(buf, t, tab, 0.7, out=buf)
    u = (0.1 * torch.randn(C, rp, generator=g)).cuda()
    e = ops.rowdot(x, u)
    torch.cuda.synchronize()
    rel = lambda a, b: float((a.float() - b.float()).norm() / b.float().norm())
    assert rel(got, want) < 4e-3 and torch.equal(got, buf)
    assert rel(e, x.float() @ u) < 1e-5


# ------------------------------------------------------------------------------------------------ 4
@pytest.mark.parametrize("case", check_variants.CASE_NAMES)
def test_general_chain_matches_oracle(case):
    """Wirings of /root/reference/models.py:118-431 beyond the fused one-launch path (post_add inside stacked chains, ranks > 8, control
    ranks > 4, stacked ControlLoRA processors, concat_hidden + stacking), the standard wirings forced through the same path, two UNet
    calls before one backward, control batch 1 under a CFG batch of 2."""
    assert check_variants.CASES[case]()


# ------------------------------------------------------------------------------------------------ 5
@pytest.mark.parametrize("case", check_eager.CASE_NAMES)
def test_processor_called_like_diffusers_matches_oracle(case):
    """`processor(attn, hidden_states, encoder_hidden_states, None, scale)` on a stand-alone attention module (models.py:118-152,
    222-287, 357-431 as diffusers' CrossAttention.forward invokes them) and LoRALinearLayer.forward."""
    assert check_eager.CASES[case]()
