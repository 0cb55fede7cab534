"""Short-K GEMMs at two CTAs per SM (pytest -m gpu).  The planner runs unsplit launches with few k-blocks per tile two CTAs
per SM; these tests check the results against torch fp32, that the cases really are planned that way and that the device
keeps two of those CTAs resident, and that the occupancy (and tile width) leaves every output bit-identical."""
import pytest
import torch

from tools import check_gemm
from tools.gemm_occupancy import _Recorder

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.mark.parametrize("case", ["two_cta_plain", "two_cta_epilogue", "two_cta_conv"])
def test_two_cta_gemm(case):
    check_gemm.CASES[case]()


def _plans(fn):
    """Run fn with every cl_gemm call recorded; returns the plans (block_n, splits, ctas_per_sm, resident_per_sm)."""
    from controllora_b200 import _lib

    rec = _Recorder(_lib.lib())
    _lib._lib = rec
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        _lib._lib = rec.real
    return [r[1] for r in rec.rows]


def _bf16(*s):
    return torch.randn(*s, device="cuda").to(torch.bfloat16)


@pytest.mark.parametrize("M,N,K,conv_c", [(16384, 384, 320, 0), (32700, 384, 320, 0), (2 * 256 * 256, 32, 288, 32),
                                         (2 * 256 * 256, 64, 288, 32), (2 * 256 * 256, 128, 576, 64)])
def test_short_k_cases_run_two_ctas_per_sm(M, N, K, conv_c):
    from controllora_b200 import ops

    kw = {}
    if conv_c:
        side = int((M // 2) ** 0.5)
        a, kw["conv_stride"] = _bf16(2, side, side, conv_c), 1
    else:
        a = _bf16(M, K)
    (plan,) = _plans(lambda: ops.gemm(a, _bf16(N, K), **kw))
    assert plan[1] == 1 and plan[2] == 2, plan
    assert plan[3] == 2, f"the device keeps {plan[3]} CTAs of this kernel resident per SM"


def test_occupancy_and_tile_width_leave_outputs_bit_identical():
    """Tile width and CTAs per SM change neither the k-block order nor the MMA sequence of an output element."""
    from controllora_b200 import ops

    torch.manual_seed(0)
    M, N, K = 8192, 640, 320
    a, b = _bf16(M, K), (torch.randn(N, K, device="cuda") / K**0.5).to(torch.bfloat16)
    bias, res = torch.randn(N, device="cuda"), _bf16(M, N)
    outs, plans = [], []
    for bn in (128, 64):                       # plain: BN 128 runs two CTAs per SM, BN 64 one
        plans += _plans(lambda: outs.append(ops.gemm(a, b, bias=bias, residual=res, block_n=bn)))
    assert [p[2] for p in plans] == [2, 1], plans
    assert torch.equal(outs[0], outs[1])
    x, w = _bf16(8, 128, 128, 64), (torch.randn(128, 576, device="cuda") / 24).to(torch.bfloat16)
    outs, plans = [], []
    for bn in (128, 64):                       # 64-channel conv: BN 128 runs two CTAs per SM, BN 64 one
        plans += _plans(lambda: outs.append(ops.gemm(x, w, conv_stride=1, bias=bias[:128], block_n=bn)))
    assert [p[2] for p in plans] == [2, 1], plans
    assert torch.equal(outs[0], outs[1])
