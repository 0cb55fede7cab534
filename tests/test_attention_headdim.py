"""Head-dim sizing of the attention MMAs (pytest -m gpu).  The kernels issue only the ceil(d / 16) K16 steps that hold data
and size the last output chunk's MMA to d rounded up to 16; the columns they skip are zero fill.  So attention on heads
of width d must equal, bit for bit on the real columns, the same call on heads zero-padded to the width of the class
(64, 128 or 192) with the same scale: o, lse, dq, dk and dv."""
import pytest
import torch

from controllora_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _pad_heads(t, heads, d, dp):
    B, N, _ = t.shape
    out = torch.zeros(B, N, heads, dp, device=t.device, dtype=t.dtype)
    out[..., :d] = t.view(B, N, heads, d)
    return out.view(B, N, heads * dp)


def _real(t, heads, d, dp):
    B, N, _ = t.shape
    return t.view(B, N, heads, dp)[..., :d]


@pytest.mark.parametrize("d", [24, 40, 80, 160])
@pytest.mark.parametrize("nq,nk", [(293, 200), (256, 77)])
def test_head_dim_sizing_only_skips_zero_columns(d, nq, nk):
    B, H = 2, 3
    dp = 64 * ((d + 63) // 64)
    g = torch.Generator(device="cuda").manual_seed(d * 1000 + nk)
    q, k, v = (torch.randn(B, n, H * d, device="cuda", generator=g).to(torch.bfloat16) for n in (nq, nk, nk))
    do = torch.randn(B, nq, H * d, device="cuda", generator=g).to(torch.bfloat16)
    scale = d ** -0.5

    o, lse = ops.attention_fwd(q, k, v, H, scale)
    dq, dk, dv = ops.attention_bwd(q, k, v, o, do, lse, H, scale)

    qp, kp, vp, dop = (_pad_heads(t, H, d, dp) for t in (q, k, v, do))
    op, lsep = ops.attention_fwd(qp, kp, vp, H, scale)
    dqp, dkp, dvp = ops.attention_bwd(qp, kp, vp, op, dop, lsep, H, scale)
    torch.cuda.synchronize()

    assert torch.equal(lse, lsep)
    assert torch.equal(o.view(B, nq, H, d), _real(op, H, d, dp))
    assert torch.equal(dq.view(B, nq, H, d), _real(dqp, H, d, dp))
    assert torch.equal(dk.view(B, nk, H, d), _real(dkp, H, d, dp))
    assert torch.equal(dv.view(B, nk, H, d), _real(dvp, H, d, dp))
    for t in (o, dq, dk, dv):
        assert torch.isfinite(t.float()).all()
    assert float(dk.float().abs().max()) > 0 and float(dq.float().abs().max()) > 0
