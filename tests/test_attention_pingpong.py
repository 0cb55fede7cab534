"""Attention at the shapes where the two consumer warpgroups' turns diverge (pytest -m gpu): a CTA with a single key or query
tile, odd numbers of streamed tiles, and token counts that are not multiples of the key tile (128 / 64 keys forward) or the
streamed tile of the backward (64 / 32 rows), so the masking of the last, partial tile is exercised on both sides.  Each
case is checked against fp32 torch with the tolerances of tools/check_ops.py / check_ops2.py, and two identical calls
must give bit-identical o, lse, dq, dk and dv."""
import pytest
import torch

from controllora_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _rel(a, b):
    return float((a.detach().float() - b.detach().float()).norm() / (b.detach().float().norm() + 1e-30))


def _run(q, k, v, do, H, scale):
    o, lse = ops.attention_fwd(q, k, v, H, scale)
    dq, dk, dv = ops.attention_bwd(q, k, v, o, do, lse, H, scale)
    torch.cuda.synchronize()
    return o, lse, dq, dk, dv


@pytest.mark.parametrize("d", [24, 40, 80])
@pytest.mark.parametrize("nq,nk", [
    (100, 77),     # one query block and one key tile forward; two streamed query tiles in dK/dV
    (40, 300),     # one streamed query tile (partial) in dK/dV; three key tiles forward, the last partial
    (320, 320),    # odd tile counts: 3 key tiles forward, 5 (or 10) streamed tiles backward
    (4096, 77),    # cross-attention: many query blocks, one key tile forward, a partial last key tile in dQ
    (293, 200),
])
def test_attention_matches_fp32_and_repeats_bitwise(d, nq, nk):
    B, H = 1, 2
    g = torch.Generator(device="cuda").manual_seed(7 * d + nq + 3 * nk)
    q = torch.randn(B, nq, H * d, device="cuda", generator=g).to(torch.bfloat16)
    k = torch.randn(B, nk, H * d, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn(B, nk, H * d, device="cuda", generator=g).to(torch.bfloat16)
    do = torch.randn(B, nq, H * d, device="cuda", generator=g).to(torch.bfloat16)
    scale = d ** -0.5

    first = _run(q, k, v, do, H, scale)
    second = _run(q, k, v, do, H, scale)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    o, lse, dq, dk, dv = first

    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    qh = qf.view(B, nq, H, d).transpose(1, 2)
    kh = kf.view(B, nk, H, d).transpose(1, 2)
    vh = vf.view(B, nk, H, d).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) * scale
    oref = (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, nq, H * d)
    lse_ref = torch.logsumexp(s, -1) * 1.4426950408889634
    oref.backward(do.float())

    assert _rel(o, oref) < 6e-3
    assert float((lse - lse_ref).abs().max()) < 2e-2
    assert _rel(dq, qf.grad) < 1e-2
    assert _rel(dk, kf.grad) < 1e-2
    assert _rel(dv, vf.grad) < 1e-2
