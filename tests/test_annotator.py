"""Canny annotator: the numpy oracle against cv2.Canny and the stored goldens (CPU), the C-ABI argument checks (CPU), and
the CUDA kernel against both, bit for bit (GPU)."""
import ctypes
from pathlib import Path

import numpy as np
import pytest

from oracle import annotator_ref as A
from tests.golden.make_canny_golden import checkerboard, shapes, smooth_noise, spiral

GOLDEN = Path(__file__).resolve().parent / "golden" / "canny_golden.npz"


def golden():
    z = np.load(GOLDEN)
    return {str(n): (z[f"img_{n}"], tuple(float(v) for v in z[f"thr_{n}"]), z[f"edges_{n}"]) for n in z["names"]}


def nms_plateau(H=48, W=64):
    """Ramps and two-pixel-wide steps: runs of equal gradient magnitude along and across the NMS direction, where the
    strict and non-strict comparisons of rule 4 decide."""
    y, x = np.mgrid[0:H, 0:W]
    img = np.where(x < W // 3, (x * 6) % 256, 0) + np.where((x // 2) % 4 == 0, 90, 20) * (x >= W // 3)
    img = img + np.where(y > H // 2, (y // 2) * 9, 0)
    return np.clip(img, 0, 255).astype(np.uint8)


def channel_tie(rng, H=40, W=56):
    """Three channels whose gradient magnitudes tie with different directions (mirror and transpose of one pattern)."""
    base = smooth_noise(rng, max(H, W), max(H, W), 1, cell=5)[:, :, 0]
    c0 = base[:H, :W]
    c1 = base[:H, ::-1][:, -W:]            # dx sign flipped, same |dx| + |dy| where the mirror lines up
    c2 = base.T[:H, :W]
    img = np.stack([c0, np.ascontiguousarray(c1), c2], axis=2)
    img[:, : W // 2, 1] = img[:, : W // 2, 0][:, ::-1]
    return np.ascontiguousarray(img)


def random_cases(n=220):
    """Seeded (image, lo, hi) cases: 1x1, 1xN, Nx1, up to 1024^2; 1 and 3 channels; thresholds 0-300 incl. swapped,
    fractional and equal; NMS plateaus and channel ties."""
    rng = np.random.default_rng(7)
    sizes = [(1, 1), (1, 17), (23, 1), (2, 2), (3, 3), (1, 300), (300, 1), (33, 65), (64, 64), (31, 97), (129, 40)]
    out = []
    for i in range(n):
        H, W = sizes[i] if i < len(sizes) else (int(rng.integers(1, 160)), int(rng.integers(1, 160)))
        C = 3 if i % 3 else 1
        kind = i % 5
        if kind == 0:
            img = rng.integers(0, 256, (H, W, C), dtype=np.uint8)
        elif kind in (1, 2):
            img = smooth_noise(rng, H, W, C, cell=int(rng.integers(2, 12)), noise=float(rng.uniform(0, 8)))
        elif kind == 3:
            img = shapes(rng, H, W, C, n=12, patch=max(1, min(H, W) // 2))
        else:
            img = np.clip(checkerboard(H, W, square=int(rng.integers(1, 9))).astype(int) + rng.integers(-3, 4, (H, W)), 0, 255)
            img = np.repeat(img.astype(np.uint8)[:, :, None], C, axis=2)
        if C == 1 and i % 2:
            img = img[:, :, 0]
        lo, hi = rng.uniform(0, 300, 2)
        mode = i % 4
        if mode == 0:
            lo, hi = float(np.floor(lo)), float(np.floor(hi))
        elif mode == 1:
            lo, hi = max(lo, hi), min(lo, hi)          # swapped
        elif mode == 2:
            hi = lo                                     # equal
        out.append((np.ascontiguousarray(img), float(lo), float(hi)))
    for k in range(6):
        out.append((nms_plateau(), 10.0 * k, 10.0 * k + 40.0))
        out.append((channel_tie(rng), 20.0 + 15 * k, 120.0 - 10 * k))
    big = shapes(rng, 1024, 1024, 3, n=200, patch=300)
    out += [(big, 30.0, 90.0), (big[:, :, 1].copy(), 95.5, 12.25)]
    return out


# -------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    cases = random_cases()
    assert len(cases) >= 200
    bad = [(img.shape, lo, hi) for img, lo, hi in cases if not np.array_equal(A.canny(img, lo, hi), cv2.Canny(img, lo, hi))]
    assert not bad, bad


def test_oracle_reproduces_golden():
    for name, (img, (lo, hi), edges) in golden().items():
        assert np.array_equal(A.canny(img, lo, hi), edges), name


def test_golden_cases_are_regenerated_exactly():
    """The stored images are the seeded constructors' output, so the generator stays the record of how they were made."""
    from tests.golden.make_canny_golden import cases

    g = golden()
    for name, img, thr in cases():
        assert np.array_equal(g[name][0], img) and g[name][1] == thr, name


def test_spiral_golden_needs_hysteresis_across_the_image():
    img, (lo, hi), edges = golden()["spiral"]
    cand, strong = A.candidates(img, lo, hi)
    ys, xs = np.nonzero(edges)
    assert strong.sum() < 16 and np.all(np.abs(np.argwhere(strong) - 512) < 4)
    assert ys.min() < 32 and ys.max() > 1024 - 32 and xs.min() < 32 and xs.max() > 1024 - 32


def test_pixel_and_guide_arithmetic_restates_the_reference():
    """oracle.pixel_values / guide_values = the float32 operations of process/diffusiondb_canny.py:40-45 and
    apps/gradio_canny2image.py:72-74, run here with torch / numpy on the host, for every uint8 value."""
    import torch

    img = np.arange(256, dtype=np.uint8).reshape(16, 16, 1).repeat(3, axis=2)
    img[:, :, 1] = img[:, :, 1][::-1]
    ref_pix = (torch.tensor(img.astype("float32").copy()).float().permute(2, 0, 1) / 127.5 - 1).numpy()
    assert np.array_equal(A.pixel_values(img).view(np.int32), ref_pix.view(np.int32))
    edges = np.where(np.arange(256).reshape(16, 16) % 3 == 0, 255, 0).astype(np.uint8)
    ds = torch.tensor((np.asarray(edges).astype("float32") / 127.5 - 1).copy())[None].repeat(3, 1, 1).float().numpy()
    hwc3 = np.concatenate([edges[:, :, None]] * 3, axis=2)
    app = (torch.from_numpy(hwc3[..., ::-1].copy().transpose([2, 0, 1])).float()[None] / 127.5 - 1)[0].numpy()
    got = A.guide_values(edges)
    assert np.array_equal(got, ds) and np.array_equal(got, app)
    assert set(np.unique(got).tolist()) == {-1.0, 1.0}


def test_cl_canny_rejects_bad_arguments_without_a_gpu(built_lib):
    from controllora_b200 import _lib

    lib = _lib.lib()
    P = ctypes.c_void_p(64)      # never dereferenced: every check runs before any CUDA call
    N = None

    def call(img=P, B=2, H=8, W=8, C=3, thr=P, labels=P, edges=P, guide=N, pixels=N):
        return lib.cl_canny(img, B, H, W, C, thr, labels, edges, guide, pixels, N)

    cases = {
        "img": dict(img=N), "thresholds": dict(thr=N), "labels": dict(labels=N),
        "no output": dict(edges=N), "C = 2": dict(C=2), "C = 4": dict(C=4), "pixels needs": dict(C=1, pixels=P),
        "B=0": dict(B=0), "H=-1": dict(H=-1), "W=0": dict(W=0), "2^31": dict(B=1 << 15, H=1 << 8, W=1 << 8),
    }
    for what, kw in cases.items():
        assert call(**kw) == -1, what
        msg = lib.cl_last_error().decode()
        assert msg.startswith("cl_canny"), (what, msg)
    assert "null" in (call(img=N), lib.cl_last_error().decode())[1]
    assert "2^31" in (call(B=1 << 15, H=1 << 8, W=1 << 8), lib.cl_last_error().decode())[1]


# -------------------------------------------------------------------------------------------------------------- GPU
def _edges(img, lo, hi):
    import torch
    from controllora_b200 import ops

    x = torch.from_numpy(img if img.ndim == 3 else img[:, :, None]).cuda()[None].contiguous()
    thr = torch.tensor([[lo, hi]], dtype=torch.float32, device="cuda")
    e = torch.empty(1, x.shape[1], x.shape[2], dtype=torch.uint8, device="cuda")
    ops.canny(x, thr, edges=e)
    return e[0].cpu().numpy()


@pytest.mark.gpu
def test_gpu_batch_512_dataset_thresholds():
    import torch
    from controllora_b200 import ops

    g = golden()
    rng = np.random.default_rng(11)
    imgs = [g["rgb512_a"][0], g["rgb512_b"][0]] + [shapes(rng, 512, 512) for _ in range(3)] + \
           [smooth_noise(rng, 512, 512, 3, cell=int(c)) for c in (4, 9, 17)]
    thr = rng.integers(1, 255, (8, 2)).astype(np.float32)     # randint(1, 255) twice: either order
    thr[0], thr[1] = g["rgb512_a"][1], g["rgb512_b"][1]
    x = torch.from_numpy(np.stack(imgs)).cuda()
    edges = torch.empty(8, 512, 512, dtype=torch.uint8, device="cuda")
    ops.canny(x, torch.from_numpy(thr).cuda(), edges=edges)
    got = edges.cpu().numpy()
    assert np.array_equal(got[0], g["rgb512_a"][2]) and np.array_equal(got[1], g["rgb512_b"][2])
    for b in range(8):
        assert np.array_equal(got[b], A.canny(imgs[b], *thr[b])), b


@pytest.mark.gpu
def test_gpu_goldens():
    """517x333, constant, checkerboard, grey, fractional / swapped / equal thresholds, and the 1024^2 spiral whose only
    strong pixels sit at its centre: every edge crosses tile borders by the union-find merge alone."""
    for name, (img, (lo, hi), edges) in golden().items():
        assert np.array_equal(_edges(img, lo, hi), edges), name


@pytest.mark.gpu
def test_gpu_shapes_and_constructed_cases():
    rng = np.random.default_rng(12)
    cases = [(shapes(rng, 768, 512), 40.0, 120.0), (shapes(rng, 512, 768, 1)[:, :, 0], 70.0, 20.0),
             (np.full((1, 1, 3), 9, np.uint8), 0.0, 0.0), (rng.integers(0, 256, (1, 1), dtype=np.uint8), -5.0, 10.0),
             (rng.integers(0, 256, (1, 777, 3), dtype=np.uint8), 50.0, 150.0), (rng.integers(0, 256, (611, 1), dtype=np.uint8), 80.0, 20.0),
             (smooth_noise(rng, 33, 1000, 3, cell=3), 25.5, 60.75), (smooth_noise(rng, 1000, 31, 1, cell=3), 60.0, 60.0),
             (np.full((300, 200), 200, np.uint8), 0.0, 1.0)]
    cases += [(nms_plateau(), 10.0 * k, 10.0 * k + 40.0) for k in range(6)]
    cases += [(channel_tie(rng), 20.0 + 15 * k, 120.0 - 10 * k) for k in range(6)]
    for i, (img, lo, hi) in enumerate(cases):
        assert np.array_equal(_edges(img, lo, hi), A.canny(img, lo, hi)), (i, img.shape, lo, hi)


@pytest.mark.gpu
def test_gpu_canny_batch_pixels_and_guide_are_bit_identical():
    import torch
    from controllora_b200 import canny_batch

    rng = np.random.default_rng(13)
    imgs = np.stack([shapes(rng, 96, 160) for _ in range(3)])
    imgs[0, :16, :16] = np.arange(256, dtype=np.uint8).reshape(16, 16, 1)      # every uint8 value
    thr = np.array([[30, 90], [120, 40], [10.5, 10.5]], np.float32)
    pix, guide = canny_batch(torch.from_numpy(imgs).cuda(), torch.from_numpy(thr).cuda())
    assert pix.shape == guide.shape == (3, 3, 96, 160) and pix.dtype == guide.dtype == torch.float32
    for b in range(3):
        e = A.canny(imgs[b], *thr[b])
        assert np.array_equal(pix[b].cpu().numpy().view(np.int32), A.pixel_values(imgs[b]).view(np.int32)), b
        assert np.array_equal(guide[b].cpu().numpy().view(np.int32), A.guide_values(e).view(np.int32)), b
    only = canny_batch(torch.from_numpy(imgs[:, :, :, :1].copy()).cuda(), (40, 100), pixel_values=False)
    for b in range(3):
        assert np.array_equal(only[b].cpu().numpy(), A.guide_values(A.canny(imgs[b, :, :, :1], 40, 100))), b


@pytest.mark.gpu
def test_gpu_canny_detector_matches_golden():
    import torch
    from controllora_b200 import CannyDetector

    det = CannyDetector()
    for name in ("smooth_rgb", "smooth_grey", "odd_517x333"):
        img, (lo, hi), edges = golden()[name]
        got = det(img, lo, hi)
        assert isinstance(got, np.ndarray) and got.dtype == np.uint8 and np.array_equal(got, edges), name
        got_t = det(torch.from_numpy(img).cuda(), lo, hi)
        assert got_t.is_cuda and np.array_equal(got_t.cpu().numpy(), edges), name


@pytest.mark.gpu
def test_gpu_canny_batch_cuda_graph_replays_with_new_images_and_thresholds():
    import torch
    from controllora_b200 import canny_batch

    rng = np.random.default_rng(14)
    B, H, W = 4, 256, 320
    static_img = torch.from_numpy(np.stack([shapes(rng, H, W) for _ in range(B)])).cuda()
    static_thr = torch.tensor([[20, 80]] * B, dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        canny_batch(static_img, static_thr)                    # warm-up outside capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        pix, guide = canny_batch(static_img, static_thr)
    for step in range(3):
        imgs = np.stack([shapes(rng, H, W) if b % 2 else smooth_noise(rng, H, W, 3, cell=7) for b in range(B)])
        thr = rng.integers(1, 255, (B, 2)).astype(np.float32)
        static_img.copy_(torch.from_numpy(imgs))
        static_thr.copy_(torch.from_numpy(thr))
        graph.replay()
        torch.cuda.synchronize()
        e_pix, e_guide = canny_batch(torch.from_numpy(imgs).cuda(), torch.from_numpy(thr).cuda())
        assert torch.equal(pix, e_pix) and torch.equal(guide, e_guide), step
        for b in range(B):
            assert np.array_equal(guide[b].cpu().numpy(), A.guide_values(A.canny(imgs[b], *thr[b]))), (step, b)
