"""Pose renderer (cl_pose_render, controllora_b200.pose): the numpy oracle against OpenCV rule by rule and against the
reference's own draw_bodypose and the stored goldens (CPU), the C-ABI argument checks and descriptor layout (CPU), and
the CUDA kernel against both, bit for bit (GPU)."""
import ctypes
import math
from pathlib import Path

import numpy as np
import pytest

from controllora_b200 import pose as PZ
from oracle import pose_ref as R
from tests.golden.make_pose_golden import background, cases as golden_cases, import_reference_util, skeleton
from tests.golden.reference_import import REFERENCE_ROOT as REFERENCE

GOLDEN = Path(__file__).resolve().parent / "golden" / "pose_golden.npz"


def golden():
    z = np.load(GOLDEN)
    assert [str(n) for n in z["names"]] == [c[0] for c in golden_cases()]
    return {str(n): (z[f"bg_{n}"], z[f"cand_{n}"], z[f"subset_{n}"], z[f"out_{n}"]) for n in z["names"]}


def reference_available():
    try:
        return (REFERENCE / "annotator" / "openpose" / "util.py").is_file()
    except OSError:
        return False


def pin_skeletons(n=300):
    """Seeded (canvas, candidate, subset): 0-6 persons, missing keypoints, overlapping limbs, keypoints outside the
    canvas, integer and fractional coordinates, square and non-square canvases, zero and random backgrounds."""
    rng = np.random.default_rng(11)
    out = []
    for i in range(n):
        H, W = (int(v) for v in rng.integers(8, 200 if i % 10 else 520, 2))
        if i % 5 == 0:
            W = H
        cand, sub = skeleton(rng, H, W, i % 7, integer=i % 3 == 0, outside=0.25 if i % 4 == 1 else 0.0,
                             missing=0.3 if i % 2 else 0.05)
        bg = background(rng, H, W) if i % 6 == 5 else np.zeros((H, W, 3), np.uint8)
        out.append((bg, cand, sub))
    return out


# -------------------------------------------------------------------------------------------------------------- CPU
def test_sin_table_is_opencv_s():
    q = R.sin_table_q30()
    assert q.shape == (451,) and q[0] == 0 and q[90] == 1 << 30 and q[450] == 1 << 30
    assert np.abs(q / 2.0 ** 30 - np.sin(np.radians(np.arange(451)))).max() < 1e-7
    pytest.importorskip("cv2")
    from tools.make_pose_sin_table import recover, render
    assert np.array_equal(recover(), q)
    assert render(q) == (Path(R.__file__).resolve().parent.parent / "controllora_b200" / "csrc" / "pose_sin_table.h").read_text()


def test_ellipse2poly_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    cases = [(a, ax) for a in range(-360, 361) for ax in (0, 1, 4, 37)]
    cases += [(int(rng.integers(-180, 181)), int(ax)) for ax in rng.integers(0, 1001, 600)]
    for angle, ax in cases:
        c = (int(rng.integers(-300, 900)), int(rng.integers(-300, 900)))
        assert np.array_equal(cv2.ellipse2Poly(c, (ax, 4), angle, 0, 360, 1), R.ellipse2poly(c, (ax, 4), angle)), (c, ax, angle)


def test_line_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2)
    for _ in range(3000):
        H, W = (int(v) for v in rng.integers(1, 60, 2))
        p1, p2 = (tuple(int(v) for v in rng.integers(-50, 110, 2)) for _ in range(2))
        img = np.zeros((H, W), np.uint8)
        cv2.line(img, p1, p2, 255, 1, cv2.LINE_8)
        m = np.zeros((H, W), bool)
        xs, ys = R.line_pixels(W, H, p1, p2)
        m[ys, xs] = True
        assert np.array_equal(img > 0, m), (H, W, p1, p2)


def test_fill_convex_poly_matches_cv2_on_limb_ellipses():
    """The thin rotated ellipses draw_bodypose fills, inside the canvas, clipped on every edge and wholly outside."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for i in range(1200):
        H, W = (int(v) for v in rng.integers(1, 160, 2))
        half = int(rng.integers(0, 3)) if i % 10 == 0 else int(rng.integers(0, 200))
        c = (int(rng.integers(-half - 20, W + half + 20)), int(rng.integers(-half - 20, H + half + 20)))
        poly = cv2.ellipse2Poly(c, (half, 4), int(rng.integers(-180, 181)), 0, 360, 1)
        img = np.zeros((H, W), np.uint8)
        cv2.fillConvexPoly(img, poly, 255)
        assert np.array_equal(img > 0, R.fill_convex_poly_mask(H, W, poly)), (H, W, c, half)


def test_circle_matches_cv2_near_every_border():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    assert R.circle_spans(4) == {0: 4, 1: 3, -1: 3, 2: 3, -2: 3, 3: 2, -3: 2, 4: 0, -4: 0}   # the kernel's table
    for _ in range(2000):
        H, W = (int(v) for v in rng.integers(1, 40, 2))
        c = (int(rng.integers(-9, W + 9)), int(rng.integers(-9, H + 9)))
        img = np.zeros((H, W), np.uint8)
        cv2.circle(img, c, 4, 255, thickness=-1)
        assert np.array_equal(img > 0, R.circle_mask(H, W, *c)), (H, W, c)


def test_add_weighted_exhaustive():
    cv2 = pytest.importorskip("cv2")
    a = np.arange(256, dtype=np.uint8)
    A, B = np.meshgrid(a, a, indexing="ij")
    assert np.array_equal(cv2.addWeighted(A, 0.4, B, 0.6, 0), R.add_weighted(A, B))
    assert np.array_equal(cv2.addWeighted(a[None], 0.4, a[None], 0.6, 0)[0], a)     # an uncovered pixel keeps its value
    assert np.array_equal(R.add_weighted(a, a), a)


def test_inter_nearest_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    from controllora_b200.transforms import resize_image_size

    rng = np.random.default_rng(5)
    pairs = [tuple(int(v) for v in rng.integers(1, 1300, 4)) for _ in range(400)]
    for h, w in [(512, 512), (1024, 768), (480, 640), (333, 517), (1000, 1500)]:      # the app: detect -> image size
        for det, res in [(512, 512), (256, 512), (512, 768), (384, 1024)]:
            dh, dw, _ = resize_image_size(h, w, det)
            ih, iw, _ = resize_image_size(h, w, res)
            pairs.append((dh, dw, ih, iw))
    for h, w, H, W in pairs:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        assert np.array_equal(cv2.resize(img, (W, H), interpolation=cv2.INTER_NEAREST), R.resize_nearest(img, H, W)), (h, w, H, W)


def test_host_limb_parameters_are_the_reference_s():
    """pose.limb_params (Python floats) against the reference's numpy scalar expressions, including limbs whose angle or
    half length lands on an integer and limbs far outside the canvas."""
    rng = np.random.default_rng(6)
    pts = [rng.uniform(-600, 1200, 4) for _ in range(3000)]
    pts += [np.round(rng.uniform(-600, 1200, 4)) for _ in range(2000)]
    pts += [np.array([0.0, 0.0, 3.0, 4.0]), np.array([5.0, 5.0, 5.0, 5.0]), np.array([1.0, 1.0, 1.0 + 1e-300, 1.0])]
    for k in range(1, 90):
        t = math.radians(k)
        pts.append(np.array([10.0, 20.0, 10.0 + 50 * math.cos(t), 20.0 + 50 * math.sin(t)]))
    for x0, y0, x1, y1 in pts:
        cand = np.array([[x0, y0, 1, 0], [x1, y1, 1, 1]], np.float64)
        assert PZ.limb_params(float(x0), float(y0), float(x1), float(y1)) == R.limb_params(cand, 0, 1), (x0, y0, x1, y1)


def test_oracle_matches_the_reference_draw_bodypose():
    if not reference_available():
        pytest.skip("reference tree not present: the goldens pin the oracle instead")
    pytest.importorskip("cv2")
    util = import_reference_util()
    for k, (bg, cand, sub) in enumerate(pin_skeletons()):
        want = util.draw_bodypose(bg.copy(), cand, sub)
        assert np.array_equal(R.draw_bodypose(bg, cand, sub), want), k


def test_oracle_reproduces_golden():
    for name, (bg, cand, sub, out) in golden().items():
        assert np.array_equal(R.draw_bodypose(bg, cand, sub), out), name


def test_golden_inputs_are_regenerated_exactly():
    g = golden()
    for name, bg, cand, sub in golden_cases():
        gb, gc, gs, _ = g[name]
        assert np.array_equal(bg, gb) and np.array_equal(cand, gc) and np.array_equal(sub, gs), name


def test_cl_pose_render_rejects_bad_arguments_without_a_gpu(built_lib):
    from controllora_b200 import _lib

    lib = _lib.lib()
    P = ctypes.c_void_p(64)      # never dereferenced: every check runs before any CUDA call

    def img(**kw):
        d = _lib.PoseImage(bg_off=-1, Hc=16, Wc=16, y0=0, x0=0, h=16, w=16, circle0=0, n_circles=1, limb0=0, n_limbs=1)
        for k, v in kw.items():
            setattr(d, k, v)
        return (_lib.PoseImage * 1)(d)

    def limb(**kw):
        d = _lib.PoseLimb(mask_off=0, image=0, cx=8, cy=8, half_len=5, angle=30, color=255, bx0=0, by0=0, bw=16, bh=16)
        for k, v in kw.items():
            setattr(d, k, v)
        return (_lib.PoseLimb * 1)(d)

    circ = (_lib.PoseCircle * 1)(_lib.PoseCircle(x=3, y=4, color=7))

    def call(i=None, B=1, c=circ, nc=1, l=None, nl=1, bg=None, bg_bytes=0, mask=P, words=16, oh=16, ow=16, flip=1,
             canvas=P, guide=None):
        return lib.cl_pose_render(ctypes.cast(i if i is not None else img(), ctypes.c_void_p), P, B, ctypes.cast(c, ctypes.c_void_p),
                                  P, nc, ctypes.cast(l if l is not None else limb(), ctypes.c_void_p), P, nl, bg, bg_bytes, mask,
                                  words, oh, ow, flip, canvas, guide, None)

    cases = {
        "no output": dict(canvas=None), "B": dict(B=0), "out size": dict(oh=0), "out too big": dict(ow=5000),
        "flip": dict(flip=2), "canvas": dict(i=img(Hc=0)), "canvas too big": dict(i=img(Wc=4097, w=16)),
        "crop": dict(i=img(y0=1)), "background": dict(i=img(bg_off=0)), "background bytes": dict(i=img(bg_off=0), bg=P, bg_bytes=767),
        "circle range": dict(i=img(n_circles=2)), "limb range": dict(i=img(limb0=1)), "limb image": dict(l=limb(image=1)),
        "angle": dict(l=limb(angle=361)), "half length": dict(l=limb(half_len=-1)), "centre": dict(l=limb(cx=1 << 23)),
        "box": dict(l=limb(bx0=1)), "mask": dict(words=15), "null mask": dict(mask=None), "colour": dict(l=limb(color=1 << 24)),
        "circle colour": dict(c=(_lib.PoseCircle * 1)(_lib.PoseCircle(x=3, y=4, color=-1))),
    }
    for what, kw in cases.items():
        assert call(**kw) == -1, what
        assert lib.cl_last_error().decode().startswith("cl_pose_render"), what


def test_pose_desc_layout_matches_c(built_lib, tmp_path):
    import subprocess

    from controllora_b200 import _lib

    root = Path(__file__).resolve().parent.parent
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "controllora_b200.h"\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(cl_pose_image), offsetof(cl_pose_image, limb0),'
                   ' sizeof(cl_pose_circle), offsetof(cl_pose_circle, color), sizeof(cl_pose_limb), offsetof(cl_pose_limb, image),'
                   ' offsetof(cl_pose_limb, color), offsetof(cl_pose_limb, bh));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", str(root / "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [ctypes.sizeof(_lib.PoseImage), _lib.PoseImage.limb0.offset, ctypes.sizeof(_lib.PoseCircle),
                   _lib.PoseCircle.color.offset, ctypes.sizeof(_lib.PoseLimb), _lib.PoseLimb.image.offset,
                   _lib.PoseLimb.color.offset, _lib.PoseLimb.bh.offset]


def test_wrappers_reject_bad_arguments():
    from controllora_b200._lib import CLError

    kp = np.zeros((1, 1, 18, 3))
    with pytest.raises(CLError):
        PZ._windows(1, (0, 10), None, None, "t")
    with pytest.raises(CLError):
        PZ._windows(1, (10, 10), [(0, 0, 11, 10)], None, "t")
    with pytest.raises(CLError):
        PZ._windows(2, [(10, 10), (12, 12)], None, None, "t")          # windows differ and no out_hw
    with pytest.raises(CLError):
        PZ._dense_prims(np.zeros((1, 1, 17, 3)), "t")
    kp[0, 0, 0] = (np.nan, 1.0, 1.0)
    with pytest.raises(CLError):
        PZ._dense_prims(kp, "t")
    with pytest.raises(CLError):
        PZ._prims_from_candidate(np.array([[3e6, 1.0, 1, 0]]), np.r_[[0.0], -np.ones(19)][None], "t")


def test_dense_keypoints_give_the_candidate_subset_primitives():
    rng = np.random.default_rng(7)
    for _ in range(20):
        P = int(rng.integers(0, 5))
        kp = np.zeros((P, 18, 3))
        cand, rows = [], []
        for n in range(P):
            row = -np.ones(20)
            for k in range(18):
                if rng.uniform() < 0.8:
                    kp[n, k] = (*rng.uniform(-50, 300, 2), 1.0)
                    row[k] = len(cand)
                    cand.append([kp[n, k, 0], kp[n, k, 1], 1.0, len(cand)])
            rows.append(row)
        a = PZ._prims_from_dense(kp, "t")
        b = PZ._prims_from_candidate(np.array(cand).reshape(-1, 4), np.array(rows).reshape(-1, 20), "t")
        assert a == b


# -------------------------------------------------------------------------------------------------------------- GPU
def _ragged_batch(rng):
    """8 images: mixed canvas sizes, 0-6 persons, crops and nearest resizes to one output size."""
    sizes = [(512, 512), (384, 640), (700, 500), (256, 256), (97, 131), (1024, 768), (300, 451), (64, 64)]
    out_hw = (192, 256)
    P = 6
    kp = np.zeros((8, P, 18, 3))
    crops = []
    for b, (H, W) in enumerate(sizes):
        n = b % 7
        cand, sub = skeleton(rng, H, W, n, integer=b % 2 == 0, outside=0.2 if b % 3 == 0 else 0.0)
        for p in range(n):
            for k in range(18):
                if sub[p, k] >= 0:
                    kp[b, p, k] = (*cand[int(sub[p, k]), :2], 1.0)
        h, w = int(rng.integers(H // 2, H + 1)), int(rng.integers(W // 2, W + 1))
        crops.append((int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w))
    return sizes, kp, crops, out_hw


def _oracle_dense(kp_b, H, W, bg=None):
    cand, rows = [], []
    for p in range(kp_b.shape[0]):
        row = -np.ones(20)
        for k in range(18):
            if kp_b[p, k, 2] > 0:
                row[k] = len(cand)
                cand.append([kp_b[p, k, 0], kp_b[p, k, 1], 1.0, len(cand)])
        rows.append(row)
    canvas = np.zeros((H, W, 3), np.uint8) if bg is None else bg
    return R.draw_bodypose(canvas, np.array(cand).reshape(-1, 4), np.array(rows).reshape(-1, 20))


@pytest.mark.gpu
def test_gpu_ragged_batch_matches_the_oracle():
    rng = np.random.default_rng(50)
    sizes, kp, crops, out_hw = _ragged_batch(rng)
    bgs = [background(rng, H, W) if b % 3 == 2 else None for b, (H, W) in enumerate(sizes)]
    for flip in (True, False):
        guide, u8 = PZ.pose_batch(kp, sizes, crops=crops, out_hw=out_hw, backgrounds=bgs, flip=flip, canvas=True)
        assert guide.shape == (8, 3, *out_hw) and u8.shape == (8, *out_hw, 3)
        for b, (H, W) in enumerate(sizes):
            want = R.window(_oracle_dense(kp[b], H, W, bgs[b]), crops[b], out_hw)
            assert np.array_equal(u8[b].cpu().numpy(), want), b
            assert np.array_equal(guide[b].cpu().numpy().view(np.int32), R.guide(want, flip).view(np.int32)), b
    # the crop window equals rendering the full canvas, then cropping
    full, = [PZ.pose_batch(kp[:1], sizes[0], canvas=True)[1]]
    y0, x0, h, w = crops[0]
    part = PZ.pose_batch(kp[:1], sizes[0], crops=[crops[0]], canvas=True)[1]
    assert np.array_equal(part[0].cpu().numpy(), full[0, y0:y0 + h, x0:x0 + w].cpu().numpy())


@pytest.mark.gpu
def test_gpu_draw_bodypose_matches_goldens_and_oracle():
    import torch

    for name, (bg, cand, sub, out) in golden().items():
        got = PZ.draw_bodypose(bg, cand, sub)
        assert isinstance(got, np.ndarray) and np.array_equal(got, out), name
        got_t = PZ.draw_bodypose(torch.from_numpy(bg).cuda(), cand, sub)
        assert got_t.is_cuda and np.array_equal(got_t.cpu().numpy(), out), name
    for k, (bg, cand, sub) in enumerate(pin_skeletons(120)):
        assert np.array_equal(PZ.draw_bodypose(bg, cand, sub), R.draw_bodypose(bg, cand, sub)), k


@pytest.mark.gpu
def test_gpu_pose_control_at_the_app_sizes():
    from controllora_b200.transforms import resize_image_size

    rng = np.random.default_rng(51)
    for (h, w), det, res in [((512, 512), 512, 512), ((768, 1024), 512, 768), ((1000, 667), 256, 512), ((480, 640), 384, 1024)]:
        dh, dw, _ = resize_image_size(h, w, det)
        ih, iw, _ = resize_image_size(h, w, res)
        cand, sub = skeleton(rng, dh, dw, 3)
        got = PZ.pose_control(cand, sub, (h, w), det, res)
        detected = R.draw_bodypose(np.zeros((dh, dw, 3), np.uint8), cand, sub)
        want = R.guide(R.resize_nearest(detected, ih, iw), True)[None]
        assert got.shape == want.shape and np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32)), (h, w, det, res)


@pytest.mark.gpu
def test_gpu_pose_buffers_graph_replay_with_new_keypoints_equals_eager():
    import torch

    rng = np.random.default_rng(52)
    sizes, kp, crops, out_hw = _ragged_batch(rng)
    buf = PZ.PoseBuffers(8, kp.shape[1], sizes, crops=crops, out_hw=out_hw)
    buf.stage(kp)
    buf.launch()
    torch.cuda.synchronize()
    assert torch.equal(buf.guide, PZ.pose_batch(kp, sizes, crops=crops, out_hw=out_hw))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        buf.launch()
    for seed in (53, 54):
        _, kp2, _, _ = _ragged_batch(np.random.default_rng(seed))
        torch.cuda.synchronize()
        buf.stage(kp2)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(buf.guide, PZ.pose_batch(kp2, sizes, crops=crops, out_hw=out_hw)), seed


@pytest.mark.gpu
def test_gpu_pose_guide_reaches_the_hint_encoder_of_mpii_pose_v2_unchanged():
    """pose_batch -> Trainer.step_from_pixels with the mpii-pose-v2 ControlLoRA at a tiny size: the hint encoder reads
    exactly the guide pose_batch produced."""
    import torch

    import controllora_b200 as cb
    from controllora_b200.configs import NAMED
    from controllora_b200.trainer import Trainer
    from oracle import clip_ref as CR
    from oracle import models_ref as MR
    from oracle import unet_ref as UR
    from oracle import vae_ref as VR
    from tests import check_unet as CU

    ounet = UR.UNet2DConditionModel(**CU.TINY)
    UR.init_synthetic_(ounet, seed=1)
    munet = cb.UNet2DConditionModel.from_state_dict({k: v.detach().clone() for k, v in ounet.state_dict().items()}, "cuda", CU.TINY)
    kw = dict(CU.TINY_LORA)
    kw.update(NAMED["mpii-pose-v2"])
    mcl = cb.ControlLoRA(**kw)
    mcl.load_state_dict(MR.ControlLoRA(**kw).state_dict())
    mcl.to("cuda")
    MR.wire_processors(munet, mcl)
    vcfg = dict(block_out_channels=(32, 64, 64), layers_per_block=1)
    ovae = VR.AutoencoderKL(**vcfg)
    VR.init_synthetic_(ovae, seed=4)
    mvae = cb.AutoencoderKL.from_state_dict({k: v.detach().clone() for k, v in ovae.state_dict().items()}, "cuda", vcfg)
    ccfg = dict(CR.SD15_TEXT_CONFIG)
    ccfg.update(num_hidden_layers=2, vocab_size=1000, hidden_size=64, intermediate_size=256, num_attention_heads=4)
    mclip = cb.CLIPTextModel.from_state_dict(CR.synthetic_state_dict(ccfg, seed=0), "cuda", ccfg)
    B = 2
    rng = np.random.default_rng(55)
    kp = np.zeros((B, 3, 18, 3))
    for b in range(B):
        cand, sub = skeleton(rng, 128, 128, 3)
        for p in range(3):
            for k in range(18):
                if sub[p, k] >= 0:
                    kp[b, p, k] = (*cand[int(sub[p, k]), :2], 1.0)
    guide = PZ.pose_batch(kp, (128, 128), flip=False)
    g = torch.Generator().manual_seed(13)
    pix = (torch.rand(B, 3, 64, 64, generator=g) * 2 - 1).cuda()
    ids = torch.randint(0, ccfg["vocab_size"], (B, 77), generator=g).cuda()
    tr = Trainer(munet, mcl, lr=0.0, noise_seed=99)
    seen = []
    forward = tr.hint.forward
    tr.hint.forward = lambda ctx, x: (seen.append(x.clone()), forward(ctx, x))[1]
    loss = tr.step_from_pixels(mvae, mclip, pix, ids, guide, eager=True)
    torch.cuda.synchronize()
    assert math.isfinite(float(loss))
    assert len(seen) == 1 and torch.equal(seen[0], guide)
    for b in range(B):
        want = R.guide(_oracle_dense(kp[b], 128, 128), False)
        assert np.array_equal(seen[0][b].cpu().numpy().view(np.int32), want.view(np.int32)), b
