"""Generates tests/golden/jpeg_golden.npz: seeded JPEG streams written by Pillow and by cv2.imencode, with Pillow's decode
of each (np.asarray(Image.open(f))), so that the JPEG oracle (oracle/jpeg_ref.py) and the CUDA decoder are pinned to
Pillow where Pillow is not importable.  The large streams (a 4032 x 3024 photo-like image, 4096 x 4096 flat and
striped images) are rebuilt from their seeds where they are used; the file keeps the sha256 of each stream, which the
rebuild must reproduce, and of Pillow's decode.

    python -m tests.golden.make_jpeg_golden        (needs Pillow and cv2)

The stream constructors are also used by tests/test_jpeg.py and tools/jpeg_bench.py.
"""
import hashlib
import io
import sys
from pathlib import Path

import numpy as np

OUT = Path(__file__).resolve().parent / "jpeg_golden.npz"


def photo(rng, H, W, C=3, cell=64, edges=12, noise=4):
    """Photo-like content: a smooth field (coarse noise upsampled with cv2's fixed-point bilinear resize), flat-coloured
    rectangles with hard edges, and mild noise."""
    import cv2

    coarse = rng.integers(0, 256, (H // cell + 2, W // cell + 2, C), dtype=np.uint8)
    img = cv2.resize(coarse, (W, H), interpolation=cv2.INTER_LINEAR).reshape(H, W, C).astype(np.int16)
    for _ in range(edges):
        y0, x0 = int(rng.integers(0, H)), int(rng.integers(0, W))
        h, w = int(rng.integers(1, max(2, H // 3))), int(rng.integers(1, max(2, W // 3)))
        img[y0:y0 + h, x0:x0 + w] = rng.integers(0, 256, C)
    img += rng.integers(-noise, noise + 1, img.shape, dtype=np.int16)
    out = np.clip(img, 0, 255).astype(np.uint8)
    return out[..., 0] if C == 1 else out


def flat(H, W, colour=(200, 30, 90)):
    return np.broadcast_to(np.array(colour, np.uint8), (H, W, 3)).copy()


def striped(H, W, period=6):
    img = np.zeros((H, W, 3), np.uint8)
    img[:, (np.arange(W) % period) < period // 2] = (240, 240, 16)
    return img


def pil_jpeg(a: np.ndarray, **kw) -> bytes:
    from PIL import Image

    buf = io.BytesIO()
    Image.fromarray(a).save(buf, "JPEG", **kw)
    return buf.getvalue()


def cv2_jpeg(a: np.ndarray, quality=95, rst=0) -> bytes:
    import cv2

    ok, enc = cv2.imencode(".jpg", a, [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_RST_INTERVAL, rst])
    assert ok
    return enc.tobytes()


def dqt_edited(value: int, entry: int) -> bytes:
    """A flat 16 x 16 grey image of `value` at quality 100 whose DC quantisation entry is then set to `entry`: the
    decoded block lies far outside 0..255, where libjpeg-turbo's SIMD IDCT (Pillow's) and its C code part ways."""
    b = bytearray(pil_jpeg(np.full((16, 16), value, np.uint8), quality=100))
    b[b.index(b"\xff\xdb") + 5] = entry
    return bytes(b)


def dqt_edited_cases():
    return [(f"dqt_flat{v}_dc{e}", dqt_edited(v, e)) for v, e in ((160, 90), (160, 100), (200, 40), (30, 255), (255, 7))]


def dqt_random_edits(rng, n):
    """Photo-like 24 x 40 streams with five random entries of the luma table replaced after encoding."""
    out = []
    for _ in range(n):
        b = bytearray(pil_jpeg(photo(rng, 24, 40), quality=int(rng.integers(50, 101))))
        i = b.index(b"\xff\xdb")
        for _ in range(5):
            b[i + 5 + int(rng.integers(64))] = int(rng.integers(1, 256))
        out.append(bytes(b))
    return out


def small_cases():
    """(name, stream) of the stored streams: every layout, restart and no-restart, optimised tables, qualities 1-100,
    cv2 streams, 1 x 1 and odd sizes."""
    rng = np.random.default_rng(20261019)
    out = []
    sizes = [(1, 1), (1, 9), (13, 1), (7, 7), (17, 31), (33, 48), (61, 87)]
    for i, (h, w) in enumerate(sizes):
        a = photo(rng, h, w)
        for ss in (0, 1, 2):
            q = (1, 10, 50, 75, 95, 100)[(i + ss) % 6]
            out.append((f"pil_{h}x{w}_ss{ss}_q{q}", pil_jpeg(a, quality=q, subsampling=ss)))
        out.append((f"pil_{h}x{w}_gray", pil_jpeg(a[..., 1], quality=85)))
    a = photo(rng, 96, 130)
    out.append(("pil_opt_rstblocks", pil_jpeg(a, quality=90, optimize=True, restart_marker_blocks=5)))
    out.append(("pil_rstrows", pil_jpeg(a, quality=60, subsampling=1, restart_marker_rows=1)))
    out.append(("pil_exif_icc_com", pil_jpeg(a, exif=b"Exif\0\0MM\0*\0\0\0\x08\0\0\0\0\0\0", icc_profile=bytes(range(256)) * 80,
                                             comment=b"golden")))
    out.append(("cv2_q95", cv2_jpeg(a[..., ::-1].copy())))
    out.append(("cv2_q40_rst3", cv2_jpeg(a[..., ::-1].copy(), quality=40, rst=3)))
    out.append(("cv2_gray_rst1", cv2_jpeg(a[..., 0].copy(), quality=70, rst=1)))
    out.append(("flat_420", pil_jpeg(flat(40, 72))))
    out.append(("striped_444", pil_jpeg(striped(40, 72), subsampling=0)))
    out += dqt_edited_cases()
    out += [(f"dqt_random_{k}", b) for k, b in enumerate(dqt_random_edits(rng, 4))]
    t = [[int(v) * 255 for v in rng.integers(1, 256, 64)] for _ in range(2)]
    out.append(("qtables16_x255", pil_jpeg(photo(rng, 24, 40), qtables=t, subsampling=2)))
    return out


def large_cases():
    """(name, stream) of the streams rebuilt where they are used."""
    rng = np.random.default_rng(4032)
    return [
        ("photo_4032x3024_q92", pil_jpeg(photo(rng, 3024, 4032), quality=92)),
        ("flat_4096", pil_jpeg(flat(4096, 4096))),
        ("striped_4096", pil_jpeg(striped(4096, 4096))),
    ]


def sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


def build(with_large=True):
    from PIL import Image

    small = small_cases()
    arrays = {}
    streams = [np.frombuffer(s, np.uint8) for _, s in small]
    decoded = [np.asarray(Image.open(io.BytesIO(s))) for _, s in small]
    arrays["names"] = np.array([n for n, _ in small])
    arrays["stream_off"] = np.cumsum([0] + [len(s) for s in streams]).astype(np.int64)
    arrays["streams"] = np.concatenate(streams)
    arrays["stream_sha256"] = np.array([sha(s) for _, s in small])
    arrays["shapes"] = np.array([d.shape + (1,) * (3 - d.ndim) for d in decoded], np.int64)
    arrays["ndim"] = np.array([d.ndim for d in decoded], np.int64)
    arrays["pixels"] = np.concatenate([d.reshape(-1) for d in decoded])
    if with_large:
        large = large_cases()
        arrays["large_names"] = np.array([n for n, _ in large])
        arrays["large_stream_sha256"] = np.array([sha(s) for _, s in large])
        arrays["large_pixels_sha256"] = np.array([sha(np.asarray(Image.open(io.BytesIO(s))).tobytes()) for _, s in large])
    return arrays


def main():
    arrays = build()
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes, {len(arrays['names'])} stored streams)")


if __name__ == "__main__":
    sys.exit(main())
