"""Generates tests/golden/png_golden.npz: seeded PNG files of every colour type and bit depth, written by a hand-built
encoder (explicit per-row filters, Python's zlib with a chosen strategy, level and window) and by Pillow, with Pillow's
convert("RGB") and convert("L") of each, so that the PNG oracle (oracle/png_ref.py) and the CUDA decoder are pinned to
Pillow where Pillow is not importable.  The file keeps each stream's sha256, which the generator must reproduce.

    python -m tests.golden.make_png_golden        (needs Pillow)

The stream constructors are also used by tests/test_png.py and tools/png_bench.py.
"""
import hashlib
import io
import struct
import sys
import zlib
from pathlib import Path

import numpy as np

OUT = Path(__file__).resolve().parent / "png_golden.npz"
SAMPLES = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def chunk(ctype: bytes, body: bytes, crc=None) -> bytes:
    c = zlib.crc32(body, zlib.crc32(ctype)) if crc is None else crc
    return struct.pack(">I", len(body)) + ctype + body + struct.pack(">I", c)


def ihdr(W, H, depth, ct, interlace=0) -> bytes:
    return chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, depth, ct, 0, 0, interlace))


def filter_rows(lines: np.ndarray, bpp: int, filters) -> bytes:
    """Filter reconstructed scanlines (uint8 [H, rowbytes]) with filters[r] (0-4) per row (PNG spec 9)."""
    H, n = lines.shape
    out = bytearray()
    prev = np.zeros(n, np.int32)
    for r in range(H):
        x = lines[r].astype(np.int32)
        a = np.concatenate([np.zeros(bpp, np.int32), x[:-bpp]])[:n]
        c = np.concatenate([np.zeros(bpp, np.int32), prev[:-bpp]])[:n]
        b = prev
        ft = int(filters[r % len(filters)])
        if ft == 0:
            y = x
        elif ft == 1:
            y = x - a
        elif ft == 2:
            y = x - b
        elif ft == 3:
            y = x - ((a + b) >> 1)
        else:
            p = a + b - c
            pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
            y = x - np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        out.append(ft)
        out += (y & 255).astype(np.uint8).tobytes()
        prev = x
    return bytes(out)


def compress(raw: bytes, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15, flushes=(), mem_level=8) -> bytes:
    """A zlib stream of raw, with Z_SYNC_FLUSH / Z_FULL_FLUSH at the given (offset, mode) points."""
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, mem_level, strategy)
    out, last = [], 0
    for off, mode in flushes:
        out.append(co.compress(raw[last:off]))
        out.append(co.flush(mode))
        last = off
    out.append(co.compress(raw[last:]))
    out.append(co.flush())
    return b"".join(out)


def build_png(lines: np.ndarray, W: int, ct: int, depth: int, filters=(0,), palette=None, trns=None, zdata=None,
              idat_split=None, before=(), after=(), **zkw) -> bytes:
    """A PNG from reconstructed scanlines: IHDR, [before], PLTE, tRNS, IDAT (split into idat_split-byte chunks), [after],
    IEND."""
    bpp = max(1, SAMPLES[ct] * depth // 8)
    if zdata is None:
        zdata = compress(filter_rows(lines, bpp, filters), **zkw)
    parts = [b"\x89PNG\r\n\x1a\n", ihdr(W, lines.shape[0], depth, ct)]
    parts += [chunk(t, b) for t, b in before]
    if palette is not None:
        parts.append(chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes()))
    if trns is not None:
        parts.append(chunk(b"tRNS", trns))
    step = idat_split or max(1, len(zdata))
    parts += [chunk(b"IDAT", zdata[k:k + step]) for k in range(0, len(zdata), step)]
    parts += [chunk(t, b) for t, b in after]
    parts.append(chunk(b"IEND", b""))
    return b"".join(parts)


def scanlines(rng, H: int, W: int, ct: int, depth: int, kind="noise") -> np.ndarray:
    """Random reconstructed scanlines (uint8 [H, rowbytes]): noise, or smooth content that compresses like a photo."""
    n = (W * SAMPLES[ct] * depth + 7) // 8
    if kind == "noise":
        return rng.integers(0, 256, (H, n), dtype=np.uint8)
    base = np.add.outer(np.arange(H), np.arange(n)) // 7 + rng.integers(0, 3, (H, n))
    return (base & 255).astype(np.uint8)


def photo_png(rng, H, W, **kw) -> bytes:
    from PIL import Image

    from tests.golden.make_jpeg_golden import photo

    buf = io.BytesIO()
    Image.fromarray(photo(rng, H, W)).save(buf, "PNG", **kw)
    return buf.getvalue()


def fill50k_pair(rng, size=512):
    """A fill50k-like pair: a flat background with a filled circle (the image) and its outline (the guide), by Pillow."""
    from PIL import Image, ImageDraw

    bg, fg = tuple(int(v) for v in rng.integers(0, 256, 3)), tuple(int(v) for v in rng.integers(0, 256, 3))
    cx, cy, r = (int(v) for v in rng.integers(size // 4, 3 * size // 4, 3) // (1, 1, 2))
    img = Image.new("RGB", (size, size), bg)
    ImageDraw.Draw(img).ellipse((cx - r, cy - r, cx + r, cy + r), fill=fg)
    guide = Image.new("RGB", (size, size), (0, 0, 0))
    ImageDraw.Draw(guide).ellipse((cx - r, cy - r, cx + r, cy + r), outline=(255, 255, 255), width=3)
    out = []
    for im in (img, guide):
        buf = io.BytesIO()
        im.save(buf, "PNG")
        out.append(buf.getvalue())
    return out


def golden_cases():
    """(name, file) of the stored files: every colour type and bit depth, each filter type, tRNS, short palettes."""
    rng = np.random.default_rng(20261020)
    out = []
    for ct, depths in ((0, (1, 2, 4, 8, 16)), (2, (8, 16)), (3, (1, 2, 4, 8)), (4, (8, 16)), (6, (8, 16))):
        for depth in depths:
            H, W = 13, 21
            lines = scanlines(rng, H, W, ct, depth, "smooth" if depth >= 8 else "noise")
            pal = rng.integers(0, 256, (max(2, (1 << depth) // 2), 3)) if ct == 3 else None
            if ct == 3:
                lines = scanlines(rng, H, W, ct, depth, "noise")
            out.append((f"ct{ct}_d{depth}", build_png(lines, W, ct, depth, filters=(0, 1, 2, 3, 4), palette=pal)))
    out.append(("rgb_trns", build_png(scanlines(rng, 8, 9, 2, 8), 9, 2, 8, filters=(4,), trns=b"\0\1\0\2\0\3")))
    out.append(("pil_photo", photo_png(rng, 40, 56)))
    return out


def sha(b) -> str:
    return hashlib.sha256(bytes(b)).hexdigest()


def build():
    from PIL import Image

    cases = golden_cases()
    arrays = {"names": np.array([n for n, _ in cases]), "stream_sha256": np.array([sha(s) for _, s in cases])}
    streams = [np.frombuffer(s, np.uint8) for _, s in cases]
    arrays["stream_off"] = np.cumsum([0] + [len(s) for s in streams]).astype(np.int64)
    arrays["streams"] = np.concatenate(streams)
    for mode in ("RGB", "L"):
        dec = [np.asarray(Image.open(io.BytesIO(s)).convert(mode)) for _, s in cases]
        arrays[f"shapes_{mode}"] = np.array([d.shape[:2] for d in dec], np.int64)
        arrays[f"pixels_{mode}"] = np.concatenate([d.reshape(-1) for d in dec])
    return arrays


def main():
    arrays = build()
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes, {len(arrays['names'])} files)")


if __name__ == "__main__":
    sys.exit(main())
