"""numpy restatement of PNG decoding as Pillow runs it: Image.open(f).convert("RGB") / .convert("L") (tests only).
Pinned by tests/test_png.py to Pillow itself (Pillow 12.2, whose wheels inflate with zlib-ng).

    chunk parsing   controllora_b200/png.py parse(): the host side of the product, shared with this module so that
                    comparing the decode with Pillow pins the parser, the CRC checks and the refusals as well
    inflate         Python's zlib (an implementation independent of Pillow's zlib-ng), asked for the filtered rows'
                    size: as under Pillow, decoding stops at the first byte past the last row, so bytes after it are
                    not read and the Adler-32 is compared only when the stream ends there with its trailer
    unfiltering     None / Sub / Up / Average / Paeth per row in uint8 arithmetic (PNG spec 9); a filter type above 4
                    is corrupt
    unpacking       Pillow's modes: grey 1 -> "1" (0 / 255), grey 2 / 4 scaled by 85 / 17, grey 16 -> "I;16" (clips
                    at 255 when converted), 16-bit RGB / RGBA / grey + alpha keep the high byte, palette indices past
                    PLTE are black
    convert         RGB -> L by Pillow's fixed-point ITU-R 601 weights, palette -> L by the L of the entries, alpha
                    dropped, grey replicated to RGB

block_table(zdata) is a small pure-Python deflate block walker: (start bit, BTYPE, BFINAL, inflated bytes) per block.
"""
from __future__ import annotations

import zlib

import numpy as np

from controllora_b200.png import SAMPLES, Frame, parse


class Corrupt(ValueError):
    """Corrupt image data (Pillow raises on it); .kind names it as the device status does."""

    def __init__(self, kind: str):
        super().__init__(kind)
        self.kind = kind


def inflate(f: Frame) -> np.ndarray:
    """The filtered rows (uint8 [H, 1 + rowbytes]) as zlib under Pillow produces them."""
    raw = f.raw_bytes
    d = zlib.decompressobj()
    try:
        out = d.decompress(f.zdata, raw)
    except zlib.error as e:
        raise Corrupt("bad Adler-32" if "incorrect data check" in str(e) else "bad deflate data") from e
    if len(out) < raw:
        raise Corrupt("truncated")
    return np.frombuffer(out, np.uint8).reshape(f.H, f.rowbytes + 1)


def unfilter(rows: np.ndarray, bpp: int) -> np.ndarray:
    """Reconstructed scanlines (uint8 [H, rowbytes]) from the filtered rows."""
    H, n = rows.shape[0], rows.shape[1] - 1
    out = np.zeros((H, n), np.uint8)
    prev = np.zeros(n, np.int32)
    for r in range(H):
        ft = int(rows[r, 0])
        x = rows[r, 1:].astype(np.int32)
        if ft > 4:
            raise Corrupt("bad filter type")
        if ft == 0:
            cur = x
        elif ft == 2:
            cur = (x + prev) & 255
        elif ft == 1:                                   # per byte lane, a running sum mod 256
            cur = np.zeros(-(-n // bpp) * bpp, np.int32)
            cur[:n] = x
            cur = (np.cumsum(cur.reshape(-1, bpp), axis=0) & 255).reshape(-1)[:n]
        else:
            cur = x.copy()
            for i in range(n):
                a = int(cur[i - bpp]) if i >= bpp else 0
                b = int(prev[i])
                if ft == 3:
                    cur[i] = (cur[i] + ((a + b) >> 1)) & 255
                else:
                    c = int(prev[i - bpp]) if i >= bpp else 0
                    p = a + b - c
                    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                    cur[i] = (cur[i] + (a if pa <= pb and pa <= pc else (b if pb <= pc else c))) & 255
        out[r] = cur
        prev = cur
    return out


def rgb_to_l(rgb: np.ndarray) -> np.ndarray:
    """Pillow's convert("L"): (R * 19595 + G * 38470 + B * 7471 + 0x8000) >> 16."""
    v = rgb.astype(np.int64)
    return ((v[..., 0] * 19595 + v[..., 1] * 38470 + v[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def _samples(lines: np.ndarray, W: int, spp: int, depth: int) -> np.ndarray:
    """[H, W, spp] sample values (16-bit big-endian, or the packed 1 / 2 / 4-bit values MSB first)."""
    H = lines.shape[0]
    if depth == 16:
        v = lines[:, :2 * W * spp].astype(np.int32)
        return ((v[:, 0::2] << 8) | v[:, 1::2]).reshape(H, W, spp)
    if depth == 8:
        return lines[:, :W * spp].astype(np.int32).reshape(H, W, spp)
    bits = np.unpackbits(lines, axis=1)[:, :W * depth].reshape(H, W, depth).astype(np.int32)
    return (bits * (1 << np.arange(depth - 1, -1, -1))).sum(axis=2)[..., None]


def convert(f: Frame, lines: np.ndarray, mode: str) -> np.ndarray:
    """Pillow's unpacking of the reconstructed scanlines and its convert(mode) for mode "RGB" or "L"."""
    s = _samples(lines, f.W, SAMPLES[f.color_type], f.depth)
    ct, d = f.color_type, f.depth
    if ct in (0, 4):
        g = s[..., 0]
        if d == 16:
            g = np.minimum(g, 255) if ct == 0 else g >> 8        # "I;16" clips; grey + alpha 16 opens as RGBA
        elif d < 8:
            g = g * {1: 255, 2: 85, 4: 17}[d]
        g = g.astype(np.uint8)
        return np.repeat(g[..., None], 3, axis=2) if mode == "RGB" else g
    if ct == 3:
        pal = np.zeros((256, 3), np.uint8)
        pal[:len(f.palette)] = f.palette
        rgb = pal[s[..., 0]]
        return rgb if mode == "RGB" else rgb_to_l(pal)[s[..., 0]]
    rgb = s[..., :3]
    rgb = (rgb >> 8 if d == 16 else rgb).astype(np.uint8)
    return rgb if mode == "RGB" else rgb_to_l(rgb)


def decode(data, mode: str = "RGB") -> np.ndarray:
    """np.asarray(Image.open(f).convert(mode)); raises Corrupt where Pillow raises on the image data, and the host
    parser's CLError for refused or corrupt files."""
    f = parse(data)
    return convert(f, unfilter(inflate(f), f.bpp), mode)


# ------------------------------------------------------------------------------------------------ block walker
_LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
_LEXT = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
_DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
_CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class _Bits:
    def __init__(self, data: bytes, pos: int):
        self.data = bytes(data) + bytes(8)
        self.pos = pos

    def peek(self, n: int) -> int:
        i = self.pos >> 3
        return (int.from_bytes(self.data[i:i + 4], "little") >> (self.pos & 7)) & ((1 << n) - 1)

    def get(self, n: int) -> int:
        r = self.peek(n)
        self.pos += n
        return r


def _codes(lengths):
    """{(length, reversed code): symbol} of a canonical code."""
    count = [0] * 16
    for l in lengths:
        count[l] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    out = {}
    for s, l in enumerate(lengths):
        if l:
            c = nxt[l]
            nxt[l] += 1
            out[(l, int(format(c, f"0{l}b")[::-1], 2))] = s
    return out


def _sym(r: _Bits, table) -> int:
    v = r.peek(15)
    for l in range(1, 16):
        s = table.get((l, v & ((1 << l) - 1)))
        if s is not None:
            r.pos += l
            return s
    raise Corrupt("bad deflate data")


_FIXED = (_codes([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8), _codes([5] * 30))


def block_table(zdata: bytes) -> list:
    """(start bit in the zlib stream, BTYPE, BFINAL, inflated bytes) of every deflate block, in order, to the final
    block.  Pure Python: for the tests' and the bench's block counts, not for speed."""
    r = _Bits(zdata, 16)
    out = []
    while True:
        start = r.pos
        final, bt = r.get(1), r.get(2)
        n = 0
        if bt == 0:
            r.pos = (r.pos + 7) & ~7
            ln = r.get(16)
            r.get(16)
            r.pos += 8 * ln
            n = ln
        elif bt == 3:
            raise Corrupt("bad deflate data")
        else:
            if bt == 1:
                lit, dist = _FIXED
            else:
                nlen, ndist, ncode = r.get(5) + 257, r.get(5) + 1, r.get(4) + 4
                cl = [0] * 19
                for k in range(ncode):
                    cl[_CL_ORDER[k]] = r.get(3)
                clt, lens = _codes(cl), []
                while len(lens) < nlen + ndist:
                    s = _sym(r, clt)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + r.get(2))
                    elif s == 17:
                        lens += [0] * (3 + r.get(3))
                    else:
                        lens += [0] * (11 + r.get(7))
                lit, dist = _codes(lens[:nlen]), _codes(lens[nlen:])
            while True:
                s = _sym(r, lit)
                if s < 256:
                    n += 1
                elif s == 256:
                    break
                else:
                    n += _LBASE[s - 257] + r.get(_LEXT[s - 257])
                    r.get(_DEXT[_sym(r, dist)])
        out.append((start, bt, final, n))
        if final:
            return out
