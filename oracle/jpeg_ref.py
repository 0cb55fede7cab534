"""numpy restatement of baseline JPEG decoding as Pillow runs it (libjpeg-turbo, default settings; tests only).
Pinned by tests/test_jpeg.py to Pillow itself (Pillow 12.2, libjpeg-turbo with the libjpeg 6.2 API).

    marker parsing     controllora_b200/jpeg.py parse(): the host side of the product, shared with this module so that
                       comparing the decode with Pillow pins the parser, the refusals and the segment split as well
    Huffman decoding   sequential, one code + extra bits per symbol (jdhuff.c); an invalid code, a coefficient written
                       past index 63 or a segment that ends before its last block is corrupt (Corrupt)
    DC prediction      per component, reset at every restart segment, summed in int and stored as a 16-bit coefficient
    IDCT               jpeg_idct_islow as libjpeg-turbo's x86-64 SIMD code runs it (jidctint-sse2 / -avx2, what Pillow
                       calls): 13-bit constants, 2 extra bits after the column pass, 16-bit lanes (see idct_islow)
    upsampling         fancy (triangle) h2v1 / h2v2 at the component's own width and height (jdsample.c), replication
                       when the subsampled width is at most 2 (libjpeg-turbo picks the plain upsampler there)
    colour             jdcolor.c ycc_rgb_convert: 16-bit fixed-point tables

Out of range, the SIMD IDCT is not libjpeg's C code: the C code wraps the result to 10 bits before clamping, the SIMD
code saturates, and it dequantises and adds in 16-bit lanes.  A stream whose dequantised coefficients push a block far
outside 0..255 (a large DC table entry, say) decodes differently under the two; this module and the device decoder follow
the SIMD code, which is what np.asarray(Image.open(f)) returns.
"""
from __future__ import annotations

import numpy as np

from controllora_b200.jpeg import ZIGZAG, Frame, huffman_codes, parse


class Corrupt(ValueError):
    """Corrupt entropy-coded data (libjpeg-turbo would warn and return a degraded image, or Pillow raises)."""


# ------------------------------------------------------------------------------------------------------ Huffman
def lut16(counts, vals) -> np.ndarray:
    """int32 [65536]: (length << 8) | symbol keyed by the next 16 bits; -1 where no code matches (an invalid code)."""
    lut = np.full(1 << 16, -1, np.int32)
    lengths, codes = huffman_codes(counts, vals)
    for length, code, sym in zip(lengths, codes, vals):
        lo = int(code) << (16 - length)
        lut[lo:lo + (1 << (16 - length))] = (int(length) << 8) | int(sym)
    return lut


def _extend(v: int, s: int) -> int:
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def decode_segment(data: np.ndarray, nblocks: int, comp_of_block, dc_luts, ac_luts):
    """Decode `nblocks` blocks (MCU order) of one restart segment: int32 [nblocks, 64] natural-order coefficients with the
    DC *difference* in [:, 0].  Raises Corrupt on an invalid code, an index past 63 or data that ends early."""
    nbits = 8 * len(data)
    pad = np.concatenate([data, np.zeros(8, np.uint8)]).astype(np.int64)
    win = ((pad[:-4] << 24) | (pad[1:-3] << 16) | (pad[2:-2] << 8) | pad[3:-1]).tolist()   # 32 bits from each byte

    def peek(pos: int, n: int) -> int:
        if pos > nbits:                              # past the end: libjpeg inserts zero bits, and the block is cut short
            raise Corrupt(f"the segment ends before its last block (bit {pos} of {nbits})")
        return ((win[pos >> 3] << (pos & 7)) & 0xFFFFFFFF) >> (32 - n)

    out = np.zeros((nblocks, 64), np.int32)
    bpm = len(comp_of_block)
    pos = 0
    zz_nat = ZIGZAG.tolist()
    for blk in range(nblocks):
        c = comp_of_block[blk % bpm]
        e = dc_luts[c][peek(pos, 16)]
        if e < 0:
            raise Corrupt(f"invalid DC code at bit {pos}")
        pos += e >> 8
        s = e & 255
        out[blk, 0] = _extend(peek(pos, s), s) if s else 0
        pos += s
        ac = ac_luts[c]
        k = 1
        while k < 64:
            e = ac[peek(pos, 16)]
            if e < 0:
                raise Corrupt(f"invalid AC code at bit {pos}")
            pos += e >> 8
            r, s = (e & 255) >> 4, e & 15
            if s:
                k += r
                if k > 63:
                    raise Corrupt(f"coefficient index {k} past 63 at bit {pos}")
                out[blk, zz_nat[k]] = _extend(peek(pos, s), s)
                pos += s
                k += 1
            elif r == 15:
                k += 16
            else:
                break
        if pos > nbits:
            raise Corrupt(f"the segment ends before block {blk} of {nblocks}")
    return out


# ---------------------------------------------------------------------------------------------------------- IDCT
def _fix(x: float) -> int:
    return int(x * (1 << 13) + 0.5)


F0_298, F0_390, F0_541, F0_765 = _fix(0.298631336), _fix(0.390180644), _fix(0.541196100), _fix(0.765366865)
F0_899, F1_175, F1_501, F1_847 = _fix(0.899976223), _fix(1.175875602), _fix(1.501321110), _fix(1.847759065)
F1_961, F2_053, F2_562, F3_072 = _fix(1.961570560), _fix(2.053119869), _fix(2.562915447), _fix(3.072711026)


def _w16(v):
    return ((v + 32768) & 0xFFFF) - 32768                                   # a 16-bit lane (paddw, pmullw, psllw)


def _w32(v):
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)                       # a 32-bit lane (paddd, pmaddwd)


def _simd_1d(x, shift: int):
    """One pass of the SIMD ISLOW IDCT over 16-bit inputs: the 16-bit sums wrap (x0 +- x4, x7 + x3, x5 + x1), the
    pair products (pmaddwd) and their sums are 32-bit, and the descaled outputs saturate to 16 bits (packssdw)."""
    x0, x1, x2, x3, x4, x5, x6, x7 = x
    tmp3 = _w32(x2 * (F0_541 + F0_765) + x6 * F0_541)
    tmp2 = _w32(x2 * F0_541 + x6 * (F0_541 - F1_847))
    tmp0 = _w16(x0 + x4) << 13
    tmp1 = _w16(x0 - x4) << 13
    t10, t13, t11, t12 = _w32(tmp0 + tmp3), _w32(tmp0 - tmp3), _w32(tmp1 + tmp2), _w32(tmp1 - tmp2)
    z3, z4 = _w16(x7 + x3), _w16(x5 + x1)
    Z3 = _w32(z3 * (F1_175 - F1_961) + z4 * F1_175)
    Z4 = _w32(z3 * F1_175 + z4 * (F1_175 - F0_390))
    o0 = _w32(_w32(x7 * (F0_298 - F0_899) - x1 * F0_899) + Z3)
    o3 = _w32(_w32(-x7 * F0_899 + x1 * (F1_501 - F0_899)) + Z4)
    o1 = _w32(_w32(x5 * (F2_053 - F2_562) - x3 * F2_562) + Z4)
    o2 = _w32(_w32(-x5 * F2_562 + x3 * (F3_072 - F2_562)) + Z3)
    outs = [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]
    return [np.clip(_w32(_w32(v) + (1 << (shift - 1))) >> shift, -32768, 32767) for v in outs]


def idct_islow(coef: np.ndarray, q: np.ndarray) -> np.ndarray:
    """jpeg_idct_islow as libjpeg-turbo's SIMD code computes it, for int16-valued coefficients [N, 64] (natural order)
    and quantisation table q [64]: uint8 [N, 8, 8].  Dequantisation keeps the low 16 bits of the product (pmullw).  A block
    whose coefficients in rows 1-7 are all zero takes the column pass's shortcut, the DC row shifted left by 2 in 16 bits
    (psllw); any other block takes the full column pass.  The row pass has no shortcut.  The result saturates to
    -128..127 (packsswb) before the +128 level shift."""
    c = coef.astype(np.int64).reshape(-1, 8, 8)
    d = _w16(c * q.astype(np.int64).reshape(8, 8))
    ws = np.stack(_simd_1d([d[:, r, :] for r in range(8)], 11), axis=1)        # column pass, DESCALE by 11
    dc_only = ~np.any(c[:, 1:, :] != 0, axis=(1, 2))
    ws = np.where(dc_only[:, None, None], _w16(d[:, :1, :] << 2), ws)
    v = np.stack(_simd_1d([ws[:, :, k] for k in range(8)], 18), axis=2)       # row pass, DESCALE by 18
    return (np.clip(v, -128, 127) + 128).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ upsample + colour
def upsample(p: np.ndarray, h: int, v: int, H: int, W: int) -> np.ndarray:
    """Component plane p [ch, cw] (uint8, its real size) to [H, W]: h2v1 / h2v2 fancy upsampling (edges replicated)
    when the subsampled width exceeds 2, else plain replication."""
    if (h, v) == (1, 1):
        return p[:H, :W]
    p = p.astype(np.int32)
    ch, cw = p.shape
    if cw <= 2:
        return np.repeat(np.repeat(p, v, axis=0), h, axis=1)[:H, :W].astype(np.uint8)
    if v == 1:
        left = np.concatenate([p[:, :1], p[:, :-1]], axis=1)
        right = np.concatenate([p[:, 1:], p[:, -1:]], axis=1)
        out = np.empty((ch, 2 * cw), np.int32)
        out[:, 0::2] = (3 * p + left + 1) >> 2
        out[:, 1::2] = (3 * p + right + 2) >> 2
        return out[:H, :W].astype(np.uint8)
    up = np.concatenate([p[:1], p[:-1]], axis=0)
    down = np.concatenate([p[1:], p[-1:]], axis=0)
    rows = np.empty((2 * ch, cw), np.int32)
    rows[0::2] = 3 * p + up
    rows[1::2] = 3 * p + down
    left = np.concatenate([rows[:, :1], rows[:, :-1]], axis=1)
    right = np.concatenate([rows[:, 1:], rows[:, -1:]], axis=1)
    out = np.empty((2 * ch, 2 * cw), np.int32)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    return out[:H, :W].astype(np.uint8)


def ycc_tables():
    """jdcolor.c build_ycc_rgb_table: (Cr->R, Cb->B, Cr->G, Cb->G) int32 [256], SCALEBITS = 16."""
    x = np.arange(256, dtype=np.int64) - 128
    fix = lambda f: int(f * 65536 + 0.5)                                    # noqa: E731
    half = 1 << 15
    cr_r = (fix(1.40200) * x + half) >> 16
    cb_b = (fix(1.77200) * x + half) >> 16
    cr_g = -fix(0.71414) * x
    cb_g = -fix(0.34414) * x + half
    return cr_r, cb_b, cr_g, cb_g


def ycc_to_rgb(y: np.ndarray, cb: np.ndarray, cr: np.ndarray) -> np.ndarray:
    cr_r, cb_b, cr_g, cb_g = ycc_tables()
    y = y.astype(np.int64)
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> 16)
    b = y + cb_b[cb]
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------------------ the decode
def coefficients(f: Frame) -> list:
    """int32 [bh, bw, 64] per component: the dequantisation-ready coefficients (DC predicted, 16-bit) on each
    component's block grid, in natural order."""
    samp = f.sampling()
    mx, my = f.mcus if f.C == 3 else (-(-f.W // 8), -(-f.H // 8))
    comp_of_block = [c for c, (h, v) in enumerate(samp) for _ in range(h * v)]
    dc_luts = [lut16(*f.ht[(0, c.td)]).tolist() for c in f.comps]
    ac_luts = [lut16(*f.ht[(1, c.ta)]).tolist() for c in f.comps]
    bpm = len(comp_of_block)
    n_mcu = mx * my
    per = n_mcu if f.ri == 0 else f.ri
    if not f.restart_ok:
        raise Corrupt("restart markers out of sequence")
    blocks = []
    for s, data in enumerate(f.segments):
        nm = min(per, n_mcu - s * per)
        seg = decode_segment(data, nm * bpm, comp_of_block, dc_luts, ac_luts).reshape(nm, bpm, 64)
        off = 0
        for c, (h, v) in enumerate(samp):            # DC prediction, reset per segment, one running sum per component
            dc = seg[:, off:off + h * v, 0].reshape(-1)
            seg[:, off:off + h * v, 0] = np.cumsum(dc).reshape(nm, h * v)
            off += h * v
        blocks.append(seg)
    allb = np.concatenate(blocks).astype(np.int16).astype(np.int32)     # (JCOEF) s
    out, off = [], 0
    for h, v in samp:
        cb = allb[:, off:off + h * v].reshape(my, mx, v, h, 64).transpose(0, 2, 1, 3, 4).reshape(my * v, mx * h, 64)
        out.append(cb)
        off += h * v
    return out


def decode_frame(f: Frame) -> np.ndarray:
    coefs = coefficients(f)
    planes = []
    for c, comp in enumerate(f.comps):
        ch, cw = f.comp_size(c)
        by, bx = -(-ch // 8), -(-cw // 8)
        blk = coefs[c][:by, :bx].reshape(-1, 64)
        px = idct_islow(blk, f.qt[comp.tq]).reshape(by, bx, 8, 8).transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)
        planes.append(px[:ch, :cw])
    if f.C == 1:
        return planes[0]
    hm, vm = f.hmax, f.vmax
    y = planes[0]
    cb = upsample(planes[1], hm, vm, f.H, f.W)
    cr = upsample(planes[2], hm, vm, f.H, f.W)
    return ycc_to_rgb(y, cb, cr)


def decode(data) -> np.ndarray:
    """np.asarray(Image.open(io.BytesIO(data))) for an accepted stream: uint8 [H, W] or [H, W, 3]."""
    return decode_frame(parse(data))
