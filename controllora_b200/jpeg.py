"""Baseline JPEG decoding on the device, bit for bit with Pillow (kernel K12, cl_jpeg_decode), and the DreamBooth image
transform on the resampler (K10).

    decode_jpeg(sources)                     = [np.asarray(Image.open(src)) for src in sources] as uint8 CUDA tensors,
                                               [H, W] (grayscale) or [H, W, 3]; the decode of train_dreambooth_lora.py:
                                               463-478, process/mpii_pose.py:26-27 and process/danbooru_sketch.py:33-34
    dreambooth_crops(sizes, size, center)    = the (top, left) of torchvision's CenterCrop / RandomCrop after Resize(size)
    dreambooth_transform(images, size, ...)  = train_dreambooth_lora.py:449-456: convert("RGB"), Resize(size, BILINEAR),
                                               CenterCrop or RandomCrop, ToTensor, Normalize([0.5], [0.5])

The host parses the marker structure (refusing, before any upload, every stream kind the kernels do not decode), builds
the Huffman lookup tables and the quantisation tables, removes the byte stuffing and splits the entropy-coded data at
its restart markers with vectorised numpy; all of it goes to the device in one pinned upload.  What the decode computes
is restated in numpy in oracle/jpeg_ref.py, which pins it to Pillow's libjpeg-turbo.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Sequence

import numpy as np
import torch

from . import ops
from ._lib import CLError, JpegImage, JpegSegment, require_cuda
from .transforms import PIL_BILINEAR, resample, torchvision_resized_size

MAX_SIDE = 16384              # largest accepted width or height
MAX_SEGMENT_BYTES = 1 << 27   # entropy-coded bytes of one restart segment (bit positions stay below 2^31)
WINDOW_BITS = 1024            # bits of entropy-coded data per decoding window (one GPU thread each)
HUFF_WORDS = 512 + 17 + 17 + 256 + 8   # int32 words of one Huffman table: 9-bit lookup, maxcode, valoff, values, pad
STATUS_OK, STATUS_BAD_CODE, STATUS_BAD_INDEX, STATUS_TRUNCATED, STATUS_BAD_RESTART = 0, 1, 2, 4, 8

# zig-zag index -> natural (row-major) index
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
    62, 63], np.int32)

_SOF_REFUSED = {
    0xC2: "progressive (SOF2)", 0xC3: "lossless (SOF3)", 0xC5: "hierarchical (SOF5)", 0xC6: "hierarchical progressive (SOF6)",
    0xC7: "hierarchical lossless (SOF7)", 0xC9: "arithmetic-coded (SOF9)", 0xCA: "arithmetic-coded progressive (SOF10)",
    0xCB: "arithmetic-coded lossless (SOF11)", 0xCD: "arithmetic-coded hierarchical (SOF13)",
    0xCE: "arithmetic-coded hierarchical progressive (SOF14)", 0xCF: "arithmetic-coded hierarchical lossless (SOF15)",
    0xCC: "arithmetic coding conditioning (DAC)", 0xDE: "hierarchical (DHP)", 0xDF: "hierarchical (EXP)",
}


class JpegRefused(CLError):
    """A stream kind cl_jpeg_decode does not decode (decode it with Pillow)."""


@dataclass
class Component:
    cid: int
    h: int
    v: int
    tq: int
    td: int = 0
    ta: int = 0


@dataclass
class Frame:
    """One parsed baseline stream: geometry, tables and the entropy-coded segments (stuffing removed)."""
    H: int
    W: int
    comps: list
    qt: dict                        # table id -> int32 [64], natural order
    ht: dict                        # (class 0 DC / 1 AC, id) -> (counts [16], values)
    ri: int                         # restart interval in MCUs, 0 = none
    segments: list = field(default_factory=list)   # uint8 arrays, one per restart segment found
    restart_ok: bool = True         # the RST markers come in sequence and their number matches the MCU count

    @property
    def C(self) -> int:
        return len(self.comps)

    @property
    def hmax(self) -> int:
        return max(c.h for c in self.comps) if self.C == 3 else 1

    @property
    def vmax(self) -> int:
        return max(c.v for c in self.comps) if self.C == 3 else 1

    def sampling(self):
        """(h, v) per component as the scan interleaves them: a one-component scan has one block per MCU."""
        return [(1, 1)] if self.C == 1 else [(c.h, c.v) for c in self.comps]

    @property
    def mcus(self) -> tuple[int, int]:
        return -(-self.W // (8 * self.hmax)), -(-self.H // (8 * self.vmax))

    @property
    def blocks_per_mcu(self) -> int:
        return sum(h * v for h, v in self.sampling())

    @property
    def n_segments(self) -> int:
        mx, my = self.mcus
        return 1 if self.ri == 0 else -(-(mx * my) // self.ri)

    def comp_size(self, c: int) -> tuple[int, int]:
        """(height, width) of component c's samples (libjpeg's downsampled_height / width)."""
        h, v = self.sampling()[c]
        return -(-self.H * v // self.vmax), -(-self.W * h // self.hmax)


def _u16(b, i) -> int:
    return (int(b[i]) << 8) | int(b[i + 1])


def _check_huffman(tc: int, counts: np.ndarray, vals: np.ndarray, what: str) -> None:
    """jpeg_make_d_derived_tbl's checks: at most 256 symbols, canonical codes that fit their lengths, DC symbols <= 15."""
    if counts.sum() > 256:
        raise JpegRefused(f"{what}: invalid Huffman table ({int(counts.sum())} symbols)")
    code = 0
    for length in range(1, 17):
        code += int(counts[length - 1])
        if code >= (1 << length):                  # the all-ones code is reserved
            raise JpegRefused(f"{what}: invalid Huffman table (codes of length {length} overflow)")
        code <<= 1
    if tc == 0 and len(vals) and int(vals.max()) > 15:
        raise JpegRefused(f"{what}: invalid Huffman table (DC symbol {int(vals.max())} > 15)")


def _entropy_segments(d: np.ndarray):
    """Split entropy-coded data at its RSTn markers and remove the stuffed zero bytes and fill bytes with vectorised
    numpy: (segments, end offset = the first byte of the marker that ends the scan (or len(d)), restart numbers in
    order)."""
    ff = np.flatnonzero(d[:-1] == 0xFF)
    nxt = d[ff + 1]
    is_marker = (nxt != 0x00) & (nxt != 0xFF)
    is_rst = is_marker & (nxt >= 0xD0) & (nxt <= 0xD7)
    term = ff[is_marker & ~is_rst]
    end = int(term[0]) if len(term) else len(d)
    inside = ff < end
    ff, nxt, is_rst = ff[inside], nxt[inside], is_rst[inside]
    keep = np.ones(end, bool)
    keep[ff[nxt == 0x00] + 1] = False          # the stuffed 0x00 after a data 0xFF
    keep[ff[nxt == 0xFF]] = False              # fill bytes before a marker
    rst = ff[is_rst]
    keep[rst] = False
    keep[rst + 1] = False
    data = d[:end][keep]
    cuts = np.cumsum(keep)[rst] if len(rst) else np.zeros(0, np.int64)   # kept bytes before each marker
    pieces = np.split(data, cuts) if len(cuts) else [data]
    return pieces, end, (nxt[is_rst] - 0xD0).astype(np.int64)


def parse(data, what: str = "jpeg") -> Frame:
    """Parse one JPEG stream.  Raises JpegRefused (a CLError) naming the feature for every kind cl_jpeg_decode does not
    decode and for malformed marker structure; corrupt entropy-coded data is left for the decoder to report."""
    b = np.frombuffer(bytes(data), np.uint8)
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise JpegRefused(f"{what}: not a JPEG stream (no SOI marker)")
    i = 2
    qt, ht, ri = {}, {}, 0
    frame = None
    jfif = False
    adobe = None
    while True:
        if i >= n:
            raise JpegRefused(f"{what}: malformed marker structure (the stream ends before its scan)")
        if b[i] != 0xFF:
            raise JpegRefused(f"{what}: malformed marker structure (byte {i} is not a marker)")
        while i < n and b[i] == 0xFF:
            i += 1
        if i >= n:
            raise JpegRefused(f"{what}: malformed marker structure (the stream ends in fill bytes)")
        m = int(b[i])
        i += 1
        if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise JpegRefused(f"{what}: malformed marker structure (marker 0x{m:02X} before the scan)")
        if i + 2 > n:
            raise JpegRefused(f"{what}: malformed marker structure (segment length past the end)")
        L = _u16(b, i)
        if L < 2 or i + L > n:
            raise JpegRefused(f"{what}: malformed marker structure (segment 0x{m:02X} of length {L} at byte {i})")
        seg = b[i + 2:i + L]
        i += L
        if m in _SOF_REFUSED:
            raise JpegRefused(f"{what}: {_SOF_REFUSED[m]} JPEG is not supported; decode it with Pillow")
        if m == 0xDC:
            raise JpegRefused(f"{what}: DNL marker is not supported; decode it with Pillow")
        if 0xE0 <= m <= 0xEF or m == 0xFE:
            if m == 0xE0 and len(seg) >= 5 and bytes(seg[:5]) == b"JFIF\0":
                jfif = True
            if m == 0xEE and len(seg) >= 12 and bytes(seg[:5]) == b"Adobe":
                adobe = int(seg[11])
            continue
        if m == 0xDB:
            j = 0
            while j < len(seg):
                pq, tq = int(seg[j]) >> 4, int(seg[j]) & 15
                size = 64 * (pq + 1)
                if pq > 1 or tq > 3 or j + 1 + size > len(seg):
                    raise JpegRefused(f"{what}: invalid quantisation table (precision {pq}, id {tq})")
                q = seg[j + 1:j + 1 + size]
                vals = (q[0::2].astype(np.int32) << 8 | q[1::2]) if pq else q.astype(np.int32)
                t = np.zeros(64, np.int32)
                t[ZIGZAG] = vals
                qt[tq] = t
                j += 1 + size
            continue
        if m == 0xC4:
            j = 0
            while j < len(seg):
                if j + 17 > len(seg):
                    raise JpegRefused(f"{what}: invalid Huffman table (short DHT segment)")
                tc, th = int(seg[j]) >> 4, int(seg[j]) & 15
                counts = seg[j + 1:j + 17].astype(np.int32)
                cnt = int(counts.sum())
                if tc > 1 or th > 3 or j + 17 + cnt > len(seg):
                    raise JpegRefused(f"{what}: invalid Huffman table (class {tc}, id {th}, {cnt} symbols)")
                vals = seg[j + 17:j + 17 + cnt].astype(np.int32)
                ht[(tc, th)] = (counts, vals)
                j += 17 + cnt
            continue
        if m == 0xDD:
            if len(seg) != 2:
                raise JpegRefused(f"{what}: malformed marker structure (DRI of length {L})")
            ri = _u16(seg, 0)
            continue
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise JpegRefused(f"{what}: malformed marker structure (two frame headers)")
            if len(seg) < 6:
                raise JpegRefused(f"{what}: malformed marker structure (short SOF)")
            P, H, W, Nf = int(seg[0]), _u16(seg, 1), _u16(seg, 3), int(seg[5])
            if P != 8:
                raise JpegRefused(f"{what}: {P}-bit samples are not supported; decode it with Pillow")
            if H == 0:
                raise JpegRefused(f"{what}: DNL (height defined after the scan) is not supported; decode it with Pillow")
            if len(seg) != 6 + 3 * Nf or Nf == 0:
                raise JpegRefused(f"{what}: malformed marker structure (SOF with {Nf} components)")
            if Nf not in (1, 3):
                kind = "CMYK / YCCK" if Nf == 4 else f"{Nf}-component"
                raise JpegRefused(f"{what}: {kind} JPEG is not supported; decode it with Pillow")
            if W == 0 or W > MAX_SIDE or H > MAX_SIDE:
                raise JpegRefused(f"{what}: size {W} x {H} outside 1..{MAX_SIDE}; decode it with Pillow")
            comps = []
            for k in range(Nf):
                cid, hv, tq = int(seg[6 + 3 * k]), int(seg[7 + 3 * k]), int(seg[8 + 3 * k])
                comps.append(Component(cid, hv >> 4, hv & 15, tq))
                if not (1 <= hv >> 4 <= 4 and 1 <= hv & 15 <= 4) or tq > 3:
                    raise JpegRefused(f"{what}: malformed marker structure (component {cid}: sampling 0x{hv:02X}, table {tq})")
            if Nf == 3:
                if jfif:
                    pass
                elif adobe is not None:
                    if adobe == 0:
                        raise JpegRefused(f"{what}: Adobe RGB JPEG (transform 0) is not supported; decode it with Pillow")
                elif [c.cid for c in comps] == [82, 71, 66]:
                    raise JpegRefused(f"{what}: Adobe RGB JPEG (component ids R, G, B) is not supported; decode it with Pillow")
                y, cb, cr = comps
                if (y.h, y.v) not in ((1, 1), (2, 1), (2, 2)) or (cb.h, cb.v, cr.h, cr.v) != (1, 1, 1, 1):
                    s = "/".join(f"{c.h}x{c.v}" for c in comps)
                    raise JpegRefused(f"{what}: chroma sampling {s} is not supported (4:4:4, 4:2:2 and 4:2:0 are); "
                                      "decode it with Pillow")
            frame = Frame(H, W, comps, qt, ht, ri)
            continue
        if m == 0xDA:
            if frame is None:
                raise JpegRefused(f"{what}: malformed marker structure (scan before the frame header)")
            Ns = int(seg[0]) if len(seg) else 0
            if len(seg) != 4 + 2 * Ns:
                raise JpegRefused(f"{what}: malformed marker structure (SOS of length {L})")
            if Ns != frame.C:
                raise JpegRefused(f"{what}: more than one scan (a scan of {Ns} of {frame.C} components) is not "
                                  "supported; decode it with Pillow")
            for k, c in enumerate(frame.comps):
                cs, t = int(seg[1 + 2 * k]), int(seg[2 + 2 * k])
                if cs != c.cid:
                    raise JpegRefused(f"{what}: malformed marker structure (scan component {cs}, frame component {c.cid})")
                c.td, c.ta = t >> 4, t & 15
                if c.td > 3 or c.ta > 3:
                    raise JpegRefused(f"{what}: invalid Huffman table (scan selects table {c.td} / {c.ta})")
            Ss, Se, A = (int(v) for v in seg[1 + 2 * Ns:4 + 2 * Ns])
            if (Ss, Se, A) != (0, 63, 0):
                raise JpegRefused(f"{what}: spectral selection {Ss}..{Se} / approximation 0x{A:02X} is not sequential; "
                                  "decode it with Pillow")
            for c in frame.comps:
                if c.tq not in qt:
                    raise JpegRefused(f"{what}: quantisation table {c.tq} is missing")
                if (0, c.td) not in ht or (1, c.ta) not in ht:
                    raise JpegRefused(f"{what}: Huffman table {c.td} (DC) / {c.ta} (AC) is missing")
                if int(ht[(0, c.td)][0].sum()) == 0 or int(ht[(1, c.ta)][0].sum()) == 0:
                    raise JpegRefused(f"{what}: invalid Huffman table (empty)")
                for tc, th in ((0, c.td), (1, c.ta)):       # as libjpeg, only the tables the scan uses are checked
                    _check_huffman(tc, *ht[(tc, th)], what)
            frame.qt = {k: v.copy() for k, v in qt.items()}
            frame.ht = dict(ht)
            frame.ri = ri
            pieces, end, numbers = _entropy_segments(b[i:])
            i += end
            _check_after_scan(b, i, what)
            want = frame.n_segments
            frame.restart_ok = (len(pieces) <= want and
                                bool(np.all(numbers == np.arange(len(numbers)) % 8)))
            if len(pieces) < want:          # missing data: the decoder finds those segments empty (truncated)
                pieces = pieces + [np.zeros(0, np.uint8)] * (want - len(pieces))
            frame.segments = pieces[:want]
            for p in frame.segments:
                if len(p) >= MAX_SEGMENT_BYTES:
                    raise JpegRefused(f"{what}: a restart segment of {len(p)} bytes (limit {MAX_SEGMENT_BYTES - 1})")
            return frame
        raise JpegRefused(f"{what}: malformed marker structure (unknown marker 0x{m:02X})")


def _check_after_scan(b: np.ndarray, i: int, what: str) -> None:
    """Markers after the scan: EOI ends the image; another scan or a DNL is refused; a stream cut short is the decoder's
    to report (truncated)."""
    n = len(b)
    while i + 1 < n:
        while i < n and b[i] == 0xFF:
            i += 1
        if i >= n:
            return
        m = int(b[i])
        i += 1
        if m == 0xD9:
            return
        if m == 0xDA:
            raise JpegRefused(f"{what}: more than one scan is not supported; decode it with Pillow")
        if m == 0xDC:
            raise JpegRefused(f"{what}: DNL marker is not supported; decode it with Pillow")
        if m in _SOF_REFUSED or m in (0xC0, 0xC1, 0xD8):
            raise JpegRefused(f"{what}: malformed marker structure (marker 0x{m:02X} after the scan)")
        if i + 2 > n:
            return
        i += _u16(b, i)


# ------------------------------------------------------------------------------------------------------ tables
def huffman_codes(counts: np.ndarray, vals: np.ndarray):
    """Canonical codes (JPEG Annex C): (lengths, codes) in symbol order of `vals`."""
    lengths = np.repeat(np.arange(1, 17), counts)
    codes = np.zeros(len(vals), np.int64)
    code, k = 0, 0
    for length in range(1, 17):
        for _ in range(int(counts[length - 1])):
            codes[k] = code
            code += 1
            k += 1
        code <<= 1
    return lengths, codes


def huffman_table(counts: np.ndarray, vals: np.ndarray) -> np.ndarray:
    """The device form of one table, int32 [HUFF_WORDS]: lut[512] = (length << 8) | symbol for codes of at most 9 bits
    keyed by the next 9 bits (0: longer code or none), maxcode[17] (-1: no code of that length), valoff[17] (index in
    values = code + valoff[length]), values[256]."""
    out = np.zeros(HUFF_WORDS, np.int32)
    lengths, codes = huffman_codes(counts, vals)
    lut = out[:512]
    for length, code, sym in zip(lengths, codes, vals):
        if length <= 9:
            lo = int(code) << (9 - length)
            lut[lo:lo + (1 << (9 - length))] = (int(length) << 8) | int(sym)
    maxcode = out[512:529]
    valoff = out[529:546]
    maxcode[:] = -1
    k = 0
    for length in range(1, 17):
        c = int(counts[length - 1])
        if c:
            valoff[length] = k - int(codes[k])
            maxcode[length] = int(codes[k + c - 1])
            k += c
    out[546:546 + len(vals)] = vals
    return out


# ------------------------------------------------------------------------------------------------------- packing
_SEGMENT_DTYPE = np.dtype([(name, np.int64 if ctype == C.c_int64 else np.int32) for name, ctype in JpegSegment._fields_])
assert _SEGMENT_DTYPE.itemsize == C.sizeof(JpegSegment)

@dataclass
class Packed:
    images: object                   # ctypes array of JpegImage
    segments: object                 # ctypes array of JpegSegment
    host: np.ndarray                 # uint8: images, segments, int32 tables, entropy-coded bytes
    tables_off: int
    tables_len: int                  # int32 words
    n_windows: int
    data_off: int
    data_len: int
    coef_blocks: int                 # coefficient blocks of the batch (64 int16 each)
    plane_bytes: int
    out_bytes: int
    shapes: list


def pack(frames: Sequence[Frame]) -> Packed:
    """Host side of one cl_jpeg_decode call for parsed frames."""
    B = len(frames)
    imgs = (JpegImage * B)()
    segs_desc, tables, data = [], [], []
    n_windows = n_segs = 0
    tab_len = data_len = coef = plane = out = 0
    shapes = []

    def table(arr):
        nonlocal tab_len
        tables.append(arr)
        tab_len += len(arr)
        return tab_len - len(arr)

    for bi, f in enumerate(frames):
        d = imgs[bi]
        mx, my = f.mcus
        d.H, d.W, d.C = f.H, f.W, f.C
        d.hmax, d.vmax = f.hmax, f.vmax
        d.mcux, d.mcuy = (mx, my) if f.C == 3 else (-(-f.W // 8), -(-f.H // 8))
        d.bpm = f.blocks_per_mcu
        d.ri = f.ri
        d.status0 = 0 if f.restart_ok else STATUS_BAD_RESTART
        d.out_off, d.coef_off, d.plane_off = out, coef, plane
        qcache, hcache = {}, {}
        for c, comp in enumerate(f.comps):
            if comp.tq not in qcache:
                qcache[comp.tq] = table(f.qt[comp.tq])
            for key in ((0, comp.td), (1, comp.ta)):
                if key not in hcache:
                    hcache[key] = table(huffman_table(*f.ht[key]))
            d.qt[c] = qcache[comp.tq]
            d.dc_tab[c], d.ac_tab[c] = hcache[(0, comp.td)], hcache[(1, comp.ta)]
            ch, cw = f.comp_size(c)
            d.ch[c], d.cw[c] = ch, cw
            d.pitch[c] = -(-cw // 8) * 8
            d.comp_plane[c] = plane - d.plane_off
            plane += d.pitch[c] * (-(-ch // 8) * 8)
        d.seg0, d.nseg = n_segs, len(f.segments)
        n_mcu = d.mcux * d.mcuy
        per = n_mcu if f.ri == 0 else f.ri
        sd = np.zeros(len(f.segments), _SEGMENT_DTYPE)          # the image's segment descriptors, built column-wise
        nbytes = np.fromiter((len(x) for x in f.segments), np.int64, len(f.segments))
        nwin = np.maximum(1, -(-8 * nbytes // WINDOW_BITS))
        sd["data_off"] = data_len + np.cumsum(nbytes) - nbytes
        sd["nbytes"], sd["image"] = nbytes, bi
        sd["mcu0"] = np.arange(len(f.segments), dtype=np.int64) * per
        sd["nmcu"] = np.minimum(per, n_mcu - sd["mcu0"])
        sd["block0"] = coef + sd["mcu0"].astype(np.int64) * d.bpm
        sd["win0"] = n_windows + np.cumsum(nwin) - nwin
        sd["nwin"] = nwin
        segs_desc.append(sd)
        data += f.segments
        n_segs += len(f.segments)
        data_len += int(nbytes.sum())
        n_windows += int(nwin.sum())
        d.nblocks = n_mcu * d.bpm
        coef += d.nblocks
        out += f.H * f.W * f.C
        shapes.append((f.H, f.W) if f.C == 1 else (f.H, f.W, 3))
    segs = (JpegSegment * n_segs).from_buffer_copy(np.concatenate(segs_desc).tobytes())
    parts = [np.frombuffer(bytes(imgs), np.uint8), np.frombuffer(bytes(segs), np.uint8)]
    tables_off = sum(len(p) for p in parts)
    tab = np.concatenate(tables).astype(np.int32)
    parts.append(tab.view(np.uint8))
    data_off = tables_off + tab.nbytes
    parts += data
    parts.append(np.zeros(8, np.uint8))            # a batch of empty segments still has a data pointer
    host = np.concatenate(parts)
    return Packed(imgs, segs, host, tables_off, len(tab), n_windows, data_off, data_len, coef, plane, out, shapes)


# ------------------------------------------------------------------------------------------------------- public API
def _read_source(src, i: int, what: str = "decode_jpeg") -> bytes:
    if isinstance(src, dict) and "bytes" in src:           # a datasets Image column loaded with decode=False
        src = src["bytes"] if src["bytes"] is not None else src.get("path")
    if isinstance(src, (bytes, bytearray)):
        return bytes(src)
    if isinstance(src, memoryview):
        return src.tobytes()
    if isinstance(src, (str, os.PathLike)):
        with open(src, "rb") as fh:
            return fh.read()
    raise CLError(f"{what}: source {i} is a {type(src).__name__}, expected bytes, bytearray, memoryview or a path")


def _name(src, i: int) -> str:
    if isinstance(src, (str, os.PathLike)):
        return f"image {i} ({os.fspath(src)})"
    return f"image {i}"


def decode_jpeg(sources: Sequence, device=None) -> list:
    """Decode baseline JPEG streams on the device: one uint8 CUDA tensor per source, [H, W] for grayscale and [H, W, 3]
    for colour, equal to np.asarray(Image.open(src)) (Pillow's libjpeg-turbo, default settings).  Sources are bytes,
    bytearray, memoryview, paths, or {"bytes": ...} dicts.  Kinds the kernels do not decode (progressive, arithmetic,
    lossless, 12-bit, multi-scan, CMYK / YCCK / Adobe RGB, 4:4:0 / 4:1:1 sampling, DNL, malformed markers or tables)
    raise CLError naming the feature before anything is uploaded; corrupt entropy-coded data raises CLError naming the
    image after the decode.  One host synchronisation per call."""
    sources = list(sources)
    if not sources:
        return []
    device = torch.device(device if device is not None else "cuda")
    require_cuda(device, "decode_jpeg")
    frames = [parse(_read_source(s, i), f"decode_jpeg: {_name(s, i)}") for i, s in enumerate(sources)]
    p = pack(frames)
    staged = torch.empty(len(p.host), dtype=torch.uint8, pin_memory=True)
    staged.numpy()[:] = p.host
    packed = staged.to(device, non_blocking=True)
    out = torch.empty(max(p.out_bytes, 1), dtype=torch.uint8, device=device)
    status, _ = ops.jpeg_decode(p, packed, out)
    bad = [i for i, s in enumerate(status) if s]
    if bad:
        i, s = bad[0], status[bad[0]]
        kinds = [k for bit, k in ((STATUS_BAD_CODE, "an invalid Huffman code"), (STATUS_BAD_INDEX, "a coefficient index past 63"),
                                  (STATUS_TRUNCATED, "entropy-coded data that ends before its last MCU"),
                                  (STATUS_BAD_RESTART, "restart markers out of sequence")) if s & bit]
        raise CLError(f"decode_jpeg: {_name(sources[i], i)} is corrupt ({', '.join(kinds)})"
                      + (f"; {len(bad) - 1} more corrupt image(s): {bad[1:]}" if len(bad) > 1 else ""))
    res, off = [], 0
    for shape in p.shapes:
        n = math.prod(shape)
        res.append(out[off:off + n].view(shape))
        off += n
    return res


def dreambooth_crops(sizes: Sequence[tuple[int, int]], size: int, center_crop: bool, generator=None) -> list:
    """(top, left) per image of torchvision's CenterCrop(size) / RandomCrop(size) after Resize(size) of an image of
    `sizes[b]` = (h, w): CenterCrop rounds int(round((h - size) / 2.0)); RandomCrop draws nothing when the resized image
    already is size x size, else torch.randint(0, h - size + 1) for the top, then for the left, from `generator` (torch's
    global generator when None)."""
    out = []
    for h, w in sizes:
        rh, rw = torchvision_resized_size(h, w, size)
        if center_crop:
            out.append((int(round((rh - size) / 2.0)), int(round((rw - size) / 2.0))))
        elif rh == size and rw == size:
            out.append((0, 0))
        else:
            top = int(torch.randint(0, rh - size + 1, size=(1,), generator=generator).item())
            left = int(torch.randint(0, rw - size + 1, size=(1,), generator=generator).item())
            out.append((top, left))
    return out


def dreambooth_transform(images: Sequence, size: int, center_crop: bool = False, crops=None, generator=None, device=None):
    """train_dreambooth_lora.py:449-456 for a batch of decoded images (uint8 [H, W] or [H, W, 3], numpy or torch, e.g.
    decode_jpeg's output): convert("RGB") (grey replicated), Resize(size, BILINEAR), CenterCrop(size) or RandomCrop(size)
    at crops[b] = (top, left) (drawn by dreambooth_crops when not given), ToTensor, Normalize([0.5], [0.5]).  Returns fp32
    [B, 3, size, size] on `device` (the current CUDA device by default), bit-identical to the torchvision pipeline."""
    images = list(images)
    if not images:
        raise CLError("dreambooth_transform: no images")
    device = torch.device(device if device is not None else "cuda")
    require_cuda(device, "dreambooth_transform")
    sizes = [tuple(x.shape[:2]) for x in images]
    for x in images:
        if len(x.shape) == 3 and x.shape[2] not in (1, 3):
            raise CLError(f"dreambooth_transform: C = {x.shape[2]}, expected 1 or 3")
    if crops is None:
        crops = dreambooth_crops(sizes, size, center_crop, generator)
    crops = [tuple(int(v) for v in c) for c in crops]
    resized = [torchvision_resized_size(h, w, size) for h, w in sizes]
    out, _ = resample(PIL_BILINEAR, images, resized, crops, size, size, device)
    return out
