"""PNG decoding on the device, bit for bit with Pillow (kernel K13, cl_png_decode), and decoding of mixed PNG / JPEG
sources.

    decode_png(sources, mode="RGB")     = [np.asarray(Image.open(src).convert(mode)) for src in sources] as uint8 CUDA
                                          tensors, [H, W, 3] for "RGB" and [H, W] for "L"; the decode of
                                          train_text_to_image_control_lora.py:615-619 (fill50k images and guides),
                                          process/diffusiondb_canny.py:15-35 and process/danbooru_sketch.py:34
    decode_images(sources, mode="RGB")  = the same for a mix of PNG and JPEG sources, picked by signature: one
                                          decode_png and one decode_jpeg call, JPEGs converted by the same device stage

The host walks the chunks, checks the CRCs Pillow checks and the zlib header, refuses (before any upload) what the
kernels do not decode, and sends descriptors, palettes and the concatenated IDAT data to the device in one pinned upload.
What the decode computes is restated in oracle/png_ref.py, which pins it to Pillow.
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass
from typing import Sequence

import numpy as np
import torch

from . import ops
from ._lib import CLError, PngImage, require_cuda
from .jpeg import _name, _read_source, decode_jpeg

SIGNATURE = b"\x89PNG\r\n\x1a\n"
MAX_SIDE = 16384
MAX_STREAM_BYTES = 1 << 28
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
SAMPLES = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
MODES = {"RGB": 3, "L": 1}
STATUS_OK, STATUS_BAD_DEFLATE, STATUS_TRUNCATED, STATUS_BAD_FILTER, STATUS_BAD_ADLER = 0, 1, 2, 4, 8
STATUS_KINDS = ((STATUS_BAD_DEFLATE, "bad deflate data"), (STATUS_TRUNCATED, "image data that ends before the last row"),
                (STATUS_BAD_FILTER, "a filter type above 4"), (STATUS_BAD_ADLER, "a wrong Adler-32"))


class PngRefused(CLError):
    """A file kind cl_png_decode does not decode (decode it with Pillow)."""


class PngCorrupt(CLError):
    """A file the host finds corrupt before any upload (Pillow raises on it as well)."""


@dataclass
class Frame:
    """One parsed PNG: IHDR, the palette (uint8 [n, 3], colour type 3) and the zlib stream (the IDAT payloads)."""
    H: int
    W: int
    color_type: int
    depth: int
    palette: np.ndarray | None
    zdata: bytes

    @property
    def rowbytes(self) -> int:
        return (self.W * SAMPLES[self.color_type] * self.depth + 7) // 8

    @property
    def bpp(self) -> int:
        return max(1, SAMPLES[self.color_type] * self.depth // 8)

    @property
    def raw_bytes(self) -> int:
        return self.H * (self.rowbytes + 1)


def parse(data, what: str = "png") -> Frame:
    """Parse one PNG file.  Raises PngRefused naming the feature for the kinds cl_png_decode does not decode and for
    malformed chunks, PngCorrupt for a bad CRC where Pillow checks one (the chunks before the first IDAT) and for a bad
    zlib header.  The IDAT payloads of the first run of IDAT chunks are concatenated (later ones are ignored, as Pillow
    ignores them); corrupt compressed data is left for the decoder to report."""
    b = bytes(data)
    n = len(b)
    if b[:8] != SIGNATURE:
        raise PngRefused(f"{what}: not a PNG file (no signature)")
    i, hdr, palette, idat, state = 8, None, None, [], 0      # state: 0 before IDAT, 1 in the IDAT run, 2 after it
    while True:
        if i + 8 > n:
            if state:
                break                                      # Pillow reads the image data without IEND
            raise PngRefused(f"{what}: malformed chunks (the file ends before its image data); decode it with Pillow")
        length = int.from_bytes(b[i:i + 4], "big")
        ctype = b[i + 4:i + 8]
        if length >= 1 << 31 or not ctype.isalpha():
            raise PngRefused(f"{what}: malformed chunks (chunk {ctype!r} of length {length} at byte {i}); decode it with Pillow")
        body = b[i + 8:i + 8 + length]
        if i + 12 + length > n:
            if ctype == b"IDAT" and state < 2:
                idat.append(body)                         # cut short: the decoder reports the missing rows
                break
            if state:
                break
            raise PngRefused(f"{what}: malformed chunks ({ctype.decode()} runs past the end of the file); decode it with Pillow")
        if state == 0 and ctype != b"IDAT":
            crc = int.from_bytes(b[i + 8 + length:i + 12 + length], "big")
            if zlib.crc32(body, zlib.crc32(ctype)) != crc:
                raise PngCorrupt(f"{what} is corrupt (bad CRC in the {ctype.decode()} chunk)")
        if hdr is None and ctype != b"IHDR":
            raise PngRefused(f"{what}: malformed chunks (the first chunk is {ctype.decode()}, not IHDR); decode it with Pillow")
        i += 12 + length
        if ctype == b"IHDR":
            if hdr is not None or length != 13:
                raise PngRefused(f"{what}: malformed chunks (IHDR of length {length}); decode it with Pillow")
            W, H = int.from_bytes(body[0:4], "big"), int.from_bytes(body[4:8], "big")
            depth, ct, comp, filt, interlace = body[8:13]
            if W == 0 or H == 0:
                raise PngRefused(f"{what}: malformed chunks (size {W} x {H}); decode it with Pillow")
            if ct not in DEPTHS or depth not in DEPTHS[ct]:
                raise PngRefused(f"{what}: colour type {ct} with bit depth {depth} is not a PNG format; decode it with Pillow")
            if comp != 0 or filt != 0 or interlace > 1:
                raise PngRefused(f"{what}: malformed chunks (compression {comp}, filter method {filt}, interlace {interlace}); "
                                 "decode it with Pillow")
            if interlace == 1:
                raise PngRefused(f"{what}: Adam7 interlaced PNG is not supported; decode it with Pillow")
            if W > MAX_SIDE or H > MAX_SIDE:
                raise PngRefused(f"{what}: size {W} x {H} outside 1..{MAX_SIDE}; decode it with Pillow")
            hdr = (H, W, ct, depth)
        elif ctype == b"acTL":
            raise PngRefused(f"{what}: APNG (acTL chunk) is not supported; decode it with Pillow")
        elif ctype == b"PLTE":
            if length == 0 or length % 3 or length > 768:
                raise PngRefused(f"{what}: malformed chunks (PLTE of length {length}); decode it with Pillow")
            palette = np.frombuffer(body, np.uint8).reshape(-1, 3)
        elif ctype == b"IDAT":
            if state < 2:
                state = 1
                idat.append(body)
        elif ctype == b"IEND":
            break
        elif state == 1:
            state = 2
    if not idat:
        raise PngRefused(f"{what}: malformed chunks (no IDAT chunk); decode it with Pillow")
    H, W, ct, depth = hdr
    if ct == 3 and palette is None:
        raise PngRefused(f"{what}: palette image without a PLTE chunk; decode it with Pillow")
    z = b"".join(idat)
    if len(z) >= MAX_STREAM_BYTES:
        raise PngRefused(f"{what}: {len(z)} bytes of image data (limit {MAX_STREAM_BYTES - 1}); decode it with Pillow")
    if len(z) < 2:
        raise PngCorrupt(f"{what} is corrupt (image data that ends before the last row)")
    cmf, flg = z[0], z[1]
    if cmf & 15 != 8 or cmf >> 4 > 7 or (cmf * 256 + flg) % 31 or flg & 0x20:
        kind = ("a preset dictionary (FDICT)" if cmf & 15 == 8 and cmf >> 4 <= 7 and (cmf * 256 + flg) % 31 == 0 else
                f"a bad zlib header 0x{cmf:02X} 0x{flg:02X}")
        raise PngCorrupt(f"{what} is corrupt ({kind})")
    frame = Frame(H, W, ct, depth, palette if ct == 3 else None, z)
    if frame.raw_bytes >= 1 << 31:
        raise PngRefused(f"{what}: {frame.raw_bytes} bytes of filtered rows (limit 2^31 - 1); decode it with Pillow")
    return frame


# ------------------------------------------------------------------------------------------------------- packing
@dataclass
class Packed:
    images: object                   # ctypes array of PngImage
    host: np.ndarray                 # uint8: images, palettes, zlib streams
    tables_off: int
    tables_len: int
    data_off: int
    data_len: int
    words: int                       # candidate words of the batch (32 bit offsets each)
    cand_slots: int
    block_slots: int
    raw_bytes: int                   # filtered rows of the batch
    out_bytes: int
    shapes: list


def pack(frames: Sequence[Frame], channels: int) -> Packed:
    """Host side of one cl_png_decode call for parsed frames, output with `channels` = 3 (RGB) or 1 (L)."""
    B = len(frames)
    imgs = (PngImage * B)()
    pals, data = [], []
    data_len = tab = raw = out = words = cands = blks = 0
    shapes = []
    for bi, f in enumerate(frames):
        d = imgs[bi]
        nb = len(f.zdata)
        d.data_off, d.raw_off, d.out_off, d.nbytes = data_len, raw, out, nb
        d.H, d.W, d.color_type, d.depth, d.rowbytes, d.bpp = f.H, f.W, f.color_type, f.depth, f.rowbytes, f.bpp
        d.word0, d.cand0, d.ncand, d.blk0, d.nblk = words, cands, nb // 8 + 16, blks, nb // 2 + 64
        if f.palette is not None:
            p = np.zeros(768, np.uint8)                    # entries past PLTE are black, as Pillow reads them
            p[:f.palette.size] = f.palette.reshape(-1)
            d.pal_off = tab
            pals.append(p)
            tab += 768
        words += (nb + 3) // 4
        cands += d.ncand
        blks += d.nblk
        data.append(np.frombuffer(f.zdata, np.uint8))
        data_len += nb
        raw += f.raw_bytes
        out += f.H * f.W * channels
        shapes.append((f.H, f.W, 3) if channels == 3 else (f.H, f.W))
    head = np.frombuffer(bytes(imgs), np.uint8)
    pals.append(np.zeros(8, np.uint8))                     # a batch without palettes still has a tables pointer
    tables = np.concatenate(pals)
    host = np.concatenate([head, tables] + data + [np.zeros(8, np.uint8)])
    return Packed(imgs, host, len(head), len(tables), len(head) + len(tables), data_len, words, cands, blks, raw, out, shapes)


# ------------------------------------------------------------------------------------------------------- public API
def _channels(mode: str, what: str) -> int:
    if mode not in MODES:
        raise CLError(f"{what}: mode {mode!r}, expected 'RGB' or 'L' (the conversions the training scripts apply)")
    return MODES[mode]


def _upload(host: np.ndarray, device) -> torch.Tensor:
    staged = torch.empty(len(host), dtype=torch.uint8, pin_memory=True)
    staged.numpy()[:] = host
    return staged.to(device, non_blocking=True)


def _views(out: torch.Tensor, shapes) -> list:
    res, off = [], 0
    for shape in shapes:
        n = math.prod(shape)
        res.append(out[off:off + n].view(shape))
        off += n
    return res


def _decode_png(datas: list, names: list, what: str, mode: str, device) -> list:
    channels = _channels(mode, what)
    frames = [parse(d, f"{what}: {name}") for d, name in zip(datas, names)]
    p = pack(frames, channels)
    packed = _upload(p.host, device)
    out = torch.empty(max(p.out_bytes, 1), dtype=torch.uint8, device=device)
    status, _, _ = ops.png_decode(p, packed, out, channels)
    bad = [i for i, s in enumerate(status) if s]
    if bad:
        i, s = bad[0], status[bad[0]]
        kinds = [k for bit, k in STATUS_KINDS if s & bit]
        raise CLError(f"{what}: {names[i]} is corrupt ({', '.join(kinds)})"
                      + (f"; {len(bad) - 1} more corrupt image(s): {[names[k] for k in bad[1:]]}" if len(bad) > 1 else ""))
    return _views(out, p.shapes)


def decode_png(sources: Sequence, mode: str = "RGB", device=None) -> list:
    """Decode PNG files on the device: one uint8 CUDA tensor per source, equal to np.asarray(Image.open(src).convert(mode))
    with mode "RGB" ([H, W, 3]) or "L" ([H, W]).  Sources are bytes, bytearray, memoryview, paths, or {"bytes": ...} dicts.
    Every non-interlaced colour type and bit depth is decoded; Adam7, APNG, malformed chunks and sides above 16384 raise
    CLError naming the feature before anything is uploaded; corrupt image data raises CLError naming the image after the
    decode.  Results are views into one output buffer.  One host synchronisation per call."""
    sources = list(sources)
    if not sources:
        return []
    device = torch.device(device if device is not None else "cuda")
    require_cuda(device, "decode_png")
    datas = [_read_source(s, i, "decode_png") for i, s in enumerate(sources)]
    return _decode_png(datas, [_name(s, i) for i, s in enumerate(sources)], "decode_png", mode, device)


def _convert(images: list, channels: int, device) -> list:
    """cl_png_convert of decode_jpeg's outputs ([H, W] grey or [H, W, 3] RGB views of one buffer) to `channels`."""
    src = torch.empty(0, dtype=torch.uint8, device=device).set_(images[0].untyped_storage())
    B = len(images)
    imgs = (PngImage * B)()
    out = 0
    for k, t in enumerate(images):
        d = imgs[k]
        c = 1 if t.dim() == 2 else 3
        d.H, d.W, d.color_type, d.depth, d.rowbytes, d.bpp = t.shape[0], t.shape[1], 0 if c == 1 else 2, 8, t.shape[1] * c, c
        d.raw_off = t.data_ptr() - src.data_ptr()
        d.out_off = out
        out += t.shape[0] * t.shape[1] * channels
    packed = torch.from_numpy(np.frombuffer(bytes(imgs), np.uint8).copy()).to(device)
    buf = torch.empty(max(out, 1), dtype=torch.uint8, device=device)
    ops.png_convert(imgs, packed, src, buf, channels)
    return _views(buf, [(t.shape[0], t.shape[1], 3) if channels == 3 else tuple(t.shape[:2]) for t in images])


def decode_images(sources: Sequence, mode: str = "RGB", device=None) -> list:
    """Decode a mix of PNG and JPEG files, picked by signature, in source order: equal to
    np.asarray(Image.open(src).convert(mode)) for mode "RGB" or "L".  At most one decode_png and one decode_jpeg call;
    JPEG outputs whose channels differ from the mode go through the PNG path's conversion stage (grey replicated to RGB,
    RGB to L by Pillow's weights).  Any other signature raises CLError; there is no Pillow fallback."""
    sources = list(sources)
    if not sources:
        return []
    channels = _channels(mode, "decode_images")
    device = torch.device(device if device is not None else "cuda")
    require_cuda(device, "decode_images")
    datas = [_read_source(s, i, "decode_images") for i, s in enumerate(sources)]
    png_idx, jpg_idx = [], []
    for i, d in enumerate(datas):
        if d[:8] == SIGNATURE:
            png_idx.append(i)
        elif d[:2] == b"\xff\xd8":
            jpg_idx.append(i)
        else:
            raise CLError(f"decode_images: {_name(sources[i], i)} is neither a PNG nor a JPEG file; decode it with Pillow")
    res = [None] * len(sources)
    if png_idx:
        outs = _decode_png([datas[i] for i in png_idx], [_name(sources[i], i) for i in png_idx], "decode_images", mode, device)
        for i, t in zip(png_idx, outs):
            res[i] = t
    if jpg_idx:
        try:
            outs = decode_jpeg([datas[i] for i in jpg_idx], device)
        except CLError as e:
            raise CLError(f"decode_images: JPEG sources {jpg_idx} (numbered 0.. in the message): {e}") from e
        conv = [k for k, t in enumerate(outs) if (1 if t.dim() == 2 else 3) != channels]
        if conv:
            for k, t in zip(conv, _convert([outs[k] for k in conv], channels, device)):
                outs[k] = t
        for i, t in zip(jpg_idx, outs):
            res[i] = t
    return res
