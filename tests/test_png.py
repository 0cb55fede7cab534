"""PNG decoding (kernel K13, controllora_b200/png.py) and decode_images.

CPU: the numpy oracle (oracle/png_ref.py) equals Pillow's convert("RGB") / convert("L") bit for bit on seeded files of
every colour type and bit depth, every filter type, Pillow / zlib / cv2 writers, flushes, window sizes and chunk
layouts, and reproduces the goldens; its block walker accounts for every inflated byte; refused kinds raise CLError
naming the feature before anything is uploaded; corrupt files are corrupt exactly where Pillow raises; cl_png_decode
and cl_png_convert validate their arguments without a GPU and the descriptors have the C layout; RGB -> L equals Pillow
over all 2^24 triples; decode_images routes by signature.
GPU: decode_png equals Pillow / the goldens on a ragged batch inside sentinel-filled output and scratch, lists the
oracle's blocks, decodes the worst cases, is repeatable, names corrupt images without touching the rest, and feeds
train_transform, canny_batch and one training step as the reference's host pipeline does."""
import ctypes
import io
import subprocess
import sys
import zlib
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from controllora_b200 import png as P  # noqa: E402
from controllora_b200._lib import CLError  # noqa: E402
from oracle import png_ref  # noqa: E402
from tests.golden import make_png_golden as G  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "png_golden.npz"

try:
    from PIL import Image
except ImportError:                                   # the goldens stand in for Pillow
    Image = None

needs_pil = pytest.mark.skipif(Image is None, reason="needs Pillow")


def pil(b: bytes, mode: str) -> np.ndarray:
    return np.asarray(Image.open(io.BytesIO(b)).convert(mode))


def golden():
    z = np.load(GOLDEN)
    off = z["stream_off"]
    out, p = [], {"RGB": 0, "L": 0}
    for i, name in enumerate(z["names"]):
        want = {}
        for mode, c in (("RGB", 3), ("L", 1)):
            h, w = (int(v) for v in z[f"shapes_{mode}"][i])
            n = h * w * c
            want[mode] = z[f"pixels_{mode}"][p[mode]:p[mode] + n].reshape((h, w, 3) if c == 3 else (h, w))
            p[mode] += n
        out.append((str(name), z["streams"][off[i]:off[i + 1]].tobytes(), want))
    return out


# ------------------------------------------------------------------------------------------------ seeded files
def seeded_files():
    """(id, file) of the CPU sweep."""
    rng = np.random.default_rng(11)
    out = []
    fmts = [(0, 1), (0, 2), (0, 4), (0, 8), (0, 16), (2, 8), (2, 16), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (4, 16),
            (6, 8), (6, 16)]
    sizes = [(1, 1), (1, 13), (17, 1), (5, 7), (9, 33), (31, 30)]
    for k, (ct, d) in enumerate(fmts):
        for j, (h, w) in enumerate(sizes):
            lines = G.scanlines(rng, h, w, ct, d, "noise" if (j + k) % 2 else "smooth")
            pal = None
            if ct == 3:
                npal = int(rng.integers(1, (1 << d) + 1)) if j % 2 else (1 << d)       # short palettes included
                pal = rng.integers(0, 256, (npal, 3))
            trns = None
            if j % 3 == 1:
                trns = {0: b"\0\1", 2: b"\0\1\0\2\0\3", 3: b"\x10\x80"}.get(ct)
            out.append((f"ct{ct}_d{d}_{h}x{w}", G.build_png(lines, w, ct, d, filters=tuple(rng.integers(0, 5, 7)),
                                                               palette=pal, trns=trns)))
    for ct, d in fmts:                                 # each filter type on every bpp
        for ft in range(5):
            lines = G.scanlines(rng, 6, 11, ct, d, "smooth")
            pal = rng.integers(0, 256, (1 << d, 3)) if ct == 3 else None
            out.append((f"filter{ft}_ct{ct}_d{d}", G.build_png(lines, 11, ct, d, filters=(ft,), palette=pal)))
    a = G.scanlines(rng, 40, 50, 2, 8, "smooth")
    for name, kw in (("default", {}), ("filtered", dict(strategy=zlib.Z_FILTERED)),
                     ("huffman", dict(strategy=zlib.Z_HUFFMAN_ONLY)), ("rle", dict(strategy=zlib.Z_RLE)),
                     ("fixed", dict(strategy=zlib.Z_FIXED)), ("level0", dict(level=0)), ("level1", dict(level=1)),
                     ("level9", dict(level=9)), ("memlevel1", dict(mem_level=1)),
                     ("sync_flush", dict(flushes=((1000, zlib.Z_SYNC_FLUSH), (3000, zlib.Z_FULL_FLUSH))))):
        out.append((f"zlib_{name}", G.build_png(a, 50, 2, 8, filters=(1, 2, 3, 4), **kw)))
    for wbits in range(9, 16):
        out.append((f"zlib_wbits{wbits}", G.build_png(a, 50, 2, 8, filters=(4,), wbits=wbits)))
    big = G.scanlines(rng, 100, 700, 2, 8, "noise")                      # stored blocks of 65 535 bytes
    out.append(("stored_65535", G.build_png(big, 700, 2, 8, level=0)))
    out.append(("empty_stored", G.build_png(a, 50, 2, 8, flushes=((0, zlib.Z_SYNC_FLUSH), (6000, zlib.Z_SYNC_FLUSH)))))
    out.append(("idat_1byte", G.build_png(a[:6], 50, 2, 8, filters=(4,), idat_split=1)))
    z = G.compress(G.filter_rows(a, 3, (2,)))
    out.append(("idat_thirds", G.build_png(a, 50, 2, 8, zdata=z, idat_split=len(z) // 3 + 1)))
    parts = [z[:1], z[1:]]                                              # split inside the 2-byte zlib header
    head = b"\x89PNG\r\n\x1a\n" + G.ihdr(50, 40, 8, 2)
    out.append(("idat_split_in_header", head + b"".join(G.chunk(b"IDAT", p) for p in parts) + G.chunk(b"IEND", b"")))
    anc = ((b"tEXt", b"Comment\0seeded"), (b"gAMA", b"\0\0\xb1\x8f"))
    out.append(("ancillary", G.build_png(a, 50, 2, 8, before=anc, after=((b"tEXt", b"After\0idat"),))))
    out.append(("wide_2049", G.build_png(G.scanlines(rng, 3, 2049, 2, 8, "smooth"), 2049, 2, 8, filters=(1, 3, 4))))
    far = rng.integers(0, 256, (2, 16383), dtype=np.uint8)         # rows 2-3 repeat rows 0-1: distance 32 768, length 258
    out.append(("distance_32768", G.build_png(np.concatenate([far, far]), 16383, 0, 8, level=9)))
    for lvl in range(10):
        out.append((f"pil_level{lvl}", G.photo_png(rng, 37, 45, compress_level=lvl)))
    out.append(("pil_optimize", G.photo_png(rng, 37, 45, optimize=True)))
    import cv2

    from tests.golden.make_jpeg_golden import photo
    for k, img in enumerate((photo(rng, 33, 47), photo(rng, 20, 30, C=1))):
        ok, enc = cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, 3 + 3 * k])
        out.append((f"cv2_{k}", enc.tobytes()))
    return out


@needs_pil
def test_oracle_equals_pillow_on_seeded_files():
    bad = []
    files = seeded_files()
    for name, b in files:
        for mode in ("RGB", "L"):
            if not np.array_equal(png_ref.decode(b, mode), pil(b, mode)):
                bad.append((name, mode))
    assert len(files) > 150 and not bad, bad


@needs_pil
def test_seeded_files_cover_what_they_claim():
    files = dict(seeded_files())
    assert Image.open(io.BytesIO(files["stored_65535"])).size == (700, 100)
    assert any(t[1] == 0 and t[3] == 65535 for t in png_ref.block_table(P.parse(files["stored_65535"]).zdata))
    assert any(t[1] == 0 and t[3] == 0 for t in png_ref.block_table(P.parse(files["empty_stored"]).zdata))
    assert {t[1] for t in png_ref.block_table(P.parse(files["zlib_fixed"]).zdata)} == {1}


def test_oracle_reproduces_the_goldens_and_the_walker_sums_to_the_rows():
    for name, b, want in golden():
        for mode in ("RGB", "L"):
            assert np.array_equal(png_ref.decode(b, mode), want[mode]), (name, mode)
        f = P.parse(b)
        assert sum(t[3] for t in png_ref.block_table(f.zdata)) == f.raw_bytes, name


def test_golden_generator_rebuilds_the_files():
    z = np.load(GOLDEN)
    assert [G.sha(b) for _, b in G.golden_cases()] == list(z["stream_sha256"])


def test_block_walker_sums_to_the_inflated_size():
    for name, b in seeded_files()[::7]:
        f = P.parse(b)
        t = png_ref.block_table(f.zdata)
        assert sum(x[3] for x in t) == len(zlib.decompress(f.zdata)) and t[-1][2] == 1, name


# ------------------------------------------------------------------------------------------------ refused / corrupt
def _base(**kw) -> bytes:
    return G.build_png(G.scanlines(np.random.default_rng(5), 6, 8, 2, 8), 8, 2, 8, **kw)


def _refused():
    ok = _base()
    lines = G.scanlines(np.random.default_rng(5), 6, 8, 2, 8)
    z = G.compress(G.filter_rows(lines, 3, (0,)))
    head = b"\x89PNG\r\n\x1a\n"
    return [
        ("adam7", head + G.chunk(b"IHDR", bytes.fromhex("000000080000000608020000") + b"\x01") + G.chunk(b"IDAT", z)
         + G.chunk(b"IEND", b""), "Adam7"),
        ("apng", _base(before=((b"acTL", b"\0\0\0\1\0\0\0\0"),)), "APNG"),
        ("bad_format", head + G.ihdr(8, 6, 4, 2) + G.chunk(b"IDAT", z) + G.chunk(b"IEND", b""), "colour type 2 with bit depth 4"),
        ("no_plte", head + G.ihdr(8, 6, 8, 3) + G.chunk(b"IDAT", z) + G.chunk(b"IEND", b""), "PLTE"),
        ("too_wide", head + G.ihdr(16385, 1, 8, 0) + G.chunk(b"IDAT", z) + G.chunk(b"IEND", b""), "16384"),
        ("not_ihdr_first", head + G.chunk(b"IDAT", z) + G.chunk(b"IEND", b""), "malformed chunks"),
        ("no_idat", head + G.ihdr(8, 6, 8, 2) + G.chunk(b"IEND", b""), "malformed chunks"),
        ("cut_before_idat", ok[:40], "malformed chunks"),
        ("plte_len", head + G.ihdr(8, 6, 8, 3) + G.chunk(b"PLTE", b"\0" * 4) + G.chunk(b"IDAT", z), "malformed chunks"),
        ("not_png", b"GIF89a" + ok[6:], "not a PNG"),
    ]


@pytest.mark.parametrize("name,stream,feature", _refused(), ids=[c[0] for c in _refused()])
def test_refused_kinds_raise_before_upload(name, stream, feature):
    with pytest.raises(CLError, match=feature):
        P.parse(stream)


def test_refused_message_points_to_pillow():
    with pytest.raises(CLError, match="decode it with Pillow"):
        P.parse(_refused()[0][1])


def _with_idat(b: bytes, z: bytes) -> bytes:
    i = b.index(b"IDAT") - 4
    n = int.from_bytes(b[i:i + 4], "big")
    return b[:i] + G.chunk(b"IDAT", z) + b[i + 12 + n:]


def corrupt_files():
    """(id, file, accepted by Pillow): the corrupt kinds, and the near-corrupt files Pillow decodes."""
    rng = np.random.default_rng(9)
    lines = G.scanlines(rng, 6, 8, 2, 8, "smooth")
    raw = G.filter_rows(lines, 3, (1,))
    ok = G.build_png(lines, 8, 2, 8, filters=(1,))
    z = G.compress(raw)
    i = ok.index(b"IHDR")
    bad_ihdr = ok[:i + 17] + bytes([ok[i + 17] ^ 1]) + ok[i + 18:]
    j = ok.index(b"IDAT")
    bad_idat_crc = ok[:j + 4 + len(z)] + bytes([ok[j + 4 + len(z)] ^ 1]) + ok[j + 5 + len(z):]
    adler = z[:-4] + bytes([z[-4] ^ 1]) + z[-3:]
    stored = bytearray(G.compress(raw, level=0))
    stored[5] ^= 1                                     # NLEN of the first stored block
    btype3 = bytes([0x78, 0x9C, 0x07]) + z[3:]         # BFINAL 1, BTYPE 3
    fdict = bytes([0x78, 0xBB]) + z[2:]
    bad_filter = G.compress(bytes([5]) + raw[1:])
    extra = G.compress(raw + b"\x01\x02\x03")
    return [
        ("bad_ihdr_crc", bad_ihdr, False), ("bad_idat_crc", bad_idat_crc, True), ("no_adler", _with_idat(ok, z[:-4]), True),
        ("extra_bytes", _with_idat(ok, extra), True), ("wrong_adler", _with_idat(ok, adler), False),
        ("filter5", _with_idat(ok, bad_filter), False), ("ends_early", _with_idat(ok, G.compress(raw[:-5])), False),
        ("cut_stream", _with_idat(ok, z[:len(z) // 2]), False), ("btype3", _with_idat(ok, btype3), False),
        ("stored_nlen", _with_idat(ok, bytes(stored)), False), ("fdict", _with_idat(ok, fdict), False),
    ]


@needs_pil
@pytest.mark.parametrize("name,stream,accepted", corrupt_files(), ids=[c[0] for c in corrupt_files()])
def test_oracle_is_corrupt_exactly_where_pillow_raises(name, stream, accepted):
    try:
        want = pil(stream, "RGB")
    except (OSError, SyntaxError, ValueError, zlib.error):
        want = None
    assert (want is not None) == accepted, f"Pillow on this machine {'decodes' if want is not None else 'raises on'} {name}"
    if accepted:
        assert np.array_equal(png_ref.decode(stream, "RGB"), want)
    else:
        with pytest.raises((png_ref.Corrupt, CLError)):
            png_ref.decode(stream, "RGB")


# ------------------------------------------------------------------------------------------------ conversions
def test_rgb_to_l_equals_pillow_on_every_triple():
    v = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)
    if Image is not None:
        assert np.array_equal(png_ref.rgb_to_l(rgb), np.asarray(Image.fromarray(rgb).convert("L")))
    assert png_ref.rgb_to_l(np.array([[10, 20, 30], [40, 50, 60]], np.uint8)).tolist() == [18, 48]


def test_decode_images_routes_by_signature_before_any_upload(monkeypatch):
    monkeypatch.setenv("CLB_DRYRUN", "1")              # past the CUDA check: the routing raises before any device work
    with pytest.raises(CLError, match="neither a PNG nor a JPEG"):
        P.decode_images([_base(), b"GIF89a...."], device="cpu")
    with pytest.raises(CLError, match="mode"):
        P.decode_images([_base()], mode="RGBA", device="cpu")


# ------------------------------------------------------------------------------------------------ C ABI
def test_descriptor_layout_matches_c(built_lib, tmp_path):
    from controllora_b200 import _lib

    src = tmp_path / "sz.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "controllora_b200.h"\n'
        'int main(){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(cl_png_image), sizeof(cl_png_block),'
        " offsetof(cl_png_image, nbytes), offsetof(cl_png_image, pal_off), offsetof(cl_png_block, start),"
        " offsetof(cl_png_block, type));return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    I, Bk = _lib.PngImage, _lib.PngBlock
    assert got == [ctypes.sizeof(I), ctypes.sizeof(Bk), I.nbytes.offset, I.pal_off.offset, Bk.start.offset, Bk.type.offset]


def test_cl_png_decode_rejects_bad_arguments_without_a_gpu(built_lib):
    """Every check runs before the first CUDA call: a status < 0 and a message naming the problem."""
    from controllora_b200 import _lib

    lib = _lib.lib()
    p = P.pack([P.parse(_base()), P.parse(G.golden_cases()[7][1])], 3)
    fake = ctypes.c_void_p(1 << 40)

    def call(images=None, B=2, out_bytes=None, data_len=None, table_len=None, ch=3, slots=None, scratch_bytes=1 << 40):
        return lib.cl_png_decode(ctypes.cast(images if images is not None else p.images, ctypes.c_void_p), fake, B, fake,
                                 p.data_len if data_len is None else data_len, fake,
                                 p.tables_len if table_len is None else table_len, fake, scratch_bytes, fake,
                                 p.block_slots if slots is None else slots, fake, ch, fake,
                                 p.out_bytes if out_bytes is None else out_bytes, fake, None)

    assert lib.cl_png_decode(None, None, 1, None, 0, None, 0, None, 0, None, 0, None, 3, None, 0, None, None) == -1
    assert b"null" in lib.cl_last_error()
    assert call(B=0) == -1
    assert call(ch=2) == -1 and b"out_channels" in lib.cl_last_error()
    assert call(out_bytes=p.out_bytes - 1) == -1 and b"output" in lib.cl_last_error()
    assert call(data_len=p.data_len - 1) == -1 and b"data" in lib.cl_last_error()
    assert call(slots=p.block_slots - 1) == -1 and b"block slots" in lib.cl_last_error()
    imgs = (P.PngImage * 2)(*p.images)
    imgs[1].depth = 3                                  # no colour type has 3-bit samples
    assert call(images=imgs) == -1 and b"bit depth" in lib.cl_last_error()
    imgs = (P.PngImage * 2)(*p.images)
    imgs[1].rowbytes += 1
    assert call(images=imgs) == -1 and b"rowbytes" in lib.cl_last_error()
    imgs = (P.PngImage * 2)(*p.images)
    imgs[1].raw_off -= 1
    assert call(images=imgs) == -1 and b"back to back" in lib.cl_last_error()
    imgs = (P.PngImage * 2)(*p.images)
    imgs[1].out_off -= 1
    assert call(images=imgs) == -1 and b"overlaps" in lib.cl_last_error()
    imgs = (P.PngImage * 2)(*p.images)
    imgs[1].pal_off = p.tables_len                     # image 1 is a palette image: its palette past the tables
    assert imgs[1].color_type == 3 and call(images=imgs) == -1 and b"palette" in lib.cl_last_error()
    conv = (P.PngImage * 1)(p.images[0])
    conv[0].color_type = 3
    assert lib.cl_png_convert(ctypes.cast(conv, ctypes.c_void_p), fake, 1, fake, 1 << 30, 1, fake, 1 << 30, None) == -1


# ================================================================================================ GPU
def _sentinel_decode(files, mode="RGB", gap=37, sentinel=0xA5):
    """decode through ops.png_decode with each image's output window `gap` bytes apart in a sentinel-filled buffer and the
    scratch inside a sentinel-filled one: (images, status, counts, blocks, out buffer, out mask, scratch guard intact)."""
    import torch

    from controllora_b200 import _lib, ops

    ch = P.MODES[mode]
    p = P.pack([P.parse(s) for s in files], ch)
    off, wins = gap, []
    for d in p.images:
        n = d.H * d.W * ch
        d.out_off = off
        wins.append((off, n))
        off += n + gap
    p.host[:ctypes.sizeof(p.images)] = np.frombuffer(bytes(p.images), np.uint8)
    packed = torch.from_numpy(p.host.copy()).cuda()
    out = torch.full((off,), sentinel, dtype=torch.uint8, device="cuda")
    need = _lib.lib().cl_png_scratch_bytes(p.words, p.cand_slots, p.raw_bytes, len(p.images))
    guard = torch.full((need + 2 * 4096,), sentinel, dtype=torch.uint8, device="cuda")
    status, counts, blocks = ops.png_decode(p, packed, out, ch, scratch=guard[4096:4096 + need])
    g = guard.cpu().numpy()
    guard_ok = bool(np.all(g[:4096] == sentinel) and np.all(g[4096 + need:] == sentinel))
    buf = out.cpu().numpy()
    imgs = [buf[o:o + n].reshape(shape) for (o, n), shape in zip(wins, p.shapes)]
    mask = np.ones(len(buf), bool)
    for o, n in wins:
        mask[o:o + n] = False
    return imgs, status, counts, blocks.cpu().numpy(), p, buf, mask, guard_ok


def _gpu_batch():
    rng = np.random.default_rng(77)
    out = [(n, b) for n, b, _ in golden()]
    out += [(n, b) for n, b in seeded_files()[::5]]
    out.append(("photo_512", G.photo_png(rng, 512, 512)))
    out.append(("photo_768", G.photo_png(rng, 768, 640, compress_level=9)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_gpu_ragged_batch_equals_pillow_and_goldens_inside_sentinels(mode):
    batch = _gpu_batch()
    imgs, status, counts, blocks, p, buf, mask, guard_ok = _sentinel_decode([b for _, b in batch], mode)
    assert status == [0] * len(batch), [(n, s) for (n, _), s in zip(batch, status) if s]
    assert np.all(buf[mask] == 0xA5), "bytes outside the output windows were written"
    assert guard_ok, "bytes outside the scratch were written"
    gold = {n: w for n, _, w in golden()}
    bad = []
    for (name, b), got in zip(batch, imgs):
        want = gold[name][mode] if name in gold else png_ref.decode(b, mode)
        if not np.array_equal(got, want) or (Image is not None and not np.array_equal(got, pil(b, mode))):
            bad.append(name)
    assert not bad, bad


@pytest.mark.gpu
def test_gpu_block_table_equals_the_oracle_walker():
    batch = _gpu_batch()
    _, status, counts, blocks, p, _, _, _ = _sentinel_decode([b for _, b in batch])
    assert status == [0] * len(batch)
    bad, taken = [], 0
    for k, ((name, b), d) in enumerate(zip(batch, p.images)):
        want = [(s, bt, f, n) for s, bt, f, n in png_ref.block_table(P.parse(b).zdata)]
        rows = blocks[d.blk0:d.blk0 + counts[k]]
        got = [(int(r[2] & 0xFFFFFFFF), int(r[2] >> 32) & 3, (int(r[2] >> 32) >> 2) & 1, int(r[1])) for r in rows]
        taken += sum(int(r[2] >> 32) >> 3 & 1 for r in rows)
        if got != want:
            bad.append(name)
    assert not bad, bad
    print(f"{int(sum(counts))} blocks, {taken} from confirmed candidates")


def _worst_cases():
    rng = np.random.default_rng(4096)
    flat = np.full((4096, 4096 * 3), 0, np.uint8)
    flat[:, 0::3], flat[:, 1::3], flat[:, 2::3] = 200, 30, 90
    noise = rng.integers(0, 256, (4096, 4096 * 3), dtype=np.uint8)
    a = G.scanlines(rng, 256, 256, 2, 8, "smooth")
    return [("flat_4096", G.build_png(flat, 4096, 2, 8, filters=(1,))),
            ("noise_4096", G.build_png(noise, 4096, 2, 8, filters=(0,), level=1)),
            ("zfixed", G.build_png(a, 256, 2, 8, filters=(4,), strategy=zlib.Z_FIXED)),
            ("single_block", G.build_png(a, 256, 2, 8, filters=(4,), level=9, mem_level=9))]


@pytest.mark.gpu
def test_gpu_worst_cases_decode_exactly():
    for name, b in _worst_cases():
        imgs, status, counts, _, _, buf, mask, guard_ok = _sentinel_decode([b])
        assert status == [0] and guard_ok and np.all(buf[mask] == 0xA5), name
        assert np.array_equal(imgs[0], png_ref.decode(b, "RGB")), name
        print(name, "blocks", counts[0])


@pytest.mark.gpu
def test_gpu_decode_is_repeatable():
    import torch

    files = [b for _, b in _gpu_batch()]
    a = P.decode_png(files)
    b = P.decode_png(files)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_gpu_corrupt_files_are_named_and_leave_the_rest_alone():
    good = [b for _, b, _ in golden()[:6]]
    for name, bad, accepted in corrupt_files():
        if name in ("bad_ihdr_crc", "fdict"):          # refused on the host, before any upload
            with pytest.raises(CLError, match="corrupt"):
                P.decode_png(good[:3] + [bad])
            continue
        files = good[:3] + [bad] + good[3:]
        imgs, status, _, _, _, buf, mask, guard_ok = _sentinel_decode(files)
        assert (status[3] == 0) == accepted and all(s == 0 for k, s in enumerate(status) if k != 3), (name, status)
        assert np.all(buf[mask] == 0xA5) and guard_ok, name
        for k in (0, 1, 2, 4, 5, 6):
            assert np.array_equal(imgs[k], png_ref.decode(files[k], "RGB")), (name, k)
        if not accepted:
            with pytest.raises(CLError, match="image 3"):
                P.decode_png(files)


@pytest.mark.gpu
@needs_pil
def test_gpu_decode_then_train_transform_equals_the_fill50k_path():
    """train_text_to_image_control_lora.py:607-634 on fill50k-like image / guide PNGs: Pillow + torchvision vs
    decode_png + train_transform."""
    import torch
    from torchvision import transforms

    import controllora_b200 as cb

    res = 256
    rng = np.random.default_rng(50)
    pairs = [G.fill50k_pair(rng, 512) for _ in range(3)]
    imgs, guides = [a for a, _ in pairs], [g for _, g in pairs]
    tf = transforms.Compose([transforms.Resize(res, interpolation=transforms.InterpolationMode.BILINEAR),
                             transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])
    torch.manual_seed(5)
    crops = cb.reference_crops([(512, 512)] * 3, res)
    want_p = torch.stack([tf(Image.open(io.BytesIO(s)).convert("RGB"))[:, y:y + res, x:x + res] for s, (y, x) in zip(imgs, crops)])
    want_g = torch.stack([tf(Image.open(io.BytesIO(s)).convert("RGB"))[:, y:y + res, x:x + res] for s, (y, x) in zip(guides, crops)])
    pix, gd = cb.train_transform(P.decode_png(imgs), P.decode_png(guides), res, crops=crops)
    assert torch.equal(pix.cpu(), want_p) and torch.equal(gd.cpu(), want_g)


@pytest.mark.gpu
@needs_pil
def test_gpu_decode_then_canny_equals_the_diffusiondb_path():
    """process/diffusiondb_canny.py:15-35 on photo-like PNGs: np.asarray + cv2.Canny vs decode_png + canny_batch."""
    import cv2
    import torch

    import controllora_b200 as cb

    rng = np.random.default_rng(51)
    files = [G.photo_png(rng, 512, 512) for _ in range(3)]
    pv, guide = cb.canny_batch(torch.stack(P.decode_png(files)), (100, 200))
    for k, b in enumerate(files):
        a = np.asarray(Image.open(io.BytesIO(b)))
        edges = cv2.Canny(a, 100, 200)
        want_g = np.repeat((edges.astype(np.float32) / np.float32(127.5) - np.float32(1))[None], 3, axis=0)
        want_p = (a.astype(np.float32) / np.float32(127.5) - np.float32(1)).transpose(2, 0, 1)
        assert np.array_equal(guide[k].cpu().numpy(), want_g) and np.array_equal(pv[k].cpu().numpy(), want_p)


@pytest.mark.gpu
@needs_pil
@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_gpu_decode_images_on_a_mixed_batch_equals_pillow(mode):
    from tests.golden import make_jpeg_golden as J

    rng = np.random.default_rng(52)
    files = [G.photo_png(rng, 40, 60), J.pil_jpeg(J.photo(rng, 48, 32)), J.pil_jpeg(J.photo(rng, 30, 30, C=1)),
             golden()[3][1], J.pil_jpeg(J.photo(rng, 17, 23), quality=60)]
    got = P.decode_images(files, mode)
    for b, g in zip(files, got):
        assert np.array_equal(g.cpu().numpy(), pil(b, mode))


@pytest.mark.gpu
@needs_pil
def test_gpu_decode_then_training_step_equals_the_torchvision_batch():
    """decode_png -> train_transform -> one step_from_pixels gives what the step fed the torchvision tensors gives, to
    the tolerances tests/test_jpeg.py uses."""
    import torch
    from torchvision import transforms

    from tests.test_jpeg import _dreambooth_step

    size = 64
    rng = np.random.default_rng(53)
    files = [G.photo_png(rng, 64, 64), G.fill50k_pair(rng, 64)[0]]
    tv = transforms.Compose([transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])
    want = torch.stack([tv(Image.open(io.BytesIO(s)).convert("RGB")) for s in files])
    import controllora_b200 as cb
    got, _ = cb.train_transform(P.decode_png(files), P.decode_png(files), size, crops=[(0, 0), (0, 0)])
    got = got.cpu()
    assert torch.equal(got, want)
    loss_a, p_a = _dreambooth_step(got)
    loss_b, p_b = _dreambooth_step(want)
    rel = float((p_a - p_b).norm() / p_b.norm())
    assert abs(loss_a - loss_b) <= 2e-3 * abs(loss_b) and rel < 2e-3
