"""Baseline JPEG decoding (kernel K12, controllora_b200/jpeg.py) and the DreamBooth transform.

CPU: the numpy oracle (oracle/jpeg_ref.py) equals Pillow bit for bit on seeded streams of every accepted kind and
reproduces the goldens; refused kinds raise CLError naming the feature before anything is uploaded; corrupt entropy-coded
data is reported; cl_jpeg_decode validates its arguments without a GPU and its descriptors have the C layout;
dreambooth_crops and the oracle chain equal torchvision.
GPU: decode_jpeg equals Pillow / the goldens on a ragged batch inside sentinel-filled memory, is repeatable, reports
corrupt images by name without touching the rest, and feeds dreambooth_transform and train_transform bit for bit with the
reference's host pipeline, and one DreamBooth-LoRA training step as the torchvision pipeline's batch does."""
import ctypes
import io
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from controllora_b200 import jpeg as J  # noqa: E402
from controllora_b200._lib import CLError  # noqa: E402
from oracle import jpeg_ref  # noqa: E402
from tests.golden import make_jpeg_golden as G  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "jpeg_golden.npz"

try:
    from PIL import Image
except ImportError:                                   # the goldens stand in for Pillow
    Image = None

needs_pil = pytest.mark.skipif(Image is None, reason="needs Pillow")


def pil_decode(b: bytes) -> np.ndarray:
    return np.asarray(Image.open(io.BytesIO(b)))


def golden():
    z = np.load(GOLDEN)
    off, px = z["stream_off"], z["pixels"]
    out, p = [], 0
    for i, name in enumerate(z["names"]):
        shape = tuple(int(v) for v in z["shapes"][i][:int(z["ndim"][i])])
        n = int(np.prod(shape))
        out.append((str(name), z["streams"][off[i]:off[i + 1]].tobytes(), px[p:p + n].reshape(shape)))
        p += n
    return out


# ------------------------------------------------------------------------------------------------ seeded streams
def seeded_streams():
    """(id, stream) of the CPU sweep: layouts, qualities 1-100 and custom tables, optimised tables, restart intervals
    (Pillow's blocks / rows, cv2's RST interval), cv2 streams, EXIF / ICC / COM segments, small and odd sizes, a few
    above 2000 px, flat and striped content."""
    rng = np.random.default_rng(7)
    out = []
    sizes = [(1, 1), (1, 17), (23, 1), (2, 3), (7, 8), (8, 9), (15, 16), (16, 17), (17, 15), (31, 33), (47, 24), (40, 65)]
    layouts = [dict(subsampling=0), dict(subsampling=1), dict(subsampling=2), "L"]
    for i, (h, w) in enumerate(sizes):
        a = G.photo(rng, h, w)
        for lay in layouts:
            for q in (1, 10, 50, 75, 95, 100):
                if lay == "L":
                    out.append((f"{h}x{w}_L_q{q}", G.pil_jpeg(a[..., 0], quality=q)))
                else:
                    out.append((f"{h}x{w}_ss{lay['subsampling']}_q{q}", G.pil_jpeg(a, quality=q, **lay)))
    a = G.photo(rng, 37, 70)
    tables = [[int(v) for v in rng.integers(1, 256, 64)] for _ in range(2)]
    for lay in layouts[:3]:
        out.append((f"qtables_ss{lay['subsampling']}", G.pil_jpeg(a, qtables=tables, **lay)))
        for mul in (16, 97, 255):                      # 16-bit tables, up to entries of 65025
            out.append((f"qtables16x{mul}_ss{lay['subsampling']}",
                        G.pil_jpeg(a, qtables=[[v * mul for v in t] for t in tables], **lay)))
        out.append((f"optimize_ss{lay['subsampling']}", G.pil_jpeg(a, quality=88, optimize=True, **lay)))
        for n in (1, 3, 7):
            out.append((f"rstblocks{n}_ss{lay['subsampling']}", G.pil_jpeg(a, quality=80, restart_marker_blocks=n, **lay)))
        out.append((f"rstrows_ss{lay['subsampling']}", G.pil_jpeg(a, quality=70, restart_marker_rows=2, **lay)))
        out.append((f"segments_ss{lay['subsampling']}", G.pil_jpeg(a, exif=b"Exif\0\0II*\0\x08\0\0\0\0\0\0\0\0\0",
                                                                  icc_profile=bytes(range(256)) * 300, comment=b"x" * 100, **lay)))
    out.append(("optimize_rst_L", G.pil_jpeg(a[..., 2], quality=60, optimize=True, restart_marker_blocks=2)))
    for q in (5, 50, 97):
        for rst in (0, 1, 4):
            for (h, w) in ((33, 47), (9, 130)):
                b = G.photo(rng, h, w)
                out.append((f"cv2_{h}x{w}_q{q}_rst{rst}", G.cv2_jpeg(b, quality=q, rst=rst)))
                out.append((f"cv2_gray_{h}x{w}_q{q}_rst{rst}", G.cv2_jpeg(b[..., 0].copy(), quality=q, rst=rst)))
    for ss in (0, 1, 2):
        out.append((f"tall_2049x11_ss{ss}", G.pil_jpeg(G.photo(rng, 2049, 11), quality=75, subsampling=ss)))
        out.append((f"wide_5x2100_ss{ss}", G.pil_jpeg(G.photo(rng, 5, 2100), quality=90, subsampling=ss)))
        out.append((f"flat_ss{ss}", G.pil_jpeg(G.flat(24, 56, (int(rng.integers(256)), 7, 250)), subsampling=ss)))
        out.append((f"striped_ss{ss}", G.pil_jpeg(G.striped(24, 56, period=4 + ss), subsampling=ss)))
    return out


@needs_pil
def test_oracle_equals_pillow_on_seeded_streams():
    cases = seeded_streams()
    assert len(cases) >= 300
    bad = []
    for name, b in cases:
        got, ref = jpeg_ref.decode(b), pil_decode(b)
        if got.shape != ref.shape or not np.array_equal(got, ref):
            bad.append(name)
    assert not bad, f"{len(bad)} of {len(cases)} streams differ from Pillow: {bad[:10]}"


@needs_pil
def test_oracle_equals_pillow_far_out_of_range():
    """Streams whose blocks decode far outside 0..255 (8-bit DQT entries edited after encoding, so a flat block's DC
    lands at thousands): Pillow's SIMD IDCT saturates, wraps its 16-bit sums and takes a DC-only shortcut in 16 bits,
    where libjpeg's C code would wrap the result at 10 bits; the oracle follows Pillow."""
    cases = G.dqt_edited_cases() + [(f"random_{k}", b) for k, b in enumerate(G.dqt_random_edits(np.random.default_rng(3), 40))]
    bad = [name for name, b in cases if not np.array_equal(jpeg_ref.decode(b), pil_decode(b))]
    assert not bad, bad
    flat_160_q90 = dict(G.dqt_edited_cases())["dqt_flat160_dc90"]
    assert np.all(jpeg_ref.decode(flat_160_q90) == 255)     # the C code's 10-bit wrap would give 0 here


def test_oracle_reproduces_the_goldens():
    for name, b, ref in golden():
        assert np.array_equal(jpeg_ref.decode(b), ref), name


@needs_pil
def test_golden_generator_rebuilds_the_file():
    z = np.load(GOLDEN)
    fresh = G.build(with_large=False)
    for k, v in fresh.items():
        assert np.array_equal(z[k], v), k


# ------------------------------------------------------------------------------------------------ refusals
def _base() -> bytes:
    return G.pil_jpeg(G.photo(np.random.default_rng(1), 24, 40), quality=80)


def _find(b: bytes, marker: int) -> int:
    i = b.index(bytes([0xFF, marker]))
    return i


def _edit_sof(b: bytes, pos: int, value: int) -> bytes:
    i = _find(b, 0xC0) + 4 + pos
    return b[:i] + bytes([value]) + b[i + 1:]


def _dc_table_two_1bit_codes(base: bytes) -> bytes:
    """The stream with its luma DC table (table 0) redefined, just before the scan, as two 1-bit codes, the second of
    them all ones: libjpeg refuses the table when the scan uses it, and Pillow raises."""
    seg = b"\x00" + bytes([2] + [0] * 15) + b"\x00\x01"
    dht = bytes([0xFF, 0xC4, 0, 2 + len(seg)]) + seg
    i = _find(base, 0xDA)
    return base[:i] + dht + base[i:]


def _refused():
    a = G.photo(np.random.default_rng(2), 24, 40)
    base = _base()
    sof = _find(base, 0xC0)
    sos = _find(base, 0xDA)
    dht = _find(base, 0xC4)
    dht_len = (base[dht + 2] << 8) | base[dht + 3]
    cmyk = io.BytesIO()
    if Image is not None:
        Image.fromarray(a).convert("CMYK").save(cmyk, "JPEG")
    prog = G.pil_jpeg(a, progressive=True) if Image is not None else None
    jfif_end = 2 + 2 + ((base[4] << 8) | base[5])
    no_jfif = base[:2] + base[jfif_end:]                   # without JFIF, libjpeg reads the colour space from Adobe / ids
    adobe0 = no_jfif[:2] + b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00" + no_jfif[2:]
    k = no_jfif.index(b"\xff\xc0") + 10
    rgb_ids = no_jfif[:k] + b"R" + no_jfif[k + 1:k + 3] + b"G" + no_jfif[k + 4:k + 6] + b"B" + no_jfif[k + 7:]
    eoi = base.rindex(b"\xff\xd9")
    two_scans = base[:eoi] + base[sos:eoi] + b"\xff\xd9"
    cases = [
        ("progressive", prog, "progressive"),
        ("cmyk", cmyk.getvalue() or None, "CMYK"),
        ("arithmetic", base[:sof + 1] + b"\xc9" + base[sof + 2:], "arithmetic"),
        ("lossless", base[:sof + 1] + b"\xc3" + base[sof + 2:], "lossless"),
        ("12-bit", _edit_sof(base, 0, 12).replace(b"\xff\xc0", b"\xff\xc1", 1), "12-bit"),
        ("two scans", two_scans, "more than one scan"),
        ("adobe transform 0", adobe0, "Adobe RGB"),
        ("rgb component ids", rgb_ids, "Adobe RGB"),
        ("4:4:0", _edit_sof(base, 7, 0x12), "sampling"),
        ("4:1:1", _edit_sof(base, 7, 0x41), "sampling"),
        ("dnl", _edit_sof(_edit_sof(base, 1, 0), 2, 0), "DNL"),
        ("two components", base[:sof + 4] + bytes([base[sof + 4]]) + base[sof + 5:sof + 9] + b"\x02" + base[sof + 10:], "malformed"),
        ("malformed", base[:sof + 6], "malformed"),
        ("not a jpeg", b"\x89PNG\r\n\x1a\n" + bytes(20), "not a JPEG"),
        ("missing huffman", base[:dht] + base[dht + 2 + dht_len:], "Huffman table"),
        ("invalid huffman", base[:dht + 5] + b"\x05" + base[dht + 6:], "Huffman table"),
        ("all-ones huffman code", _dc_table_two_1bit_codes(base), "Huffman table"),
        ("missing quantisation", _edit_sof(base, 8, 3), "quantisation table 3 is missing"),
    ]
    return [c for c in cases if c[1] is not None]


@pytest.mark.parametrize("name,stream,feature", _refused(), ids=[c[0] for c in _refused()])
def test_refused_kinds_raise_before_upload(name, stream, feature):
    """decode_jpeg raises CLError naming the feature from the host parser: no GPU is needed to see it."""
    with pytest.raises(CLError) as e:
        J.decode_jpeg([_base(), stream])
    assert feature in str(e.value) and "image 1" in str(e.value), str(e.value)


@needs_pil
def test_all_ones_huffman_code_is_refused_as_pillow_refuses_it():
    b = _dc_table_two_1bit_codes(_base())
    with pytest.raises(OSError):
        pil_decode(b)


def test_refused_stream_message_points_to_pillow():
    with pytest.raises(CLError, match="Pillow"):
        J.parse(_base().replace(b"\xff\xc0", b"\xff\xc2", 1))


# ------------------------------------------------------------------------------------------------ corruption
def _entropy_span(b: bytes):
    sos = _find(b, 0xDA)
    start = sos + 2 + ((b[sos + 2] << 8) | b[sos + 3])
    return start, b.rindex(b"\xff\xd9")


def corrupt_streams():
    big = G.pil_jpeg(G.photo(np.random.default_rng(5), 64, 96), quality=90)
    s, e = _entropy_span(big)
    truncated = big[:s + (e - s) // 2]
    bad_code = big[:s] + b"\xff\x00" * 12 + big[s + 12:]           # sixteen and more 1 bits: no code of the tables
    return [("truncated", truncated), ("invalid code", bad_code)]


@pytest.mark.parametrize("name,stream", corrupt_streams(), ids=[c[0] for c in corrupt_streams()])
def test_oracle_reports_corrupt_entropy_data(name, stream):
    with pytest.raises(jpeg_ref.Corrupt):
        jpeg_ref.decode(stream)
    if Image is not None and name == "truncated":
        with pytest.raises(OSError):
            pil_decode(stream)


# ------------------------------------------------------------------------------------------------ C ABI
def test_descriptor_layout_matches_c(built_lib, tmp_path):
    from controllora_b200 import _lib

    src = tmp_path / "sz.c"
    src.write_text(
        '#include <stdio.h>\n#include <stddef.h>\n#include "controllora_b200.h"\n'
        'int main(){printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(cl_jpeg_image), sizeof(cl_jpeg_segment),'
        " offsetof(cl_jpeg_image, status0), offsetof(cl_jpeg_image, comp_plane), offsetof(cl_jpeg_segment, nbytes),"
        " offsetof(cl_jpeg_segment, nwin), (size_t)CL_JPEG_HUFF_WORDS);return 0;}\n")
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    I, S = _lib.JpegImage, _lib.JpegSegment
    assert got == [ctypes.sizeof(I), ctypes.sizeof(S), I.status0.offset, I.comp_plane.offset, S.nbytes.offset, S.nwin.offset,
                   J.HUFF_WORDS]


def _packed(streams):
    return J.pack([J.parse(s) for s in streams])


def test_cl_jpeg_decode_rejects_bad_arguments_without_a_gpu(built_lib):
    """Every check runs before the first CUDA call: a status < 0 and a message naming the problem."""
    from controllora_b200 import _lib

    lib = _lib.lib()
    p = _packed([_base(), G.pil_jpeg(G.photo(np.random.default_rng(3), 20, 9), restart_marker_blocks=1)])
    fake = ctypes.c_void_p(1 << 40)

    def call(images=None, segments=None, B=2, S=None, out_bytes=None, table_len=None, scratch_bytes=1 << 40):
        return lib.cl_jpeg_decode(ctypes.cast(images if images is not None else p.images, ctypes.c_void_p), fake, B,
                                  ctypes.cast(segments if segments is not None else p.segments, ctypes.c_void_p), fake,
                                  len(p.segments) if S is None else S, fake, p.tables_len if table_len is None else table_len,
                                  fake, p.data_len, fake, scratch_bytes, fake, p.out_bytes if out_bytes is None else out_bytes,
                                  fake, None, None)

    assert lib.cl_jpeg_decode(None, None, 1, None, None, 1, None, 0, None, 0, None, 0, None, 0, None, None, None) == -1
    assert b"null" in lib.cl_last_error()
    assert call(B=0) == -1
    assert call(out_bytes=p.out_bytes - 1) == -1 and b"output" in lib.cl_last_error()
    assert call(table_len=100) == -1 and b"tables" in lib.cl_last_error()
    assert call(S=len(p.segments) - 1) == -1
    imgs = (J.JpegImage * 2)(*p.images)
    imgs[1].C = 2
    assert call(images=imgs) == -1 and b"C = 2" in lib.cl_last_error()
    imgs = (J.JpegImage * 2)(*p.images)
    imgs[0].hmax = 1
    assert call(images=imgs) == -1 and b"sampling" in lib.cl_last_error()
    segs = (J.JpegSegment * len(p.segments))(*p.segments)
    segs[1].nbytes += 1 << 20
    assert call(segments=segs) == -1 and b"data" in lib.cl_last_error()
    segs = (J.JpegSegment * len(p.segments))(*p.segments)
    segs[-1].nwin += 1
    assert call(segments=segs) == -1 and b"windows" in lib.cl_last_error()
    imgs = (J.JpegImage * 2)(*p.images)
    imgs[1].plane_off += 4                             # a misaligned, overlapping plane range
    assert call(images=imgs) == -1 and b"back to back" in lib.cl_last_error()
    imgs = (J.JpegImage * 2)(*p.images)
    imgs[1].coef_off -= 1                              # overlapping coefficient blocks
    assert call(images=imgs) == -1 and b"back to back" in lib.cl_last_error()
    imgs = (J.JpegImage * 2)(*p.images)
    imgs[1].out_off -= 1                               # output windows that overlap
    assert call(images=imgs) == -1 and b"overlaps" in lib.cl_last_error()


def test_pack_splits_restart_segments_and_removes_stuffing():
    b = G.pil_jpeg(G.photo(np.random.default_rng(4), 40, 40), quality=100, restart_marker_blocks=1)
    f = J.parse(b)
    assert f.ri == 1 and len(f.segments) == f.n_segments == 9 and f.restart_ok
    s, e = _entropy_span(b)
    raw = b[s:e]
    assert sum(len(x) for x in f.segments) == len(raw) - 2 * (len(f.segments) - 1) - raw.count(b"\xff\x00")
    p = J.pack([f])
    assert p.n_windows == sum(max(1, -(-8 * len(x) // J.WINDOW_BITS)) for x in f.segments)


def test_pack_is_linear_in_restart_segments():
    """A 4032 x 3024 stream with a restart marker after every MCU (47 628 segments): parse + pack build the segment
    descriptors column-wise, in a fraction of a second where a per-segment pass over the batch took seconds."""
    import time

    b = G.cv2_jpeg(G.photo(np.random.default_rng(6), 3024, 4032), quality=90, rst=1)
    t0 = time.perf_counter()
    p = J.pack([J.parse(b)])
    dt = time.perf_counter() - t0
    segs = np.frombuffer(bytes(p.segments), J._SEGMENT_DTYPE)
    assert len(segs) == 47628 and np.all(segs["mcu0"] == np.arange(len(segs)))
    assert np.all(segs["win0"][1:] == np.cumsum(segs["nwin"])[:-1]) and segs["win0"][0] == 0
    assert np.all(segs["data_off"][1:] == np.cumsum(segs["nbytes"])[:-1]) and p.n_windows == int(segs["nwin"].sum())
    assert dt < 2.0, f"parse + pack took {dt:.2f} s"


# ------------------------------------------------------------------------------------------------ DreamBooth crops
@needs_pil
@pytest.mark.parametrize("center", [True, False])
def test_dreambooth_crops_and_oracle_chain_equal_torchvision(center):
    import torch
    from torchvision import transforms

    from oracle import resample_ref as RR

    size = 64
    rng = np.random.default_rng(8)
    imgs = [G.photo(rng, h, w) for h, w in ((64, 64), (80, 64), (64, 97), (121, 75), (50, 50))]
    imgs.append(G.photo(rng, 90, 70, C=1))
    pil = [Image.fromarray(a) for a in imgs]
    crop = transforms.CenterCrop(size) if center else transforms.RandomCrop(size)
    tv = transforms.Compose([transforms.Resize(size, interpolation=transforms.InterpolationMode.BILINEAR), crop,
                             transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])
    torch.manual_seed(1234)
    want = torch.stack([tv(im.convert("RGB")) for im in pil])
    torch.manual_seed(1234)
    crops = J.dreambooth_crops([a.shape[:2] for a in imgs], size, center)
    got = []
    for a, (top, left) in zip(imgs, crops):
        rgb = np.repeat(a[..., None], 3, axis=2) if a.ndim == 2 else a
        got.append(torch.from_numpy(RR.train_transform(rgb, size, top, left)))
    assert torch.equal(torch.stack(got), want)


# ================================================================================================ GPU
def _sentinel_decode(streams, gap=37, sentinel=0xA5):
    """decode through ops.jpeg_decode with each image's output window `gap` bytes apart in a sentinel-filled buffer:
    (images, status, rounds, buffer, windows)."""
    import torch

    from controllora_b200 import ops

    p = J.pack([J.parse(s) for s in streams])
    off, wins = gap, []
    for k, d in enumerate(p.images):
        n = d.H * d.W * d.C
        d.out_off = off
        wins.append((off, n))
        off += n + gap
    p.host[:ctypes.sizeof(p.images)] = np.frombuffer(bytes(p.images), np.uint8)
    staged = torch.from_numpy(p.host.copy())
    packed = staged.cuda()
    out = torch.full((off,), sentinel, dtype=torch.uint8, device="cuda")
    status, rounds = ops.jpeg_decode(p, packed, out)
    buf = out.cpu().numpy()
    imgs = [buf[o:o + n].reshape(shape) for (o, n), shape in zip(wins, p.shapes)]
    mask = np.ones(len(buf), bool)
    for o, n in wins:
        mask[o:o + n] = False
    return imgs, status, rounds, buf, mask


def _gpu_batch():
    rng = np.random.default_rng(99)
    out = [(n, b, ref) for n, b, ref in golden()]
    z = np.load(GOLDEN)
    large = G.large_cases()
    for (name, b), want_sha, px_sha in zip(large, z["large_stream_sha256"], z["large_pixels_sha256"]):
        assert G.sha(b) == want_sha, f"{name}: the rebuilt stream differs from the golden's"
        out.append((name, b, str(px_sha)))
    out.append(("extra_rst_420", G.pil_jpeg(G.photo(rng, 300, 451), quality=67, restart_marker_rows=3), None))
    return out


@pytest.mark.gpu
def test_gpu_ragged_batch_equals_pillow_and_goldens_inside_sentinels():
    batch = _gpu_batch()
    imgs, status, rounds, buf, mask = _sentinel_decode([b for _, b, _ in batch])
    assert status == [0] * len(batch)
    assert np.all(buf[mask] == 0xA5), "bytes outside the output windows were written"
    bad = []
    for (name, b, ref), got in zip(batch, imgs):
        if isinstance(ref, str):
            ok = G.sha(np.ascontiguousarray(got).tobytes()) == ref
        else:
            ok = np.array_equal(got, ref if ref is not None else jpeg_ref.decode(b))
        if Image is not None:
            ok = ok and np.array_equal(got, pil_decode(b))
        if not ok:
            bad.append(name)
    assert not bad, bad
    print(f"sync rounds: {rounds}")


@pytest.mark.gpu
def test_gpu_decode_is_repeatable():
    import torch

    streams = [b for _, b, _ in _gpu_batch()]
    a = J.decode_jpeg(streams)
    b = J.decode_jpeg(streams)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_gpu_corrupt_streams_are_named_and_leave_the_rest_alone():
    good = [b for _, b, _ in golden()[:6]]
    for name, bad in corrupt_streams():
        streams = good[:3] + [bad] + good[3:]
        imgs, status, _, buf, mask = _sentinel_decode(streams)
        assert status[3] != 0 and all(s == 0 for k, s in enumerate(status) if k != 3), (name, status)
        assert np.all(buf[mask] == 0xA5), name
        for k in (0, 1, 2, 4, 5, 6):
            assert np.array_equal(imgs[k], jpeg_ref.decode(streams[k])), (name, k)
        with pytest.raises(CLError, match="image 3"):
            J.decode_jpeg(streams)


def _db_sources():
    rng = np.random.default_rng(31)
    srcs = [G.pil_jpeg(G.photo(rng, 3024 // 4, 4032 // 4), quality=92),
            G.pil_jpeg(G.photo(rng, 512, 512)),                      # as sample_class_images writes: Image.save, defaults
            G.pil_jpeg(G.photo(rng, 700, 513), quality=85, subsampling=1),
            G.pil_jpeg(G.photo(rng, 600, 777, C=1), quality=90)]
    return srcs


@pytest.mark.gpu
@needs_pil
@pytest.mark.parametrize("center", [True, False])
def test_gpu_decode_then_dreambooth_transform_equals_torchvision(center):
    import torch
    from torchvision import transforms

    size = 512
    srcs = _db_sources()
    crop = transforms.CenterCrop(size) if center else transforms.RandomCrop(size)
    tv = transforms.Compose([transforms.Resize(size, interpolation=transforms.InterpolationMode.BILINEAR), crop,
                             transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])
    torch.manual_seed(77)
    want = torch.stack([tv(Image.open(io.BytesIO(s)).convert("RGB")) for s in srcs])
    torch.manual_seed(77)
    got = J.dreambooth_transform(J.decode_jpeg(srcs), size, center_crop=center)
    assert torch.equal(got.cpu(), want)


@pytest.mark.gpu
@needs_pil
def test_gpu_decode_then_train_transform_equals_the_generic_path():
    """train_text_to_image_control_lora.py:607-634 on JPEG images and guides decoded by Pillow vs by decode_jpeg."""
    import torch
    from torchvision import transforms

    import controllora_b200 as cb

    res = 256
    rng = np.random.default_rng(12)
    imgs = [G.pil_jpeg(G.photo(rng, 360, 480), quality=90), G.pil_jpeg(G.photo(rng, 300, 300), quality=75)]
    guides = [G.pil_jpeg(G.photo(rng, 360, 480, C=1), quality=95), G.pil_jpeg(G.photo(rng, 300, 300), quality=60)]
    tf = transforms.Compose([transforms.Resize(res, interpolation=transforms.InterpolationMode.BILINEAR),
                             transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])
    torch.manual_seed(5)
    crops = cb.reference_crops([pil_decode(s).shape[:2] for s in imgs], res)
    want_p, want_g = [], []
    for s, gsrc, (y1, x1) in zip(imgs, guides, crops):
        p = tf(Image.open(io.BytesIO(s)).convert("RGB"))[:, y1:y1 + res, x1:x1 + res]
        g = tf(Image.open(io.BytesIO(gsrc)).convert("RGB"))[:, y1:y1 + res, x1:x1 + res]
        want_p.append(p)
        want_g.append(g)
    pix, gd = cb.train_transform(J.decode_jpeg(imgs), J.decode_jpeg(guides), res, crops=crops)
    assert torch.equal(pix.cpu(), torch.stack(want_p)) and torch.equal(gd.cpu(), torch.stack(want_g))


def _dreambooth_step(pixels):
    """One Trainer(unet, None, prior_loss_weight=1.0).step_from_pixels on the tiny config with fixed weights, token ids,
    latent noise and noise seed: (loss, trained LoRA parameters), both on the host."""
    import torch

    import controllora_b200 as cb
    from controllora_b200.trainer import Trainer
    from oracle import clip_ref as CR
    from oracle import models_ref as MR
    from oracle import unet_ref as UR
    from oracle import vae_ref as VR
    from tests.check_unet import TINY

    torch.manual_seed(0)                               # module construction draws from the global generator
    ounet = UR.UNet2DConditionModel(**TINY)
    UR.init_synthetic_(ounet, seed=1)
    sd = {k: v.to(torch.bfloat16).float() for k, v in ounet.state_dict().items()}
    munet = cb.UNet2DConditionModel.from_state_dict(sd, "cuda", TINY)
    g = torch.Generator().manual_seed(7)
    procs = {}
    for name in ounet.attn_processors.keys():
        C = dict(ounet._attn_modules())[name].to_q.weight.shape[0]
        xd = None if name.endswith("attn1.processor") else TINY["cross_attention_dim"]
        op = MR.LoRACrossAttnProcessor(C, xd, rank=4)
        with torch.no_grad():
            for n_, p_ in op.named_parameters():
                if n_.endswith("up.weight"):
                    p_.copy_(0.05 * torch.randn(p_.shape, generator=g))
        mp = cb.LoRACrossAttnProcessor(C, xd, rank=4)
        mp.load_state_dict(op.state_dict())
        procs[name] = mp.to("cuda")
    munet.set_attn_processor(procs)
    vcfg = dict(block_out_channels=(32, 64, 64), layers_per_block=1)      # 64 x 64 pixels -> 16 x 16 latents
    ovae = VR.AutoencoderKL(**vcfg)
    VR.init_synthetic_(ovae, seed=4)
    mvae = cb.AutoencoderKL.from_state_dict({k: v.detach().clone() for k, v in ovae.state_dict().items()}, "cuda", vcfg)
    ccfg = dict(CR.SD15_TEXT_CONFIG)
    ccfg.update(num_hidden_layers=2, vocab_size=1000, hidden_size=64, intermediate_size=256, num_attention_heads=4)
    mclip = cb.CLIPTextModel.from_state_dict(CR.synthetic_state_dict(ccfg, seed=0), "cuda", ccfg)
    B = pixels.shape[0]
    ids = torch.randint(0, ccfg["vocab_size"], (B, 77), generator=g)
    eps = torch.randn(B, 4, 16, 16, generator=g)
    tr = Trainer(munet, None, lr=1e-3, prior_loss_weight=1.0, noise_seed=21)
    loss = tr.step_from_pixels(mvae, mclip, pixels.to("cuda"), ids.to("cuda"), None, latent_noise=eps)
    torch.cuda.synchronize()
    return float(loss), tr.flat_p[:tr.numel].detach().cpu().clone()


@pytest.mark.gpu
@needs_pil
def test_gpu_decode_then_dreambooth_step_equals_the_torchvision_batch():
    """decode_jpeg -> dreambooth_transform -> one DreamBooth-LoRA step (instance + class image, prior_loss_weight 1.0)
    gives the loss and trained parameters of the same step fed the torchvision pipeline's pixel_values
    (train_dreambooth_lora.py:449-478, 880-918): the pixels bit for bit, the loss bit for bit when the step repeats it
    exactly, and the parameters to the tolerance of the step's atomically reduced gradients."""
    import torch
    from torchvision import transforms

    size = 64
    rng = np.random.default_rng(41)
    srcs = [G.pil_jpeg(G.photo(rng, 120, 90), quality=92), G.pil_jpeg(G.photo(rng, 64, 64))]
    tv = transforms.Compose([transforms.Resize(size, interpolation=transforms.InterpolationMode.BILINEAR),
                             transforms.RandomCrop(size), transforms.ToTensor(), transforms.Normalize([0.5], [0.5])])
    torch.manual_seed(3)
    want = torch.stack([tv(Image.open(io.BytesIO(s)).convert("RGB")) for s in srcs])
    torch.manual_seed(3)
    got = J.dreambooth_transform(J.decode_jpeg(srcs), size).cpu()
    assert torch.equal(got, want)
    loss_a, p_a = _dreambooth_step(got)
    loss_b, p_b = _dreambooth_step(want)
    loss_c, p_c = _dreambooth_step(want)
    # The step's weight gradients are reduced with atomics, so its parameters are not bit-reproducible even for the same
    # pixels (the repeat shows it); they are held to the tolerance the project's resume check uses (2e-3 relative).
    rel = lambda x, y: float((x - y).norm() / y.norm())       # noqa: E731
    print(f"loss {loss_a!r} vs {loss_b!r} (repeat {loss_c!r}); parameters rel {rel(p_a, p_b):.2e} (repeat {rel(p_c, p_b):.2e})")
    assert loss_a == loss_b if loss_b == loss_c else abs(loss_a - loss_b) <= 2e-3 * abs(loss_b)
    assert rel(p_a, p_b) < 2e-3 and rel(p_c, p_b) < 2e-3
