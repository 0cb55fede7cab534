// PNG decoder for a ragged batch, bit for bit with Pillow's Image.open(f).convert("RGB") / .convert("L"): every
// non-interlaced colour type and bit depth.  The rules are restated in oracle/png_ref.py; the host
// (controllora_b200/png.py) parses the chunks and the zlib header and refuses what is not decoded here.
//
// Inflate runs in parallel inside one stream by speculative block discovery (pugz: Kerbiriou & Chikhi, 2019; PAPERS.md)
// and pointer jumping; unfiltering runs as a wavefront.  Launches, a number fixed by the batch's sizes, no host sync:
//   0. cudaMemsetAsync: status and the Adler-32 sums.  png_init_kernel: inflated bytes 0, source index p -> p.
//   1. png_find_kernel: one thread per bit offset of each stream tests whether a dynamic-Huffman block header that
//      zlib accepts starts there (BTYPE 2, HLIT / HDIST in range, a complete code-length code, code lengths that decode
//      inside their count, EOB coded, literal / length and distance codes complete or incomplete as zlib allows), and
//      sets the offset's bit in a 32-bit word.
//   2. cub::DeviceScan::ExclusiveSum of the words' popcounts: the rank of every candidate in its stream.
//   3. png_count_kernel: one thread per candidate (up to the stream's slots) decodes the block without output and
//      records its end bit, its inflated length and whether it decoded cleanly to its end-of-block code.
//   4. png_walk_kernel: one thread per stream follows the chain from the first block.  A block that starts on a clean
//      candidate is taken from its slot in O(1) (the candidate bit and the rank); any other block (stored, fixed
//      Huffman, a candidate that did not decode cleanly) is decoded inline.  The chain from the stream's start is
//      authoritative whatever the data: speculation only saves time.  Here, as zlib under Pillow does, decoding stops
//      at the first byte past the last row, and corrupt data is reported on this path only.
//   5. png_write_kernel: one thread per chain block stores its literals and, per inflated byte, a source index: p for a
//      literal, p - distance for a match byte.
//   6. ceil(log2(largest inflated size)) rounds of png_jump_kernel (src[p] = src[src[p]]) resolve every byte to a
//      literal whatever the data; png_gather_kernel copies the literals and sums the Adler-32 in parallel.
//   7. png_unfilter_kernel: one CTA per image, one thread per (row, byte lane of a pixel), each row one step behind the
//      row above, 1024 / bpp rows in flight per band, one barrier per step.
//   8. png_unpack_kernel: one thread per pixel, Pillow's unpackers and convert("RGB") / convert("L"); compares the
//      Adler-32.
// Every index taken from a stream is bounds-checked: reads past a stream's end read zero bits and stop the decode, writes
// are bounded by the image's inflated size, source indices by the byte being resolved.
#include <stdio.h>

#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

constexpr int PNG_THREADS = 128;
constexpr int PNG_UNFILTER_THREADS = 1024;

__constant__ uint16_t kPngLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                         31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kPngLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t kPngDistBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                          193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kPngDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kPngClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// ------------------------------------------------------------------------------------------------ bit reader
// LSB-first over one stream; bytes past its end read as zero, and pos > nbits tells the decode that it ran out.
struct PngBits {
    const uint8_t* p;
    int64_t nbytes, next, pos;
    uint64_t buf;
    int valid;

    __device__ __forceinline__ void fill() {
        while (valid <= 56) {
            const uint64_t b = next < nbytes ? (uint64_t)__ldg(p + next) : 0ull;
            buf |= b << valid;
            valid += 8;
            ++next;
        }
    }
    __device__ __forceinline__ void init(const uint8_t* p_, int64_t n, int64_t bitpos) {
        p = p_; nbytes = n; next = bitpos >> 3; buf = 0; valid = 0; pos = bitpos;
        fill();
        const int s = (int)(bitpos & 7);
        buf >>= s;
        valid -= s;
    }
    __device__ __forceinline__ void skip(int n) {
        buf >>= n;
        valid -= n;
        pos += n;
        if (valid < 32) fill();
    }
    __device__ __forceinline__ uint32_t get(int n) {   // n in 0..24
        const uint32_t v = (uint32_t)(buf & ((1ull << n) - 1));
        skip(n);
        return v;
    }
};

// ------------------------------------------------------------------------------------------------ Huffman codes
// Canonical code of up to 15 bits (RFC 1951 3.2.2): counts per length, symbols by (length, value), and a lookup of the
// next LUT_BITS stream bits for the short codes ((symbol << 4) | length, 0 for a longer code or none).
template <int NSYM, int LUT_BITS>
struct PngHuff {
    uint16_t lut[1 << LUT_BITS];
    uint16_t count[16];
    uint16_t sym[NSYM];
};

// zlib's inflate_table verdict: -1 over-subscribed, else 1 when incomplete, 0 when complete; maxlen = the longest code.
template <int NSYM, int LUT_BITS>
__device__ __forceinline__ int png_build(const uint8_t* len, int n, PngHuff<NSYM, LUT_BITS>& h, bool lut, int& maxlen) {
    for (int l = 0; l < 16; ++l) h.count[l] = 0;
    for (int s = 0; s < n; ++s) h.count[len[s]]++;
    h.count[0] = 0;
    maxlen = 0;
    int left = 1;
    for (int l = 1; l < 16; ++l) {
        if (h.count[l]) maxlen = l;
        left = (left << 1) - h.count[l];
        if (left < 0) return -1;
    }
    uint16_t offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
    for (int s = 0; s < n; ++s)
        if (len[s]) h.sym[offs[len[s]]++] = (uint16_t)s;
    if (lut) {
        for (int i = 0; i < (1 << LUT_BITS); ++i) h.lut[i] = 0;
        int code = 0, k = 0;
        for (int l = 1; l <= LUT_BITS; ++l) {
            for (int i = 0; i < h.count[l]; ++i, ++code, ++k) {
                const int rev = (int)(__brev((unsigned)code) >> (32 - l));
                for (int j = rev; j < (1 << LUT_BITS); j += 1 << l) h.lut[j] = (uint16_t)((h.sym[k] << 4) | l);
            }
            code <<= 1;
        }
    }
    return left > 0 ? 1 : 0;
}

// The next symbol, or -1 for a bit pattern no code has (possible in an incomplete code).
template <int NSYM, int LUT_BITS>
__device__ __forceinline__ int png_decode(PngBits& r, const PngHuff<NSYM, LUT_BITS>& h) {
    const int e = h.lut[r.buf & ((1u << LUT_BITS) - 1)];
    if (e) {
        r.skip(e & 15);
        return e >> 4;
    }
    uint64_t b = r.buf;
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; ++l) {
        code |= (int)(b & 1);
        b >>= 1;
        const int c = h.count[l];
        if (code - c < first) {
            r.skip(l);
            return h.sym[index + (code - first)];
        }
        index += c;
        first = (first + c) << 1;
        code <<= 1;
    }
    return -1;
}

using PngLit = PngHuff<288, 9>;
using PngDist = PngHuff<32, 8>;
using PngCl = PngHuff<19, 7>;

// A dynamic block's header from HLIT on: 0 with the two codes built, -1 when zlib rejects it (or it runs past nbits).
// With lut = false only the verdict is computed (the find pass).
__device__ __forceinline__ int png_dynamic_header(PngBits& r, int64_t nbits, PngLit& lit, PngDist& dist, bool lut) {
    const int nlen = (int)r.get(5) + 257, ndist = (int)r.get(5) + 1, ncode = (int)r.get(4) + 4;
    if (nlen > 286 || ndist > 30) return -1;
    uint8_t lens[320];
    for (int i = 0; i < 19; ++i) lens[i] = 0;
    for (int i = 0; i < ncode; ++i) lens[kPngClOrder[i]] = (uint8_t)r.get(3);
    if (r.pos > nbits) return -1;
    PngCl cl;
    int mx;
    if (png_build(lens, 19, cl, true, mx) != 0 || mx == 0) return -1;   // the code-length code must be complete
    const int n = nlen + ndist;
    int i = 0;
    while (i < n) {
        const int s = png_decode(r, cl);
        if (s < 0 || r.pos > nbits) return -1;
        if (s < 16) {
            lens[i++] = (uint8_t)s;
            continue;
        }
        int rep;
        uint8_t v = 0;
        if (s == 16) {
            if (i == 0) return -1;
            v = lens[i - 1];
            rep = 3 + (int)r.get(2);
        } else if (s == 17) {
            rep = 3 + (int)r.get(3);
        } else {
            rep = 11 + (int)r.get(7);
        }
        if (i + rep > n || r.pos > nbits) return -1;
        while (rep--) lens[i++] = v;
    }
    if (lens[256] == 0) return -1;                                       // no end-of-block code
    int v = png_build(lens, nlen, lit, lut, mx);
    if (v < 0 || (v > 0 && mx != 1)) return -1;
    v = png_build(lens + nlen, ndist, dist, lut, mx);
    if (v < 0 || (v > 0 && mx > 1)) return -1;                           // an empty distance code is accepted
    return 0;
}

// Fixed Huffman codes (RFC 1951 3.2.6) from the next 9 stream bits.
__device__ __forceinline__ int png_fixed_lit(PngBits& r) {
    const unsigned b = (unsigned)(r.buf & 511);
    const unsigned c7 = __brev(b & 127) >> 25;
    if (c7 <= 23) { r.skip(7); return 256 + (int)c7; }
    const unsigned c8 = __brev(b & 255) >> 24;
    if (c8 >= 48 && c8 <= 191) { r.skip(8); return (int)c8 - 48; }
    if (c8 >= 192 && c8 <= 199) { r.skip(8); return 280 + (int)c8 - 192; }
    r.skip(9);
    return 144 + (int)(__brev(b) >> 23) - 400;
}

enum { PNG_DONE = 0, PNG_ERR = 1, PNG_EXHAUSTED = 2, PNG_STOP = 3 };
enum { PNG_COUNT = 0, PNG_WALK = 1, PNG_WRITE = 2 };

// The codes of one Huffman block up to and including end-of-block.  out: the inflated bytes so far (block-relative
// in PNG_COUNT, image-relative otherwise).  PNG_WALK / PNG_WRITE stop where zlib under Pillow stops: at a literal or
// match that would write byte raw or later (after decoding the match's distance); PNG_WRITE stores bytes below raw.
template <int MODE>
__device__ __forceinline__ int png_codes(PngBits& r, int64_t nbits, bool fixed, const PngLit& lit, const PngDist& dist, int64_t& out,
                         int64_t raw, uint8_t* rows, int32_t* src, int64_t cap) {
    for (;;) {
        const int s = fixed ? png_fixed_lit(r) : png_decode(r, lit);
        if (s < 0 || s > 285) return r.pos > nbits ? PNG_EXHAUSTED : PNG_ERR;
        if (r.pos > nbits) return PNG_EXHAUSTED;
        if (s < 256) {
            if (MODE != PNG_COUNT && out >= raw) return PNG_STOP;
            if (MODE == PNG_WRITE) {
                rows[out] = (uint8_t)s;
                src[out] = (int32_t)out;
            }
            ++out;
        } else if (s == 256) {
            return PNG_DONE;
        } else {
            const int li = s - 257;
            const int len = kPngLenBase[li] + (int)r.get(kPngLenExtra[li]);
            int ds;
            if (fixed) {
                ds = (int)(__brev((unsigned)(r.buf & 31)) >> 27);
                r.skip(5);
            } else {
                ds = png_decode(r, dist);
            }
            if (ds < 0 || ds > 29) return r.pos > nbits ? PNG_EXHAUSTED : PNG_ERR;
            const int64_t d = kPngDistBase[ds] + (int)r.get(kPngDistExtra[ds]);
            if (r.pos > nbits) return PNG_EXHAUSTED;
            if (MODE != PNG_COUNT) {
                if (out >= raw) return PNG_STOP;
                if (d > out) return PNG_ERR;                             // a distance before the stream's start
            }
            if (MODE == PNG_WRITE) {
                const int64_t e = min(out + len, raw);
                for (int64_t p = out; p < e; ++p) src[p] = (int32_t)(p - d);
            }
            out += len;
        }
        if (MODE == PNG_COUNT && out > cap) return PNG_ERR;              // longer than the image: not worth a slot
    }
}

// A stored block after its 3 header bits: byte-align, LEN / NLEN, then the bytes.
template <int MODE>
__device__ __forceinline__ int png_stored(PngBits& r, int64_t nbits, int64_t& out, int64_t raw, uint8_t* rows, int32_t* src) {
    r.skip((int)((8 - (r.pos & 7)) & 7));
    const uint32_t len = r.get(16), nlen = r.get(16);
    if (r.pos > nbits) return PNG_EXHAUSTED;
    if (len != (~nlen & 0xFFFFu)) return PNG_ERR;
    if (len == 0) return PNG_DONE;
    if (out >= raw) return PNG_STOP;
    const int64_t avail = (nbits - r.pos) >> 3;
    const int64_t n = min((int64_t)len, avail);
    if (MODE == PNG_WRITE) {
        const int64_t b0 = r.pos >> 3;
        const int64_t e = min(out + n, raw);
        for (int64_t p = out; p < e; ++p) {
            rows[p] = __ldg(r.p + b0 + (p - out));
            src[p] = (int32_t)p;
        }
    }
    out += n;
    if (n < (int64_t)len) return PNG_EXHAUSTED;
    r.init(r.p, r.nbytes, r.pos + 8 * n);
    return PNG_DONE;
}

// One whole block from its header (the walker's inline decode and the write pass).
template <int MODE>
__device__ __forceinline__ int png_block(PngBits& r, int64_t nbits, int64_t& out, int64_t raw, uint8_t* rows, int32_t* src, int& type) {
    const int bfinal = (int)r.get(1), bt = (int)r.get(2);
    type = bt | (bfinal << 2);
    if (r.pos > nbits) return PNG_EXHAUSTED;
    if (bt == 3) return PNG_ERR;
    if (bt == 0) return png_stored<MODE>(r, nbits, out, raw, rows, src);
    PngLit lit;
    PngDist dist;
    if (bt == 2 && png_dynamic_header(r, nbits, lit, dist, true) != 0) return r.pos > nbits ? PNG_EXHAUSTED : PNG_ERR;
    return png_codes<MODE>(r, nbits, bt == 1, lit, dist, out, raw, rows, src, 0);
}

__host__ __device__ __forceinline__ int64_t png_raw_bytes(const cl_png_image& im) { return (int64_t)im.H * (im.rowbytes + 1); }

// The image whose candidate words contain word w.
__device__ __forceinline__ int png_image_of_word(const cl_png_image* __restrict__ img, int B, int64_t w) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (img[mid].word0 <= w) lo = mid; else hi = mid - 1;
    }
    return lo;
}

struct PngCand {
    int32_t end;      // bit after the block's end-of-block code
    int32_t flags;    // 1: decoded cleanly, 2: BFINAL
    int64_t len;      // inflated bytes
};

// ------------------------------------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(PNG_THREADS) png_init_kernel(const cl_png_image* __restrict__ img, uint8_t* rows, int32_t* src) {
    const cl_png_image& im = img[blockIdx.y];
    const int64_t n = png_raw_bytes(im);
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
        rows[im.raw_off + p] = 0;
        src[im.raw_off + p] = (int32_t)p;
    }
}

__global__ void __launch_bounds__(PNG_THREADS) png_find_kernel(const cl_png_image* __restrict__ img, int B,
                                                               const uint8_t* __restrict__ data, int64_t n_words,
                                                               uint32_t* mask, int32_t* popc) {
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t w = g >> 5;
    bool ok = false;
    if (w < n_words) {
        const cl_png_image& im = img[png_image_of_word(img, B, w)];
        const int64_t bit = (w - im.word0) * 32 + (g & 31), nbits = 8ll * im.nbytes;
        if (bit >= 16 && bit + 17 <= nbits) {
            PngBits r;
            r.init(data + im.data_off, im.nbytes, bit);
            r.skip(1);
            if (r.get(2) == 2) {
                PngLit lit;
                PngDist dist;
                ok = png_dynamic_header(r, nbits, lit, dist, false) == 0;
            }
        }
    }
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, ok);
    if ((threadIdx.x & 31) == 0 && w < n_words) {
        mask[w] = m;
        popc[w] = __popc(m);
    }
}

__global__ void __launch_bounds__(PNG_THREADS, 2) png_count_kernel(const cl_png_image* __restrict__ img, int B,
                                                                const uint8_t* __restrict__ data, int64_t n_words,
                                                                const uint32_t* __restrict__ mask,
                                                                const int32_t* __restrict__ rank, PngCand* cand) {
    for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x) {
        uint32_t m = mask[w];
        if (!m) continue;
        const cl_png_image& im = img[png_image_of_word(img, B, w)];
        const int64_t nbits = 8ll * im.nbytes, raw = png_raw_bytes(im);
        int k = rank[w] - rank[im.word0];
        while (m) {
            const int b = __ffs(m) - 1;
            m &= m - 1;
            if (k >= im.ncand) break;
            PngBits r;
            r.init(data + im.data_off, im.nbytes, (w - im.word0) * 32 + b);
            const int bfinal = (int)r.get(1);
            r.get(2);
            PngLit lit;
            PngDist dist;
            int64_t out = 0;
            int res = png_dynamic_header(r, nbits, lit, dist, true) == 0 ? PNG_DONE : PNG_ERR;
            if (res == PNG_DONE) res = png_codes<PNG_COUNT>(r, nbits, false, lit, dist, out, raw, nullptr, nullptr, raw);
            PngCand c;
            c.end = (int32_t)r.pos;
            c.flags = res == PNG_DONE ? 1 | (bfinal << 1) : 0;
            c.len = out;
            cand[im.cand0 + k] = c;
            ++k;
        }
    }
}

__global__ void png_walk_kernel(const cl_png_image* __restrict__ img, int B, const uint8_t* __restrict__ data,
                                const uint32_t* __restrict__ mask, const int32_t* __restrict__ rank,
                                const PngCand* __restrict__ cand, cl_png_block* blocks, int32_t* block_count,
                                uint32_t* adler_want, int32_t* status) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const cl_png_image& im = img[b];
    const int64_t nbits = 8ll * im.nbytes, raw = png_raw_bytes(im);
    const uint8_t* d = data + im.data_off;
    int64_t pos = 16, out = 0;
    int nb = 0, st = 0;
    bool ended = false;                       // the final block's end-of-block code was reached
    for (;;) {
        if (out > raw) break;                 // zlib stopped inside the last block
        const int64_t w = im.word0 + (pos >> 5);
        const uint32_t m = pos < nbits ? mask[w] : 0u;
        const int bit = (int)(pos & 31);
        cl_png_block e;
        e.out_off = out;
        e.start = (int32_t)pos;
        int res;
        if ((m >> bit) & 1) {
            const int k = rank[w] - rank[im.word0] + __popc(m & ((1u << bit) - 1));
            if (k < im.ncand && (cand[im.cand0 + k].flags & 1)) {
                const PngCand c = cand[im.cand0 + k];
                if (out >= raw && c.len > 0) break;
                e.type = 2 | ((c.flags & 2) << 1) | 8;
                e.out_len = c.len;
                out += c.len;
                pos = c.end;
                res = PNG_DONE;
                goto record;
            }
        }
        {
            PngBits r;
            r.init(d, im.nbytes, pos);
            int type = 0;
            res = png_block<PNG_WALK>(r, nbits, out, raw, nullptr, nullptr, type);
            e.type = type;
            e.out_len = out - e.out_off;
            pos = r.pos;
        }
    record:
        // an empty block is listed only while the slots later non-empty blocks (17 bits or more each) could need remain
        if (e.out_len > 0 || nb < im.nblk - 1 - (nbits - pos) / 17) {
            if (nb < im.nblk) blocks[im.blk0 + nb++] = e;
        }
        if (res == PNG_ERR) { st |= CL_PNG_BAD_DEFLATE; break; }
        if (res == PNG_EXHAUSTED) { if (out < raw) st |= CL_PNG_TRUNCATED; break; }
        if (res == PNG_STOP) break;
        if (e.type & 4) { ended = true; break; }
    }
    uint32_t want = 0;
    int check = 0;
    if (ended && out < raw) st |= CL_PNG_TRUNCATED;
    if (ended && out == raw) {
        const int64_t byte = (pos + 7) >> 3;
        if (byte + 4 <= im.nbytes) {
            want = ((uint32_t)d[byte] << 24) | ((uint32_t)d[byte + 1] << 16) | ((uint32_t)d[byte + 2] << 8) | d[byte + 3];
            check = 1;
        }
    }
    adler_want[2 * b] = want;
    adler_want[2 * b + 1] = (uint32_t)check;
    block_count[b] = nb;
    if (st) atomicOr(status + b, st);
}

__global__ void __launch_bounds__(PNG_THREADS, 2) png_write_kernel(const cl_png_image* __restrict__ img,
                                                                const uint8_t* __restrict__ data,
                                                                const cl_png_block* __restrict__ blocks,
                                                                const int32_t* __restrict__ block_count, uint8_t* rows,
                                                                int32_t* src, int32_t* status) {
    const int b = blockIdx.y;
    const cl_png_image& im = img[b];
    const int64_t nbits = 8ll * im.nbytes, raw = png_raw_bytes(im);
    const int n = block_count[b];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const cl_png_block e = blocks[im.blk0 + i];
        if (e.out_len == 0) continue;
        PngBits r;
        r.init(data + im.data_off, im.nbytes, e.start);
        int64_t out = e.out_off;
        int type;
        const int res = png_block<PNG_WRITE>(r, nbits, out, raw, rows + im.raw_off, src + im.raw_off, type);
        if (res == PNG_ERR) atomicOr(status + b, CL_PNG_BAD_DEFLATE);   // a distance before the stream's start
    }
}

__global__ void __launch_bounds__(PNG_THREADS) png_jump_kernel(const cl_png_image* __restrict__ img, int32_t* src) {
    const cl_png_image& im = img[blockIdx.y];
    const int64_t n = png_raw_bytes(im);
    int32_t* s = src + im.raw_off;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
        const int32_t q = s[p];
        if (q != p) s[p] = s[q];              // any value read is an ancestor of q: in place is safe
    }
}

__global__ void __launch_bounds__(PNG_THREADS) png_gather_kernel(const cl_png_image* __restrict__ img,
                                                                 const int32_t* __restrict__ src, uint8_t* rows,
                                                                 unsigned long long* adler) {
    const int b = blockIdx.y;
    const cl_png_image& im = img[b];
    const int64_t n = png_raw_bytes(im);
    uint8_t* r = rows + im.raw_off;
    const int32_t* s = src + im.raw_off;
    uint64_t s1 = 0, s2 = 0;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
        const int32_t q = s[p];
        const uint8_t v = r[q];               // a literal: never rewritten
        if (q != p) r[p] = v;
        s1 += v;
        s2 += (uint64_t)((n - p) % 65521) * v;
    }
    s1 %= 65521;
    s2 %= 65521;
    for (int o = 16; o; o >>= 1) {
        s1 += __shfl_down_sync(0xFFFFFFFFu, s1, o);
        s2 += __shfl_down_sync(0xFFFFFFFFu, s2, o);
    }
    if ((threadIdx.x & 31) == 0 && (s1 | s2)) {
        atomicAdd(adler + 2 * b, (unsigned long long)s1);
        atomicAdd(adler + 2 * b + 1, (unsigned long long)s2);
    }
}

// Rows of image blockIdx.x in place: a thread per (row in the band, byte lane), row rr handling pixel t - rr at step t.
__global__ void __launch_bounds__(PNG_UNFILTER_THREADS) png_unfilter_kernel(const cl_png_image* __restrict__ img,
                                                                           uint8_t* rows, int32_t* status) {
    __shared__ uint8_t pub[2][PNG_UNFILTER_THREADS];
    const int b = blockIdx.x;
    const cl_png_image& im = img[b];
    const int bpp = im.bpp, rb = im.rowbytes;
    const int64_t pitch = (int64_t)rb + 1;
    const int R = PNG_UNFILTER_THREADS / bpp;
    const int tid = threadIdx.x, rr = tid / bpp, lane = tid - rr * bpp;
    const int npix = (rb + bpp - 1) / bpp;
    uint8_t* base = rows + im.raw_off;
    bool bad = false;
    for (int r0 = 0; r0 < im.H; r0 += R) {
        const int r = r0 + rr;
        const bool active = rr < R && r < im.H;
        uint8_t* row = base + (int64_t)r * pitch;
        int ft = 0;
        if (active) {
            ft = row[0];
            if (ft > 4) {
                bad = true;
                ft = 0;
            }
        }
        int left = 0, upleft = 0;
        for (int t = 0; t < npix + R - 1; ++t) {
            const int x = t - rr;
            if (active && x >= 0 && x < npix) {
                const int i = x * bpp + lane;
                int up = 0;
                if (r > 0) up = rr > 0 ? pub[(t - 1) & 1][tid - bpp] : row[i + 1 - pitch];
                int v = row[i + 1];
                switch (ft) {
                case 1: v += left; break;
                case 2: v += up; break;
                case 3: v += (left + up) >> 1; break;
                case 4: {
                    const int p = left + up - upleft, pa = abs(p - left), pb = abs(p - up), pc = abs(p - upleft);
                    v += (pa <= pb && pa <= pc) ? left : (pb <= pc ? up : upleft);
                    break;
                }
                default: break;
                }
                v &= 255;
                row[i + 1] = (uint8_t)v;
                pub[t & 1][tid] = (uint8_t)v;
                left = v;
                upleft = up;
            }
            __syncthreads();
        }
    }
    if (bad) atomicOr(status + b, CL_PNG_BAD_FILTER);
}

__device__ __forceinline__ int png_l(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

__device__ __forceinline__ int png_bits(const uint8_t* row, int x, int depth) {
    const int per = 8 / depth;
    return (row[x / per] >> (8 - depth * (x % per + 1))) & ((1 << depth) - 1);
}

// Pillow's unpackers and convert: the pixel's (r, g, b) (grey and palette L from their own rules) into out.
__global__ void __launch_bounds__(256) png_unpack_kernel(const cl_png_image* __restrict__ img, const uint8_t* __restrict__ rows,
                                                         const uint8_t* __restrict__ tables, int filtered, int out_ch,
                                                         uint8_t* out, const unsigned long long* __restrict__ adler,
                                                         const uint32_t* __restrict__ adler_want, int32_t* status) {
    const int b = blockIdx.y;
    const cl_png_image& im = img[b];
    const int64_t n = (int64_t)im.H * im.W;
    const int64_t pitch = (int64_t)im.rowbytes + filtered;
    const uint8_t* pal = tables + im.pal_off;
    uint8_t* o = out + im.out_off;
    const int ct = im.color_type, dep = im.depth;
    if (adler && blockIdx.x == 0 && threadIdx.x == 0 && adler_want[2 * b + 1]) {
        const uint64_t raw = (uint64_t)png_raw_bytes(im);
        const uint32_t a = (uint32_t)((1 + adler[2 * b]) % 65521), s = (uint32_t)((raw % 65521 + adler[2 * b + 1]) % 65521);
        if (((s << 16) | a) != adler_want[2 * b]) atomicOr(status + b, CL_PNG_BAD_ADLER);
    }
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / im.W), x = (int)(i - (int64_t)y * im.W);
        const uint8_t* row = rows + im.raw_off + (int64_t)y * pitch + filtered;
        int R, G, Bc, L = -1;
        if (ct == 0 || ct == 4) {
            int g;
            const int spp = ct == 0 ? 1 : 2;
            if (dep == 16) g = ct == 0 ? min(((int)row[2 * x] << 8) | row[2 * x + 1], 255) : row[4 * x];   // I;16 clips
            else if (dep == 8) g = row[spp * x];
            else g = png_bits(row, x, dep) * (dep == 1 ? 255 : dep == 2 ? 85 : 17);
            R = G = Bc = L = g;
        } else if (ct == 3) {
            const int k = dep == 8 ? row[x] : png_bits(row, x, dep);
            R = pal[3 * k];
            G = pal[3 * k + 1];
            Bc = pal[3 * k + 2];
        } else {
            const int spp = ct == 2 ? 3 : 4, bs = dep / 8;   // 16-bit samples keep their high byte
            R = row[(spp * x) * bs];
            G = row[(spp * x + 1) * bs];
            Bc = row[(spp * x + 2) * bs];
        }
        if (out_ch == 3) {
            o[3 * i] = (uint8_t)R;
            o[3 * i + 1] = (uint8_t)G;
            o[3 * i + 2] = (uint8_t)Bc;
        } else {
            o[i] = (uint8_t)(L >= 0 ? L : png_l(R, G, Bc));
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
struct PngScratch {
    size_t mask, popc, rank, cand, rows, src, adler, want, temp, total, temp_bytes;
};

static size_t png_align(size_t v) { return (v + 255) & ~(size_t)255; }

static int png_layout(int64_t words, int64_t cand_slots, int64_t raw, int B, PngScratch& L) {
    size_t t = 0;
    CL_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, t, (const int32_t*)nullptr, (int32_t*)nullptr, (int)words));
    size_t off = 0;
    L.mask = off; off = png_align(off + (size_t)words * 4);
    L.popc = off; off = png_align(off + (size_t)words * 4);
    L.rank = off; off = png_align(off + (size_t)words * 4);
    L.cand = off; off = png_align(off + (size_t)cand_slots * sizeof(PngCand));
    L.rows = off; off = png_align(off + (size_t)raw);
    L.src = off; off = png_align(off + (size_t)raw * 4);
    L.adler = off; off = png_align(off + (size_t)B * 16);
    L.want = off; off = png_align(off + (size_t)B * 8);
    L.temp = off;
    L.temp_bytes = t;
    L.total = png_align(off + t);
    return CL_OK;
}

static bool png_depth_ok(int ct, int d) {
    switch (ct) {
    case 0: return d == 1 || d == 2 || d == 4 || d == 8 || d == 16;
    case 3: return d == 1 || d == 2 || d == 4 || d == 8;
    case 2: case 4: case 6: return d == 8 || d == 16;
    default: return false;
    }
}

static int png_samples(int ct) { return ct == 2 ? 3 : ct == 4 ? 2 : ct == 6 ? 4 : 1; }

// Checks shared by decode and convert: sizes, formats, output windows.
static int png_check_images(const char* what, const cl_png_image* img, int B, int out_channels, int64_t out_bytes) {
    if (B <= 0 || B > 65535) return set_error(CL_ERR_INVALID, "%s: B = %d, expected 1..65535", what, B);
    if (out_channels != 1 && out_channels != 3)
        return set_error(CL_ERR_INVALID, "%s: out_channels = %d, expected 1 (L) or 3 (RGB)", what, out_channels);
    int64_t out_end = 0;
    for (int b = 0; b < B; ++b) {
        const cl_png_image& d = img[b];
        if (d.H <= 0 || d.W <= 0 || d.H > CL_PNG_MAX_SIDE || d.W > CL_PNG_MAX_SIDE)
            return set_error(CL_ERR_INVALID, "%s: image %d: size %d x %d outside 1..%d", what, b, d.W, d.H, CL_PNG_MAX_SIDE);
        if (!png_depth_ok(d.color_type, d.depth))
            return set_error(CL_ERR_INVALID, "%s: image %d: colour type %d with bit depth %d", what, b, d.color_type, d.depth);
        const int bits = png_samples(d.color_type) * d.depth;
        if (d.rowbytes != (int)(((int64_t)d.W * bits + 7) / 8) || d.bpp != std::max(1, bits / 8))
            return set_error(CL_ERR_INVALID, "%s: image %d: rowbytes %d / bpp %d do not fit %d x %d-bit pixels", what, b, d.rowbytes,
                             d.bpp, d.W, bits);
        if ((int64_t)d.H * (d.rowbytes + 1) >= (1ll << 31))
            return set_error(CL_ERR_INVALID, "%s: image %d: %lld inflated bytes (limit 2^31 - 1)", what, b,
                             (long long)d.H * (d.rowbytes + 1));
        const int64_t n = (int64_t)d.H * d.W * out_channels;
        if (d.out_off < out_end || d.out_off + n > out_bytes)
            return set_error(CL_ERR_INVALID, "%s: image %d: output %lld + %lld overlaps image %d or lies outside the %lld-byte output",
                             what, b, (long long)d.out_off, (long long)n, b - 1, (long long)out_bytes);
        out_end = d.out_off + n;
    }
    return CL_OK;
}

static int png_grid(int64_t n, int threads) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, (int64_t)num_sms() * 8)); }

}  // namespace clb

using namespace clb;

extern "C" int64_t cl_png_scratch_bytes(int64_t words, int64_t cand_slots, int64_t raw_bytes, int B) {
    if (words <= 0 || words >= (1ll << 31) || cand_slots <= 0 || raw_bytes <= 0 || B <= 0)
        return set_error(CL_ERR_INVALID, "cl_png_scratch_bytes: %lld words, %lld candidate slots, %lld inflated bytes, B = %d",
                         (long long)words, (long long)cand_slots, (long long)raw_bytes, B);
    PngScratch L;
    CL_CHECK(png_layout(words, cand_slots, raw_bytes, B, L));
    return (int64_t)L.total;
}

extern "C" int cl_png_decode(const cl_png_image* img, const cl_png_image* img_dev, int B, const uint8_t* data, int64_t data_bytes,
                             const uint8_t* tables, int64_t table_bytes, void* scratch, int64_t scratch_bytes, cl_png_block* blocks,
                             int64_t n_block_slots, int32_t* block_count, int out_channels, uint8_t* out, int64_t out_bytes,
                             int32_t* status, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!img || !img_dev || !data || !tables || !scratch || !blocks || !block_count || !out || !status)
        return set_error(CL_ERR_INVALID, "cl_png_decode: null img, img_dev, data, tables, scratch, blocks, block_count, out or status");
    CL_CHECK(png_check_images("cl_png_decode", img, B, out_channels, out_bytes));
    int64_t words = 0, cands = 0, raw = 0, blks = 0, max_raw = 1;
    for (int b = 0; b < B; ++b) {
        const cl_png_image& d = img[b];
        if (d.nbytes < 2 || d.nbytes >= CL_PNG_MAX_STREAM_BYTES || d.data_off < 0 || d.data_off + d.nbytes > data_bytes)
            return set_error(CL_ERR_INVALID, "cl_png_decode: image %d: %d stream bytes at %lld outside the %lld-byte data", b, d.nbytes,
                             (long long)d.data_off, (long long)data_bytes);
        if (d.color_type == 3 ? (d.pal_off < 0 || d.pal_off + 768ll > table_bytes) : d.pal_off != 0)
            return set_error(CL_ERR_INVALID, "cl_png_decode: image %d: palette at %d outside the %lld-byte tables", b, d.pal_off,
                             (long long)table_bytes);
        if (d.word0 != words || d.cand0 != cands || d.blk0 != blks || d.raw_off != raw || d.ncand != d.nbytes / 8 + 16 ||
            d.nblk != d.nbytes / 2 + 64)
            return set_error(CL_ERR_INVALID, "cl_png_decode: image %d: words %d, candidates [%d, +%d), blocks [%d, +%d), rows at %lld "
                             "are not the back to back ranges of the batch", b, d.word0, d.cand0, d.ncand, d.blk0, d.nblk,
                             (long long)d.raw_off);
        words += (d.nbytes + 3) / 4;
        cands += d.ncand;
        blks += d.nblk;
        raw += png_raw_bytes(d);
        max_raw = std::max<int64_t>(max_raw, png_raw_bytes(d));
    }
    if (words >= (1ll << 31) / 32 || blks > n_block_slots)
        return set_error(CL_ERR_INVALID, "cl_png_decode: %lld candidate words, %lld block slots of %lld", (long long)words,
                         (long long)blks, (long long)n_block_slots);
    PngScratch L;
    CL_CHECK(png_layout(words, cands, raw, B, L));
    if ((int64_t)L.total > scratch_bytes)
        return set_error(CL_ERR_INVALID, "cl_png_decode: scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)L.total);

    char* sp = static_cast<char*>(scratch);
    uint32_t* mask = reinterpret_cast<uint32_t*>(sp + L.mask);
    int32_t* popc = reinterpret_cast<int32_t*>(sp + L.popc);
    int32_t* rank = reinterpret_cast<int32_t*>(sp + L.rank);
    PngCand* cand = reinterpret_cast<PngCand*>(sp + L.cand);
    uint8_t* rows = reinterpret_cast<uint8_t*>(sp + L.rows);
    int32_t* src = reinterpret_cast<int32_t*>(sp + L.src);
    unsigned long long* adler = reinterpret_cast<unsigned long long*>(sp + L.adler);
    uint32_t* want = reinterpret_cast<uint32_t*>(sp + L.want);

    CL_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int32_t) * B, stream));
    CL_CUDA_CHECK(cudaMemsetAsync(adler, 0, 16ull * B, stream));
    const int gx = png_grid(max_raw, PNG_THREADS);
    launch_k(png_init_kernel, dim3(gx, B), PNG_THREADS, 0, stream, img_dev, rows, src);
    launch_k(png_find_kernel, dim3((unsigned)((words * 32 + PNG_THREADS - 1) / PNG_THREADS)), PNG_THREADS, 0, stream, img_dev, B,
             data, words, mask, popc);
    size_t tb = L.temp_bytes;
    CL_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(sp + L.temp, tb, (const int32_t*)popc, rank, (int)words, stream));
    launch_k(png_count_kernel, dim3(png_grid(words, PNG_THREADS)), PNG_THREADS, 0, stream, img_dev, B, data, words,
             (const uint32_t*)mask, (const int32_t*)rank, cand);
    launch_k(png_walk_kernel, dim3((B + 31) / 32), 32, 0, stream, img_dev, B, data, (const uint32_t*)mask, (const int32_t*)rank,
             (const PngCand*)cand, blocks, block_count, want, status);
    launch_k(png_write_kernel, dim3(8, B), PNG_THREADS, 0, stream, img_dev, data, (const cl_png_block*)blocks,
             (const int32_t*)block_count, rows, src, status);
    int rounds = 0;
    while ((1ll << rounds) < max_raw) ++rounds;
    for (int k = 0; k < rounds; ++k) launch_k(png_jump_kernel, dim3(gx, B), PNG_THREADS, 0, stream, img_dev, src);
    launch_k(png_gather_kernel, dim3(gx, B), PNG_THREADS, 0, stream, img_dev, (const int32_t*)src, rows, adler);
    launch_k(png_unfilter_kernel, dim3(B), PNG_UNFILTER_THREADS, 0, stream, img_dev, rows, status);
    int64_t max_px = 1;
    for (int b = 0; b < B; ++b) max_px = std::max<int64_t>(max_px, (int64_t)img[b].H * img[b].W);
    launch_k(png_unpack_kernel, dim3(png_grid(max_px, 256), B), 256, 0, stream, img_dev, (const uint8_t*)rows, tables, 1,
             out_channels, out, (const unsigned long long*)adler, (const uint32_t*)want, status);
    count_launch(10 + rounds);
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

extern "C" int cl_png_convert(const cl_png_image* img, const cl_png_image* img_dev, int B, const uint8_t* src, int64_t src_bytes,
                              int out_channels, uint8_t* out, int64_t out_bytes, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!img || !img_dev || !src || !out) return set_error(CL_ERR_INVALID, "cl_png_convert: null img, img_dev, src or out");
    CL_CHECK(png_check_images("cl_png_convert", img, B, out_channels, out_bytes));
    int64_t max_px = 1;
    for (int b = 0; b < B; ++b) {
        const cl_png_image& d = img[b];
        if ((d.color_type != 0 && d.color_type != 2) || d.depth != 8)
            return set_error(CL_ERR_INVALID, "cl_png_convert: image %d: colour type %d, depth %d (8-bit grey or RGB only)", b,
                             d.color_type, d.depth);
        if (d.raw_off < 0 || d.raw_off + (int64_t)d.H * d.rowbytes > src_bytes)
            return set_error(CL_ERR_INVALID, "cl_png_convert: image %d: rows at %lld outside the %lld-byte source", b,
                             (long long)d.raw_off, (long long)src_bytes);
        max_px = std::max<int64_t>(max_px, (int64_t)d.H * d.W);
    }
    launch_k(png_unpack_kernel, dim3(png_grid(max_px, 256), B), 256, 0, stream, img_dev, src, src, 0, out_channels, out,
             (const unsigned long long*)nullptr, (const uint32_t*)nullptr, (int32_t*)nullptr);
    count_launch(1);
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
