// Baseline JPEG decoder for a ragged batch, bit for bit with Pillow's libjpeg-turbo (default settings): sequential
// Huffman, 8-bit samples, one scan, grayscale or YCbCr 4:4:4 / 4:2:2 / 4:2:0, restart intervals.  The rules are
// restated in oracle/jpeg_ref.py; the host (controllora_b200/jpeg.py) parses the markers, refuses what is not decoded
// here, builds the Huffman lookup tables and removes the byte stuffing.
//
// The entropy-coded data of each restart segment is cut into windows of JPEG_WINDOW_BITS bits, one thread each, and
// decoded by self-synchronising subsequences (Weissenberger & Schmidt, ICPP 2018; PAPERS.md).  The decoder state
// between two symbols is (bit position, zig-zag index, block within the MCU); a window's end state is the state at
// the first symbol boundary at or past its last bit.  Launches, all of them whatever the data, no host synchronisation:
//   0. cudaMemsetAsync: the coefficient blocks and the DC differences to zero.
//   1. jpeg_sync_kernel (cooperative): every window decodes from the guess (its first bit, index 0, block 0) - exact
//      for a segment's first window - and records its end state.  Then rounds: a window whose predecessor's end state
//      changed in the last round decodes again from it, and while its own end state changes it goes on into the next
//      window of the segment.  A round in which nothing changes leaves every recorded state a fixpoint, which is the
//      sequential decoder's state; windows whose predecessors are all exact never change again, so at most one round
//      per window is needed however long the decoders take to lock in (flat and periodic images), and usually two or
//      three.  Finally each window counts the blocks that start in it.
//   2. cub::DeviceScan::ExclusiveSum of the counts: the scan index of each window's first block.
//   3. jpeg_write_kernel: each window decodes from its exact start state and writes the coefficients of the blocks
//      that start in it (finishing the last one past its end) and the DC differences, grouped per segment and component.
//      Corrupt data (an invalid code, a coefficient index past 63, a segment that ends before its last block) sets the
//      image's status; only the sequential decoder's path reports, never a window's guess.
//   4. cub::DeviceScan::InclusiveSum of the DC differences (uint32, wrapping): a group's DC values are the differences
//      from the sum before the group, and only their low 16 bits are kept, as libjpeg stores (JCOEF) last_dc_val.
//   5. jpeg_idct_kernel: dequantisation and jpeg_idct_islow per block into the component planes, with the 16-bit
//      lanes of libjpeg-turbo's SIMD IDCT that Pillow runs.
//   6. jpeg_color_kernel: fancy upsampling (h2v1 / h2v2) and the YCbCr -> RGB tables into the packed uint8 output.
// Reads of the entropy-coded data are bounded by each segment's length (bytes past it read as zero bits, as libjpeg
// inserts them), coefficient writes by the segment's block count, pixel writes by the image's output window.
#include <cooperative_groups.h>
#include <stdio.h>

#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace cg = cooperative_groups;

namespace clb {

constexpr int JPEG_THREADS = 128;
constexpr int JPEG_HUFF_WORDS = 810;     // 9-bit lookup [512], maxcode [17], valoff [17], values [256], pad [8]
constexpr int JPEG_MAX_SIDE = 16384;

__constant__ int kJpegNatural[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
    62, 63};

// ------------------------------------------------------------------------------------------------ bit reader
struct JpegBits {
    const uint8_t* p;
    int64_t nbytes, next;   // segment length, next byte to load
    uint64_t buf;           // MSB-aligned look-ahead
    int valid;              // bits in buf
    int64_t pos;            // bit position of buf's first bit in the segment

    __device__ __forceinline__ void fill() {
        while (valid <= 56) {
            const uint64_t b = next < nbytes ? (uint64_t)__ldg(p + next) : 0ull;
            buf |= b << (56 - valid);
            valid += 8;
            ++next;
        }
    }
    __device__ __forceinline__ void init(const uint8_t* p_, int64_t n, int64_t bitpos) {
        p = p_; nbytes = n; next = bitpos >> 3; buf = 0; valid = 0; pos = bitpos;
        fill();
        const int s = (int)(bitpos & 7);
        buf <<= s;
        valid -= s;
    }
    __device__ __forceinline__ void skip(int n) {
        buf <<= n;
        valid -= n;
        pos += n;
        if (valid < 32) fill();
    }
    __device__ __forceinline__ int get(int n) {   // n in 0..15
        const int v = n ? (int)(buf >> (64 - n)) : 0;
        skip(n);
        return v;
    }
};

// Huffman symbol of the next bits (c16 = the next 16), or -1 for an invalid code (jdhuff.c jpeg_huff_decode).
__device__ __forceinline__ int jpeg_huff(const int32_t* __restrict__ t, uint32_t c16, int& len) {
    const int e = __ldg(t + (c16 >> 7));
    if (e) {
        len = e >> 8;
        return e & 255;
    }
#pragma unroll 1
    for (int l = 10; l <= 16; ++l) {
        const int code = (int)(c16 >> (16 - l));
        if (code <= __ldg(t + 512 + l)) {
            len = l;
            return __ldg(t + 546 + ((code + __ldg(t + 529 + l)) & 255));
        }
    }
    len = 1;
    return -1;
}

__device__ __forceinline__ int jpeg_extend(int v, int s) { return (s && v < (1 << (s - 1))) ? v - (1 << s) + 1 : v; }

struct JpegTabs {
    const int32_t* dc[6];
    const int32_t* ac[6];
    int bpm;
};

__device__ __forceinline__ void jpeg_tabs(const cl_jpeg_image& im, const int32_t* __restrict__ tables, JpegTabs& T) {
    T.bpm = im.bpm;
    const int ny = im.C == 1 ? 1 : im.hmax * im.vmax;
    for (int k = 0; k < 6; ++k) {
        const int c = k < ny ? 0 : (k == ny ? 1 : 2);
        const int cc = im.C == 1 ? 0 : c;
        T.dc[k] = tables + im.dc_tab[cc];
        T.ac[k] = tables + im.ac_tab[cc];
    }
}

// One symbol: a DC difference when zz == 0, else one AC run / size or EOB / ZRL.  Advances (bits, zz, blk); k = the
// zig-zag index of the coefficient produced (0: DC difference) or -1.  Returns the CL_JPEG_* error of the symbol (the
// decode goes on deterministically: an invalid code skips one bit, an index past 63 ends the block).
__device__ __forceinline__ int jpeg_symbol(JpegBits& r, int& zz, int& blk, const JpegTabs& T, int& k, int& v) {
    k = -1;
    const uint32_t c16 = (uint32_t)(r.buf >> 48);
    int len;
    if (zz == 0) {
        const int s = jpeg_huff(T.dc[blk], c16, len);
        if (s < 0) {
            r.skip(1);
            return CL_JPEG_BAD_CODE;
        }
        r.skip(len);
        v = jpeg_extend(r.get(s), s);
        k = 0;
        zz = 1;
        return 0;
    }
    const int rs = jpeg_huff(T.ac[blk], c16, len);
    if (rs < 0) {
        r.skip(1);
        return CL_JPEG_BAD_CODE;
    }
    r.skip(len);
    const int run = rs >> 4, s = rs & 15;
    int err = 0;
    if (s) {
        const int kk = zz + run;
        const int bits = r.get(s);
        if (kk > 63) {
            err = CL_JPEG_BAD_INDEX;
            zz = 64;
        } else {
            k = kk;
            v = jpeg_extend(bits, s);
            zz = kk + 1;
        }
    } else {
        zz = run == 15 ? zz + 16 : 64;
    }
    if (zz >= 64) {
        zz = 0;
        blk = blk + 1 == T.bpm ? 0 : blk + 1;
    }
    return err;
}

__device__ __forceinline__ uint64_t jpeg_pack(int64_t pos, int zz, int blk) {
    return ((uint64_t)pos << 16) | ((uint64_t)zz << 8) | (uint64_t)blk;
}

// The segment of window w (segments hold contiguous window ranges in order).
__device__ __forceinline__ int jpeg_seg_of(const cl_jpeg_segment* __restrict__ seg, int n_seg, int w) {
    int lo = 0, hi = n_seg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (seg[mid].win0 <= w) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Decode window w from `start` until the first symbol boundary at or past its end: the end state (and, when count is
// given, the number of blocks that start in the window).
__device__ uint64_t jpeg_run_window(const cl_jpeg_segment& S, const JpegTabs& T, const uint8_t* __restrict__ data, int w,
                                    uint64_t start, int* count) {
    const int64_t wend = (int64_t)(w - S.win0 + 1) * CL_JPEG_WINDOW_BITS;
    JpegBits r;
    r.init(data + S.data_off, S.nbytes, (int64_t)(start >> 16));
    int zz = (int)((start >> 8) & 255), blk = (int)(start & 255);
    int n = 0, k, v;
    while (r.pos < wend) {
        n += zz == 0;
        jpeg_symbol(r, zz, blk, T, k, v);
    }
    if (count) *count = n;
    return jpeg_pack(r.pos, zz, blk);
}

__global__ void __launch_bounds__(JPEG_THREADS) jpeg_sync_kernel(const cl_jpeg_image* __restrict__ img, int B,
                                                                 const cl_jpeg_segment* __restrict__ seg, int n_seg,
                                                                 const int32_t* __restrict__ tables,
                                                                 const uint8_t* __restrict__ data, int n_windows,
                                                                 uint64_t* state, int32_t* stamp, int32_t* count,
                                                                 int32_t* flags, int32_t* status, int32_t* rounds_out) {
    cg::grid_group grid = cg::this_grid();
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int nthr = gridDim.x * blockDim.x;
    for (int b = tid; b < B; b += nthr) status[b] = img[b].status0;
    if (tid == 0) flags[1] = 0;
    JpegTabs T;
    for (int w = tid; w < n_windows; w += nthr) {           // the guess: the window's first bit, index 0, block 0
        const cl_jpeg_segment& S = seg[jpeg_seg_of(seg, n_seg, w)];
        jpeg_tabs(img[S.image], tables, T);
        const uint64_t guess = jpeg_pack((int64_t)(w - S.win0) * CL_JPEG_WINDOW_BITS, 0, 0);
        __stcg(state + w, jpeg_run_window(S, T, data, w, guess, nullptr));
        __stcg(stamp + w, 0);
    }
    grid.sync();
    int round = 0;
    for (;;) {
        ++round;
        if (tid == 0) flags[(round + 1) % 3] = 0;
        bool changed = false;
        for (int w = tid; w < n_windows; w += nthr) {
            const cl_jpeg_segment& S = seg[jpeg_seg_of(seg, n_seg, w)];
            if (w == S.win0 || __ldcg(stamp + w - 1) != round - 1) continue;
            jpeg_tabs(img[S.image], tables, T);
            uint64_t st = __ldcg(state + w - 1);
            for (int u = w; u < S.win0 + S.nwin; ++u) {       // while the end state changes, go on into the next window
                const uint64_t e = jpeg_run_window(S, T, data, u, st, nullptr);
                if (e == __ldcg(state + u)) break;
                __stcg(state + u, e);
                __stcg(stamp + u, round);
                changed = true;
                st = e;
            }
        }
        if (__syncthreads_or(changed) && threadIdx.x == 0) atomicAdd(flags + round % 3, 1);
        grid.sync();
        if (*(volatile int32_t*)(flags + round % 3) == 0 || round > n_windows) break;
    }
    for (int w = tid; w < n_windows; w += nthr) {
        const cl_jpeg_segment& S = seg[jpeg_seg_of(seg, n_seg, w)];
        jpeg_tabs(img[S.image], tables, T);
        int n;
        jpeg_run_window(S, T, data, w, w == S.win0 ? 0ull : __ldcg(state + w - 1), &n);
        count[w] = n;
    }
    if (tid == 0 && rounds_out) *rounds_out = round;
}

// Component layout of block k of an MCU: (component, its first block in the MCU, its blocks per MCU).
__device__ __forceinline__ void jpeg_block_comp(const cl_jpeg_image& im, int k, int& c, int& off, int& nb) {
    const int ny = im.C == 1 ? 1 : im.hmax * im.vmax;
    if (k < ny) { c = 0; off = 0; nb = ny; }
    else { c = k - ny + 1; off = k; nb = 1; }
}

__global__ void __launch_bounds__(JPEG_THREADS) jpeg_write_kernel(const cl_jpeg_image* __restrict__ img,
                                                                  const cl_jpeg_segment* __restrict__ seg, int n_seg,
                                                                  const int32_t* __restrict__ tables,
                                                                  const uint8_t* __restrict__ data, int n_windows,
                                                                  const uint64_t* __restrict__ state,
                                                                  const int32_t* __restrict__ base, int16_t* coef,
                                                                  uint32_t* dc, int32_t* status) {
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < n_windows; w += gridDim.x * blockDim.x) {
        const cl_jpeg_segment& S = seg[jpeg_seg_of(seg, n_seg, w)];
        const cl_jpeg_image& im = img[S.image];
        JpegTabs T;
        jpeg_tabs(im, tables, T);
        const uint64_t st = w == S.win0 ? 0ull : state[w - 1];
        const bool last = w == S.win0 + S.nwin - 1;
        const int64_t wend = last ? INT64_MAX : (int64_t)(w - S.win0 + 1) * CL_JPEG_WINDOW_BITS;
        const int64_t nbits = 8ll * S.nbytes, nbl = (int64_t)S.nmcu * im.bpm;
        JpegBits r;
        r.init(data + S.data_off, S.nbytes, (int64_t)(st >> 16));
        int zz = (int)((st >> 8) & 255), blk = (int)(st & 255);
        int64_t bi = base[w] - base[S.win0], cur = -1;
        int c = 0, off = 0, nb = 1;
        int64_t m = 0;
        int err = 0;
        for (;;) {
            if (zz == 0) {
                if (r.pos >= wend || bi >= nbl) break;
                cur = bi++;
                m = cur / im.bpm;
                jpeg_block_comp(im, (int)(cur - m * im.bpm), c, off, nb);
            }
            int k, v;
            err = jpeg_symbol(r, zz, blk, T, k, v);
            if (cur < 0) continue;                     // the tail of a block the previous window writes
            if (!err && r.pos > nbits) err = CL_JPEG_TRUNCATED;
            if (err) break;
            if (k == 0) {
                const int kk = (int)(cur - m * im.bpm);
                dc[S.block0 + (int64_t)off * S.nmcu + m * nb + (kk - off)] = (uint32_t)v;
            } else if (k > 0) {
                coef[(S.block0 + cur) * 64 + kJpegNatural[k]] = (int16_t)v;
            }
        }
        if (err) atomicOr(status + S.image, err);
    }
}

// jpeg_idct_islow as libjpeg-turbo's x86-64 SIMD code computes it (jidctint-sse2 / -avx2, what Pillow runs), which out
// of range differs from the C code: dequantisation keeps the low 16 bits of the product (pmullw), the sums x0 +- x4,
// x7 + x3 and x5 + x1 wrap at 16 bits (paddw), the pair products and their sums are 32-bit (pmaddwd, paddd), each pass's
// descaled outputs saturate to 16 bits (packssdw) and the result to -128..127 before the level shift (packsswb).  The
// 32-bit sums are formed in unsigned arithmetic so that they wrap as the lanes do.  Restated in oracle/jpeg_ref.py.
constexpr int F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373, F1_175 = 9633, F1_501 = 12299,
              F1_847 = 15137, F1_961 = 16069, F2_053 = 16819, F2_562 = 20995, F3_072 = 25172;

__device__ __forceinline__ int jpeg_w16(int v) { return (int)(int16_t)(uint16_t)(uint32_t)v; }
__device__ __forceinline__ int jpeg_add(int a, int b) { return (int)((uint32_t)a + (uint32_t)b); }
__device__ __forceinline__ int jpeg_sub(int a, int b) { return (int)((uint32_t)a - (uint32_t)b); }

// One pass over 16-bit inputs x: outputs saturate(((sum + 2^(shift-1)) >> shift), 16 bits).
template <int SHIFT>
__device__ __forceinline__ void jpeg_idct_1d(const int x[8], int o[8]) {
    const int tmp3 = jpeg_add(x[2] * (F0_541 + F0_765), x[6] * F0_541);
    const int tmp2 = jpeg_add(x[2] * F0_541, x[6] * (F0_541 - F1_847));
    const int tmp0 = jpeg_w16(x[0] + x[4]) * 8192, tmp1 = jpeg_w16(x[0] - x[4]) * 8192;
    const int t10 = jpeg_add(tmp0, tmp3), t13 = jpeg_sub(tmp0, tmp3), t11 = jpeg_add(tmp1, tmp2), t12 = jpeg_sub(tmp1, tmp2);
    const int z3 = jpeg_w16(x[7] + x[3]), z4 = jpeg_w16(x[5] + x[1]);
    const int Z3 = jpeg_add(z3 * (F1_175 - F1_961), z4 * F1_175), Z4 = jpeg_add(z3 * F1_175, z4 * (F1_175 - F0_390));
    const int o0 = jpeg_add(jpeg_add(x[7] * (F0_298 - F0_899), x[1] * -F0_899), Z3);
    const int o3 = jpeg_add(jpeg_add(x[7] * -F0_899, x[1] * (F1_501 - F0_899)), Z4);
    const int o1 = jpeg_add(jpeg_add(x[5] * (F2_053 - F2_562), x[3] * -F2_562), Z4);
    const int o2 = jpeg_add(jpeg_add(x[5] * -F2_562, x[3] * (F3_072 - F2_562)), Z3);
    const int v[8] = {jpeg_add(t10, o3), jpeg_add(t11, o2), jpeg_add(t12, o1), jpeg_add(t13, o0),
                      jpeg_sub(t13, o0), jpeg_sub(t12, o1), jpeg_sub(t11, o2), jpeg_sub(t10, o3)};
#pragma unroll
    for (int r = 0; r < 8; ++r) o[r] = min(max(jpeg_add(v[r], 1 << (SHIFT - 1)) >> SHIFT, -32768), 32767);
}

__device__ __forceinline__ uint32_t jpeg_level_shift(int v) { return (uint32_t)(min(max(v, -128), 127) + 128); }

__global__ void __launch_bounds__(JPEG_THREADS) jpeg_idct_kernel(const cl_jpeg_image* __restrict__ img,
                                                                 const cl_jpeg_segment* __restrict__ seg,
                                                                 const int32_t* __restrict__ tables,
                                                                 const int16_t* __restrict__ coef,
                                                                 const uint32_t* __restrict__ dcsum, uint8_t* plane) {
    const cl_jpeg_image& im = img[blockIdx.y];
    int64_t nblk[3] = {0, 0, 0}, total = 0;
    for (int c = 0; c < im.C; ++c) {
        nblk[c] = (int64_t)(im.pitch[c] >> 3) * ((im.ch[c] + 7) >> 3);
        total += nblk[c];
    }
    const int ny = im.C == 1 ? 1 : im.hmax * im.vmax;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int c = 0;
        int64_t j = i;
        while (j >= nblk[c]) j -= nblk[c++];
        const int nbx = im.pitch[c] >> 3;
        const int bx = (int)(j % nbx), by = (int)(j / nbx);
        const int h = c == 0 && im.C == 3 ? im.hmax : 1, v = c == 0 && im.C == 3 ? im.vmax : 1;
        const int off = c == 0 ? 0 : ny + c - 1, nb = c == 0 ? ny : 1;
        const int k = off + (by % v) * h + bx % h;
        const int64_t mcu = (int64_t)(by / v) * im.mcux + bx / h;
        const int s = im.ri ? (int)(mcu / im.ri) : 0;
        if (s >= im.nseg) continue;
        const cl_jpeg_segment& S = seg[im.seg0 + s];
        const int64_t ml = mcu - S.mcu0;
        const int64_t gs = S.block0 + (int64_t)off * S.nmcu;
        const uint32_t dcv = dcsum[gs + ml * nb + (k - off)] - (gs > 0 ? dcsum[gs - 1] : 0u);
        const int16_t* cp = coef + (S.block0 + ml * im.bpm + k) * 64;
        const int32_t* q = tables + im.qt[c];
        int ws[64];
        bool ac_rows = false;                          // any coefficient in rows 1-7: the full column pass
#pragma unroll
        for (int n = 8; n < 64; ++n) ac_rows |= cp[n] != 0;
#pragma unroll
        for (int col = 0; col < 8; ++col) {
            int x[8], o[8];
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const int n = r * 8 + col;
                const int cv = n == 0 ? (int)(int16_t)(dcv & 0xFFFF) : (int)cp[n];
                x[r] = jpeg_w16((int)((uint32_t)cv * (uint32_t)__ldg(q + n)));
            }
            if (ac_rows) {
                jpeg_idct_1d<11>(x, o);
            } else {                                   // rows 1-7 zero: the DC row shifted left by 2 in 16 bits
#pragma unroll
                for (int r = 0; r < 8; ++r) o[r] = jpeg_w16(x[0] * 4);
            }
#pragma unroll
            for (int r = 0; r < 8; ++r) ws[r * 8 + col] = o[r];
        }
        uint8_t* dst = plane + im.plane_off + im.comp_plane[c] + (int64_t)by * 8 * im.pitch[c] + bx * 8;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            int o[8];
            jpeg_idct_1d<18>(ws + r * 8, o);
            uint2 packed;
            packed.x = jpeg_level_shift(o[0]) | jpeg_level_shift(o[1]) << 8 | jpeg_level_shift(o[2]) << 16 |
                       jpeg_level_shift(o[3]) << 24;
            packed.y = jpeg_level_shift(o[4]) | jpeg_level_shift(o[5]) << 8 | jpeg_level_shift(o[6]) << 16 |
                       jpeg_level_shift(o[7]) << 24;
            *reinterpret_cast<uint2*>(dst + (int64_t)r * im.pitch[c]) = packed;
        }
    }
}

// Chroma sample at output pixel (y, x): h2v1 / h2v2 fancy upsampling of jdsample.c at the component's own size (edges
// replicated), or replication when the component is at most 2 samples wide (libjpeg-turbo's plain upsampler there).
__device__ __forceinline__ int jpeg_chroma(const uint8_t* __restrict__ p, int pitch, int ch, int cw, int hmax, int vmax,
                                           int y, int x) {
    if (hmax == 1) return p[(int64_t)y * pitch + x];
    const int i = x >> 1;
    if (cw <= 2) return p[(int64_t)(vmax == 2 ? y >> 1 : y) * pitch + i];
    const int in = (x & 1) ? min(i + 1, cw - 1) : max(i - 1, 0);
    if (vmax == 1) {
        const uint8_t* row = p + (int64_t)y * pitch;
        return (x & 1) ? (3 * row[i] + row[in] + 2) >> 2 : (3 * row[i] + row[in] + 1) >> 2;
    }
    const int j = y >> 1;
    const int jn = (y & 1) ? min(j + 1, ch - 1) : max(j - 1, 0);
    const uint8_t* r0 = p + (int64_t)j * pitch;
    const uint8_t* r1 = p + (int64_t)jn * pitch;
    const int cs = 3 * r0[i] + r1[i], csn = 3 * r0[in] + r1[in];
    return (x & 1) ? (3 * cs + csn + 7) >> 4 : (3 * cs + csn + 8) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color_kernel(const cl_jpeg_image* __restrict__ img,
                                                         const uint8_t* __restrict__ plane, uint8_t* out) {
    const cl_jpeg_image& im = img[blockIdx.y];
    const int64_t n = (int64_t)im.H * im.W;
    const uint8_t* py = plane + im.plane_off + im.comp_plane[0];
    uint8_t* o = out + im.out_off;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / im.W), x = (int)(i - (int64_t)y * im.W);
        const int Y = py[(int64_t)y * im.pitch[0] + x];
        if (im.C == 1) {
            o[i] = (uint8_t)Y;
            continue;
        }
        const int cb = jpeg_chroma(plane + im.plane_off + im.comp_plane[1], im.pitch[1], im.ch[1], im.cw[1], im.hmax, im.vmax, y, x) - 128;
        const int cr = jpeg_chroma(plane + im.plane_off + im.comp_plane[2], im.pitch[2], im.ch[2], im.cw[2], im.hmax, im.vmax, y, x) - 128;
        // jdcolor.c build_ycc_rgb_table / ycc_rgb_convert: FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414)
        const int rr = Y + ((91881 * cr + 32768) >> 16);
        const int gg = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
        const int bb = Y + ((116130 * cb + 32768) >> 16);
        o[3 * i] = (uint8_t)min(max(rr, 0), 255);
        o[3 * i + 1] = (uint8_t)min(max(gg, 0), 255);
        o[3 * i + 2] = (uint8_t)min(max(bb, 0), 255);
    }
}

// ------------------------------------------------------------------------------------------------ host side
struct JpegScratch {
    size_t coef, dc, dcsum, plane, state, stamp, count, base, flags, temp, total, temp_bytes;
};

static size_t jpeg_align(size_t v) { return (v + 255) & ~(size_t)255; }

static int jpeg_layout(int64_t coef_blocks, int64_t plane_bytes, int n_windows, JpegScratch& L) {
    size_t t1 = 0, t2 = 0;
    CL_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, t1, (const int32_t*)nullptr, (int32_t*)nullptr, n_windows));
    CL_CUDA_CHECK(cub::DeviceScan::InclusiveSum(nullptr, t2, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)coef_blocks));
    size_t off = 0;
    L.coef = off; off = jpeg_align(off + (size_t)coef_blocks * 128);
    L.dc = off; off = jpeg_align(off + (size_t)coef_blocks * 4);
    L.dcsum = off; off = jpeg_align(off + (size_t)coef_blocks * 4);
    L.plane = off; off = jpeg_align(off + (size_t)plane_bytes);
    L.state = off; off = jpeg_align(off + (size_t)n_windows * 8);
    L.stamp = off; off = jpeg_align(off + (size_t)n_windows * 4);
    L.count = off; off = jpeg_align(off + (size_t)n_windows * 4);
    L.base = off; off = jpeg_align(off + (size_t)n_windows * 4);
    L.flags = off; off = jpeg_align(off + 16);
    L.temp = off;
    L.temp_bytes = std::max(t1, t2);
    L.total = jpeg_align(off + L.temp_bytes);
    return CL_OK;
}

}  // namespace clb

using namespace clb;

extern "C" int64_t cl_jpeg_scratch_bytes(int64_t coef_blocks, int64_t plane_bytes, int n_windows) {
    if (coef_blocks <= 0 || coef_blocks >= (1ll << 31) || plane_bytes <= 0 || n_windows <= 0)
        return set_error(CL_ERR_INVALID, "cl_jpeg_scratch_bytes: %lld blocks, %lld plane bytes, %d windows", (long long)coef_blocks,
                         (long long)plane_bytes, n_windows);
    JpegScratch L;
    CL_CHECK(jpeg_layout(coef_blocks, plane_bytes, n_windows, L));
    return (int64_t)L.total;
}

extern "C" int cl_jpeg_decode(const cl_jpeg_image* img, const cl_jpeg_image* img_dev, int B, const cl_jpeg_segment* seg,
                              const cl_jpeg_segment* seg_dev, int n_seg, const int32_t* tables, int64_t table_len,
                              const uint8_t* data, int64_t data_bytes, void* scratch, int64_t scratch_bytes, uint8_t* out,
                              int64_t out_bytes, int32_t* status, int32_t* sync_rounds, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!img || !img_dev || !seg || !seg_dev || !tables || !data || !scratch || !out || !status)
        return set_error(CL_ERR_INVALID, "cl_jpeg_decode: null img, img_dev, seg, seg_dev, tables, data, scratch, out or status");
    if (B <= 0 || B > 65535) return set_error(CL_ERR_INVALID, "cl_jpeg_decode: B = %d, expected 1..65535", B);
    if (n_seg < B) return set_error(CL_ERR_INVALID, "cl_jpeg_decode: %d segments for %d images", n_seg, B);
    int64_t coef_blocks = 0, plane_bytes = 0, out_end = 0, max_px = 0, max_blk = 0;
    int n_windows = 0;
    for (int b = 0; b < B; ++b) {
        const cl_jpeg_image& d = img[b];
        if (d.C != 1 && d.C != 3) return set_error(CL_ERR_INVALID, "cl_jpeg_decode: image %d has C = %d, expected 1 or 3", b, d.C);
        if (d.H <= 0 || d.W <= 0 || d.H > JPEG_MAX_SIDE || d.W > JPEG_MAX_SIDE)
            return set_error(CL_ERR_INVALID, "cl_jpeg_decode: image %d: size %d x %d outside 1..%d", b, d.W, d.H, JPEG_MAX_SIDE);
        const bool samp_ok = d.C == 1 ? (d.hmax == 1 && d.vmax == 1)
                                      : ((d.hmax == 1 && d.vmax == 1) || (d.hmax == 2 && (d.vmax == 1 || d.vmax == 2)));
        const int bpm = d.C == 1 ? 1 : d.hmax * d.vmax + 2;
        const int mx = d.C == 1 ? (d.W + 7) / 8 : (d.W + 8 * d.hmax - 1) / (8 * d.hmax);
        const int my = d.C == 1 ? (d.H + 7) / 8 : (d.H + 8 * d.vmax - 1) / (8 * d.vmax);
        if (!samp_ok || d.bpm != bpm || d.mcux != mx || d.mcuy != my)
            return set_error(CL_ERR_INVALID, "cl_jpeg_decode: image %d: sampling %d x %d, %d blocks per MCU, %d x %d MCUs do not fit %d x %d x %d",
                             b, d.hmax, d.vmax, d.bpm, d.mcux, d.mcuy, d.W, d.H, d.C);
        const int64_t n_mcu = (int64_t)mx * my;
        if (d.nblocks != n_mcu * bpm || d.ri < 0 || d.nseg != (d.ri ? (n_mcu + d.ri - 1) / d.ri : 1) || d.seg0 < 0 ||
            d.seg0 + (int64_t)d.nseg > n_seg || (b > 0 && d.seg0 != img[b - 1].seg0 + img[b - 1].nseg) || (b == 0 && d.seg0 != 0))
            return set_error(CL_ERR_INVALID, "cl_jpeg_decode: image %d: %d blocks, restart interval %d, segments [%d, +%d) do not fit",
                             b, d.nblocks, d.ri, d.seg0, d.nseg);
        if (d.out_off < out_end || d.out_off + (int64_t)d.H * d.W * d.C > out_bytes)
            return set_error(CL_ERR_INVALID, "cl_jpeg_decode: image %d: output %lld + %d x %d x %d overlaps image %d or lies outside the "
                             "%lld-byte output", b, (long long)d.out_off, d.H, d.W, d.C, b - 1, (long long)out_bytes);
        out_end = d.out_off + (int64_t)d.H * d.W * d.C;
        if (d.coef_off != coef_blocks || d.plane_off != plane_bytes)   // scratch ranges back to back; planes 8-byte aligned
            return set_error(CL_ERR_INVALID, "cl_jpeg_decode: image %d: coefficient block %lld / plane byte %lld, expected %lld / %lld "
                             "(the images' scratch ranges back to back)", b, (long long)d.coef_off, (long long)d.plane_off,
                             (long long)coef_blocks, (long long)plane_bytes);
        int64_t pl = 0;
        for (int c = 0; c < d.C; ++c) {
            const int h = d.C == 3 && c == 0 ? d.hmax : 1, v = d.C == 3 && c == 0 ? d.vmax : 1;
            const int ch = (int)(((int64_t)d.H * v + d.vmax - 1) / d.vmax), cw = (int)(((int64_t)d.W * h + d.hmax - 1) / d.hmax);
            if (d.ch[c] != ch || d.cw[c] != cw || d.pitch[c] != (cw + 7) / 8 * 8 || d.comp_plane[c] != pl)
                return set_error(CL_ERR_INVALID, "cl_jpeg_decode: image %d component %d: plane %d x %d (pitch %d at %d) does not fit", b, c,
                                 d.ch[c], d.cw[c], d.pitch[c], d.comp_plane[c]);
            pl += (int64_t)d.pitch[c] * ((ch + 7) / 8 * 8);
            if (d.qt[c] < 0 || d.qt[c] + 64ll > table_len || d.dc_tab[c] < 0 || d.dc_tab[c] + (int64_t)JPEG_HUFF_WORDS > table_len ||
                d.ac_tab[c] < 0 || d.ac_tab[c] + (int64_t)JPEG_HUFF_WORDS > table_len)
                return set_error(CL_ERR_INVALID, "cl_jpeg_decode: image %d component %d: tables (%d, %d, %d) outside the %lld-word tables", b,
                                 c, d.qt[c], d.dc_tab[c], d.ac_tab[c], (long long)table_len);
        }
        coef_blocks = d.coef_off + d.nblocks;
        plane_bytes = d.plane_off + pl;
        max_px = std::max<int64_t>(max_px, (int64_t)d.H * d.W);
        max_blk = std::max<int64_t>(max_blk, pl / 64);
        for (int s = 0; s < d.nseg; ++s) {
            const cl_jpeg_segment& S = seg[d.seg0 + s];
            const int per = d.ri ? d.ri : (int)n_mcu;
            const int nm = (int)std::min<int64_t>(per, n_mcu - (int64_t)s * per);
            const int nwin = S.nbytes > 0 ? (int)((8ll * S.nbytes + CL_JPEG_WINDOW_BITS - 1) / CL_JPEG_WINDOW_BITS) : 1;
            if (S.image != b || S.mcu0 != s * per || S.nmcu != nm || S.block0 != d.coef_off + (int64_t)S.mcu0 * bpm)
                return set_error(CL_ERR_INVALID, "cl_jpeg_decode: segment %d: image %d, MCUs [%d, +%d), block %lld do not fit image %d", d.seg0 + s,
                                 S.image, S.mcu0, S.nmcu, (long long)S.block0, b);
            if (S.nbytes < 0 || S.nbytes >= CL_JPEG_MAX_SEGMENT_BYTES || S.data_off < 0 || S.data_off + S.nbytes > data_bytes)
                return set_error(CL_ERR_INVALID, "cl_jpeg_decode: segment %d: %d bytes at %lld outside the %lld-byte data", d.seg0 + s,
                                 S.nbytes, (long long)S.data_off, (long long)data_bytes);
            if (S.win0 != n_windows || S.nwin != nwin)
                return set_error(CL_ERR_INVALID, "cl_jpeg_decode: segment %d: windows [%d, +%d), expected [%d, +%d)", d.seg0 + s, S.win0,
                                 S.nwin, n_windows, nwin);
            n_windows += nwin;
        }
    }
    if (img[B - 1].seg0 + img[B - 1].nseg != n_seg)
        return set_error(CL_ERR_INVALID, "cl_jpeg_decode: the images cover %d of %d segments", img[B - 1].seg0 + img[B - 1].nseg, n_seg);
    if (coef_blocks >= (1ll << 31)) return set_error(CL_ERR_INVALID, "cl_jpeg_decode: %lld coefficient blocks", (long long)coef_blocks);
    JpegScratch L;
    CL_CHECK(jpeg_layout(coef_blocks, plane_bytes, n_windows, L));
    if ((int64_t)L.total > scratch_bytes)
        return set_error(CL_ERR_INVALID, "cl_jpeg_decode: scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)L.total);

    char* sp = static_cast<char*>(scratch);
    int16_t* coef = reinterpret_cast<int16_t*>(sp + L.coef);
    uint32_t* dc = reinterpret_cast<uint32_t*>(sp + L.dc);
    uint32_t* dcsum = reinterpret_cast<uint32_t*>(sp + L.dcsum);
    uint8_t* plane = reinterpret_cast<uint8_t*>(sp + L.plane);
    uint64_t* state = reinterpret_cast<uint64_t*>(sp + L.state);
    int32_t* stamp = reinterpret_cast<int32_t*>(sp + L.stamp);
    int32_t* count = reinterpret_cast<int32_t*>(sp + L.count);
    int32_t* base = reinterpret_cast<int32_t*>(sp + L.base);
    int32_t* flags = reinterpret_cast<int32_t*>(sp + L.flags);
    void* temp = sp + L.temp;

    CL_CUDA_CHECK(cudaMemsetAsync(sp + L.coef, 0, L.dcsum - L.coef, stream));
    int dev = 0, per_sm = 0;
    CL_CUDA_CHECK(cudaGetDevice(&dev));
    CL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, jpeg_sync_kernel, JPEG_THREADS, 0));
    const int sync_grid = (int)std::max<int64_t>(1, std::min<int64_t>((n_windows + JPEG_THREADS - 1) / JPEG_THREADS, (int64_t)per_sm * num_sms()));
    {
        const cl_jpeg_image* a0 = img_dev;
        int a1 = B;
        const cl_jpeg_segment* a2 = seg_dev;
        int a3 = n_seg;
        const int32_t* a4 = tables;
        const uint8_t* a5 = data;
        int a6 = n_windows;
        uint64_t* a7 = state;
        int32_t* a8 = stamp;
        int32_t* a9 = count;
        int32_t* a10 = flags;
        int32_t* a11 = status;
        int32_t* a12 = sync_rounds;
        void* args[] = {&a0, &a1, &a2, &a3, &a4, &a5, &a6, &a7, &a8, &a9, &a10, &a11, &a12};
        CL_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)jpeg_sync_kernel, dim3(sync_grid), dim3(JPEG_THREADS), args, 0, stream));
    }
    size_t tb = L.temp_bytes;
    CL_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(temp, tb, count, base, n_windows, stream));
    const int wgrid = (int)std::min<int64_t>((n_windows + JPEG_THREADS - 1) / JPEG_THREADS, (int64_t)num_sms() * 16);
    launch_k(jpeg_write_kernel, dim3(wgrid), JPEG_THREADS, 0, stream, img_dev, seg_dev, n_seg, tables, data, n_windows,
             (const uint64_t*)state, (const int32_t*)base, coef, dc, status);
    tb = L.temp_bytes;
    CL_CUDA_CHECK(cub::DeviceScan::InclusiveSum(temp, tb, (const uint32_t*)dc, dcsum, (int)coef_blocks, stream));
    const int cap = num_sms() * 8;
    const int g1 = (int)std::min<int64_t>((max_blk + JPEG_THREADS - 1) / JPEG_THREADS, cap);
    launch_k(jpeg_idct_kernel, dim3(std::max(g1, 1), B), JPEG_THREADS, 0, stream, img_dev, seg_dev, tables, (const int16_t*)coef,
             (const uint32_t*)dcsum, plane);
    const int g2 = (int)std::min<int64_t>((max_px + 255) / 256, cap);
    launch_k(jpeg_color_kernel, dim3(std::max(g2, 1), B), 256, 0, stream, img_dev, (const uint8_t*)plane, out);
    count_launch(7);
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
