// Canny edge annotator: cv2.Canny(img, lo, hi) with aperture 3 and L2gradient = false, bit for bit, plus the float32
// guide / pixel tensors the reference builds from it (process/diffusiondb_canny.py:35-45, apps/gradio_canny2image.py:71-74,
// annotator/canny/__init__.py:6).  The rules are restated in oracle/annotator_ref.py.
//
// Four launches, independent of the data, no host synchronisation (the call can be captured in a CUDA graph):
//   1. canny_local_kernel: one CTA per 32x32 tile.  The uint8 tile plus a 2-pixel halo (replicate border) goes to shared
//      memory; Sobel + channel selection for the tile and a 1-pixel ring, non-maximum suppression, thresholds read from
//      the device table.  Candidates are labelled by union-find in shared memory (8-connectivity) and flattened; each
//      local root carries FLAG when its tile-local component holds a strong pixel.  labels[] receives, per pixel, the
//      global index of its local root (| FLAG on a flagged root), or -1 for a non-candidate.
//   2. canny_merge_kernel: the top row and left column of each tile are united with their 8-neighbours in the adjacent
//      tiles (lock-free union: the larger root is linked under the smaller one by atomicCAS).
//   3. canny_mark_kernel: each flagged former local root sets FLAG on its global root (atomicOr).
//   4. canny_resolve_kernel: a candidate is an edge iff its root carries FLAG; writes edges / guide / pixels.
// Labels are union-find parent pointers in bits 0..30 (B*H*W < 2^31); bit 31 of an entry is that pixel's own flag, kept
// when the entry is relinked, so a flag is never lost.  Which root a component ends with depends on the scheduling of the
// atomics; the set of edge pixels does not.
#include <stdio.h>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

constexpr int CT_W = 32, CT_H = 32, CT_THREADS = 256;
constexpr int CT_PER_THREAD = CT_W * CT_H / CT_THREADS;
constexpr int CANNY_FLAG = (int)0x80000000u;
constexpr int CANNY_IDX = 0x7fffffff;
constexpr int CANNY_TG22 = 13573;  // round(tan(22.5 deg) * 2^15), OpenCV's constant

// Sobel of the pixel at (sy, sx) of the shared tile (row pitch CT_W + 4 pixels); channel of largest |dx| + |dy|, the first
// one on a tie.
template <int C>
__device__ __forceinline__ int canny_grad(const uint8_t* simg, int sy, int sx, int& dx, int& dy) {
    constexpr int P = (CT_W + 4) * C;
    int best = -1;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const uint8_t* p = simg + sy * P + sx * C + c;
        const int a = p[-P - C], b = p[-P], d = p[-P + C];
        const int l = p[-C], r = p[C];
        const int e = p[P - C], f = p[P], g = p[P + C];
        const int gx = (d + 2 * r + g) - (a + 2 * l + e);
        const int gy = (e + 2 * f + g) - (a + 2 * b + d);
        const int m = abs(gx) + abs(gy);
        if (m > best) { best = m; dx = gx; dy = gy; }
    }
    return best;
}

// m in [0, 2040], so clamping keeps every comparison and makes the float -> int conversion defined
__device__ __forceinline__ int canny_floor_thr(float t) { return (int)floorf(fminf(fmaxf(t, -1.f), 4096.f)); }

__device__ __forceinline__ int find_s(volatile int* s, int x) {
    while (true) {
        const int p = s[x];
        if (p == x) return x;
        x = p;
    }
}

__device__ __forceinline__ void union_s(volatile int* s, int a, int b) {
    while (true) {
        a = find_s(s, a);
        b = find_s(s, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = atomicMin((int*)&s[a], b);
        if (old == a) return;
        a = old;
    }
}

// Root of x, with path halving: a node that is not a root is pointed at its current grandparent.  Every parent index is
// smaller than its node and each store keeps that so (no cycle can form); only entries that are not roots are rewritten,
// and such an entry never becomes a root again, so the plain stores cannot undo a concurrent link.  Loads bypass L1:
// other CTAs write the table.
__device__ __forceinline__ int find_g(int* L, int x) {
    while (true) {
        const int v = __ldcg(L + x);
        const int p = v & CANNY_IDX;
        if (p == x) return x;
        const int g = __ldcg(L + p) & CANNY_IDX;
        if (g == p) return p;
        __stcg(L + x, g | (v & CANNY_FLAG));
        x = g;
    }
}

__device__ __forceinline__ void union_g(int* L, int a, int b) {
    while (true) {
        a = find_g(L, a);
        b = find_g(L, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = __ldcg(L + a);
        if ((old & CANNY_IDX) != a) continue;
        if (atomicCAS(L + a, old, b | (old & CANNY_FLAG)) == old) return;
    }
}

template <int C>
__global__ void __launch_bounds__(CT_THREADS)
canny_local_kernel(const uint8_t* __restrict__ img, int H, int W, int tiles_x, int tiles_per_img, const float* __restrict__ thr,
                   int* __restrict__ labels) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ uint8_t simg[(CT_H + 4) * (CT_W + 4) * C];
    __shared__ int smag[(CT_H + 2) * (CT_W + 2)];
    __shared__ int slab[CT_H * CT_W];
    const int tid = threadIdx.x;
    const int b = blockIdx.x / tiles_per_img;
    const int t = blockIdx.x % tiles_per_img;
    const int y0 = (t / tiles_x) * CT_H, x0 = (t % tiles_x) * CT_W;
    const uint8_t* im = img + (size_t)b * H * W * C;

    for (int i = tid; i < (CT_H + 4) * (CT_W + 4); i += CT_THREADS) {
        const int gy = min(max(y0 + i / (CT_W + 4) - 2, 0), H - 1);
        const int gx = min(max(x0 + i % (CT_W + 4) - 2, 0), W - 1);
        const uint8_t* p = im + ((size_t)gy * W + gx) * C;
#pragma unroll
        for (int c = 0; c < C; ++c) simg[i * C + c] = p[c];
    }
    __syncthreads();
    for (int i = tid; i < (CT_H + 2) * (CT_W + 2); i += CT_THREADS) {
        const int sy = i / (CT_W + 2), sx = i % (CT_W + 2);
        const int gy = y0 + sy - 1, gx = x0 + sx - 1;
        int dx, dy, m = 0;
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) m = canny_grad<C>(simg, sy + 1, sx + 1, dx, dy);
        smag[i] = m;
    }
    float lo = thr[2 * b], hi = thr[2 * b + 1];
    if (lo > hi) { const float s = lo; lo = hi; hi = s; }
    const int low = canny_floor_thr(lo), high = canny_floor_thr(hi);
    __syncthreads();

    unsigned cand_bits = 0, strong_bits = 0;
#pragma unroll
    for (int k = 0; k < CT_PER_THREAD; ++k) {
        const int i = tid + k * CT_THREADS;
        const int ly = i / CT_W, lx = i % CT_W;
        bool cand = false;
        if (y0 + ly < H && x0 + lx < W) {
            int dx, dy;
            const int m = canny_grad<C>(simg, ly + 2, lx + 2, dx, dy);
            if (m > low) {
                const int* mc = smag + (ly + 1) * (CT_W + 2) + lx + 1;
                constexpr int MP = CT_W + 2;
                const int xs = abs(dx), ys = abs(dy);
                const int tg22x = xs * CANNY_TG22;
                const int yy = ys << 15;
                if (yy < tg22x) {
                    cand = m > mc[-1] && m >= mc[1];
                } else if (yy > tg22x + (xs << 16)) {
                    cand = m > mc[-MP] && m >= mc[MP];
                } else if ((dx ^ dy) < 0) {
                    cand = m > mc[-MP + 1] && m > mc[MP - 1];
                } else {
                    cand = m > mc[-MP - 1] && m > mc[MP + 1];
                }
                if (cand && m > high) strong_bits |= 1u << k;
            }
        }
        if (cand) cand_bits |= 1u << k;
        slab[i] = cand ? i : -1;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < CT_PER_THREAD; ++k) {
        if (!(cand_bits >> k & 1u)) continue;
        const int i = tid + k * CT_THREADS;
        const int ly = i / CT_W, lx = i % CT_W;
        if (lx > 0 && slab[i - 1] >= 0) union_s(slab, i, i - 1);
        if (ly > 0) {
            if (lx > 0 && slab[i - CT_W - 1] >= 0) union_s(slab, i, i - CT_W - 1);
            if (slab[i - CT_W] >= 0) union_s(slab, i, i - CT_W);
            if (lx + 1 < CT_W && slab[i - CT_W + 1] >= 0) union_s(slab, i, i - CT_W + 1);
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < CT_PER_THREAD; ++k) {
        const int i = tid + k * CT_THREADS;
        if (cand_bits >> k & 1u) slab[i] = find_s(slab, i);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < CT_PER_THREAD; ++k) {
        const int i = tid + k * CT_THREADS;
        if (strong_bits >> k & 1u) atomicOr(&slab[slab[i] & CANNY_IDX], CANNY_FLAG);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < CT_PER_THREAD; ++k) {
        const int i = tid + k * CT_THREADS;
        const int ly = i / CT_W, lx = i % CT_W;
        if (y0 + ly >= H || x0 + lx >= W) continue;
        const int v = slab[i];
        int out = -1;
        if (v != -1) {
            const int r = v & CANNY_IDX;
            out = ((b * H + y0 + r / CT_W) * W + x0 + r % CT_W) | (v & CANNY_FLAG);
        }
        labels[(b * H + y0 + ly) * W + x0 + lx] = out;
    }
}

// one CTA per tile, thread t < CT_W: top-row pixel t, else left-column pixel t - CT_W
__global__ void __launch_bounds__(CT_W + CT_H)
canny_merge_kernel(int H, int W, int tiles_x, int tiles_per_img, int* labels) {
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.x / tiles_per_img;
    const int t = blockIdx.x % tiles_per_img;
    const int y0 = (t / tiles_x) * CT_H, x0 = (t % tiles_x) * CT_W;
    const int base = b * H * W;
    const bool row = threadIdx.x < CT_W;
    const int y = row ? y0 : y0 + threadIdx.x - CT_W;
    const int x = row ? x0 + threadIdx.x : x0;
    if (row ? (y0 == 0 || x >= W) : (x0 == 0 || y >= H)) return;
    const int p = base + y * W + x;
    if (__ldcg(labels + p) == -1) return;
    // the three neighbours in the tile row above (x - 1 .. x + 1) or the tile column to the left (y - 1 .. y + 1)
    for (int j = -1; j <= 1; ++j) {
        const int qy = row ? y - 1 : y + j, qx = row ? x + j : x - 1;
        if (qy < 0 || qy >= H || qx < 0 || qx >= W) continue;
        const int q = base + qy * W + qx;
        if (__ldcg(labels + q) != -1) union_g(labels, p, q);
    }
}

__global__ void __launch_bounds__(256) canny_mark_kernel(int* labels, int n) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long ii = blockIdx.x * blockDim.x + threadIdx.x; ii < n; ii += gridDim.x * blockDim.x) {
        const int i = (int)ii;
        const int v = __ldcg(labels + i);
        if (v == -1 || !(v & CANNY_FLAG)) continue;
        const int r = find_g(labels, i);
        if (r != i) atomicOr(labels + r, CANNY_FLAG);
    }
}

// pixels: x / 127.5 - 1 with the division and the subtraction each rounded to fp32, as torch / numpy compute it on the host
template <bool PIXELS>
__global__ void __launch_bounds__(256)
canny_resolve_kernel(const uint8_t* __restrict__ img, int* labels, int n, int HW, uint8_t* __restrict__ edges,
                     float* __restrict__ guide, float* __restrict__ pixels) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long ii = blockIdx.x * blockDim.x + threadIdx.x; ii < n; ii += gridDim.x * blockDim.x) {
        const int i = (int)ii;
        bool e = false;
        if (__ldcg(labels + i) != -1) e = (__ldcg(labels + find_g(labels, i)) & CANNY_FLAG) != 0;
        if (edges != nullptr) edges[i] = e ? 255 : 0;
        const int b = i / HW, hw = i % HW;
        const size_t o = (size_t)b * 3 * HW + hw;
        if (guide != nullptr) {
            const float g = e ? 1.f : -1.f;
            guide[o] = g; guide[o + HW] = g; guide[o + 2 * (size_t)HW] = g;
        }
        if (PIXELS) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                pixels[o + c * (size_t)HW] = __fsub_rn(__fdiv_rn((float)img[(size_t)i * 3 + c], 127.5f), 1.f);
        }
    }
}

}  // namespace clb

using namespace clb;

extern "C" int cl_canny(const uint8_t* img, int B, int H, int W, int C, const float* thresholds, int32_t* labels,
                        uint8_t* edges, float* guide, float* pixels, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!img || !thresholds || !labels) return set_error(CL_ERR_INVALID, "cl_canny: null img, thresholds or labels");
    if (!edges && !guide && !pixels) return set_error(CL_ERR_INVALID, "cl_canny: no output requested (edges, guide, pixels all null)");
    if (C != 1 && C != 3) return set_error(CL_ERR_INVALID, "cl_canny: C = %d, expected 1 or 3", C);
    if (pixels && C != 3) return set_error(CL_ERR_INVALID, "cl_canny: pixels needs a 3-channel image (C = %d)", C);
    if (B <= 0 || H <= 0 || W <= 0) return set_error(CL_ERR_INVALID, "cl_canny: non-positive size B=%d H=%d W=%d", B, H, W);
    const long long n = (long long)B * H * W;
    if (n >= (1ll << 31)) return set_error(CL_ERR_INVALID, "cl_canny: B*H*W = %lld must be below 2^31", n);
    const int tiles_x = (W + CT_W - 1) / CT_W, tiles_y = (H + CT_H - 1) / CT_H;
    const long long tiles = (long long)tiles_x * tiles_y;   // <= n
    const int grid_tiles = (int)(tiles * B);
    if (C == 3)
        launch_k(canny_local_kernel<3>, grid_tiles, CT_THREADS, 0, stream, img, H, W, tiles_x, (int)tiles, thresholds, labels);
    else
        launch_k(canny_local_kernel<1>, grid_tiles, CT_THREADS, 0, stream, img, H, W, tiles_x, (int)tiles, thresholds, labels);
    launch_k(canny_merge_kernel, grid_tiles, CT_W + CT_H, 0, stream, H, W, tiles_x, (int)tiles, labels);
    int blocks = (int)((n + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(canny_mark_kernel, blocks, 256, 0, stream, labels, (int)n);
    if (pixels)
        launch_k(canny_resolve_kernel<true>, blocks, 256, 0, stream, img, labels, (int)n, H * W, edges, guide, pixels);
    else
        launch_k(canny_resolve_kernel<false>, blocks, 256, 0, stream, img, labels, (int)n, H * W, edges, guide, pixels);
    count_launch(4);
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
