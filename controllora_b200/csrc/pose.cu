// OpenPose body-skeleton renderer: the reference's draw_bodypose (annotator/openpose/util.py:37-70) for a ragged batch,
// bit for bit, and the guide arithmetic of apps/gradio_pose2image.py:70-78 and process/mpii_pose.py:29-44.  The OpenCV
// rules (ellipse2Poly, Line, FillConvexPoly, Circle, addWeighted, INTER_NEAREST) are restated in oracle/pose_ref.py.
//
// Two launches per call, no host synchronisation:
//   1. pose_limb_kernel, one CTA per limb slot: the ellipse2Poly polygon (361 points in double from OpenCV's float sine
//      table, cvRound, consecutive duplicates dropped), its edges stroked with OpenCV's clipped 8-connected lines
//      (one thread per edge, atomicOr into the limb's bitmask), then FillConvexPoly's scanline walk (one thread, rows
//      above the canvas skipped in closed form) whose spans are OR-ed in by the whole CTA.
//   2. pose_render_kernel, one thread per output pixel: the pixel's canvas position through crop and nearest resize,
//      the background, the circles in draw order (last write wins), then every limb whose bitmask covers the pixel,
//      in draw order, blended as addWeighted(canvas, 0.4, colour, 0.6) in fp32; then the outputs.
// A limb that does not cover a pixel leaves it unchanged: addWeighted(a, 0.4, a, 0.6, 0) == a for every uint8 a.
#include <stdio.h>

#include "common.cuh"
#include "host_common.h"
#include "pose_sin_table.h"
#include "../../include/controllora_b200.h"

namespace clb {

constexpr int PS_LIMB_THREADS = 384;   // >= 361 ellipse points
constexpr int PS_NPTS = 361;
constexpr int PS_MAX_CANVAS = 4096;
constexpr int PS_MAX_COORD = 1 << 22;  // |centre|, half length: keeps every fixed-point product inside int64
constexpr int PS_XY_SHIFT = 16;

__constant__ int ps_sin_q30[CL_POSE_SIN_Q30_N] = CL_POSE_SIN_Q30;

__device__ __forceinline__ float ps_sin(int deg) { return (float)ps_sin_q30[deg] * 0x1p-30f; }  // exact

__device__ __forceinline__ void ps_set(uint32_t* __restrict__ m, int words, const cl_pose_limb& L, int x, int y) {
    const int c = x - L.bx0, r = y - L.by0;
    if ((unsigned)c < (unsigned)L.bw && (unsigned)r < (unsigned)L.bh)
        atomicOr(m + (size_t)r * words + (c >> 5), 1u << (c & 31));
}

// drawing.cpp Line(img, p1, p2, colour, 8): LineIterator(leftToRight) after clipLine on a W x H image.
__device__ void ps_line(uint32_t* m, int words, const cl_pose_limb& L, int W, int H, long long x1, long long y1, long long x2,
                        long long y2) {
    if (x1 < 0 || x1 >= W || x2 < 0 || x2 >= W || y1 < 0 || y1 >= H || y2 < 0 || y2 >= H) {
        const long long right = W - 1, bottom = H - 1;
        int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
        int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            long long a;
            if (c1 & 12) {
                a = c1 < 8 ? 0 : bottom;
                x1 += __double2ll_rz(__ddiv_rn(__dmul_rn((double)(a - y1), (double)(x2 - x1)), (double)(y2 - y1)));
                y1 = a;
                c1 = (x1 < 0) + (x1 > right) * 2;
            }
            if (c2 & 12) {
                a = c2 < 8 ? 0 : bottom;
                x2 += __double2ll_rz(__ddiv_rn(__dmul_rn((double)(a - y2), (double)(x2 - x1)), (double)(y2 - y1)));
                y2 = a;
                c2 = (x2 < 0) + (x2 > right) * 2;
            }
            if ((c1 & c2) == 0 && (c1 | c2) != 0) {
                if (c1) {
                    a = c1 == 1 ? 0 : right;
                    y1 += __double2ll_rz(__ddiv_rn(__dmul_rn((double)(a - x1), (double)(y2 - y1)), (double)(x2 - x1)));
                    x1 = a;
                    c1 = 0;
                }
                if (c2) {
                    a = c2 == 1 ? 0 : right;
                    y2 += __double2ll_rz(__ddiv_rn(__dmul_rn((double)(a - x2), (double)(y2 - y1)), (double)(x2 - x1)));
                    x2 = a;
                    c2 = 0;
                }
            }
        }
        if (c1 | c2) return;
    }
    int sx = 1, sy = 1;
    int dx = (int)(x2 - x1), dy = (int)(y2 - y1);
    int x = (int)x1, y = (int)y1;
    if (dx < 0) { dx = -dx; dy = -dy; x = (int)x2; y = (int)y2; }
    if (dy < 0) { dy = -dy; sy = -1; }
    const bool vert = dy > dx;
    if (vert) { const int t = dx; dx = dy; dy = t; sx = sy; sy = 1; }
    int err = dx - (dy + dy);
    for (int k = 0; k <= dx; ++k) {
        ps_set(m, words, L, x, y);
        const bool neg = err < 0;
        err += -(dy + dy) + (neg ? dx + dx : 0);
        if (vert) { y += sx; x += neg ? sy : 0; }
        else      { x += sx; y += neg ? sy : 0; }
    }
}

__global__ void __launch_bounds__(PS_LIMB_THREADS) pose_limb_kernel(const cl_pose_image* __restrict__ imgs, int B,
                                                                     const cl_pose_limb* __restrict__ limbs, int n_limbs,
                                                                     uint32_t* __restrict__ mask, long long mask_words) {
    __shared__ int2 s_pt[PS_NPTS + 1];
    __shared__ int s_woff[PS_LIMB_THREADS / 32 + 1];
    __shared__ int s_lo[PS_MAX_CANVAS], s_hi[PS_MAX_CANVAS];
    const int li = blockIdx.x, t = threadIdx.x;
    if (li >= n_limbs) return;
    const cl_pose_limb L = limbs[li];
    if (L.image < 0 || L.image >= B || L.bw <= 0 || L.bh <= 0) return;
    const cl_pose_image I = imgs[L.image];
    const int W = I.Wc, H = I.Hc;
    const int words = (L.bw + 31) >> 5;
    if (W <= 0 || H <= 0 || W > PS_MAX_CANVAS || H > PS_MAX_CANVAS || L.bx0 < 0 || L.by0 < 0 || L.bx0 + L.bw > W ||
        L.by0 + L.bh > H || L.mask_off < 0 || L.mask_off + (long long)L.bh * words > mask_words)
        return;
    uint32_t* m = mask + L.mask_off;

    // ellipse2Poly((cx, cy), (half_len, 4), angle, 0, 360, 1): its while loops bring the angle into [0, 360]
    int ang = L.angle;
    if (ang < 0) ang = ((ang % 360) + 360) % 360;
    else if (ang > 360) ang = (ang - 1) % 360 + 1;
    const double alpha = (double)ps_sin(450 - ang), beta = (double)ps_sin(ang);
    int2 pt = make_int2(0, 0);
    if (t < PS_NPTS) {
        const double x = __dmul_rn((double)L.half_len, (double)ps_sin(450 - t));
        const double y = __dmul_rn(4.0, (double)ps_sin(t));
        pt.x = __double2int_rn(__dsub_rn(__dadd_rn((double)L.cx, __dmul_rn(x, alpha)), __dmul_rn(y, beta)));
        pt.y = __double2int_rn(__dadd_rn(__dadd_rn((double)L.cy, __dmul_rn(x, beta)), __dmul_rn(y, alpha)));
        s_pt[t] = pt;
    }
    for (int r = t; r < L.bh; r += PS_LIMB_THREADS) { s_lo[r] = 1; s_hi[r] = 0; }
    for (long long i = t; i < (long long)L.bh * words; i += PS_LIMB_THREADS) m[i] = 0u;
    __syncthreads();
    // drop consecutive duplicates, keeping order: one ballot per warp, warp offsets by a serial prefix
    const bool keep = t < PS_NPTS && (t == 0 || pt.x != s_pt[t - 1].x || pt.y != s_pt[t - 1].y);
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    const int lane = t & 31, warp = t >> 5;
    if (lane == 0) s_woff[warp + 1] = __popc(bal);
    __syncthreads();
    if (t == 0) {
        s_woff[0] = 0;
        for (int w = 1; w <= PS_LIMB_THREADS / 32; ++w) s_woff[w] += s_woff[w - 1];
    }
    __syncthreads();
    if (keep) s_pt[s_woff[warp] + __popc(bal & ((1u << lane) - 1))] = pt;
    int n = s_woff[PS_LIMB_THREADS / 32];
    __syncthreads();
    if (n == 1) {                       // a zero-size polygon: the centre twice
        n = 2;
        if (t == 0) s_pt[0] = s_pt[1] = make_int2(L.cx, L.cy);
        __syncthreads();
    }

    // FillConvexPoly, part 1: every edge (v[i - 1], v[i]) stroked with Line()
    if (t < n) {
        const int2 p0 = s_pt[t == 0 ? n - 1 : t - 1], p1 = s_pt[t];
        ps_line(m, words, L, W, H, p0.x, p0.y, p1.x, p1.y);
    }

    // part 2: the scanline walk of both edge chains from the topmost vertex (16-bit fixed point, spans rounded)
    if (t == 0) {
        long long xmin = s_pt[0].x, xmax = xmin, ymin = s_pt[0].y, ymax = ymin;
        int imin = 0;
        for (int i = 0; i < n; ++i) {
            const int2 p = s_pt[i];
            if (p.y < ymin) { ymin = p.y; imin = i; }
            ymax = max(ymax, (long long)p.y);
            xmax = max(xmax, (long long)p.x);
            xmin = min(xmin, (long long)p.x);
        }
        if (!(n < 3 || xmax < 0 || ymax < 0 || xmin >= W || ymin >= H)) {
            ymax = min(ymax, (long long)H - 1);
            int e_idx[2] = {imin, imin}, e_di[2] = {1, n - 1};
            long long e_x[2] = {-(1ll << PS_XY_SHIFT), -(1ll << PS_XY_SHIFT)}, e_dx[2] = {0, 0}, e_ye[2] = {ymin, ymin};
            long long y = ymin;
            int edges = n;
            const long long half = 1ll << (PS_XY_SHIFT - 1);
            while (true) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    if (y >= e_ye[i]) {
                        int idx0 = e_idx[i], di = e_di[i];
                        int idx = idx0 + di;
                        if (idx >= n) idx -= n;
                        for (; edges-- > 0;) {
                            const long long ty = s_pt[idx].y;
                            if (ty > y) {
                                const long long xs = (long long)s_pt[idx0].x << PS_XY_SHIFT;
                                const long long xe = (long long)s_pt[idx].x << PS_XY_SHIFT;
                                e_ye[i] = ty;
                                e_dx[i] = ((xe - xs) * 2 + (ty - y)) / (2 * (ty - y));
                                e_x[i] = xs;
                                e_idx[i] = idx;
                                break;
                            }
                            idx0 = idx;
                            idx += di;
                            if (idx >= n) idx -= n;
                        }
                    }
                }
                if (edges < 0) break;
                long long step = 1;
                if (y >= 0) {
                    const bool swap = e_x[0] > e_x[1];
                    const long long xx1 = ((swap ? e_x[1] : e_x[0]) + half) >> PS_XY_SHIFT;
                    const long long xx2 = ((swap ? e_x[0] : e_x[1]) + half) >> PS_XY_SHIFT;
                    const int r = (int)(y - L.by0);
                    if (xx2 >= 0 && xx1 < W && (unsigned)r < (unsigned)L.bh) {
                        s_lo[r] = (int)max(xx1, 0ll);
                        s_hi[r] = (int)min(xx2, (long long)W - 1);
                    }
                } else {                // rows above the canvas: no edge changes before min(ye, 0)
                    step = min(min(e_ye[0], e_ye[1]), 0ll) - y;
                }
                e_x[0] += e_dx[0] * step;
                e_x[1] += e_dx[1] * step;
                y += step;
                if (y > ymax) break;
            }
        }
    }
    __syncthreads();
    // OR the spans into the bitmask: one thread per word
    for (long long i = t; i < (long long)L.bh * words; i += PS_LIMB_THREADS) {
        const int r = (int)(i / words), c0 = (int)(i % words) * 32 + L.bx0;
        const int lo = max(s_lo[r], c0), hi = min(s_hi[r], c0 + 31);
        if (lo > hi) continue;
        const int a = lo - c0, b = hi - c0;
        const uint32_t bits = (b == 31 ? 0xffffffffu : ((1u << (b + 1)) - 1u)) & ~((1u << a) - 1u);
        atomicOr(m + i, bits);
    }
}

__device__ __forceinline__ int ps_blend(int a, int c) {
    // cv2.addWeighted(a, 0.4, b, 0.6, 0) on uint8: float32 products and sum, rounded half to even, saturated
    const float v = __fadd_rn(__fmul_rn(0.4f, (float)a), __fmul_rn(0.6f, (float)c));
    return min(max(__float2int_rn(v), 0), 255);
}

__device__ __forceinline__ int ps_nearest(int o, int src, int dst) {
    // cv2.resize INTER_NEAREST: min(floor(o * (1 / (dst / src))), src - 1) in double
    const double inv = __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src));
    return min((int)floor(__dmul_rn((double)o, inv)), src - 1);
}

__global__ void __launch_bounds__(256) pose_render_kernel(const cl_pose_image* __restrict__ imgs,
                                                          const cl_pose_circle* __restrict__ circles, int n_circles,
                                                          const cl_pose_limb* __restrict__ limbs, int n_limbs,
                                                          const uint8_t* __restrict__ bg, const uint32_t* __restrict__ mask,
                                                          long long mask_words, int out_h, int out_w, int flip,
                                                          uint8_t* __restrict__ out_canvas, float* __restrict__ out_guide) {
    const int ox = blockIdx.x * 32 + threadIdx.x, oy = blockIdx.y * 8 + threadIdx.y, b = blockIdx.z;
    if (ox >= out_w || oy >= out_h) return;
    const cl_pose_image I = imgs[b];
    if (I.Hc <= 0 || I.Wc <= 0 || I.h <= 0 || I.w <= 0) return;
    const int y = min(max(I.y0 + ps_nearest(oy, I.h, out_h), 0), I.Hc - 1);
    const int x = min(max(I.x0 + ps_nearest(ox, I.w, out_w), 0), I.Wc - 1);
    int c0 = 0, c1 = 0, c2 = 0;
    if (bg && I.bg_off >= 0) {
        const uint8_t* p = bg + I.bg_off + ((size_t)y * I.Wc + x) * 3;
        c0 = p[0]; c1 = p[1]; c2 = p[2];
    }
    // cv2.circle radius 4, filled: half-width of the span on row centre + dy, |dy| = 0..4
    const int cend = min(I.circle0 + I.n_circles, n_circles);
    for (int i = max(I.circle0, 0); i < cend; ++i) {
        const cl_pose_circle C = circles[i];
        const int dy = abs(y - C.y), dx = abs(x - C.x);
        if (dy <= 4 && dx <= (dy == 0 ? 4 : dy <= 2 ? 3 : dy == 3 ? 2 : 0)) {
            c0 = C.color & 255; c1 = (C.color >> 8) & 255; c2 = (C.color >> 16) & 255;
        }
    }
    const int lend = min(I.limb0 + I.n_limbs, n_limbs);
    for (int i = max(I.limb0, 0); i < lend; ++i) {
        const cl_pose_limb& L = limbs[i];
        const int c = x - L.bx0, r = y - L.by0;
        if ((unsigned)c >= (unsigned)L.bw || (unsigned)r >= (unsigned)L.bh || L.image != b) continue;
        const int words = (L.bw + 31) >> 5;
        const long long w = L.mask_off + (long long)r * words + (c >> 5);
        if (L.mask_off < 0 || L.mask_off + (long long)L.bh * words > mask_words) continue;
        if ((mask[w] >> (c & 31)) & 1u) {
            c0 = ps_blend(c0, L.color & 255);
            c1 = ps_blend(c1, (L.color >> 8) & 255);
            c2 = ps_blend(c2, (L.color >> 16) & 255);
        }
    }
    const size_t pix = (size_t)oy * out_w + ox;
    if (out_canvas) {
        uint8_t* o = out_canvas + ((size_t)b * out_h * out_w + pix) * 3;
        o[0] = (uint8_t)c0; o[1] = (uint8_t)c1; o[2] = (uint8_t)c2;
    }
    if (out_guide) {
        const size_t plane = (size_t)out_h * out_w;
        float* g = out_guide + (size_t)b * 3 * plane + pix;
        const int v[3] = {flip ? c2 : c0, c1, flip ? c0 : c2};
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) g[ch * plane] = __fsub_rn(__fdiv_rn((float)v[ch], 127.5f), 1.f);
    }
}

}  // namespace clb

using namespace clb;

extern "C" int cl_pose_render(const cl_pose_image* img, const cl_pose_image* img_dev, int B, const cl_pose_circle* circles,
                              const cl_pose_circle* circles_dev, int n_circles, const cl_pose_limb* limbs,
                              const cl_pose_limb* limbs_dev, int n_limbs, const uint8_t* bg, int64_t bg_bytes, uint32_t* mask,
                              int64_t mask_words, int out_h, int out_w, int flip, uint8_t* out_canvas, float* out_guide,
                              void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!img || !img_dev) return set_error(CL_ERR_INVALID, "cl_pose_render: null img or img_dev");
    if (n_circles < 0 || n_limbs < 0 || (n_circles > 0 && (!circles || !circles_dev)) ||
        (n_limbs > 0 && (!limbs || !limbs_dev || !mask)))
        return set_error(CL_ERR_INVALID, "cl_pose_render: %d circles, %d limbs with null descriptors or mask", n_circles, n_limbs);
    if (!out_canvas && !out_guide) return set_error(CL_ERR_INVALID, "cl_pose_render: no output requested (out_canvas, out_guide both null)");
    if (B <= 0 || B > 65535) return set_error(CL_ERR_INVALID, "cl_pose_render: B = %d, expected 1..65535", B);
    if (out_h <= 0 || out_w <= 0 || out_h > PS_MAX_CANVAS || out_w > PS_MAX_CANVAS)
        return set_error(CL_ERR_INVALID, "cl_pose_render: output size %d x %d, expected 1..%d", out_h, out_w, PS_MAX_CANVAS);
    if (flip != 0 && flip != 1) return set_error(CL_ERR_INVALID, "cl_pose_render: flip = %d, expected 0 or 1", flip);
    if (mask_words < 0) return set_error(CL_ERR_INVALID, "cl_pose_render: mask_words = %lld", (long long)mask_words);
    for (int b = 0; b < B; ++b) {
        const cl_pose_image& d = img[b];
        if (d.Hc <= 0 || d.Wc <= 0 || d.Hc > PS_MAX_CANVAS || d.Wc > PS_MAX_CANVAS)
            return set_error(CL_ERR_INVALID, "cl_pose_render: image %d: canvas %d x %d, expected 1..%d", b, d.Hc, d.Wc, PS_MAX_CANVAS);
        if (d.h <= 0 || d.w <= 0 || d.y0 < 0 || d.x0 < 0 || d.y0 + d.h > d.Hc || d.x0 + d.w > d.Wc)
            return set_error(CL_ERR_INVALID, "cl_pose_render: image %d: crop (%d, %d) + %d x %d outside the %d x %d canvas", b, d.y0,
                             d.x0, d.h, d.w, d.Hc, d.Wc);
        if (d.bg_off != -1 && (!bg || d.bg_off < 0 || d.bg_off + 3ll * d.Hc * d.Wc > bg_bytes))
            return set_error(CL_ERR_INVALID, "cl_pose_render: image %d: background at byte %lld outside the %lld-byte bg", b,
                             (long long)d.bg_off, (long long)bg_bytes);
        if (d.circle0 < 0 || d.n_circles < 0 || (long long)d.circle0 + d.n_circles > n_circles || d.limb0 < 0 || d.n_limbs < 0 ||
            (long long)d.limb0 + d.n_limbs > n_limbs)
            return set_error(CL_ERR_INVALID, "cl_pose_render: image %d: circles [%d, +%d) or limbs [%d, +%d) outside %d / %d", b,
                             d.circle0, d.n_circles, d.limb0, d.n_limbs, n_circles, n_limbs);
        for (int i = d.circle0; i < d.circle0 + d.n_circles; ++i) {
            const cl_pose_circle& c = circles[i];
            if (c.x < -PS_MAX_COORD || c.x > PS_MAX_COORD || c.y < -PS_MAX_COORD || c.y > PS_MAX_COORD || c.color < 0 || c.color >= (1 << 24))
                return set_error(CL_ERR_INVALID, "cl_pose_render: circle %d: centre (%d, %d) or colour %d out of range", i, c.x, c.y, c.color);
        }
        for (int i = d.limb0; i < d.limb0 + d.n_limbs; ++i)
            if (limbs[i].image != b)
                return set_error(CL_ERR_INVALID, "cl_pose_render: limb %d is in image %d's range but names image %d", i, b, limbs[i].image);
    }
    for (int i = 0; i < n_limbs; ++i) {
        const cl_pose_limb& l = limbs[i];
        if (l.image == -1) continue;
        if (l.image < 0 || l.image >= B) return set_error(CL_ERR_INVALID, "cl_pose_render: limb %d: image %d of %d", i, l.image, B);
        const cl_pose_image& d = img[l.image];
        if (l.cx < -PS_MAX_COORD || l.cx > PS_MAX_COORD || l.cy < -PS_MAX_COORD || l.cy > PS_MAX_COORD || l.half_len < 0 ||
            l.half_len > PS_MAX_COORD || l.angle < -360 || l.angle > 360 || l.color < 0 || l.color >= (1 << 24))
            return set_error(CL_ERR_INVALID, "cl_pose_render: limb %d: centre (%d, %d), half length %d, angle %d or colour %d out of range",
                             i, l.cx, l.cy, l.half_len, l.angle, l.color);
        if (l.bw < 0 || l.bh < 0 || l.bx0 < 0 || l.by0 < 0 || (long long)l.bx0 + l.bw > d.Wc || (long long)l.by0 + l.bh > d.Hc)
            return set_error(CL_ERR_INVALID, "cl_pose_render: limb %d: box (%d, %d) + %d x %d outside the %d x %d canvas", i, l.bx0,
                             l.by0, l.bw, l.bh, d.Wc, d.Hc);
        if (l.mask_off < 0 || l.mask_off + (long long)l.bh * ((l.bw + 31) / 32) > mask_words)
            return set_error(CL_ERR_INVALID, "cl_pose_render: limb %d: bitmask at word %lld outside the %lld-word mask", i,
                             (long long)l.mask_off, (long long)mask_words);
    }
    launch_k(pose_limb_kernel, dim3(n_limbs > 0 ? n_limbs : 1), PS_LIMB_THREADS, 0, stream, img_dev, B, limbs_dev, n_limbs, mask,
             (long long)mask_words);
    launch_k(pose_render_kernel, dim3((out_w + 31) / 32, (out_h + 7) / 8, B), dim3(32, 8), 0, stream, img_dev, circles_dev,
             n_circles, limbs_dev, n_limbs, bg, mask, (long long)mask_words, out_h, out_w, flip, out_canvas, out_guide);
    count_launch(2);
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
