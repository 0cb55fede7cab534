// K6 — weight gradients of the (trainable) hint-encoder convolutions on wgmma, plus the small helper kernels the
// hint encoder needs every step (weight re-layout fp32 -> bf16, bias gradient, conv_in weight gradient).
//
//   dW[co, ci, ky, kx] += sum_{n,h,w} dY[n, h, w, co] * X[n, s*h + ky - pad, s*w + kx - pad, ci]
//
// As a GEMM per tap: D[co, ci] = dY^T[co, P] * X_tap[P, ci] with the reduction over pixels P.  Both operands are
// "pixel-major" in HBM (NHWC), i.e. MN-major for the tensor core, so the same TMA box loads as in the forward implicit
// GEMM land directly in the canonical MN-major 128B-swizzled layout; the 3x3 window shift is again a TMA coordinate
// offset with zero fill.  The pixel range is split across CTAs (split-K) and partial sums are reduced with fp32 RED.
//
// Replaces autograd's cudnn_convolution_backward_weight for models.py:470 (ConvBlock2D.conv1), :594 (Downsample2D).
#include <stdio.h>
#include <string.h>

#include "common.cuh"
#include "wgmma.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

struct WgradParams {
    int n_img, Ho, Wo, Cout, Cin, C_in_map;   // output-space geometry
    int mode;          // 1: stride 1 pad 1 ; 2: stride 2 pad_lo 0/1 (5-D strided view) ; 0: 1x1 (no shift)
    int pad_lo;
    int ksize;         // 3 or 1
    int bw, bh, bn, tiles_w, tiles_h, tiles_n, num_pix_blocks;
    int blocks_per_split;
    int cin_tiles, cout_tiles, tap_groups;
    float* dw;         // fp32 [Cout][Cin][k][k], accumulated
    float alpha;
};

static constexpr int WG_NT = 64;          // input-channel tile (wgmma N)
static constexpr int WG_TG = 3;           // taps per group
static constexpr int WG_STAGES = 2;
static constexpr int WG_THREADS = 384;    // producer warpgroup + two consumer warpgroups (64 output channels each)
static constexpr int WG_A_BYTES = 2 * 128 * 128;              // dY tile: 2 chunks x [128 px x 64 ch]
static constexpr int WG_B_BYTES = 128 * 128;                  // one X tile: [128 px x 64 ch]
static constexpr int WG_STAGE_BYTES = WG_A_BYTES + WG_TG * WG_B_BYTES;
static constexpr int WG_SMEM = 1024 + WG_STAGES * WG_STAGE_BYTES + 256;

__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, const WgradParams p) {
    pdl_launch_dependents();
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + WG_STAGES * WG_STAGE_BYTES);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + WG_STAGES;
    const int warp_idx = uniform_warp_idx(), lane = threadIdx.x & 31;
    const int wg = warp_idx >> 2;

    // work decomposition: blockIdx.y -> (cout tile, cin tile, tap group); blockIdx.x -> pixel split
    int wy = blockIdx.y;
    const int tg = wy % p.tap_groups; wy /= p.tap_groups;
    const int cit = wy % p.cin_tiles;
    const int cot = wy / p.cin_tiles;
    const int ntaps_total = p.ksize * p.ksize;
    const int tap0 = tg * WG_TG;
    const int ntaps = min(WG_TG, ntaps_total - tap0);
    const int pb0 = blockIdx.x * p.blocks_per_split;
    const int pb1 = min(p.num_pix_blocks, pb0 + p.blocks_per_split);

    if (warp_idx == 0 && lane == 0) {
        tma_prefetch_desc(&tmDY);
        tma_prefetch_desc(&tmX);
        for (int i = 0; i < WG_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();   // the prologue above touched only shared memory and kernel parameters

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (warp_idx == 0 && elect_one_sync()) {
            int stage = 0; uint32_t phase = 0;
            for (int pb = pb0; pb < pb1; ++pb) {
                const int tw = pb % p.tiles_w, th = (pb / p.tiles_w) % p.tiles_h, tn = pb / (p.tiles_w * p.tiles_h);
                mbar_wait(&empty_bar[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], WG_A_BYTES + ntaps * WG_B_BYTES);
                uint8_t* sa = smem + stage * WG_STAGE_BYTES;
                for (int c = 0; c < 2; ++c)
                    tma_load_4d(&tmDY, &full_bar[stage], sa + c * (128 * 128), cot * 128 + c * 64, tw * p.bw, th * p.bh, tn * p.bn);
                for (int t = 0; t < ntaps; ++t) {
                    uint8_t* sb = sa + WG_A_BYTES + t * WG_B_BYTES;
                    const int tap = tap0 + t;
                    const int ky = (p.ksize == 3) ? tap / 3 : 1, kx = (p.ksize == 3) ? tap % 3 : 1;
                    if (p.mode != 2) {
                        tma_load_4d(&tmX, &full_bar[stage], sb, cit * WG_NT, tw * p.bw + kx - 1, th * p.bh + ky - 1, tn * p.bn);
                    } else {
                        const int iy = ky - p.pad_lo, ix = kx - p.pad_lo;
                        tma_load_5d(&tmX, &full_bar[stage], sb, (ix & 1) * p.C_in_map + cit * WG_NT, tw * p.bw + (ix >> 1), iy & 1,
                                    th * p.bh + (iy >> 1), tn * p.bn);
                    }
                }
                if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    setmaxnreg_inc<232>();
    // D[co, ci] (per tap) = dY^T X over the tile's 128 pixels: A = dY chunk (wg - 1), B = X tap tile, both MN-major
    float acc[WG_TG][WG_NT / 2];
#pragma unroll
    for (int t = 0; t < WG_TG; ++t)
#pragma unroll
        for (int i = 0; i < WG_NT / 2; ++i) acc[t][i] = 0.f;
    {
        int stage = 0; uint32_t phase = 0;
        for (int pb = pb0; pb < pb1; ++pb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * WG_STAGE_BYTES) + (wg - 1) * (128 * 128);
            const uint32_t sb0 = smem_u32(smem + stage * WG_STAGE_BYTES) + WG_A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int t = 0; t < WG_TG; ++t) {
                if (t < ntaps) {
#pragma unroll
                    for (int kk = 0; kk < 8; ++kk)   // 128 pixels = 8 x K16
                        Wgmma<WG_NT, 1, 1>::mma(acc[t], make_smem_desc(sa + kk * 2048, 128 * 128, 1024, SWZ_128B),
                                                make_smem_desc(sb0 + t * WG_B_BYTES + kk * 2048, 128 * 128, 1024, SWZ_128B), 1);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);
            if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
        }
#pragma unroll
        for (int t = 0; t < WG_TG; ++t) wgmma_fence_acc(acc[t]);
    }
    if (pb1 <= pb0) return;
    // acc[t][j*4 + i*2 + c] = D[co row w*16 + lane/4 + 8i][ci col 8j + 2*(lane%4) + c]
    const int w4 = warp_idx & 3, q = lane & 3;
    const int kk2 = p.ksize * p.ksize;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int co = cot * 128 + (wg - 1) * 64 + w4 * 16 + (lane >> 2) + 8 * i;
        if (co >= p.Cout) continue;
#pragma unroll
        for (int t = 0; t < WG_TG; ++t) {
            if (t >= ntaps) continue;
#pragma unroll
            for (int j = 0; j < WG_NT / 8; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int ci = cit * WG_NT + 8 * j + 2 * q + c;
                    if (ci < p.Cin)
                        atomicAdd(&p.dw[((long long)co * p.Cin + ci) * kk2 + tap0 + t], p.alpha * acc[t][j * 4 + i * 2 + c]);
                }
        }
    }
}

// ---------------------------------------------------------------------------------------------- weight re-layout
// w fp32 [Cout][Cin][k][k] -> wf bf16 [Cout][k*k][Cin]  and  wd bf16 [Cin][k*k (flipped)][Cout]
__global__ void conv_weight_prep_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ wf, __nv_bfloat16* __restrict__ wd,
                                        int Cout, int Cin, int kk) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)Cout * Cin * kk;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % kk);
        const int ci = (int)((i / kk) % Cin);
        const int co = (int)(i / ((long long)kk * Cin));
        const __nv_bfloat16 v = __float2bfloat16(w[i]);
        wf[((long long)co * kk + t) * Cin + ci] = v;
        if (wd != nullptr) wd[((long long)ci * kk + (kk - 1 - t)) * Cout + co] = v;
    }
}

// ---------------------------------------------------------------------------------------------- column sums (bias grad)
// out[c] += alpha * sum_m x[m, c]
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ out, long long M, int C, float alpha, int rows_per_cta) {
    pdl_launch_dependents();
    pdl_wait();
    // thread -> column chunk of 8; CTA -> slab of rows; block-level smem reduction, then C global atomics per CTA
    __shared__ float sh[2048];
    for (int i = threadIdx.x; i < C; i += blockDim.x) sh[i] = 0.f;
    __syncthreads();
    const int chunks = C / 8;
    const int rows_par = blockDim.x / chunks;
    const int chunk = threadIdx.x % chunks, rsub = threadIdx.x / chunks;
    if (rsub < rows_par) {
        const long long r0 = (long long)blockIdx.x * rows_per_cta;
        const long long r1 = min(M, r0 + rows_per_cta);
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (long long m = r0 + rsub; m < r1; m += rows_par) {
            const uint4 u = *reinterpret_cast<const uint4*>(x + m * C + chunk * 8);
            const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
            acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y; acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(&sh[chunk * 8 + j], acc[j]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(&out[i], alpha * sh[i]);
}

// ---------------------------------------------------------------------------------------------- conv_in weight grad
// dW[co][ci][ky][kx] += sum_pix dY[pix][co] * x[n, ci, h+ky-1, w+kx-1];  x NCHW fp32 (bf16-rounded), dY NHWC bf16.
// A CTA walks its pixel range in blocks of 64 pixels staged in shared memory (im2col rows sx[pixel][k], dY rows
// sdy[pixel][32 channels of blockIdx.y's group]).  Thread = (pixel subset, 4 channels, 4 taps): 16 accumulators fed by
// two 16-byte shared loads per pixel, i.e. 8 FMAs per shared-memory instruction (the first version did 0.5).
template <int CIN>
__global__ void __launch_bounds__(256)
conv_in_wgrad_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ dy, float* __restrict__ dw, int n, int H, int W,
                     int Cout, int pix_per_cta) {
    pdl_launch_dependents();
    pdl_wait();
    constexpr int KK = 9 * CIN, KP = (KK + 3) / 4 * 4, KG = KP / 4, TPS = 8 * KG;
    constexpr int PS = (CIN == 3) ? 4 : 2;          // pixel subsets (PS * TPS <= 256)
    constexpr int PB = 64, PPS = PB / PS;
    static_assert(PS * TPS <= 256, "thread layout");
    __shared__ __align__(16) float sx[PB][KP];
    __shared__ __align__(16) float sdy[PB][32];
    __shared__ float red[PS][32][KP];
    const int tid = threadIdx.x;
    const int sub = tid / TPS, within = tid % TPS;
    const int cg = within / KG, kg = within % KG;
    const bool active = sub < PS;
    const int co0 = blockIdx.y * 32;
    const long long npix = (long long)n * H * W;
    const long long p0 = (long long)blockIdx.x * pix_per_cta;
    const long long p1 = min(npix, p0 + pix_per_cta);
    float acc[4][4];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[c][k] = 0.f;
    for (int i = tid; i < PB * (KP - KK); i += 256) sx[i / (KP - KK > 0 ? KP - KK : 1)][KK + i % (KP - KK > 0 ? KP - KK : 1)] = 0.f;   // pad taps
    for (long long pb = p0; pb < p1; pb += PB) {
        __syncthreads();
        for (int i = tid; i < PB * 9; i += 256) {        // one (pixel, tap) per item: the coordinate math is shared by the CIN loads
            const int pl = i / 9, tap = i % 9;
            const long long pix = pb + pl;
            bool ok = pix < p1;
            long long src = 0;
            if (ok) {
                const int b = (int)(pix / (H * W));
                const int hw = (int)(pix % (H * W));
                const int h = hw / W + tap / 3 - 1, ww = hw % W + tap % 3 - 1;
                ok = h >= 0 && h < H && ww >= 0 && ww < W;
                src = ((long long)b * CIN * H + h) * W + ww;
            }
#pragma unroll
            for (int ci = 0; ci < CIN; ++ci)
                sx[pl][tap * CIN + ci] = ok ? __bfloat162float(__float2bfloat16(__ldg(x + src + (long long)ci * H * W))) : 0.f;
        }
        for (int i = tid; i < PB * 8; i += 256) {
            const int pl = i / 8, c4 = (i % 8) * 4;
            const long long pix = pb + pl;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (pix < p1 && co0 + c4 + 4 <= Cout) {      // Cout % 4 == 0 is enforced on the host
                const uint2 u = __ldg(reinterpret_cast<const uint2*>(dy + pix * Cout + co0 + c4));
                const float2 a = unpack_bf16x2(u.x), c = unpack_bf16x2(u.y);
                v = make_float4(a.x, a.y, c.x, c.y);
            }
            *reinterpret_cast<float4*>(&sdy[pl][c4]) = v;
        }
        __syncthreads();
        if (active) {
#pragma unroll 4
            for (int pp = 0; pp < PPS; ++pp) {
                const int pl = sub * PPS + pp;
                const float4 d4 = *reinterpret_cast<const float4*>(&sdy[pl][cg * 4]);
                const float4 x4 = *reinterpret_cast<const float4*>(&sx[pl][kg * 4]);
                const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
                const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
                for (int c = 0; c < 4; ++c)
#pragma unroll
                    for (int k = 0; k < 4; ++k) acc[c][k] = fmaf(dv[c], xv[k], acc[c][k]);
            }
        }
    }
    if (active) {
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
            for (int k = 0; k < 4; ++k) red[sub][cg * 4 + c][kg * 4 + k] = acc[c][k];
    }
    __syncthreads();
    for (int o = tid; o < 32 * KK; o += 256) {
        const int co = o / KK, k = o % KK;
        if (co0 + co < Cout) {
            float v = 0.f;
#pragma unroll
            for (int s2 = 0; s2 < PS; ++s2) v += red[s2][co][k];
            const int tap = k / CIN, ci = k % CIN;
            atomicAdd(&dw[((long long)(co0 + co) * CIN + ci) * 9 + tap], v);
        }
    }
}

}  // namespace clb

using namespace clb;
#define STREAM cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_)
#define DONE()                         \
    count_launch();                    \
    CL_CUDA_CHECK(cudaGetLastError()); \
    return CL_OK

extern "C" int cl_conv_wgrad(const void* dy, const void* x, float* dw, int n_img, int H, int W, int Cin, int Cout, int ksize,
                             int stride, int pad_lo, float alpha, void* stream_) {
    STREAM;
    if (!dy || !x || !dw) return set_error(CL_ERR_INVALID, "cl_conv_wgrad: null");
    if (ksize != 1 && ksize != 3) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_wgrad: kernel size must be 1 or 3");
    if (stride != 1 && stride != 2) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_wgrad: stride must be 1 or 2");
    if (Cin % 8 || Cout % 8) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_wgrad: channels must be multiples of 8");
    if (stride == 2 && (H % 2 || W % 2 || ksize != 3)) return set_error(CL_ERR_INVALID, "cl_conv_wgrad: stride-2 needs even H, W and k=3");
    WgradParams p;
    memset(&p, 0, sizeof(p));
    p.n_img = n_img; p.Ho = H / stride; p.Wo = W / stride; p.Cout = Cout; p.Cin = Cin; p.C_in_map = Cin;
    p.mode = (stride == 2) ? 2 : 1; p.pad_lo = pad_lo; p.ksize = ksize; p.dw = dw; p.alpha = alpha;
    int bw = 128;
    while (bw > 1 && (p.Wo % bw) != 0) bw >>= 1;
    int bh = 128 / bw;
    while (bh > 1 && (p.Ho % bh) != 0) bh >>= 1;
    int bn = 128 / (bw * bh);
    p.bw = bw; p.bh = bh; p.bn = bn;
    p.tiles_w = p.Wo / bw; p.tiles_h = p.Ho / bh; p.tiles_n = (n_img + bn - 1) / bn;
    p.num_pix_blocks = p.tiles_w * p.tiles_h * p.tiles_n;
    p.cin_tiles = (Cin + WG_NT - 1) / WG_NT;
    p.cout_tiles = (Cout + 127) / 128;
    p.tap_groups = (ksize * ksize + WG_TG - 1) / WG_TG;
    const int tiles = p.cin_tiles * p.cout_tiles * p.tap_groups;
    int splits = (2 * num_sms() + tiles - 1) / tiles;
    if (splits > p.num_pix_blocks) splits = p.num_pix_blocks;
    if (splits < 1) splits = 1;
    p.blocks_per_split = (p.num_pix_blocks + splits - 1) / splits;
    splits = (p.num_pix_blocks + p.blocks_per_split - 1) / p.blocks_per_split;
    CUtensorMap tDY, tX;
    {
        const uint64_t C = Cout, Wd = p.Wo, Hd = p.Ho, NI = n_img;
        uint64_t dims[4] = {C, Wd, Hd, NI};
        uint64_t strides[3] = {C * 2, Wd * C * 2, Hd * Wd * C * 2};
        uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
        CL_CHECK(get_tensor_map(&tDY, dy, 4, dims, strides, box, 128));
    }
    {
        const uint64_t C = Cin, Wd = W, Hd = H, NI = n_img;
        if (stride == 1) {
            uint64_t dims[4] = {C, Wd, Hd, NI};
            uint64_t strides[3] = {C * 2, Wd * C * 2, Hd * Wd * C * 2};
            uint32_t box[4] = {64, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
            CL_CHECK(get_tensor_map(&tX, x, 4, dims, strides, box, 128));
        } else {
            uint64_t dims[5] = {2 * C, Wd / 2, 2, Hd / 2, NI};
            uint64_t strides[4] = {2 * C * 2, Wd * C * 2, 2 * Wd * C * 2, Hd * Wd * C * 2};
            uint32_t box[5] = {64, (uint32_t)bw, 1, (uint32_t)bh, (uint32_t)bn};
            CL_CHECK(get_tensor_map(&tX, x, 5, dims, strides, box, 128));
        }
    }
    static bool done = false;
    if (!done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(wgrad_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM));
        done = true;
    }
    launch_k(wgrad_wgmma_kernel, dim3(splits, tiles), WG_THREADS, WG_SMEM, stream, tDY, tX, p);
    DONE();
}

extern "C" int cl_conv_weight_prep(const float* w, void* wf, void* wd, int Cout, int Cin, int ksize, void* stream_) {
    STREAM;
    if (!w || !wf) return set_error(CL_ERR_INVALID, "cl_conv_weight_prep: null");
    const long long total = (long long)Cout * Cin * ksize * ksize;
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(conv_weight_prep_kernel, blocks, 256, 0, stream, w, reinterpret_cast<__nv_bfloat16*>(wf), reinterpret_cast<__nv_bfloat16*>(wd),
                                                        Cout, Cin, ksize * ksize);
    DONE();
}

extern "C" int cl_colsum(const void* x, float* out, int64_t M, int C, float alpha, void* stream_) {
    STREAM;
    if (!x || !out || C % 8 || C > 2048) return set_error(CL_ERR_INVALID, "cl_colsum: bad args");
    const int chunks = C / 8;
    int rows_par = 256 / chunks;
    if (rows_par < 1) rows_par = 1;
    int ctas = num_sms() * 4;
    int rows_per_cta = (int)((M + ctas - 1) / ctas);
    if (rows_per_cta < rows_par * 4) rows_per_cta = rows_par * 4;
    const int grid = (int)((M + rows_per_cta - 1) / rows_per_cta);
    launch_k(colsum_kernel, grid, 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x), out, M, C, alpha, rows_per_cta);
    DONE();
}

extern "C" int cl_conv_in_wgrad(const float* x, const void* dy, float* dw, int n, int Cin, int H, int W, int Cout, void* stream_) {
    STREAM;
    if (!x || !dy || !dw) return set_error(CL_ERR_INVALID, "cl_conv_in_wgrad: null");
    if (Cout % 4 != 0) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_in_wgrad: Cout must be a multiple of 4");
    const long long npix = (long long)n * H * W;
    const int groups = (Cout + 31) / 32;
    int ctas = (num_sms() * 8 + groups - 1) / groups;          // ~8 CTAs per SM over all channel groups
    long long ppc = (npix + ctas - 1) / ctas;
    ppc = ((ppc + 63) / 64) * 64;
    if (ppc < 256) ppc = 256;
    const dim3 grid((unsigned)((npix + ppc - 1) / ppc), (unsigned)groups);
    if (Cin == 3) launch_k(conv_in_wgrad_kernel<3>, grid, 256, 0, stream, x, reinterpret_cast<const __nv_bfloat16*>(dy), dw, n, H, W, Cout, (int)ppc);
    else if (Cin == 4) launch_k(conv_in_wgrad_kernel<4>, grid, 256, 0, stream, x, reinterpret_cast<const __nv_bfloat16*>(dy), dw, n, H, W, Cout, (int)ppc);
    else return set_error(CL_ERR_UNSUPPORTED, "cl_conv_in_wgrad: Cin must be 3 or 4");
    DONE();
}
