// Small SIMT kernels at the edges of the UNet: conv_in (4 -> C0), conv_out (C0 -> 4) and its input gradient, the
// timestep embedding + tiny-M linears (time MLP, all time_emb_proj layers at once), and the fused MSE loss.
// None of them is GEMM-shaped enough for tensor cores (K = 36, N = 4, or M = batch), all are weight/HBM-bound.
//
// Replaces: diffusers UNet2DConditionModel.conv_in / time_proj / time_embedding / ResnetBlock2D.time_emb_proj /
// conv_out as reached from train_text_to_image_control_lora.py:782, and F.mse_loss at :783.
#include <stdio.h>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

__device__ __forceinline__ float siluf(float z) { return z / (1.f + __expf(-z)); }

// ------------------------------------------------------------------------------------------ conv_in (3x3, Cin small)
// x: NCHW fp32 [n, Cin, H, W] (rounded to bf16 on load == the reference's cast to weight_dtype), w: bf16 [Cout][3][3][Cin],
// y: NHWC bf16 [n, H, W, Cout].  Thread = one output pixel x 32 output channels (blockIdx.y picks the channel group):
// the 9*Cin inputs and the 32 accumulators live in registers, the weights are read from shared memory as broadcast
// 16-byte loads ([k][32] layout), so the kernel is FMA-bound (~4 FMAs per shared-memory word) instead of LDS-bound.
template <int CIN>
__global__ void __launch_bounds__(256)
conv_in_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
               __nv_bfloat16* __restrict__ y, int n, int H, int W, int Cout) {
    pdl_launch_dependents();
    pdl_wait();
    constexpr int KK = 9 * CIN;
    __shared__ __align__(16) float sw[KK * 32];     // [k][32 channels of this group]
    __shared__ float sb[32];
    const int co0 = blockIdx.y * 32;
    for (int i = threadIdx.x; i < KK * 32; i += blockDim.x) {
        const int k = i / 32, c = i % 32;
        sw[i] = (co0 + c < Cout) ? __bfloat162float(w[(size_t)(co0 + c) * KK + k]) : 0.f;
    }
    if (threadIdx.x < 32) sb[threadIdx.x] = (bias != nullptr && co0 + threadIdx.x < Cout) ? bias[co0 + threadIdx.x] : 0.f;
    __syncthreads();
    const long long npix = (long long)n * H * W;
    const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= npix) return;
    const int b = (int)(pix / (H * W));
    const int hw = (int)(pix % (H * W));
    const int h0 = hw / W, w0 = hw % W;
    float xin[KK];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
        const int h = h0 + tap / 3 - 1, ww = w0 + tap % 3 - 1;
        const bool ok = h >= 0 && h < H && ww >= 0 && ww < W;
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci)
            xin[tap * CIN + ci] = ok ? __bfloat162float(__float2bfloat16(__ldg(x + (((long long)b * CIN + ci) * H + h) * W + ww))) : 0.f;
    }
    float acc[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) acc[c] = sb[c];
#pragma unroll
    for (int k = 0; k < KK; ++k) {
        const float xv = xin[k];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 w4 = *reinterpret_cast<const float4*>(sw + k * 32 + q * 4);
            acc[4 * q] = fmaf(xv, w4.x, acc[4 * q]);
            acc[4 * q + 1] = fmaf(xv, w4.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(xv, w4.z, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(xv, w4.w, acc[4 * q + 3]);
        }
    }
    __nv_bfloat16* yp = y + pix * Cout + co0;
    if (co0 + 32 <= Cout) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            uint4 o;
            o.x = pack_bf16x2(acc[8 * q], acc[8 * q + 1]); o.y = pack_bf16x2(acc[8 * q + 2], acc[8 * q + 3]);
            o.z = pack_bf16x2(acc[8 * q + 4], acc[8 * q + 5]); o.w = pack_bf16x2(acc[8 * q + 6], acc[8 * q + 7]);
            *reinterpret_cast<uint4*>(yp + 8 * q) = o;
        }
    } else {
#pragma unroll
        for (int c = 0; c < 32; ++c)
            if (co0 + c < Cout) yp[c] = __float2bfloat16(acc[c]);
    }
}

// ------------------------------------------------------------------------------------------ conv_out (3x3, Cout small)
// x: NHWC bf16 [n, H, W, C], w: bf16 [COUT][3][3][C], y: NCHW fp32 [n, COUT, H, W].  One warp per output pixel.
template <int COUT>
__global__ void __launch_bounds__(256)
conv_out_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                float* __restrict__ y, int n, int H, int W, int C) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ __nv_bfloat16 swb[];   // [COUT][9][C]
    for (int i = threadIdx.x; i < COUT * 9 * C / 8; i += blockDim.x)
        reinterpret_cast<uint4*>(swb)[i] = reinterpret_cast<const uint4*>(w)[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int chunks = C / 8;
    const long long npix = (long long)n * H * W;
    for (long long pix = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pix < npix;
         pix += (long long)gridDim.x * (blockDim.x >> 5)) {
        const int b = (int)(pix / (H * W));
        const int hw = (int)(pix % (H * W));
        const int h0 = hw / W, w0 = hw % W;
        float acc[COUT];
#pragma unroll
        for (int co = 0; co < COUT; ++co) acc[co] = 0.f;
        for (int tap = 0; tap < 9; ++tap) {
            const int h = h0 + tap / 3 - 1, ww = w0 + tap % 3 - 1;
            if (h < 0 || h >= H || ww < 0 || ww >= W) continue;
            const __nv_bfloat16* xp = x + (((long long)b * H + h) * W + ww) * C;
            for (int ch = lane; ch < chunks; ch += 32) {
                const uint4 xv = *reinterpret_cast<const uint4*>(xp + ch * 8);
                const float2 x0 = unpack_bf16x2(xv.x), x1 = unpack_bf16x2(xv.y), x2 = unpack_bf16x2(xv.z), x3 = unpack_bf16x2(xv.w);
#pragma unroll
                for (int co = 0; co < COUT; ++co) {
                    const uint4 wv = *reinterpret_cast<const uint4*>(swb + ((long long)co * 9 + tap) * C + ch * 8);
                    const float2 w0f = unpack_bf16x2(wv.x), w1f = unpack_bf16x2(wv.y), w2f = unpack_bf16x2(wv.z), w3f = unpack_bf16x2(wv.w);
                    acc[co] += x0.x * w0f.x + x0.y * w0f.y + x1.x * w1f.x + x1.y * w1f.y + x2.x * w2f.x + x2.y * w2f.y +
                               x3.x * w3f.x + x3.y * w3f.y;
                }
            }
        }
#pragma unroll
        for (int co = 0; co < COUT; ++co) {
            const float s = warp_sum(acc[co]);
            if (lane == 0) y[(((long long)b * COUT + co) * H + h0) * W + w0] = s + (bias ? bias[co] : 0.f);
        }
    }
}

// input gradient of conv_out: dy NCHW fp32 [n, COUT, H, W] -> dx NHWC bf16 [n, H, W, C]; thread = (pixel, 8 channels)
template <int COUT>
__global__ void __launch_bounds__(256)
conv_out_bwd_kernel(const float* __restrict__ dy, const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ dx, int n,
                    int H, int W, int C) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ __nv_bfloat16 swb[];   // [COUT][9][C]
    for (int i = threadIdx.x; i < COUT * 9 * C / 8; i += blockDim.x)
        reinterpret_cast<uint4*>(swb)[i] = reinterpret_cast<const uint4*>(w)[i];
    __syncthreads();
    const int chunks = C / 8;
    const long long total = (long long)n * H * W * chunks;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ch = (int)(i % chunks);
        const long long pix = i / chunks;
        const int b = (int)(pix / (H * W));
        const int hw = (int)(pix % (H * W));
        const int h0 = hw / W, w0 = hw % W;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int tap = 0; tap < 9; ++tap) {
            // y[h0 - ky + 1, w0 - kx + 1] used x[h0, w0] through tap (ky, kx)
            const int h = h0 - (tap / 3) + 1, ww = w0 - (tap % 3) + 1;
            if (h < 0 || h >= H || ww < 0 || ww >= W) continue;
#pragma unroll
            for (int co = 0; co < COUT; ++co) {
                const float g = dy[(((long long)b * COUT + co) * H + h) * W + ww];
                const uint4 wv = *reinterpret_cast<const uint4*>(swb + ((long long)co * 9 + tap) * C + ch * 8);
                const float2 a = unpack_bf16x2(wv.x), bq = unpack_bf16x2(wv.y), c = unpack_bf16x2(wv.z), d = unpack_bf16x2(wv.w);
                acc[0] += g * a.x; acc[1] += g * a.y; acc[2] += g * bq.x; acc[3] += g * bq.y;
                acc[4] += g * c.x; acc[5] += g * c.y; acc[6] += g * d.x; acc[7] += g * d.y;
            }
        }
        uint4 o;
        o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
        o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
        *reinterpret_cast<uint4*>(dx + pix * C + ch * 8) = o;
    }
}

// ------------------------------------------------------------------------------------------ timestep embedding
// out[b, :] = [cos(t * f_i) | sin(t * f_i)], f_i = exp(-ln(10000) * i / half)   (flip_sin_to_cos, freq_shift 0)
__global__ void timestep_embedding_kernel(const float* __restrict__ t, float* __restrict__ out, int B, int dim) {
    pdl_launch_dependents();
    pdl_wait();
    const int half = dim / 2;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * half; i += gridDim.x * blockDim.x) {
        const int b = i / half, j = i % half;
        const float f = expf(-9.210340371976184f * (float)j / (float)half);
        const float a = t[b] * f;
        out[b * dim + j] = cosf(a);
        out[b * dim + half + j] = sinf(a);
    }
}

// ------------------------------------------------------------------------------------------ tiny-M linear
// out[b, n] = act_out( sum_k act_in(x[b, k]) * W[n, k] + bias[n] );  x fp32 [Bt, K], W bf16 [N, K]; warp per n.
static constexpr int SL_MAXB = 8;
__global__ void __launch_bounds__(256)
small_linear_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                    float* __restrict__ out, int Bt, int N, int K, int silu_in, int silu_out) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sxs[];  // [nb][K]
    const int b0 = blockIdx.y * SL_MAXB;
    const int nb = min(SL_MAXB, Bt - b0);
    for (int i = threadIdx.x; i < nb * K; i += blockDim.x) {
        float v = x[(long long)(b0 + i / K) * K + i % K];
        sxs[i] = silu_in ? siluf(v) : v;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int nrow = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (nrow >= N) return;
    float acc[SL_MAXB];
#pragma unroll
    for (int b = 0; b < SL_MAXB; ++b) acc[b] = 0.f;
    for (int k = lane * 8; k < K; k += 256) {
        const uint4 wv = *reinterpret_cast<const uint4*>(w + (long long)nrow * K + k);
        const float2 w0 = unpack_bf16x2(wv.x), w1 = unpack_bf16x2(wv.y), w2 = unpack_bf16x2(wv.z), w3 = unpack_bf16x2(wv.w);
#pragma unroll
        for (int b = 0; b < SL_MAXB; ++b) {
            if (b < nb) {
                const float* xp = sxs + b * K + k;
                acc[b] += xp[0] * w0.x + xp[1] * w0.y + xp[2] * w1.x + xp[3] * w1.y + xp[4] * w2.x + xp[5] * w2.y +
                          xp[6] * w3.x + xp[7] * w3.y;
            }
        }
    }
#pragma unroll
    for (int b = 0; b < SL_MAXB; ++b) {
        if (b < nb) {
            float s = warp_sum(acc[b]);
            if (lane == 0) {
                s += bias ? bias[nrow] : 0.f;
                out[(long long)(b0 + b) * N + nrow] = silu_out ? siluf(s) : s;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ MSE (mean) + gradient
// loss += sum((pred - target)^2) / n ; dpred = 2 (pred - target) / n * gscale
__global__ void __launch_bounds__(256)
mse_kernel(const float* __restrict__ pred, const float* __restrict__ target, float* __restrict__ loss,
           float* __restrict__ dpred, long long n, float gscale) {
    pdl_launch_dependents();
    pdl_wait();
    float s = 0.f;
    const float inv = 1.f / (float)n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float d = pred[i] - target[i];
        s += d * d;
        if (dpred) dpred[i] = 2.f * d * inv * gscale;
    }
    s = warp_sum(s);
    __shared__ float part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += part[i];
        atomicAdd(loss, t * inv);
    }
}

}  // namespace clb

using namespace clb;
#define STREAM cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_)
#define DONE()                         \
    count_launch();                    \
    CL_CUDA_CHECK(cudaGetLastError()); \
    return CL_OK

extern "C" int cl_conv_in(const float* x, const void* w, const float* bias, void* y, int n, int Cin, int H, int W, int Cout,
                          void* stream_) {
    STREAM;
    if (!x || !w || !y) return set_error(CL_ERR_INVALID, "cl_conv_in: null");
    const long long npix = (long long)n * H * W;
    if (Cout % 8 != 0) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_in: Cout must be a multiple of 8");
    const dim3 grid((unsigned)((npix + 255) / 256), (unsigned)((Cout + 31) / 32));
#define CONV_IN_CASE(CI)                                                                                         \
    case CI:                                                                                                     \
        launch_k(conv_in_kernel<CI>, grid, 256, 0, stream, x, reinterpret_cast<const __nv_bfloat16*>(w), bias,         \
                                                     reinterpret_cast<__nv_bfloat16*>(y), n, H, W, Cout);        \
        break;
    switch (Cin) {
        CONV_IN_CASE(3)
        CONV_IN_CASE(4)
        default: return set_error(CL_ERR_UNSUPPORTED, "cl_conv_in: Cin must be 3 or 4");
    }
#undef CONV_IN_CASE
    DONE();
}

extern "C" int cl_conv_out(const void* x, const void* w, const float* bias, float* y, int n, int H, int W, int C, int Cout,
                           void* stream_) {
    STREAM;
    if (!x || !w || !y) return set_error(CL_ERR_INVALID, "cl_conv_out: null");
    if (Cout != 4 || C % 8) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_out: Cout must be 4, C %% 8 == 0");
    const size_t smem = (size_t)4 * 9 * C * 2;
    static bool done = false;
    if (!done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(conv_out_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        done = true;
    }
    if (smem > 200 * 1024) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_out: C too large");
    launch_k(conv_out_kernel<4>, num_sms() * 4, 256, smem, stream, reinterpret_cast<const __nv_bfloat16*>(x),
                                                            reinterpret_cast<const __nv_bfloat16*>(w), bias, y, n, H, W, C);
    DONE();
}

extern "C" int cl_conv_out_bwd(const float* dy, const void* w, void* dx, int n, int H, int W, int C, int Cout, void* stream_) {
    STREAM;
    if (!dy || !w || !dx) return set_error(CL_ERR_INVALID, "cl_conv_out_bwd: null");
    if (Cout != 4 || C % 8) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_out_bwd: Cout must be 4, C %% 8 == 0");
    const size_t smem = (size_t)4 * 9 * C * 2;
    static bool done = false;
    if (!done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(conv_out_bwd_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        done = true;
    }
    if (smem > 200 * 1024) return set_error(CL_ERR_UNSUPPORTED, "cl_conv_out_bwd: C too large");
    launch_k(conv_out_bwd_kernel<4>, num_sms() * 4, 256, smem, stream, dy, reinterpret_cast<const __nv_bfloat16*>(w),
                                                                reinterpret_cast<__nv_bfloat16*>(dx), n, H, W, C);
    DONE();
}

extern "C" int cl_timestep_embedding(const float* t, float* out, int B, int dim, void* stream_) {
    STREAM;
    if (!t || !out || dim % 2) return set_error(CL_ERR_INVALID, "cl_timestep_embedding: bad args");
    launch_k(timestep_embedding_kernel, (B * dim / 2 + 255) / 256, 256, 0, stream, t, out, B, dim);
    DONE();
}

extern "C" int cl_small_linear(const float* x, const void* w, const float* bias, float* out, int Bt, int N, int K,
                               int silu_in, int silu_out, void* stream_) {
    STREAM;
    if (!x || !w || !out || K % 8) return set_error(CL_ERR_INVALID, "cl_small_linear: bad args");
    const size_t smem = (size_t)SL_MAXB * K * sizeof(float);
    if (smem > 48 * 1024) return set_error(CL_ERR_UNSUPPORTED, "cl_small_linear: K too large");
    dim3 grid((N + 7) / 8, (Bt + SL_MAXB - 1) / SL_MAXB);
    launch_k(small_linear_kernel, grid, 256, smem, stream, x, reinterpret_cast<const __nv_bfloat16*>(w), bias, out, Bt, N, K,
                                                     silu_in, silu_out);
    DONE();
}

extern "C" int cl_mse_loss(const float* pred, const float* target, float* loss, float* dpred, int64_t n, float gscale,
                           void* stream_) {
    STREAM;
    if (!pred || !target || !loss) return set_error(CL_ERR_INVALID, "cl_mse_loss: null");
    CL_CUDA_CHECK(cudaMemsetAsync(loss, 0, sizeof(float), stream));
    int blocks = (int)((n + 255) / 256);
    if (blocks > num_sms() * 4) blocks = num_sms() * 4;
    launch_k(mse_kernel, blocks, 256, 0, stream, pred, target, loss, dpred, n, gscale);
    DONE();
}

// ------------------------------------------------------------------------------------------ CFG + DDIM update (eta = 0)
// eps = eps_u + g (eps_c - eps_u);  x0 = (x - sqrt(1-a_t) eps) / sqrt(a_t);  x <- sqrt(a_prev) x0 + sqrt(1-a_prev) eps
// (classifier-free guidance as in StableDiffusionPipeline + diffusers DDIMScheduler.step, the loop of
//  train_text_to_image_control_lora.py:829-843 / apps/gradio_canny2image.py:81-89 with BASELINE config 3's scheduler)
namespace clb {
__global__ void cfg_ddim_kernel(const float* __restrict__ eps2, float* __restrict__ x, long long n_half, float g, float sa_t,
                                float s1a_t, float sa_p, float s1a_p) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_half; i += (long long)gridDim.x * blockDim.x) {
        const float eu = eps2[i], ec = eps2[n_half + i];
        const float e = eu + g * (ec - eu);
        const float x0 = (x[i] - s1a_t * e) / sa_t;
        x[i] = sa_p * x0 + s1a_p * e;
    }
}
}  // namespace clb

extern "C" int cl_cfg_ddim_step(const float* eps2, float* latents, int64_t n_half, float guidance, float sqrt_at, float sqrt_1m_at,
                                float sqrt_aprev, float sqrt_1m_aprev, void* stream_) {
    STREAM;
    if (!eps2 || !latents) return set_error(CL_ERR_INVALID, "cl_cfg_ddim_step: null");
    int blocks = (int)((n_half + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(clb::cfg_ddim_kernel, blocks, 256, 0, stream, eps2, latents, n_half, guidance, sqrt_at, sqrt_1m_at, sqrt_aprev, sqrt_1m_aprev);
    DONE();
}

// ------------------------------------------------------------------------------------------ CFG + DPM-Solver++(2M) step
// eps = eps_u + g (eps_c - eps_u);  x0 = (x - sigma_s eps) / alpha_s;  x <- c_x x + c_m0 x0 + c_m1 x0_prev;  x0_prev <- x0
// (diffusers-0.13 DPMSolverMultistepScheduler.step, dpmsolver++ / midpoint / order 2, the scheduler the reference's
//  validation loop and apps use: train_text_to_image_control_lora.py:817-823, mix_lora_and_control_lora.py:80; the five
//  scalars come from controllora_b200/sampler.py:dpmpp_2m_coeffs)
namespace clb {
__global__ void cfg_dpmpp_kernel(const float* __restrict__ eps2, float* __restrict__ x, float* __restrict__ x0_prev, long long n_half,
                                 float g, float alpha_s, float sigma_s, float c_x, float c_m0, float c_m1) {
    pdl_launch_dependents();
    pdl_wait();
    const float inv_a = 1.f / alpha_s;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_half; i += (long long)gridDim.x * blockDim.x) {
        const float eu = eps2[i], ec = eps2[n_half + i];
        const float e = eu + g * (ec - eu);
        const float xv = x[i];
        const float x0 = (xv - sigma_s * e) * inv_a;
        x[i] = c_x * xv + c_m0 * x0 + c_m1 * x0_prev[i];
        x0_prev[i] = x0;
    }
}
}  // namespace clb

extern "C" int cl_cfg_dpmpp_step(const float* eps2, float* latents, float* x0_prev, int64_t n_half, float guidance, float alpha_s,
                                 float sigma_s, float c_x, float c_m0, float c_m1, void* stream_) {
    STREAM;
    if (!eps2 || !latents || !x0_prev) return set_error(CL_ERR_INVALID, "cl_cfg_dpmpp_step: null");
    int blocks = (int)((n_half + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(clb::cfg_dpmpp_kernel, blocks, 256, 0, stream, eps2, latents, x0_prev, n_half, guidance, alpha_s, sigma_s, c_x, c_m0, c_m1);
    DONE();
}

// ------------------------------------------------------------------------------------------ denoise loop as ONE replayed CUDA graph
// The per-step scalars of the loop (timestep, solver coefficients) come from device tables indexed by a device step
// counter, so the captured {prep -> UNet -> CFG + solver update -> counter + 1} sequence can be replayed num_steps times
// without host work (StableDiffusionPipeline.__call__'s loop, train_text_to_image_control_lora.py:829-843).
namespace clb {
// x2 = [latents | latents] (the CFG batch), tt[0 .. B2) = timestep_table[*step]
__global__ void sampler_prep_kernel(const float* __restrict__ latents, float* __restrict__ x2, float* __restrict__ tt,
                                    const float* __restrict__ ts_table, const unsigned long long* __restrict__ step_ctr,
                                    long long n_half, int B2) {
    pdl_launch_dependents();
    pdl_wait();
    const unsigned long long step = *step_ctr;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_half; i += (long long)gridDim.x * blockDim.x) {
        const float v = latents[i];
        x2[i] = v;
        x2[n_half + i] = v;
    }
    if (blockIdx.x == 0 && threadIdx.x < B2) tt[threadIdx.x] = ts_table[step];
}

// kind 0: DDIM (coef = sqrt_at, sqrt_1m_at, sqrt_aprev, sqrt_1m_aprev), kind 1: DPM-Solver++(2M) (coef = alpha_s, sigma_s,
// c_x, c_m0, c_m1); same arithmetic as cfg_ddim_kernel / cfg_dpmpp_kernel, coefficients read from coef[*step][8].
__global__ void cfg_solver_dev_kernel(const float* __restrict__ eps2, float* __restrict__ x, float* __restrict__ x0_prev,
                                      const float* __restrict__ coef, const unsigned long long* __restrict__ step_ctr,
                                      long long n_half, float g, int kind) {
    pdl_launch_dependents();
    pdl_wait();
    const float* c = coef + 8 * (*step_ctr);
    const float c0 = c[0], c1 = c[1], c2 = c[2], c3 = c[3], c4 = c[4];
    const float inv_a = 1.f / c0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_half; i += (long long)gridDim.x * blockDim.x) {
        const float eu = eps2[i], ec = eps2[n_half + i];
        const float e = eu + g * (ec - eu);
        const float xv = x[i];
        if (kind == 0) {
            const float x0 = (xv - c1 * e) / c0;
            x[i] = c2 * x0 + c3 * e;
        } else {
            const float x0 = (xv - c1 * e) * inv_a;
            x[i] = c2 * xv + c3 * x0 + c4 * x0_prev[i];
            x0_prev[i] = x0;
        }
    }
}

__global__ void counter_advance_kernel(unsigned long long* ctr) {
    pdl_launch_dependents();
    pdl_wait();
    *ctr += 1ull;
}
}  // namespace clb

extern "C" int cl_sampler_prep(const float* latents, float* x2, float* tt, const float* ts_table, const unsigned long long* step_ctr,
                               int64_t n_half, int B2, void* stream_) {
    STREAM;
    if (!latents || !x2 || !tt || !ts_table || !step_ctr || B2 <= 0 || B2 > 256)
        return set_error(CL_ERR_INVALID, "cl_sampler_prep: bad arguments (CFG batch <= 256)");
    int blocks = (int)((n_half + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(clb::sampler_prep_kernel, blocks, 256, 0, stream, latents, x2, tt, ts_table, step_ctr, (long long)n_half, B2);
    DONE();
}

extern "C" int cl_cfg_solver_step_dev(const float* eps2, float* latents, float* x0_prev, const float* coef,
                                      unsigned long long* step_ctr, int64_t n_half, float guidance, int kind, void* stream_) {
    STREAM;
    if (!eps2 || !latents || !coef || !step_ctr || (kind == 1 && !x0_prev) || (kind != 0 && kind != 1))
        return set_error(CL_ERR_INVALID, "cl_cfg_solver_step_dev: bad arguments");
    int blocks = (int)((n_half + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(clb::cfg_solver_dev_kernel, blocks, 256, 0, stream, eps2, latents, x0_prev, coef, (const unsigned long long*)step_ctr,
             (long long)n_half, guidance, kind);
    count_launch();
    launch_k(clb::counter_advance_kernel, 1, 1, 0, stream, step_ctr);
    DONE();
}
