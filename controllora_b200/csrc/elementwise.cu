// HBM-bound glue kernels of the UNet path (all 16-byte vectorised, grid-stride, channels-last bf16):
// GEGLU, residual adds, nearest-2x upsample (+ its adjoint), channel concat / split, zero insertion for the
// stride-2 conv adjoint, bf16<->fp32 layout changes at the UNet boundary.
#include <stdio.h>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&f)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&f)[8]) {
    uint4 u;
    u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
    u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(p) = u;
}

static inline int ew_blocks(long long work, int threads = 256) {
    long long b = (work + threads - 1) / threads;
    const long long cap = (long long)num_sms() * 16;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

#define GRID_STRIDE(i, n) \
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (long long)gridDim.x * blockDim.x)

// ---------------------------------------------------------------- GEGLU: out = a * gelu_erf(g), p = [a | g]
__device__ __forceinline__ float gelu_grad_f(float x) {
    return 0.5f * (1.f + erff(x * 0.70710678118654752f)) + x * 0.3989422804014327f * __expf(-0.5f * x * x);
}

__global__ void geglu_fwd_kernel(const __nv_bfloat16* __restrict__ p, __nv_bfloat16* __restrict__ out, long long T, int F) {
    pdl_launch_dependents();
    pdl_wait();
    const int ch = F / 8;
    GRID_STRIDE(i, T * ch) {
        const long long t = i / ch;
        const int c = (int)(i % ch) * 8;
        float a[8], g[8], o[8];
        ld8(p + t * 2 * F + c, a);
        ld8(p + t * 2 * F + F + c, g);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = a[j] * gelu_f(g[j]);
        st8(out + t * F + c, o);
    }
}
__global__ void geglu_bwd_kernel(const __nv_bfloat16* __restrict__ p, const __nv_bfloat16* __restrict__ dout,
                                 __nv_bfloat16* __restrict__ dp, long long T, int F) {
    pdl_launch_dependents();
    pdl_wait();
    const int ch = F / 8;
    GRID_STRIDE(i, T * ch) {
        const long long t = i / ch;
        const int c = (int)(i % ch) * 8;
        float a[8], g[8], d[8], da[8], dg[8];
        ld8(p + t * 2 * F + c, a);
        ld8(p + t * 2 * F + F + c, g);
        ld8(dout + t * F + c, d);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            da[j] = d[j] * gelu_f(g[j]);
            dg[j] = d[j] * a[j] * gelu_grad_f(g[j]);
        }
        st8(dp + t * 2 * F + c, da);
        st8(dp + t * 2 * F + F + c, dg);
    }
}

// ---------------------------------------------------------------- out = a + b
__global__ void add_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b,
                           __nv_bfloat16* __restrict__ out, long long n8) {
    pdl_launch_dependents();
    pdl_wait();
    GRID_STRIDE(i, n8) {
        float x[8], y[8];
        ld8(a + i * 8, x);
        ld8(b + i * 8, y);
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] += y[j];
        st8(out + i * 8, x);
    }
}

// ---------------------------------------------------------------- nearest 2x upsample and its adjoint
__global__ void upsample2x_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int n, int H, int W, int C) {
    pdl_launch_dependents();
    pdl_wait();
    const int ch = C / 8;
    const long long total = (long long)n * 2 * H * 2 * W * ch;
    GRID_STRIDE(i, total) {
        const int c = (int)(i % ch);
        long long r = i / ch;
        const int wo = (int)(r % (2 * W)); r /= 2 * W;
        const int ho = (int)(r % (2 * H));
        const int b = (int)(r / (2 * H));
        const uint4 v = *reinterpret_cast<const uint4*>(x + (((long long)b * H + ho / 2) * W + wo / 2) * C + c * 8);
        *reinterpret_cast<uint4*>(y + i * 8) = v;
    }
}
__global__ void upsample2x_bwd_kernel(const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ dx, int n, int H, int W,
                                      int C, int accumulate) {
    pdl_launch_dependents();
    pdl_wait();
    const int ch = C / 8;
    const long long total = (long long)n * H * W * ch;
    GRID_STRIDE(i, total) {
        const int c = (int)(i % ch);
        long long r = i / ch;
        const int w = (int)(r % W); r /= W;
        const int h = (int)(r % H);
        const int b = (int)(r / H);
        float acc[8];
        if (accumulate) ld8(dx + i * 8, acc);
        else {
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        }
#pragma unroll
        for (int dyy = 0; dyy < 2; ++dyy)
#pragma unroll
            for (int dxx = 0; dxx < 2; ++dxx) {
                float v[8];
                ld8(dy + (((long long)b * 2 * H + 2 * h + dyy) * 2 * W + 2 * w + dxx) * C + c * 8, v);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[j];
            }
        st8(dx + i * 8, acc);
    }
}

// ---------------------------------------------------------------- zero insertion (adjoint of stride-2 sampling)
// out [n, 2H, 2W, C] = 0 except out[b, 2h+off, 2w+off, :] = x[b, h, w, :]
__global__ void zero_insert2x_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, int n, int H, int W,
                                     int C, int off) {
    pdl_launch_dependents();
    pdl_wait();
    const int ch = C / 8;
    const long long total = (long long)n * 2 * H * 2 * W * ch;
    GRID_STRIDE(i, total) {
        const int c = (int)(i % ch);
        long long r = i / ch;
        const int wo = (int)(r % (2 * W)); r /= 2 * W;
        const int ho = (int)(r % (2 * H));
        const int b = (int)(r / (2 * H));
        uint4 v = make_uint4(0, 0, 0, 0);
        if ((ho & 1) == off && (wo & 1) == off)
            v = *reinterpret_cast<const uint4*>(x + (((long long)b * H + ho / 2) * W + wo / 2) * C + c * 8);
        *reinterpret_cast<uint4*>(y + i * 8) = v;
    }
}

// ---------------------------------------------------------------- channel concat / split on [M, C] matrices
__global__ void concat_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b,
                              __nv_bfloat16* __restrict__ out, long long M, int Ca, int Cb) {
    pdl_launch_dependents();
    pdl_wait();
    const int ch = (Ca + Cb) / 8, cha = Ca / 8;
    GRID_STRIDE(i, M * ch) {
        const long long m = i / ch;
        const int c = (int)(i % ch);
        const uint4 v = (c < cha) ? *reinterpret_cast<const uint4*>(a + m * Ca + c * 8)
                                  : *reinterpret_cast<const uint4*>(b + m * Cb + (c - cha) * 8);
        *reinterpret_cast<uint4*>(out + i * 8) = v;
    }
}
// dst[m, :] (+)= src[m, c_off : c_off + Cd]
__global__ void slice_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long M, int Cs,
                             int c_off, int Cd, int accumulate) {
    pdl_launch_dependents();
    pdl_wait();
    const int ch = Cd / 8;
    GRID_STRIDE(i, M * ch) {
        const long long m = i / ch;
        const int c = (int)(i % ch);
        float v[8];
        ld8(src + m * Cs + c_off + c * 8, v);
        if (accumulate) {
            float o[8];
            ld8(dst + i * 8, o);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] += o[j];
        }
        st8(dst + i * 8, v);
    }
}

// ---------------------------------------------------------------- layout / dtype changes at the boundary
// NCHW (fp32 or bf16) -> NHWC bf16, and NHWC bf16 -> NCHW fp32 (used for control states / their gradients)
template <typename TIn>
__global__ void nchw_to_nhwc_kernel(const TIn* __restrict__ x, __nv_bfloat16* __restrict__ y, int n, int C, int HW) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, p = p0 + threadIdx.x;
        tile[i][threadIdx.x] = (c < C && p < HW) ? (float)x[((long long)b * C + c) * HW + p] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int p = p0 + i, c = c0 + threadIdx.x;
        if (p < HW && c < C) y[((long long)b * HW + p) * C + c] = __float2bfloat16(tile[threadIdx.x][i]);
    }
}
__global__ void nhwc_to_nchw_f32_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ y, int n, int C, int HW,
                                        int accumulate) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int p = p0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (c < C && p < HW) ? __bfloat162float(x[((long long)b * HW + p) * C + c]) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, p = p0 + threadIdx.x;
        if (c < C && p < HW) {
            const long long o = ((long long)b * C + c) * HW + p;
            y[o] = accumulate ? y[o] + tile[threadIdx.x][i] : tile[threadIdx.x][i];
        }
    }
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
    pdl_launch_dependents();
    pdl_wait();
    GRID_STRIDE(i, n) y[i] = __float2bfloat16(x[i]);
}
__global__ void bf16_to_f32_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ y, long long n) {
    pdl_launch_dependents();
    pdl_wait();
    GRID_STRIDE(i, n) y[i] = __bfloat162float(x[i]);
}

}  // namespace clb

using namespace clb;
#define BF(p) reinterpret_cast<const __nv_bfloat16*>(p)
#define BFW(p) reinterpret_cast<__nv_bfloat16*>(p)
#define STREAM cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_)
#define DONE()                           \
    count_launch();                      \
    CL_CUDA_CHECK(cudaGetLastError());   \
    return CL_OK

extern "C" int cl_geglu_fwd(const void* p, void* out, int64_t T, int F, void* stream_) {
    STREAM;
    if (!p || !out || F % 8) return set_error(CL_ERR_INVALID, "cl_geglu_fwd: bad args");
    launch_k(geglu_fwd_kernel, ew_blocks(T * (F / 8)), 256, 0, stream, BF(p), BFW(out), T, F);
    DONE();
}
extern "C" int cl_geglu_bwd(const void* p, const void* dout, void* dp, int64_t T, int F, void* stream_) {
    STREAM;
    if (!p || !dout || !dp || F % 8) return set_error(CL_ERR_INVALID, "cl_geglu_bwd: bad args");
    launch_k(geglu_bwd_kernel, ew_blocks(T * (F / 8)), 256, 0, stream, BF(p), BF(dout), BFW(dp), T, F);
    DONE();
}
extern "C" int cl_add(const void* a, const void* b, void* out, int64_t n, void* stream_) {
    STREAM;
    if (!a || !b || !out || n % 8) return set_error(CL_ERR_INVALID, "cl_add: bad args (n %% 8)");
    launch_k(add_kernel, ew_blocks(n / 8), 256, 0, stream, BF(a), BF(b), BFW(out), n / 8);
    DONE();
}
extern "C" int cl_upsample2x_fwd(const void* x, void* y, int n, int H, int W, int C, void* stream_) {
    STREAM;
    if (!x || !y || C % 8) return set_error(CL_ERR_INVALID, "cl_upsample2x_fwd: bad args");
    launch_k(upsample2x_kernel, ew_blocks((long long)n * 4 * H * W * (C / 8)), 256, 0, stream, BF(x), BFW(y), n, H, W, C);
    DONE();
}
extern "C" int cl_upsample2x_bwd(const void* dy, void* dx, int n, int H, int W, int C, int accumulate, void* stream_) {
    STREAM;
    if (!dy || !dx || C % 8) return set_error(CL_ERR_INVALID, "cl_upsample2x_bwd: bad args");
    launch_k(upsample2x_bwd_kernel, ew_blocks((long long)n * H * W * (C / 8)), 256, 0, stream, BF(dy), BFW(dx), n, H, W, C, accumulate);
    DONE();
}
extern "C" int cl_zero_insert2x(const void* x, void* y, int n, int H, int W, int C, int off, void* stream_) {
    STREAM;
    if (!x || !y || C % 8 || (off != 0 && off != 1)) return set_error(CL_ERR_INVALID, "cl_zero_insert2x: bad args");
    launch_k(zero_insert2x_kernel, ew_blocks((long long)n * 4 * H * W * (C / 8)), 256, 0, stream, BF(x), BFW(y), n, H, W, C, off);
    DONE();
}
extern "C" int cl_concat_channels(const void* a, const void* b, void* out, int64_t M, int Ca, int Cb, void* stream_) {
    STREAM;
    if (!a || !b || !out || Ca % 8 || Cb % 8) return set_error(CL_ERR_INVALID, "cl_concat_channels: bad args");
    launch_k(concat_kernel, ew_blocks(M * ((Ca + Cb) / 8)), 256, 0, stream, BF(a), BF(b), BFW(out), M, Ca, Cb);
    DONE();
}
extern "C" int cl_slice_channels(const void* src, void* dst, int64_t M, int Cs, int c_off, int Cd, int accumulate,
                                 void* stream_) {
    STREAM;
    if (!src || !dst || Cs % 8 || Cd % 8 || c_off % 8 || c_off + Cd > Cs) return set_error(CL_ERR_INVALID, "cl_slice_channels: bad args");
    launch_k(slice_kernel, ew_blocks(M * (Cd / 8)), 256, 0, stream, BF(src), BFW(dst), M, Cs, c_off, Cd, accumulate);
    DONE();
}
extern "C" int cl_nchw_to_nhwc(const void* x, int x_is_fp32, void* y, int n, int C, int HW, void* stream_) {
    STREAM;
    if (!x || !y) return set_error(CL_ERR_INVALID, "cl_nchw_to_nhwc: null");
    dim3 grid((HW + 31) / 32, (C + 31) / 32, n), block(32, 8);
    if (x_is_fp32) launch_k(nchw_to_nhwc_kernel<float>, grid, block, 0, stream, reinterpret_cast<const float*>(x), BFW(y), n, C, HW);
    else launch_k(nchw_to_nhwc_kernel<__nv_bfloat16>, grid, block, 0, stream, BF(x), BFW(y), n, C, HW);
    DONE();
}
extern "C" int cl_nhwc_to_nchw_f32(const void* x, float* y, int n, int C, int HW, int accumulate, void* stream_) {
    STREAM;
    if (!x || !y) return set_error(CL_ERR_INVALID, "cl_nhwc_to_nchw_f32: null");
    dim3 grid((HW + 31) / 32, (C + 31) / 32, n), block(32, 8);
    launch_k(nhwc_to_nchw_f32_kernel, grid, block, 0, stream, BF(x), y, n, C, HW, accumulate);
    DONE();
}
extern "C" int cl_f32_to_bf16(const float* x, void* y, int64_t n, void* stream_) {
    STREAM;
    if (!x || !y) return set_error(CL_ERR_INVALID, "cl_f32_to_bf16: null");
    launch_k(f32_to_bf16_kernel, ew_blocks(n), 256, 0, stream, x, BFW(y), n);
    DONE();
}
extern "C" int cl_bf16_to_f32(const void* x, float* y, int64_t n, void* stream_) {
    STREAM;
    if (!x || !y) return set_error(CL_ERR_INVALID, "cl_bf16_to_f32: null");
    launch_k(bf16_to_f32_kernel, ew_blocks(n), 256, 0, stream, BF(x), y, n);
    DONE();
}

// ------------------------------------------------------------------------------------------ strided weight-space helpers
// (trainable dense operands of the concat_hidden control MLP, models.py:208-214: bf16 views / transposes of the fp32 masters
//  and strided accumulation of their fp32 weight gradients)
namespace clb {
// dst[i*ld + j] = bf16(alpha * src[i*s_i + j*s_j])
__global__ void cast_matrix_kernel(const float* __restrict__ src, long long s_i, long long s_j, __nv_bfloat16* __restrict__ dst,
                                   long long ld, int I, int J, float alpha) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)I * J;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(k / J), j = (int)(k % J);
        dst[i * ld + j] = __float2bfloat16(alpha * src[i * s_i + j * s_j]);
    }
}
// dst[i*ld + j] += alpha * src[i*J + j]   (fp32)
__global__ void axpy_matrix_kernel(const float* __restrict__ src, float* __restrict__ dst, long long ld, int I, int J, float alpha) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)I * J;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(k / J), j = (int)(k % J);
        dst[i * ld + j] += alpha * src[k];
    }
}
}  // namespace clb

extern "C" int cl_cast_matrix_bf16(const float* src, int64_t s_i, int64_t s_j, void* dst, int64_t ld, int I, int J, float alpha,
                                   void* stream_) {
    STREAM;
    if (!src || !dst || I <= 0 || J <= 0) return set_error(CL_ERR_INVALID, "cl_cast_matrix_bf16: bad args");
    launch_k(clb::cast_matrix_kernel, ew_blocks((long long)I * J), 256, 0, stream, src, (long long)s_i, (long long)s_j, BFW(dst),
             (long long)ld, I, J, alpha);
    DONE();
}

extern "C" int cl_axpy_matrix_f32(const float* src, float* dst, int64_t ld, int I, int J, float alpha, void* stream_) {
    STREAM;
    if (!src || !dst || I <= 0 || J <= 0) return set_error(CL_ERR_INVALID, "cl_axpy_matrix_f32: bad args");
    launch_k(clb::axpy_matrix_kernel, ew_blocks((long long)I * J), 256, 0, stream, src, dst, (long long)ld, I, J, alpha);
    DONE();
}

// ------------------------------------------------------------------------------------------ VAE helpers
// Row softmax of the one-head AttentionBlock of the VAE mid block (diffusers AttentionBlock: softmax(q k^T / sqrt(C)) in fp32):
// p[r, :] = softmax(scale * s[r, :]) written as bf16.  One CTA per row, the row cached in shared memory (cols <= 12288).
namespace clb {
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ s, __nv_bfloat16* __restrict__ p, int cols, float scale_log2) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float row[];
    __shared__ float red[8];
    const float* sr = s + (long long)blockIdx.x * cols;
    __nv_bfloat16* pr = p + (long long)blockIdx.x * cols;
    float mx = -INFINITY;
    for (int c = threadIdx.x * 4; c < cols; c += blockDim.x * 4) {
        const float4 v = *reinterpret_cast<const float4*>(sr + c);
        *reinterpret_cast<float4*>(row + c) = v;
        mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
    }
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
    __syncthreads();
    float sum = 0.f;
    for (int c = threadIdx.x * 4; c < cols; c += blockDim.x * 4) {
        float4 v = *reinterpret_cast<float4*>(row + c);
        v.x = fast_exp2((v.x - mx) * scale_log2); v.y = fast_exp2((v.y - mx) * scale_log2);
        v.z = fast_exp2((v.z - mx) * scale_log2); v.w = fast_exp2((v.w - mx) * scale_log2);
        *reinterpret_cast<float4*>(row + c) = v;
        sum += v.x + v.y + v.z + v.w;
    }
    sum = warp_sum(sum);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) sum += red[i];
    const float inv = 1.f / sum;
    for (int c = threadIdx.x * 4; c < cols; c += blockDim.x * 4) {
        const float4 v = *reinterpret_cast<float4*>(row + c);
        uint2 o;
        o.x = pack_bf16x2(v.x * inv, v.y * inv);
        o.y = pack_bf16x2(v.z * inv, v.w * inv);
        *reinterpret_cast<uint2*>(pr + c) = o;
    }
}

// y[n, c, :] = mul * x[n, c, :] + shift[c]   (NCHW fp32; the post_quant_conv bias as a shift of the latents)
__global__ void channel_affine_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, const float* __restrict__ shift,
                                           float mul, int C, long long hw, long long total) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)((i / hw) % C);
        y[i] = fmaf(mul, x[i], shift[c]);
    }
}

// ---------------------------------------------------------------------------------------------- CLIP text encoder helpers
__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
    uint4 u;
    u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
    u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(p) = u;
}
// (transformers CLIPTextModel behind train_text_to_image_control_lora.py:768 `text_encoder(batch["input_ids"])[0]`)
// x[b, t, :] = token_embedding[ids[b, t]] + position_embedding[t]     (bf16 tables, 16 bytes per thread)
__global__ void __launch_bounds__(256)
clip_embed_kernel(const long long* __restrict__ ids, const __nv_bfloat16* __restrict__ tok, const __nv_bfloat16* __restrict__ pos,
                  __nv_bfloat16* __restrict__ out, int T, int C, int vocab, long long total_chunks) {
    pdl_launch_dependents();
    pdl_wait();
    const int chunks = C / 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total_chunks; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / chunks;
        const int ch = (int)(i - row * chunks);
        long long id = ids[row];
        id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
        const int t = (int)(row % T);
        float a[8], b[8];
        load8(tok + id * C + ch * 8, a);
        load8(pos + (long long)t * C + ch * 8, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] += b[j];
        store8(out + row * C + ch * 8, a);
    }
}

// y = x * sigmoid(1.702 x) in place (CLIP's `quick_gelu`), 8 bf16 per thread
__global__ void __launch_bounds__(256)
quick_gelu_kernel(__nv_bfloat16* __restrict__ x, long long total_chunks) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total_chunks; i += (long long)gridDim.x * blockDim.x) {
        float a[8];
        load8(x + i * 8, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] = a[j] / (1.f + __expf(-1.702f * a[j]));
        store8(x + i * 8, a);
    }
}

// causal softmax(q k^T * scale) v for short sequences (T <= 128, d <= 64): one CTA per (batch, head), K and V of the head in
// shared memory as fp32, one thread per query row with an online softmax over keys 0..row (fp32 throughout).
// qkv [B*T, 3*C] bf16 (q | k | v, head h at columns h*d), out [B*T, C] bf16.
__global__ void __launch_bounds__(128)
causal_attention_small_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int C, int d, float scale) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float sm_kv[];            // [T][d] K | [T][d] V
    float* sk = sm_kv;
    float* sv = sm_kv + T * d;
    const int b = blockIdx.x, h = blockIdx.y;
    const long long ld = 3LL * C;
    const __nv_bfloat16* base = qkv + (long long)b * T * ld + h * d;
    for (int i = threadIdx.x; i < T * d; i += blockDim.x) {
        const int t = i / d, c = i - t * d;
        sk[i] = __bfloat162float(base[t * ld + C + c]);
        sv[i] = __bfloat162float(base[t * ld + 2 * C + c]);
    }
    __syncthreads();
    const int row = threadIdx.x;
    if (row >= T) return;
    float q[64], o[64];
#pragma unroll
    for (int c = 0; c < 64; ++c) { q[c] = (c < d) ? __bfloat162float(base[row * ld + c]) * scale : 0.f; o[c] = 0.f; }
    float m = -INFINITY, l = 0.f;
    for (int j = 0; j <= row; ++j) {
        float sdot = 0.f;
#pragma unroll
        for (int c = 0; c < 64; ++c)
            if (c < d) sdot = fmaf(q[c], sk[j * d + c], sdot);
        const float mn = fmaxf(m, sdot);
        const float corr = __expf(m - mn), pj = __expf(sdot - mn);
        l = l * corr + pj;
#pragma unroll
        for (int c = 0; c < 64; ++c)
            if (c < d) o[c] = fmaf(pj, sv[j * d + c], o[c] * corr);
        m = mn;
    }
    const float inv = 1.f / l;
    __nv_bfloat16* op = out + ((long long)b * T + row) * C + h * d;
#pragma unroll
    for (int c = 0; c < 64; ++c)
        if (c < d) op[c] = __float2bfloat16(o[c] * inv);
}
}  // namespace clb

extern "C" int cl_softmax_rows(const float* s, void* p, int rows, int cols, float scale, void* stream_) {
    STREAM;
    if (!s || !p || rows <= 0 || cols <= 0 || cols % 4 != 0 || cols > 12288)
        return set_error(CL_ERR_INVALID, "cl_softmax_rows: cols must be a multiple of 4, <= 12288");
    static bool done = false;
    if (!done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(clb::softmax_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 12288 * 4));
        done = true;
    }
    launch_k(clb::softmax_rows_kernel, rows, 256, (size_t)cols * 4, stream, s, BFW(p), cols, scale * 1.4426950408889634f);
    DONE();
}

extern "C" int cl_channel_affine_nchw(const float* x, float* y, const float* shift, float mul, int n, int C, int64_t hw, void* stream_) {
    STREAM;
    if (!x || !y || !shift || n <= 0 || C <= 0 || hw <= 0) return set_error(CL_ERR_INVALID, "cl_channel_affine_nchw: bad args");
    const long long total = (long long)n * C * hw;
    launch_k(clb::channel_affine_nchw_kernel, ew_blocks(total), 256, 0, stream, x, y, shift, mul, C, (long long)hw, total);
    DONE();
}

extern "C" int cl_clip_embed(const int64_t* ids, const void* tok, const void* pos, void* out, int rows, int T, int C, int vocab, void* stream_) {
    STREAM;
    if (!ids || !tok || !pos || !out || rows <= 0 || T <= 0 || C % 8 != 0 || vocab <= 0) return set_error(CL_ERR_INVALID, "cl_clip_embed: bad args");
    const long long total = (long long)rows * (C / 8);
    launch_k(clb::clip_embed_kernel, ew_blocks(total), 256, 0, stream, reinterpret_cast<const long long*>(ids), BF(tok), BF(pos), BFW(out), T, C,
             vocab, total);
    DONE();
}

extern "C" int cl_quick_gelu(void* x, int64_t n, void* stream_) {
    STREAM;
    if (!x || n <= 0 || n % 8 != 0) return set_error(CL_ERR_INVALID, "cl_quick_gelu: n must be a positive multiple of 8");
    launch_k(clb::quick_gelu_kernel, ew_blocks(n / 8), 256, 0, stream, BFW(x), (long long)(n / 8));
    DONE();
}

extern "C" int cl_causal_attention_small(const void* qkv, void* out, int B, int T, int heads, int d, float scale, void* stream_) {
    STREAM;
    if (!qkv || !out || B <= 0 || heads <= 0 || T <= 0 || T > 128 || d <= 0 || d > 64)
        return set_error(CL_ERR_INVALID, "cl_causal_attention_small: T <= 128, head dim <= 64");
    const size_t smem = (size_t)2 * T * d * sizeof(float);
    static bool done = false;
    if (!done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(clb::causal_attention_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 128 * 64 * 4));
        done = true;
    }
    launch_k(clb::causal_attention_small_kernel, dim3(B, heads), 128, smem, stream, BF(qkv), BFW(out), T, heads * d, d, scale);
    DONE();
}
