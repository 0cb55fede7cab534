// LoRA side-path kernels: operand packing for the fused GEMM epilogue and the skinny rank-r reductions of the
// backward pass (dA, dB) — everything that models.py:89-97,185 (LoRALinearLayer instances) adds to autograd, minus
// the parts already folded into the wgmma GEMM.  All HBM-bound: each activation matrix is read exactly once.
#include <stdio.h>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

// ------------------------------------------------------------------------------------------ batched packing
// One launch prepares every LoRA operand of a step from the fp32 master weights (descriptor table in device memory):
//   kind 0: ext[16, K] bf16   rows row_off+j <- hi(src(j, k)), rows 8+row_off+j <- lo(src(j, k)), j < r
//   kind 1: table[N, rp] fp32  table[n*rp + row_off + j] <- src(j, n), j < r
// with src(j, k) = mul * src[j*s_j + k*s_k].  Rows / columns not covered by any descriptor must be pre-zeroed once.
__global__ void __launch_bounds__(256)
lora_pack_kernel(const cl_pack_desc* __restrict__ descs, int n_desc) {
    pdl_launch_dependents();
    pdl_wait();
    const int di = blockIdx.y;
    if (di >= n_desc) return;
    const cl_pack_desc d = descs[di];
    const float* src = reinterpret_cast<const float*>(d.src);
    const long long total = (long long)d.r * d.K;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(i / d.K);
        const int k = (int)(i % d.K);
        const float v = d.mul * src[(long long)j * d.s_j + (long long)k * d.s_k];
        if (d.kind == 0) {
            __nv_bfloat16* ext = reinterpret_cast<__nv_bfloat16*>(d.dst);
            const __nv_bfloat16 hi = __float2bfloat16(v);
            const __nv_bfloat16 lo = __float2bfloat16(v - __bfloat162float(hi));
            ext[(long long)(d.row_off + j) * d.ld + k] = hi;
            ext[(long long)(8 + d.row_off + j) * d.ld + k] = lo;
        } else if (d.kind == 1) {
            float* tab = reinterpret_cast<float*>(d.dst);
            tab[(long long)k * d.ld + d.row_off + j] = v;
        } else {
            // kind 2: bf16 transposed table, value duplicated in the hi and lo column slots
            __nv_bfloat16* tb = reinterpret_cast<__nv_bfloat16*>(d.dst);
            const __nv_bfloat16 hi = __float2bfloat16(v);
            tb[(long long)k * d.ld + d.row_off + j] = hi;
            tb[(long long)k * d.ld + 8 + d.row_off + j] = hi;
        }
    }
}

// ------------------------------------------------------------------------------------------ out[j, c] += alpha * sum_m a[m, j] * b[m, c]
// a: fp32 [M, lda] (first r columns used), b: bf16 [M, ldb] (C columns), out fp32 with strides (so_j, so_c).
// Thread layout as in the GroupNorm reduction: a thread owns one 8-column chunk for all rows of its slab.
template <int R>
__global__ void __launch_bounds__(512)
skinny_atb_kernel(const float* __restrict__ a, int lda, const __nv_bfloat16* __restrict__ b, long long ldb,
                  float* __restrict__ out, long long so_j, long long so_c, float alpha, int M, int C, int rows_per_cta) {
    pdl_launch_dependents();
    pdl_wait();
    const int chunks = C / 8;
    const int rows_par = blockDim.x / chunks;
    const int chunk = threadIdx.x % chunks;
    const int rsub = threadIdx.x / chunks;
    const bool active = rsub < rows_par;
    const int row0 = blockIdx.x * rows_per_cta;
    const int row1 = min(M, row0 + rows_per_cta);
    float acc[R][8];
#pragma unroll
    for (int j = 0; j < R; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
    if (active) {
        for (int m = row0 + rsub; m < row1; m += rows_par) {
            const uint4 u = *reinterpret_cast<const uint4*>(b + (long long)m * ldb + chunk * 8);
            const float2 b0 = unpack_bf16x2(u.x), b1 = unpack_bf16x2(u.y), b2 = unpack_bf16x2(u.z), b3 = unpack_bf16x2(u.w);
            const float bv[8] = {b0.x, b0.y, b1.x, b1.y, b2.x, b2.y, b3.x, b3.y};
            float av[R];
#pragma unroll
            for (int j = 0; j < R; ++j) av[j] = a[(long long)m * lda + j];
#pragma unroll
            for (int j = 0; j < R; ++j)
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[j][i] += av[j] * bv[i];
        }
    }
    // combine the row-parallel partials of this CTA through shared memory with plain stores (shared-memory atomics cost
    // ~2 cycles per lane and dominated this kernel), then one global RED per output element and CTA
    extern __shared__ float sh[];   // [rows_par][R][C]
    if (active) {
#pragma unroll
        for (int j = 0; j < R; ++j) {
            float* dst = sh + ((long long)rsub * R + j) * C + chunk * 8;
            *reinterpret_cast<float4*>(dst) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
            *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[j][4], acc[j][5], acc[j][6], acc[j][7]);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < R * C; i += blockDim.x) {
        float s = 0.f;
        for (int g = 0; g < rows_par; ++g) s += sh[(long long)g * R * C + i];
        const int j = i / C, c = i % C;
        atomicAdd(&out[j * so_j + c * so_c], alpha * s);
    }
}

// ------------------------------------------------------------------------------------------ batched skinny reductions
// Up to CL_SKINNY_MAX independent  out[j, c] += alpha * sum_m a[m, j] * b[m, c]  problems in ONE launch (blockIdx.y selects
// the problem): the dA / dB reductions of all LoRA adapters of an attention layer are tiny, launch-latency-bound kernels
// when issued one by one.
struct SkinnyBatch {
    cl_skinny_desc d[CL_SKINNY_MAX];
};

// RT: compile-time bound on the rank (4 or 8); U: rows in flight per thread.  All U row loads (16 B of b, the RT
// coefficients of a) are issued before the FMAs: with one load in flight per thread the kernel ran at ~25 % of HBM speed.
template <int RT, int U>
__global__ void __launch_bounds__(512, 1)
skinny_atb_batch_kernel(const __grid_constant__ SkinnyBatch batch, int slabs) {
    pdl_launch_dependents();
    pdl_wait();
    const cl_skinny_desc& d = batch.d[blockIdx.y];
    const int C = d.C, M = d.M, R = d.r;
    const int chunks = C / 8;
    const int rows_par = blockDim.x / chunks;
    const int chunk = threadIdx.x % chunks;
    const int rsub = threadIdx.x / chunks;
    const bool active = rsub < rows_par;
    const int rows_per_cta = (M + slabs - 1) / slabs;
    const int row0 = blockIdx.x * rows_per_cta;
    const int row1 = min(M, row0 + rows_per_cta);
    if (row0 >= M) return;
    const float* a = d.a;
    const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(d.b) + chunk * 8;
    const bool vec_a = ((reinterpret_cast<uintptr_t>(a) & 15) == 0) && (d.lda % 4 == 0) && (d.lda >= RT);
    float acc[RT][8];
#pragma unroll
    for (int j = 0; j < RT; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
    if (active) {
        for (int m = row0 + rsub; m < row1; m += U * rows_par) {
            uint4 u[U];
            float av[U][RT];
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const int mk = m + k * rows_par;
                const bool ok = mk < row1;
                const long long mc = ok ? mk : (row1 - 1);      // clamp: a padded row contributes with zero coefficients
                u[k] = __ldg(reinterpret_cast<const uint4*>(b + mc * d.ldb));
                if (vec_a) {
                    // only the 4-column groups that hold one of the r columns: at RT = 8, a rank-4 t[:, 4:] view of an
                    // [M, 8] table would otherwise read 16 bytes past the table's last row
#pragma unroll
                    for (int q = 0; q < RT / 4; ++q) {
                        const float4 t4 = 4 * q < R ? __ldg(reinterpret_cast<const float4*>(a + mc * d.lda + 4 * q))
                                                    : make_float4(0.f, 0.f, 0.f, 0.f);
                        av[k][4 * q] = ok ? t4.x : 0.f; av[k][4 * q + 1] = ok ? t4.y : 0.f;
                        av[k][4 * q + 2] = ok ? t4.z : 0.f; av[k][4 * q + 3] = ok ? t4.w : 0.f;
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < RT; ++j) av[k][j] = (ok && j < R) ? a[mc * d.lda + j] : 0.f;
                }
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const float2 b0 = unpack_bf16x2(u[k].x), b1 = unpack_bf16x2(u[k].y), b2 = unpack_bf16x2(u[k].z),
                             b3 = unpack_bf16x2(u[k].w);
                const float bv[8] = {b0.x, b0.y, b1.x, b1.y, b2.x, b2.y, b3.x, b3.y};
#pragma unroll
                for (int j = 0; j < RT; ++j)
#pragma unroll
                    for (int i = 0; i < 8; ++i) acc[j][i] = fmaf(av[k][j], bv[i], acc[j][i]);
            }
        }
    }
    extern __shared__ float sh[];   // [rows_par][R][C]
    if (active) {
#pragma unroll
        for (int j = 0; j < RT; ++j) {
            if (j < R) {
                float* dst = sh + ((long long)rsub * R + j) * C + chunk * 8;
                *reinterpret_cast<float4*>(dst) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
                *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[j][4], acc[j][5], acc[j][6], acc[j][7]);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < R * C; i += blockDim.x) {
        float s = 0.f;
        for (int g = 0; g < rows_par; ++g) s += sh[(long long)g * R * C + i];
        const int j = i / C, c = i % C;
        atomicAdd(&d.out[j * d.so_j + c * d.so_c], d.alpha * s);
    }
}

// ------------------------------------------------------------------------------------------ e[m, j] = sum_n a[m, n] * u[n*rp + j]
// a bf16 [M, lda], u fp32 [N, rp]; one warp per row.
template <int RP>
__global__ void __launch_bounds__(256)
rowdot_kernel(const __nv_bfloat16* __restrict__ a, long long lda, const float* __restrict__ u, float* __restrict__ e, int M, int N) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float s_ut[];                 // [RP][N]  (transposed: conflict-free 16-byte reads along n)
    for (int i = threadIdx.x; i < N * RP; i += blockDim.x) s_ut[(i % RP) * N + i / RP] = u[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    for (int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); m < M; m += warps_total) {
        float acc[RP];
#pragma unroll
        for (int j = 0; j < RP; ++j) acc[j] = 0.f;
        for (int n = lane * 8; n < N; n += 256) {
            const uint4 v = *reinterpret_cast<const uint4*>(a + (long long)m * lda + n);
            const float2 a0 = unpack_bf16x2(v.x), a1 = unpack_bf16x2(v.y), a2 = unpack_bf16x2(v.z), a3 = unpack_bf16x2(v.w);
#pragma unroll
            for (int j = 0; j < RP; ++j) {
                const float4 u0 = *reinterpret_cast<const float4*>(s_ut + j * N + n);
                const float4 u1 = *reinterpret_cast<const float4*>(s_ut + j * N + n + 4);
                acc[j] += a0.x * u0.x + a0.y * u0.y + a1.x * u0.z + a1.y * u0.w + a2.x * u1.x + a2.y * u1.y + a3.x * u1.z + a3.y * u1.w;
            }
        }
#pragma unroll
        for (int j = 0; j < RP; ++j) {
            const float sum = warp_sum(acc[j]);
            if (lane == 0) e[(long long)m * RP + j] = sum;
        }
    }
}

// ------------------------------------------------------------------------------------------ per-row tiny matmul
// out[m, i] (+)= alpha * sum_j a[m*lda + j] * w[i*sw_i + j*sw_j],  i < I, j < J   (I, J <= 8)
// out_mode 0: fp32 out[m*ldo + i] ; out_mode 1: bf16 hi/lo pair -> out_bf[m*ldo + col_off + i], [.. + lo_off + i]
__global__ void __launch_bounds__(256)
rowmat_kernel(const float* __restrict__ a, int lda, const float* __restrict__ w, int sw_i, int sw_j, int I, int J,
              float alpha, void* __restrict__ out, int ldo, int out_mode, int col_off, int lo_off, int accumulate, int M) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float sw[64];
    if (threadIdx.x < I * J) sw[threadIdx.x] = w[(threadIdx.x / J) * sw_i + (threadIdx.x % J) * sw_j];
    __syncthreads();
    for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < M; m += gridDim.x * blockDim.x) {
        float av[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) av[j] = (j < J) ? a[(long long)m * lda + j] : 0.f;
        for (int i = 0; i < I; ++i) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (j < J) s += av[j] * sw[i * J + j];
            s *= alpha;
            if (out_mode == 0) {
                float* o = reinterpret_cast<float*>(out) + (long long)m * ldo + i;
                *o = accumulate ? *o + s : s;
            } else {
                __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out) + (long long)m * ldo + col_off + i;
                const __nv_bfloat16 hi = __float2bfloat16(s);
                o[0] = hi;
                o[lo_off] = __float2bfloat16(s - __bfloat162float(hi));
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ hi/lo combine
// src fp32 [M, 16*nb] laid out in 16-column blocks [hi0..3 | hi4..7 | lo0..3 | lo4..7] -> dst fp32 [M, 8*nb] = hi + lo
__global__ void __launch_bounds__(256)
hilo_combine_kernel(const float* __restrict__ src, float* __restrict__ dst, long long M, int nb) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = M * nb * 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long m = i / (nb * 8);
        const int c = (int)(i % (nb * 8));
        const int blk = c / 8, j = c % 8;
        const float* sp = src + m * nb * 16 + blk * 16;
        dst[i] = sp[j] + sp[8 + j];
    }
}

// ------------------------------------------------------------------------------------------ rank-r update of a bf16 matrix
// out[m, c] = x[m, c] + alpha * sum_j t[m*ldt + j] * tab[c*rp + j]
template <int RP>
__global__ void __launch_bounds__(256)
rank_update_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ t, int ldt, const float* __restrict__ tab,
                   float alpha, __nv_bfloat16* __restrict__ out, long long M, int C) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float s_tt[];                 // [RP][C] transposed table
    for (int i = threadIdx.x; i < C * RP; i += blockDim.x) s_tt[(i % RP) * C + i / RP] = tab[i];
    __syncthreads();
    const int chunks = C / 8;
    const bool vec_t = ((reinterpret_cast<uintptr_t>(t) & 15) == 0) && (ldt % 4 == 0);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M * chunks; i += (long long)gridDim.x * blockDim.x) {
        const long long m = i / chunks;
        const int c0 = (int)(i % chunks) * 8;
        const uint4 u = *reinterpret_cast<const uint4*>(x + m * C + c0);
        const float2 x0 = unpack_bf16x2(u.x), x1 = unpack_bf16x2(u.y), x2 = unpack_bf16x2(u.z), x3 = unpack_bf16x2(u.w);
        float xv[8] = {x0.x, x0.y, x1.x, x1.y, x2.x, x2.y, x3.x, x3.y};
        float tr[RP];
        if (vec_t) {
#pragma unroll
            for (int q = 0; q < RP / 4; ++q) {
                const float4 t4 = __ldg(reinterpret_cast<const float4*>(t + m * ldt + 4 * q));
                tr[4 * q] = t4.x; tr[4 * q + 1] = t4.y; tr[4 * q + 2] = t4.z; tr[4 * q + 3] = t4.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < RP; ++j) tr[j] = t[m * ldt + j];
        }
#pragma unroll
        for (int j = 0; j < RP; ++j) {
            const float tv = alpha * tr[j];
            const float4 a = *reinterpret_cast<const float4*>(s_tt + j * C + c0);
            const float4 b = *reinterpret_cast<const float4*>(s_tt + j * C + c0 + 4);
            xv[0] += tv * a.x; xv[1] += tv * a.y; xv[2] += tv * a.z; xv[3] += tv * a.w;
            xv[4] += tv * b.x; xv[5] += tv * b.y; xv[6] += tv * b.z; xv[7] += tv * b.w;
        }
        uint4 o;
        o.x = pack_bf16x2(xv[0], xv[1]); o.y = pack_bf16x2(xv[2], xv[3]);
        o.z = pack_bf16x2(xv[4], xv[5]); o.w = pack_bf16x2(xv[6], xv[7]);
        *reinterpret_cast<uint4*>(out + m * C + c0) = o;
    }
}

// ------------------------------------------------------------------------------------------ V2 control injection (fused)
// forward:  t[m, :] = hi/lo-combine(th16[m, :16]) (+ uc[m, :rc]);   out[m, c] = x[m, c] + alpha * sum_{j<4} t[m, j] * tab[c*4 + j]
// (== cl_hilo_combine + cl_rowmat(identity) + cl_rank_update in one pass: x is read once, t [M, 8] is kept for the backward)
__global__ void __launch_bounds__(256)
v2_inject_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ th16, const float* __restrict__ uc, int ldu,
                     int rc, const float* __restrict__ tab, float alpha, __nv_bfloat16* __restrict__ out,
                     float* __restrict__ t_out, long long M, int C) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float s_tt[];                 // [4][C] transposed table
    for (int i = threadIdx.x; i < C * 4; i += blockDim.x) s_tt[(i % 4) * C + i / 4] = tab[i];
    __syncthreads();
    const int chunks = C / 8;
    const bool vec_u = uc != nullptr && rc == 4 && ((reinterpret_cast<uintptr_t>(uc) & 15) == 0) && (ldu % 4 == 0);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < M * chunks; i += (long long)gridDim.x * blockDim.x) {
        const long long m = i / chunks;
        const int chunk = (int)(i - m * chunks);
        const int c0 = chunk * 8;
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + m * C + c0));
        const float4 hi = __ldg(reinterpret_cast<const float4*>(th16 + m * 16));
        const float4 lo = __ldg(reinterpret_cast<const float4*>(th16 + m * 16 + 8));
        float tv[4] = {hi.x + lo.x, hi.y + lo.y, hi.z + lo.z, hi.w + lo.w};
        if (vec_u) {
            const float4 u4 = __ldg(reinterpret_cast<const float4*>(uc + m * ldu));
            tv[0] += u4.x; tv[1] += u4.y; tv[2] += u4.z; tv[3] += u4.w;
        } else if (uc != nullptr) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (j < rc) tv[j] += uc[m * ldu + j];
        }
        if (chunk == 0) {
            const float4 hi2 = __ldg(reinterpret_cast<const float4*>(th16 + m * 16 + 4));
            const float4 lo2 = __ldg(reinterpret_cast<const float4*>(th16 + m * 16 + 12));
            *reinterpret_cast<float4*>(t_out + m * 8) = make_float4(tv[0], tv[1], tv[2], tv[3]);
            *reinterpret_cast<float4*>(t_out + m * 8 + 4) = make_float4(hi2.x + lo2.x, hi2.y + lo2.y, hi2.z + lo2.z, hi2.w + lo2.w);
        }
        const float2 x0 = unpack_bf16x2(u.x), x1 = unpack_bf16x2(u.y), x2 = unpack_bf16x2(u.z), x3 = unpack_bf16x2(u.w);
        float xv[8] = {x0.x, x0.y, x1.x, x1.y, x2.x, x2.y, x3.x, x3.y};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float tj = alpha * tv[j];
            const float4 a = *reinterpret_cast<const float4*>(s_tt + j * C + c0);
            const float4 b = *reinterpret_cast<const float4*>(s_tt + j * C + c0 + 4);
            xv[0] = fmaf(tj, a.x, xv[0]); xv[1] = fmaf(tj, a.y, xv[1]); xv[2] = fmaf(tj, a.z, xv[2]); xv[3] = fmaf(tj, a.w, xv[3]);
            xv[4] = fmaf(tj, b.x, xv[4]); xv[5] = fmaf(tj, b.y, xv[5]); xv[6] = fmaf(tj, b.z, xv[6]); xv[7] = fmaf(tj, b.w, xv[7]);
        }
        uint4 o;
        o.x = pack_bf16x2(xv[0], xv[1]); o.y = pack_bf16x2(xv[2], xv[3]);
        o.z = pack_bf16x2(xv[4], xv[5]); o.w = pack_bf16x2(xv[6], xv[7]);
        *reinterpret_cast<uint4*>(out + m * C + c0) = o;
    }
}

// backward (one warp per row, the row stays in registers between the two phases):
//   dt[m, j] = sum_c dy[m, c] * up[c*4 + j]                       (== cl_rowdot)
//   dh[m, c] = dy[m, c] + alpha * sum_j dt[m, j] * down[c*4 + j]   (== cl_rank_update), dh optional
// The same kernel serves the forward as "project, add control, update":  t = x U (+ uc);  y = x + alpha t D^T  with
// U = Ac_h^T, D = Bc  - no separate skinny GEMM for x Ac_h^T is needed, x is read exactly once.
// R rows per warp are processed together: every coefficient fetched from the shared-memory tables is used for R rows (the
// one-row version read 16 KB of table per 1.3 KB row: shared-memory bound, 37 us for a 32768 x 320 pass), and the R x IT
// 16-byte row loads are all in flight before the first use.
template <int IT, int R>
__global__ void __launch_bounds__(256)
v2_inject_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const float* __restrict__ up, const float* __restrict__ down, float alpha,
                     float* __restrict__ dt_out, __nv_bfloat16* __restrict__ dh, int M, int C, const float* __restrict__ uc, int ldu,
                     int rc) {
    pdl_launch_dependents();
    pdl_wait();
    extern __shared__ float s_tab[];                // [4][C] up (transposed) | [4][C] down (transposed)
    float* s_up = s_tab;
    float* s_dn = s_tab + 4 * C;
    for (int i = threadIdx.x; i < C * 4; i += blockDim.x) {
        s_up[(i % 4) * C + i / 4] = up[i];
        s_dn[(i % 4) * C + i / 4] = (dh != nullptr) ? down[i] : 0.f;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int chunks = C / 8;
    const int warps_total = gridDim.x * (blockDim.x >> 5);
    for (int m0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * R; m0 < M; m0 += warps_total * R) {
        float v[R][IT][8];
        float acc[R][4];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int m = min(m0 + r, M - 1);               // clamped rows are computed and dropped
#pragma unroll
            for (int it = 0; it < IT; ++it) {
                const int ch = it * 32 + lane;
                if (ch < chunks) {
                    const uint4 u = __ldg(reinterpret_cast<const uint4*>(dy + (long long)m * C + ch * 8));
                    const float2 a0 = unpack_bf16x2(u.x), a1 = unpack_bf16x2(u.y), a2 = unpack_bf16x2(u.z), a3 = unpack_bf16x2(u.w);
                    v[r][it][0] = a0.x; v[r][it][1] = a0.y; v[r][it][2] = a1.x; v[r][it][3] = a1.y;
                    v[r][it][4] = a2.x; v[r][it][5] = a2.y; v[r][it][6] = a3.x; v[r][it][7] = a3.y;
                }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[r][j] = 0.f;
        }
#pragma unroll
        for (int it = 0; it < IT; ++it) {
            const int ch = it * 32 + lane;
            if (ch < chunks) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float4 u0 = *reinterpret_cast<const float4*>(s_up + j * C + ch * 8);
                    const float4 u1 = *reinterpret_cast<const float4*>(s_up + j * C + ch * 8 + 4);
#pragma unroll
                    for (int r = 0; r < R; ++r)
                        acc[r][j] += v[r][it][0] * u0.x + v[r][it][1] * u0.y + v[r][it][2] * u0.z + v[r][it][3] * u0.w +
                                     v[r][it][4] * u1.x + v[r][it][5] * u1.y + v[r][it][6] * u1.z + v[r][it][7] * u1.w;
                }
            }
        }
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[r][j] = warp_sum(acc[r][j]);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int m = m0 + r;
            if (m < M) {
                if (uc != nullptr) {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (j < rc) acc[r][j] += uc[(long long)m * ldu + j];
                }
                if (lane == 0) *reinterpret_cast<float4*>(dt_out + (long long)m * 4) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
            }
        }
        if (dh != nullptr) {
#pragma unroll
            for (int it = 0; it < IT; ++it) {
                const int ch = it * 32 + lane;
                if (ch < chunks) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float4 d0 = *reinterpret_cast<const float4*>(s_dn + j * C + ch * 8);
                        const float4 d1 = *reinterpret_cast<const float4*>(s_dn + j * C + ch * 8 + 4);
#pragma unroll
                        for (int r = 0; r < R; ++r) {
                            const float tj = alpha * acc[r][j];
                            v[r][it][0] = fmaf(tj, d0.x, v[r][it][0]); v[r][it][1] = fmaf(tj, d0.y, v[r][it][1]);
                            v[r][it][2] = fmaf(tj, d0.z, v[r][it][2]); v[r][it][3] = fmaf(tj, d0.w, v[r][it][3]);
                            v[r][it][4] = fmaf(tj, d1.x, v[r][it][4]); v[r][it][5] = fmaf(tj, d1.y, v[r][it][5]);
                            v[r][it][6] = fmaf(tj, d1.z, v[r][it][6]); v[r][it][7] = fmaf(tj, d1.w, v[r][it][7]);
                        }
                    }
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        if (m0 + r < M) {
                            uint4 o;
                            o.x = pack_bf16x2(v[r][it][0], v[r][it][1]); o.y = pack_bf16x2(v[r][it][2], v[r][it][3]);
                            o.z = pack_bf16x2(v[r][it][4], v[r][it][5]); o.w = pack_bf16x2(v[r][it][6], v[r][it][7]);
                            *reinterpret_cast<uint4*>(dh + (long long)(m0 + r) * C + ch * 8) = o;
                        }
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ out[i, j] += alpha * sum_m a[m, i] * b[m, j]
__global__ void __launch_bounds__(256)
skinny_small_kernel(const float* __restrict__ a, int lda, int I, const float* __restrict__ b, int ldb, int J,
                    float* __restrict__ out, float alpha, int M) {
    pdl_launch_dependents();
    pdl_wait();
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < M; m += gridDim.x * blockDim.x) {
        float av[8], bv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) av[i] = (i < I) ? a[(long long)m * lda + i] : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) bv[j] = (j < J) ? b[(long long)m * ldb + j] : 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] += av[i] * bv[j];
    }
    __shared__ float sh[64];
    if (threadIdx.x < 64) sh[threadIdx.x] = 0.f;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float s = warp_sum(acc[i][j]);
            if ((threadIdx.x & 31) == 0 && i < I && j < J) atomicAdd(&sh[i * 8 + j], s);
        }
    __syncthreads();
    if (threadIdx.x < 64) {
        const int i = threadIdx.x / 8, j = threadIdx.x % 8;
        if (i < I && j < J) atomicAdd(&out[i * J + j], alpha * sh[threadIdx.x]);
    }
}

// ------------------------------------------------------------------------------------------ weight-space tiny matmul (fp32)
// out[i*so_i + k*so_k] (+)= alpha * sum_j a[i*sa_i + j*sa_j] * b[j*sb_j + k*sb_k]
// one warp per output element (the reduction length J is up to the hidden size, the outputs are few)
__global__ void __launch_bounds__(256)
small_matmul_kernel(const float* __restrict__ a, long long sa_i, long long sa_j, const float* __restrict__ b, long long sb_j,
                    long long sb_k, float* __restrict__ out, long long so_i, long long so_k, int I, int J, int K, float alpha,
                    int accumulate) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)I * K;
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long t = warp0; t < total; t += nwarps) {
        const int i = (int)(t / K), k = (int)(t % K);
        float s = 0.f;
        for (int j = lane; j < J; j += 32) s += a[i * sa_i + j * sa_j] * b[j * sb_j + k * sb_k];
        s = warp_sum(s);
        if (lane == 0) {
            float* o = out + i * so_i + k * so_k;
            *o = accumulate ? *o + alpha * s : alpha * s;
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

extern "C" int cl_lora_pack_batch(const cl_pack_desc* descs_dev, int n_desc, int max_elems, void* stream_) {
    STREAM;
    if (!descs_dev || n_desc <= 0) return set_error(CL_ERR_INVALID, "cl_lora_pack_batch: bad args");
    int bx = (max_elems + 255) / 256;
    if (bx > 16) bx = 16;
    if (bx < 1) bx = 1;
    launch_k(lora_pack_kernel, dim3(bx, n_desc), 256, 0, stream, descs_dev, n_desc);
    DONE();
}

extern "C" int cl_skinny_atb(const float* a, int lda, int r, const void* b, int64_t ldb, float* out, int64_t so_j,
                             int64_t so_c, float alpha, int M, int Ccols, void* stream_) {
    STREAM;
    if (!a || !b || !out || Ccols % 8) return set_error(CL_ERR_INVALID, "cl_skinny_atb: bad args");
    const int chunks = Ccols / 8;
    if (chunks > 512) return set_error(CL_ERR_UNSUPPORTED, "cl_skinny_atb: C too large");
    int rows_par = 512 / chunks;
    if (rows_par < 1) rows_par = 1;
    int threads = ((rows_par * chunks + 31) / 32) * 32;
    if (threads > 512) { rows_par = 1; threads = ((chunks + 31) / 32) * 32; }
    int ctas = num_sms();
    int rows_per_cta = (M + ctas - 1) / ctas;
    if (rows_per_cta < rows_par * 16) rows_per_cta = rows_par * 16;
    const int grid = (M + rows_per_cta - 1) / rows_per_cta;
    const __nv_bfloat16* bb = reinterpret_cast<const __nv_bfloat16*>(b);
#define SK_CASE(R)                                                                                                      \
    case R: {                                                                                                           \
        const size_t smem = (size_t)rows_par * R * Ccols * sizeof(float);                                               \
        static bool done = false;                                                                                       \
        if (!done) {                                                                                                    \
            CL_CUDA_CHECK(cudaFuncSetAttribute(skinny_atb_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024)); \
            done = true;                                                                                                \
        }                                                                                                               \
        launch_k(skinny_atb_kernel<R>, grid, threads, smem, stream, a, lda, bb, ldb, out, so_j, so_c, alpha, M, Ccols, rows_per_cta); \
        break;                                                                                                          \
    }
    switch (r) {
        SK_CASE(1) SK_CASE(2) SK_CASE(3) SK_CASE(4) SK_CASE(8)
        default: return set_error(CL_ERR_UNSUPPORTED, "cl_skinny_atb: r must be 1..4 or 8");
    }
#undef SK_CASE
    DONE();
}

extern "C" int cl_skinny_atb_batch(const cl_skinny_desc* descs, int n, void* stream_) {
    STREAM;
    if (!descs || n < 1 || n > CL_SKINNY_MAX) return set_error(CL_ERR_INVALID, "cl_skinny_atb_batch: 1..%d descriptors", CL_SKINNY_MAX);
    SkinnyBatch batch;
    size_t smem = 0;
    int max_m = 0;
    for (int i = 0; i < n; ++i) {
        const cl_skinny_desc& d = descs[i];
        if (!d.a || !d.b || !d.out || d.C % 8 || d.C / 8 > 512 || d.r < 1 || d.r > 8 || d.M < 1)
            return set_error(CL_ERR_INVALID, "cl_skinny_atb_batch: bad descriptor %d", i);
        batch.d[i] = d;
        const int rows_par = 512 / (d.C / 8);
        const size_t need = (size_t)(rows_par < 1 ? 1 : rows_par) * d.r * d.C * sizeof(float);
        if (need > smem) smem = need;
        if (d.M > max_m) max_m = d.M;
    }
    if (smem > 200 * 1024) return set_error(CL_ERR_UNSUPPORTED, "cl_skinny_atb_batch: shared memory");
    static bool done = false;
    if (!done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(skinny_atb_batch_kernel<4, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        CL_CUDA_CHECK(cudaFuncSetAttribute(skinny_atb_batch_kernel<8, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        done = true;
    }
    int max_r = 0;
    for (int i = 0; i < n; ++i) max_r = descs[i].r > max_r ? descs[i].r : max_r;
    // ~one wave of CTAs in total (two resident per SM for rank <= 4); every problem gets the same number of row slabs
    // one 512-thread CTA per SM, 8 (rank <= 4) or 4 rows in flight per thread; slabs * n must NOT exceed the SM count: the
    // round-1 grid (ceil: 304 CTAs on 296 slots) ran a second, almost empty wave and took twice the time (ncu: SMs active 56 %)
    int slabs = num_sms() / n;
    if (slabs > (max_m + 63) / 64) slabs = (max_m + 63) / 64;
    if (slabs < 1) slabs = 1;
    if (max_r <= 4) launch_k(skinny_atb_batch_kernel<4, 8>, dim3(slabs, n), 512, smem, stream, batch, slabs);
    else launch_k(skinny_atb_batch_kernel<8, 4>, dim3(slabs, n), 512, smem, stream, batch, slabs);
    DONE();
}

extern "C" int cl_rowdot(const void* a, int64_t lda, const float* u, int rp, float* e, int M, int N, void* stream_) {
    STREAM;
    if (!a || !u || !e || N % 8) return set_error(CL_ERR_INVALID, "cl_rowdot: bad args");
    const __nv_bfloat16* aa = reinterpret_cast<const __nv_bfloat16*>(a);
    int blocks = (M + 7) / 8;
    if (blocks > num_sms() * 4) blocks = num_sms() * 4;
    const size_t smem = (size_t)N * rp * sizeof(float);
    if (smem > 48 * 1024) return set_error(CL_ERR_UNSUPPORTED, "cl_rowdot: N * rp too large");
    if (rp == 4) launch_k(rowdot_kernel<4>, blocks, 256, smem, stream, aa, lda, u, e, M, N);
    else if (rp == 8) launch_k(rowdot_kernel<8>, blocks, 256, smem, stream, aa, lda, u, e, M, N);
    else return set_error(CL_ERR_UNSUPPORTED, "cl_rowdot: rp must be 4 or 8");
    DONE();
}

extern "C" int cl_rowmat(const float* a, int lda, const float* w, int sw_i, int sw_j, int I, int J, float alpha, void* out,
                         int ldo, int out_mode, int col_off, int lo_off, int accumulate, int M, void* stream_) {
    STREAM;
    if (!a || !w || !out || I > 8 || J > 8 || I < 1 || J < 1) return set_error(CL_ERR_INVALID, "cl_rowmat: bad args");
    int blocks = (M + 255) / 256;
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(rowmat_kernel, blocks, 256, 0, stream, a, lda, w, sw_i, sw_j, I, J, alpha, out, ldo, out_mode, col_off, lo_off, accumulate, M);
    DONE();
}

extern "C" int cl_hilo_combine(const float* src, float* dst, int64_t M, int nb, void* stream_) {
    STREAM;
    if (!src || !dst || nb < 1) return set_error(CL_ERR_INVALID, "cl_hilo_combine: bad args");
    long long total = M * nb * 8;
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(hilo_combine_kernel, blocks, 256, 0, stream, src, dst, M, nb);
    DONE();
}

extern "C" int cl_rank_update(const void* x, const float* t, int ldt, const float* tab, int rp, float alpha, void* out,
                              int64_t M, int Ccols, void* stream_) {
    STREAM;
    if (!x || !t || !tab || !out || Ccols % 8) return set_error(CL_ERR_INVALID, "cl_rank_update: bad args");
    long long total = M * (Ccols / 8);
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    const __nv_bfloat16* xx = reinterpret_cast<const __nv_bfloat16*>(x);
    __nv_bfloat16* oo = reinterpret_cast<__nv_bfloat16*>(out);
    const size_t smem = (size_t)Ccols * rp * sizeof(float);
    if (smem > 48 * 1024) return set_error(CL_ERR_UNSUPPORTED, "cl_rank_update: C * rp too large");
    if (rp == 4) launch_k(rank_update_kernel<4>, blocks, 256, smem, stream, xx, t, ldt, tab, alpha, oo, M, Ccols);
    else if (rp == 8) launch_k(rank_update_kernel<8>, blocks, 256, smem, stream, xx, t, ldt, tab, alpha, oo, M, Ccols);
    else return set_error(CL_ERR_UNSUPPORTED, "cl_rank_update: rp must be 4 or 8");
    DONE();
}

extern "C" int cl_v2_inject_fwd(const void* x, const float* th16, const float* uc, int ldu, int rc, const float* tab, float alpha,
                                void* out, float* t_out, int64_t M, int Ccols, void* stream_) {
    STREAM;
    if (!x || !th16 || !tab || !out || !t_out || Ccols % 8 || rc < 1 || rc > 4) return set_error(CL_ERR_INVALID, "cl_v2_inject_fwd: bad args");
    const size_t smem = (size_t)Ccols * 4 * sizeof(float);
    if (smem > 48 * 1024) return set_error(CL_ERR_UNSUPPORTED, "cl_v2_inject_fwd: C too large");
    long long total = M * (Ccols / 8);
    int blocks = (int)((total + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(v2_inject_fwd_kernel, blocks, 256, smem, stream, reinterpret_cast<const __nv_bfloat16*>(x), th16, uc, ldu, rc, tab, alpha,
                                                        reinterpret_cast<__nv_bfloat16*>(out), t_out, M, Ccols);
    DONE();
}

extern "C" int cl_v2_inject_bwd(const void* dy, const float* up, const float* down, float alpha, float* dt_out, void* dh, int M,
                                int Ccols, void* stream_) {
    STREAM;
    if (!dy || !up || !dt_out || (dh && !down) || Ccols % 8) return set_error(CL_ERR_INVALID, "cl_v2_inject_bwd: bad args");
    if (Ccols > 1280) return set_error(CL_ERR_UNSUPPORTED, "cl_v2_inject_bwd: C <= 1280");
    const size_t smem = (size_t)Ccols * 8 * sizeof(float);
    int blocks = (M + 15) / 16;
    // two 256-thread CTAs are resident per SM (registers): a grid beyond that only repeats the per-CTA table load
    if (blocks > num_sms() * 2) blocks = num_sms() * 2;
    const __nv_bfloat16* dd = reinterpret_cast<const __nv_bfloat16*>(dy);
    __nv_bfloat16* hh = reinterpret_cast<__nv_bfloat16*>(dh);
    if (Ccols <= 512) launch_k(v2_inject_bwd_kernel<2, 4>, blocks, 256, smem, stream, dd, up, down, alpha, dt_out, hh, M, Ccols, nullptr, 0, 0);
    else if (Ccols <= 768) launch_k(v2_inject_bwd_kernel<3, 2>, blocks, 256, smem, stream, dd, up, down, alpha, dt_out, hh, M, Ccols, nullptr, 0, 0);
    else launch_k(v2_inject_bwd_kernel<5, 2>, blocks, 256, smem, stream, dd, up, down, alpha, dt_out, hh, M, Ccols, nullptr, 0, 0);
    DONE();
}

extern "C" int cl_rank4_project_update(const void* x, const float* proj, const float* upd, const float* uc, int ldu, int rc, float alpha,
                                       float* t_out, void* y, int M, int Ccols, void* stream_) {
    STREAM;
    if (!x || !proj || !upd || !t_out || !y || Ccols % 8 || rc < 0 || rc > 4) return set_error(CL_ERR_INVALID, "cl_rank4_project_update: bad args");
    if (Ccols > 1280) return set_error(CL_ERR_UNSUPPORTED, "cl_rank4_project_update: C <= 1280");
    const size_t smem = (size_t)Ccols * 8 * sizeof(float);
    int blocks = (M + 15) / 16;
    // two 256-thread CTAs are resident per SM (registers): a grid beyond that only repeats the per-CTA table load
    if (blocks > num_sms() * 2) blocks = num_sms() * 2;
    const __nv_bfloat16* xx = reinterpret_cast<const __nv_bfloat16*>(x);
    __nv_bfloat16* yy = reinterpret_cast<__nv_bfloat16*>(y);
    if (Ccols <= 512) launch_k(v2_inject_bwd_kernel<2, 4>, blocks, 256, smem, stream, xx, proj, upd, alpha, t_out, yy, M, Ccols, uc, ldu, rc);
    else if (Ccols <= 768) launch_k(v2_inject_bwd_kernel<3, 2>, blocks, 256, smem, stream, xx, proj, upd, alpha, t_out, yy, M, Ccols, uc, ldu, rc);
    else launch_k(v2_inject_bwd_kernel<5, 2>, blocks, 256, smem, stream, xx, proj, upd, alpha, t_out, yy, M, Ccols, uc, ldu, rc);
    DONE();
}

extern "C" int cl_skinny_small(const float* a, int lda, int I, const float* b, int ldb, int J, float* out, float alpha, int M,
                               void* stream_) {
    STREAM;
    if (!a || !b || !out || I > 8 || J > 8) return set_error(CL_ERR_INVALID, "cl_skinny_small: bad args");
    int blocks = (M + 255) / 256;
    if (blocks > num_sms()) blocks = num_sms();
    launch_k(skinny_small_kernel, blocks, 256, 0, stream, a, lda, I, b, ldb, J, out, alpha, M);
    DONE();
}

extern "C" int cl_small_matmul(const float* a, int64_t sa_i, int64_t sa_j, const float* b, int64_t sb_j, int64_t sb_k, float* out,
                               int64_t so_i, int64_t so_k, int I, int J, int K, float alpha, int accumulate, void* stream_) {
    STREAM;
    if (!a || !b || !out) return set_error(CL_ERR_INVALID, "cl_small_matmul: null");
    const long long total = (long long)I * K;          // one warp per output
    int blocks = (int)((total + 7) / 8);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(small_matmul_kernel, blocks, 256, 0, stream, a, sa_i, sa_j, b, sb_j, sb_k, out, so_i, so_k, I, J, K, alpha, accumulate);
    DONE();
}
