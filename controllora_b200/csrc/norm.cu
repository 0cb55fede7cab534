// K5 — GroupNorm(+SiLU) and LayerNorm, forward and input-gradient, on channels-last bf16 tensors.  HBM-bound:
// every pass reads/writes 16-byte vectors, fully coalesced along C; statistics in fp32 (fp64 for the cross-CTA
// GroupNorm combine).  Replaces ATen native_group_norm / layer_norm (+ F.silu) called by diffusers' ResnetBlock2D,
// Transformer2DModel, BasicTransformerBlock and by models.py:515-543 (ConvBlock2D).
#include <stdio.h>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
    uint4 u;
    u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
    u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(p) = u;
}

__device__ __forceinline__ uint4 ldg16(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ float fast_sigmoid(float z) { return __fdividef(1.f, 1.f + __expf(-z)); }
__device__ __forceinline__ float silu_grad_fast(float z) {
    const float s = fast_sigmoid(z);
    return s * (1.f + z * (1.f - s));
}

// ---------------------------------------------------------------------------------------------- GroupNorm
// Layout: x [n, HW, C]; group g = channels [g*cpg, (g+1)*cpg).  One launch per direction, no workspace.
// One thread-block CLUSTER per image (up to 16 CTAs, each owning a slab of rows of all channels): phase 1 reduces the slab
// (thread == fixed 8-channel chunk, partial sums in registers), the CTAs exchange their per-group partial sums through
// distributed shared memory (fp64), every CTA derives the per-channel affine coefficients, and phase 2 streams the slab
// again - from L2, where phase 1 just left it - to write y (forward) or dx (backward).
__device__ __forceinline__ double ld_dsmem_f64(uint32_t cluster_addr) {
    double v;
    asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(cluster_addr) : "memory");
    return v;
}

static constexpr int GNC_THREADS = 512;

// BWD = 0: y = act(GN(x)), stats out.   BWD = 1: dx (+)= dGN(x, dy), stats in, optional dgamma / dbeta accumulation.
template <int BWD>
__global__ void __launch_bounds__(GNC_THREADS, 2)
gn_cluster_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, const float* gamma,
                  const float* beta, float* stats, __nv_bfloat16* __restrict__ out, float* dgamma, float* dbeta, int HW, int C, int G,
                  float eps, double inv_m, int silu, int accumulate) {
    pdl_launch_dependents();
    pdl_wait();
    // grid (CL, n_img, CS): the cluster of CL CTAs shares the rows of image blockIdx.y; blockIdx.z selects one of CS
    // contiguous channel ranges (whole groups - GroupNorm statistics never cross a group), so that n_img * CL * CS CTAs
    // cover the machine about twice even at batch 8.  Inside the kernel C / G / pointers are made LOCAL to that range.
    const int n = blockIdx.y;
    const int CL = gridDim.x;                          // cluster == the gridDim.x CTAs of one (image, channel range)
    const int crank = (CL > 1) ? (int)cluster_ctarank() : 0;
    const int Cfull = C, Gfull = G;
    const int cpg = C / G;
    G = Gfull / (int)gridDim.z;                        // groups of this CTA
    C = G * cpg;                                       // channels of this CTA
    const int cbase = (int)blockIdx.z * C;             // first channel
    const int gbase = (int)blockIdx.z * G;             // first group
    gamma += cbase; beta += cbase;
    if (dgamma != nullptr) { dgamma += cbase; dbeta += cbase; }
    stats += ((long long)n * Gfull + gbase) * 2;       // stats[(g_local) * 2 + {0,1}] below
    const int chunks = C / 8;
    const int rows_par = blockDim.x / chunks;
    const int chunk = threadIdx.x % chunks;
    const int rsub = threadIdx.x / chunks;
    const bool active = rsub < rows_par;
    const int c0 = chunk * 8;
    const int rows_cta = (HW + CL - 1) / CL;
    const int row0 = crank * rows_cta;
    const int row1 = min(HW, row0 + rows_cta);
    const __nv_bfloat16* xp = x + (long long)n * HW * Cfull + cbase + c0;
    const __nv_bfloat16* dp = BWD ? dy + (long long)n * HW * Cfull + cbase + c0 : nullptr;

    extern __shared__ __align__(16) unsigned char gnc_raw[];
    double* gpart = reinterpret_cast<double*>(gnc_raw);                    // [G][2]  this CTA's partial group sums
    float* coef = reinterpret_cast<float*>(gpart + 2 * G);                 // [4][C]  per-channel coefficients
    float* part0 = coef + 4 * C;                                           // [rows_par][C]
    float* part1 = part0 + (size_t)rows_par * C;                           // [rows_par][C]

    // ---------------- phase 1
    float a0[8], a1[8], sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { a0[j] = a1[j] = 0.f; sc[j] = sh[j] = 0.f; }
    if (BWD && active) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int g = (c0 + j) / cpg;
            const float mu = stats[g * 2], rs = stats[g * 2 + 1];
            sc[j] = rs * gamma[c0 + j];
            sh[j] = fmaf(-mu, sc[j], beta[c0 + j]);
        }
    }
    if (active) {
        if (!BWD) {
            for (int r = row0 + rsub; r < row1; r += 4 * rows_par) {       // 4 rows (64 B) in flight per thread
                uint4 u[4];
                bool ok[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int rq = r + q * rows_par;
                    ok[q] = rq < row1;
                    u[q] = ldg16(xp + (long long)(ok[q] ? rq : r) * Cfull);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (!ok[q]) continue;
                    float xv[8];
                    unpack8(u[q], xv);
#pragma unroll
                    for (int j = 0; j < 8; ++j) { a0[j] += xv[j]; a1[j] = fmaf(xv[j], xv[j], a1[j]); }
                }
            }
        } else {
            for (int r = row0 + rsub; r < row1; r += 2 * rows_par) {
                const int r1 = r + rows_par;
                const bool ok1 = r1 < row1;
                const long long o0 = (long long)r * Cfull, o1 = (long long)(ok1 ? r1 : r) * Cfull;
                const uint4 ux0 = ldg16(xp + o0), ud0 = ldg16(dp + o0), ux1 = ldg16(xp + o1), ud1 = ldg16(dp + o1);
                float xv[8], dv[8];
                unpack8(ux0, xv);
                unpack8(ud0, dv);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float dz = dv[j];
                    if (silu) dz *= silu_grad_fast(fmaf(xv[j], sc[j], sh[j]));
                    a0[j] = fmaf(dz, xv[j], a0[j]);
                    a1[j] += dz;
                }
                if (ok1) {
                    unpack8(ux1, xv);
                    unpack8(ud1, dv);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        float dz = dv[j];
                        if (silu) dz *= silu_grad_fast(fmaf(xv[j], sc[j], sh[j]));
                        a0[j] = fmaf(dz, xv[j], a0[j]);
                        a1[j] += dz;
                    }
                }
            }
        }
        float* d0 = part0 + (size_t)rsub * C + c0;
        float* d1 = part1 + (size_t)rsub * C + c0;
        *reinterpret_cast<float4*>(d0) = make_float4(a0[0], a0[1], a0[2], a0[3]);
        *reinterpret_cast<float4*>(d0 + 4) = make_float4(a0[4], a0[5], a0[6], a0[7]);
        *reinterpret_cast<float4*>(d1) = make_float4(a1[0], a1[1], a1[2], a1[3]);
        *reinterpret_cast<float4*>(d1 + 4) = make_float4(a1[4], a1[5], a1[6], a1[7]);
    }
    __syncthreads();
    // per-channel totals of this CTA -> coef planes 0 / 1 (scratch until the coefficients are written)
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s0 = 0.f, s1 = 0.f;
        for (int g = 0; g < rows_par; ++g) { s0 += part0[(size_t)g * C + c]; s1 += part1[(size_t)g * C + c]; }
        if (BWD) {
            const int g = c / cpg;
            const float mu = stats[g * 2], rs = stats[g * 2 + 1];
            const float dzxh = rs * fmaf(-mu, s1, s0);              // this slab's share of sum dz*xhat of the channel
            if (dgamma != nullptr) { atomicAdd(&dgamma[c], dzxh); atomicAdd(&dbeta[c], s1); }
            const float gm = gamma[c];
            s0 = gm * s1;                                            // -> group sum of dz*gamma
            s1 = gm * dzxh;                                          // -> group sum of dz*gamma*xhat
        }
        coef[c] = s0;
        coef[C + c] = s1;
    }
    __syncthreads();
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        double s0 = 0.0, s1 = 0.0;
        for (int c = g * cpg; c < (g + 1) * cpg; ++c) { s0 += coef[c]; s1 += coef[C + c]; }
        gpart[2 * g] = s0;
        gpart[2 * g + 1] = s1;
    }
    // ---------------- exchange: every CTA sums the partials of all CTAs of its image (distributed shared memory)
    if (CL > 1) cluster_sync_all(); else __syncthreads();
    double* gtot = reinterpret_cast<double*>(part0);                 // [G][2] (part0 / part1 are free now; sized to hold it)
    for (int g = threadIdx.x; g < 2 * G; g += blockDim.x) {
        double s = 0.0;
        if (CL > 1) {
            const uint32_t local = smem_u32(gpart + g);
            for (int rk = 0; rk < CL; ++rk) s += ld_dsmem_f64(mapa_shared(local, (uint32_t)rk));
        } else {
            s = gpart[g];
        }
        gtot[g] = s;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const int g = c / cpg;
        if (!BWD) {
            const double mu = gtot[2 * g] * inv_m;
            double var = gtot[2 * g + 1] * inv_m - mu * mu;
            if (var < 0.0) var = 0.0;
            const float rs = (float)(1.0 / sqrt(var + (double)eps));
            const float fmu = (float)mu;
            if (crank == 0 && c == g * cpg) { stats[g * 2] = fmu; stats[g * 2 + 1] = rs; }
            const float s_ = rs * gamma[c];
            coef[2 * C + c] = s_;
            coef[3 * C + c] = fmaf(-fmu, s_, beta[c]);
        } else {
            const float mu = stats[g * 2], rs = stats[g * 2 + 1];
            const float im = (float)inv_m;
            const float K2 = rs * rs * (float)gtot[2 * g + 1] * im;
            coef[2 * C + c] = fmaf(-mu, K2, rs * (float)gtot[2 * g] * im);    // K1
            coef[3 * C + c] = K2;
        }
    }
    __syncthreads();
    // ---------------- phase 2 (the slab is L2-resident: phase 1 just streamed it)
    if (active) {
        __nv_bfloat16* op = out + (long long)n * HW * Cfull + cbase + c0;
        if (!BWD) {
            float s2[8], h2[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { s2[j] = coef[2 * C + c0 + j]; h2[j] = coef[3 * C + c0 + j]; }
            for (int r = row0 + rsub; r < row1; r += 4 * rows_par) {
                uint4 u[4];
                bool ok[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int rq = r + q * rows_par;
                    ok[q] = rq < row1;
                    u[q] = ldg16(xp + (long long)(ok[q] ? rq : r) * Cfull);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (!ok[q]) continue;
                    float xv[8], o[8];
                    unpack8(u[q], xv);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float z = fmaf(xv[j], s2[j], h2[j]);
                        o[j] = silu ? z * fast_sigmoid(z) : z;
                    }
                    store8(op + (long long)(r + q * rows_par) * Cfull, o);
                }
            }
        } else {
            float k1[8], k2[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { k1[j] = coef[2 * C + c0 + j]; k2[j] = coef[3 * C + c0 + j]; }
            for (int r = row0 + rsub; r < row1; r += 2 * rows_par) {
                const int r1 = r + rows_par;
                const bool ok1 = r1 < row1;
                const long long o0 = (long long)r * Cfull, o1 = (long long)(ok1 ? r1 : r) * Cfull;
                const uint4 ux0 = ldg16(xp + o0), ud0 = ldg16(dp + o0), ux1 = ldg16(xp + o1), ud1 = ldg16(dp + o1);
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    if (q == 1 && !ok1) continue;
                    float xv[8], dv[8], o[8];
                    unpack8(q ? ux1 : ux0, xv);
                    unpack8(q ? ud1 : ud0, dv);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        float dz = dv[j];
                        if (silu) dz *= silu_grad_fast(fmaf(xv[j], sc[j], sh[j]));
                        o[j] = fmaf(-xv[j], k2[j], fmaf(dz, sc[j], -k1[j]));       // dz*A - K1 - x*K2   (A == sc)
                    }
                    __nv_bfloat16* dst = op + (q ? o1 : o0);
                    if (accumulate) {
                        float pv[8];
                        load8(dst, pv);
#pragma unroll
                        for (int j = 0; j < 8; ++j) o[j] += pv[j];
                    }
                    store8(dst, o);
                }
            }
        }
    }
    if (CL > 1) cluster_sync_all();      // peers may still be reading this CTA's gpart
}

// ---------------------------------------------------------------------------------------------- LayerNorm
// One warp per row; the row (C <= 2560) lives in registers.
static constexpr int LN_MAX_IT = 10;  // 10 * 32 lanes * 8 = 2560 channels

// ROWS rows per warp are processed together: all their 16-byte loads are issued before the first reduction, which
// doubles the bytes in flight per SM for the narrow (C = 320 / 640) rows.
template <int LN_IT, int ROWS>
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
              __nv_bfloat16* __restrict__ y, float* __restrict__ stats, int T, int C, float eps) {
    pdl_launch_dependents();
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int row0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * ROWS;
    if (row0 >= T) return;
    const int chunks = C / 8;
    float v[ROWS][LN_IT][8];
    float s[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        const int row = min(row0 + r, T - 1);
        s[r] = 0.f;
#pragma unroll
        for (int it = 0; it < LN_IT; ++it) {
            const int ch = it * 32 + lane;
            if (ch < chunks) load8(x + (long long)row * C + ch * 8, v[r][it]);
        }
    }
    float mu[ROWS], rs[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
#pragma unroll
        for (int it = 0; it < LN_IT; ++it) {
            if (it * 32 + lane < chunks) {
#pragma unroll
                for (int j = 0; j < 8; ++j) s[r] += v[r][it][j];
            }
        }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) mu[r] = warp_sum(s[r]) / C;
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        float q = 0.f;
#pragma unroll
        for (int it = 0; it < LN_IT; ++it) {
            if (it * 32 + lane < chunks) {
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float d = v[r][it][j] - mu[r]; q = fmaf(d, d, q); }
            }
        }
        s[r] = q;
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) rs[r] = rsqrtf(warp_sum(s[r]) / C + eps);
#pragma unroll
    for (int it = 0; it < LN_IT; ++it) {
        const int ch = it * 32 + lane;
        if (ch < chunks) {
            float g[8], bt[8];
            const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + ch * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + ch * 8 + 4));
            const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + ch * 8)), b1 = __ldg(reinterpret_cast<const float4*>(beta + ch * 8 + 4));
            g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
            bt[0] = b0.x; bt[1] = b0.y; bt[2] = b0.z; bt[3] = b0.w; bt[4] = b1.x; bt[5] = b1.y; bt[6] = b1.z; bt[7] = b1.w;
#pragma unroll
            for (int r = 0; r < ROWS; ++r) {
                if (row0 + r < T) {
                    float o[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) o[j] = fmaf((v[r][it][j] - mu[r]) * rs[r], g[j], bt[j]);
                    store8(y + (long long)(row0 + r) * C + ch * 8, o);
                }
            }
        }
    }
    if (lane == 0 && stats != nullptr) {
#pragma unroll
        for (int r = 0; r < ROWS; ++r)
            if (row0 + r < T) { stats[(row0 + r) * 2] = mu[r]; stats[(row0 + r) * 2 + 1] = rs[r]; }
    }
}

template <int LN_IT, int ROWS>
__global__ void __launch_bounds__(256)
ln_bwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
              const float* __restrict__ gamma, const float* __restrict__ stats, __nv_bfloat16* __restrict__ dx, int T,
              int C, int accumulate) {
    pdl_launch_dependents();
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int row0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * ROWS;
    if (row0 >= T) return;
    const int chunks = C / 8;
    float xh[ROWS][LN_IT][8], dg[ROWS][LN_IT][8];
    float mu[ROWS], rs[ROWS], s1[ROWS], s2[ROWS];
    // raw loads of every row first (bf16 data parked in the fp32 arrays' storage after unpacking)
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        const int row = min(row0 + r, T - 1);
        mu[r] = stats[row * 2];
        rs[r] = stats[row * 2 + 1];
#pragma unroll
        for (int it = 0; it < LN_IT; ++it) {
            const int ch = it * 32 + lane;
            if (ch < chunks) {
                load8(x + (long long)row * C + ch * 8, xh[r][it]);
                load8(dy + (long long)row * C + ch * 8, dg[r][it]);
            }
        }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        s1[r] = 0.f; s2[r] = 0.f;
#pragma unroll
        for (int it = 0; it < LN_IT; ++it) {
            const int ch = it * 32 + lane;
            if (ch < chunks) {
                const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + ch * 8)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + ch * 8 + 4));
                const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    xh[r][it][j] = (xh[r][it][j] - mu[r]) * rs[r];
                    dg[r][it][j] *= g[j];
                    s1[r] += dg[r][it][j];
                    s2[r] = fmaf(dg[r][it][j], xh[r][it][j], s2[r]);
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) { s1[r] = warp_sum(s1[r]) / C; s2[r] = warp_sum(s2[r]) / C; }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        if (row0 + r < T) {
#pragma unroll
            for (int it = 0; it < LN_IT; ++it) {
                const int ch = it * 32 + lane;
                if (ch < chunks) {
                    float o[8];
                    if (accumulate) load8(dx + (long long)(row0 + r) * C + ch * 8, o);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float d = rs[r] * (dg[r][it][j] - s1[r] - xh[r][it][j] * s2[r]);
                        o[j] = accumulate ? o[j] + d : d;
                    }
                    store8(dx + (long long)(row0 + r) * C + ch * 8, o);
                }
            }
        }
    }
}

}  // namespace clb

using namespace clb;

// One-launch GroupNorm: pick the channel ranges and the cluster size (CTAs per image), launch gn_cluster_kernel<BWD>.
template <int BWD>
static int gn_cluster_launch(const __nv_bfloat16* x, const __nv_bfloat16* dy, const float* gamma, const float* beta, float* stats,
                             __nv_bfloat16* out, float* dgamma, float* dbeta, int n, int HW, int C, int G, float eps, int silu,
                             int accumulate, cudaStream_t stream) {
    static const char* c_msg = "groupnorm: C must be a multiple of 8 and <= 4096";
    if (C % 8 != 0 || C < 8) return set_error(CL_ERR_UNSUPPORTED, c_msg);
    const int cpg = C / G;
    // channel ranges per image (whole groups, >= 128 channels = 256 contiguous bytes per row and a multiple of 8 channels)
    int cs = 1;
    while (G % (2 * cs) == 0 && (C / (2 * cs)) >= 128 && ((G / (2 * cs)) * cpg) % 8 == 0 && n * 16 * cs < 2 * num_sms()) cs *= 2;
    const int Cl = C / cs, Gl = G / cs;
    if (Cl / 8 > GNC_THREADS) return set_error(CL_ERR_UNSUPPORTED, c_msg);
    const int chunks = Cl / 8;
    const int rows_par = GNC_THREADS / chunks;
    // [G][2] fp64 partial group sums, [4][C] fp32 coefficients, [2][rows_par][C] fp32 partial channel sums; the [G][2] fp64
    // group totals reuse the last area after the exchange, so it is at least that large
    const size_t part_bytes = sizeof(float) * 2 * rows_par * Cl, gsum_bytes = sizeof(double) * 2 * Gl;
    const size_t smem = gsum_bytes + sizeof(float) * 4 * Cl + (part_bytes > gsum_bytes ? part_bytes : gsum_bytes);
    static int max_cluster = 0, smem_max = 0;
    static size_t smem_optin = 0;
    if (max_cluster == 0) {
        int dev = 0;
        CL_CUDA_CHECK(cudaGetDevice(&dev));
        CL_CUDA_CHECK(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        // clusters of 16 CTAs are "non-portable": opt in, and keep 8 when the device refuses
        max_cluster = cudaFuncSetAttribute(gn_cluster_kernel<BWD>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess ? 16 : 8;
        (void)cudaGetLastError();
    }
    if (smem > (size_t)smem_max)
        return set_error(CL_ERR_UNSUPPORTED, "groupnorm: C = %d, G = %d needs %zu B of shared memory per CTA, the device allows %d", C, G,
                         smem, smem_max);
    if (smem > smem_optin) {           // 100 KiB (two CTAs per SM) covers every UNet / VAE / hint-encoder shape
        const size_t optin = smem > 100 * 1024 ? smem : 100 * 1024;
        CL_CUDA_CHECK(cudaFuncSetAttribute(gn_cluster_kernel<BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)optin));
        smem_optin = optin;
    }
    // CTAs per image: enough CTAs to fill the machine once, at least ~8 rows per row-slot, a power of two <= max_cluster.
    // Above 100 KiB only one CTA fits per SM, and a cluster of 16 would need 16 free SMs in one GPC: 8 at most then.
    int cl = (smem > 100 * 1024 && max_cluster > 8) ? 8 : max_cluster;
    while (cl > 1 && (n * cl * cs > 3 * num_sms() || HW / cl < rows_par)) cl >>= 1;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(cl, n, cs);
    cfg.blockDim = dim3(GNC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cl; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = cl > 1 ? 1 : 0;
    const double inv_m = 1.0 / ((double)HW * (C / G));
    CL_CUDA_CHECK(cudaLaunchKernelEx(&cfg, gn_cluster_kernel<BWD>, x, dy, gamma, beta, stats, out, dgamma, dbeta, HW, C, G, eps, inv_m,
                                     silu, accumulate));
    count_launch();
    return CL_OK;
}

extern "C" int cl_groupnorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stats, int n, int HW, int C,
                                int G, float eps, int silu, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !gamma || !beta || !y) return set_error(CL_ERR_INVALID, "cl_groupnorm_fwd: null pointer");
    if (stats == nullptr) return set_error(CL_ERR_INVALID, "cl_groupnorm_fwd: stats buffer is required");
    if (G <= 0 || C % G != 0) return set_error(CL_ERR_INVALID, "cl_groupnorm_fwd: C %% G != 0");
    return gn_cluster_launch<0>(reinterpret_cast<const __nv_bfloat16*>(x), nullptr, gamma, beta, stats, reinterpret_cast<__nv_bfloat16*>(y),
                                nullptr, nullptr, n, HW, C, G, eps, silu, 0, stream);
}

extern "C" int cl_groupnorm_bwd(const void* x, const void* dy, const float* gamma, const float* beta, const float* stats, void* dx,
                                float* dgamma, float* dbeta, int n, int HW, int C, int G, int silu, int accumulate, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !dy || !gamma || !beta || !stats || !dx) return set_error(CL_ERR_INVALID, "cl_groupnorm_bwd: null pointer");
    if (G <= 0 || C % G != 0) return set_error(CL_ERR_INVALID, "cl_groupnorm_bwd: C %% G != 0");
    if (G > 4096) return set_error(CL_ERR_UNSUPPORTED, "cl_groupnorm_bwd: G <= 4096");
    return gn_cluster_launch<1>(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(dy), gamma, beta,
                                const_cast<float*>(stats), reinterpret_cast<__nv_bfloat16*>(dx), dgamma, dbeta, n, HW, C, G, 0.f, silu,
                                accumulate, stream);
}
extern "C" int cl_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stats, int T,
                                int C, float eps, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !gamma || !beta || !y) return set_error(CL_ERR_INVALID, "cl_layernorm_fwd: null pointer");
    if (C % 8 != 0 || C > LN_MAX_IT * 256) return set_error(CL_ERR_UNSUPPORTED, "cl_layernorm_fwd: C must be a multiple of 8, <= 2560");
#define LN_FWD(IT, R) launch_k(ln_fwd_kernel<IT, R>, (T + 8 * R - 1) / (8 * R), 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x), gamma, beta, reinterpret_cast<__nv_bfloat16*>(y), stats, T, C, eps)
    if (C <= 512) LN_FWD(2, 2); else if (C <= 768) LN_FWD(3, 2); else if (C <= 1280) LN_FWD(5, 1); else LN_FWD(10, 1);
#undef LN_FWD
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

extern "C" int cl_layernorm_bwd(const void* x, const void* dy, const float* gamma, const float* stats, void* dx, int T,
                                int C, int accumulate, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !dy || !gamma || !stats || !dx) return set_error(CL_ERR_INVALID, "cl_layernorm_bwd: null pointer");
    if (C % 8 != 0 || C > LN_MAX_IT * 256) return set_error(CL_ERR_UNSUPPORTED, "cl_layernorm_bwd: C must be a multiple of 8, <= 2560");
#define LN_BWD(IT, R) launch_k(ln_bwd_kernel<IT, R>, (T + 8 * R - 1) / (8 * R), 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<const __nv_bfloat16*>(dy), gamma, stats, reinterpret_cast<__nv_bfloat16*>(dx), T, C, accumulate)
    if (C <= 512) LN_BWD(2, 1); else if (C <= 768) LN_BWD(3, 1); else if (C <= 1280) LN_BWD(5, 1); else LN_BWD(10, 1);
#undef LN_BWD
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
