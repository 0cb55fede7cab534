// K1/K4 — warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = epilogue( A[M,K] * B[N,K]^T ),  bf16 operands, fp32 accumulation in registers.
//
// One CTA per 128 x BN output tile (x one K range under split-K), 288 threads:
//   warpgroups 0-1 consumers: rows 0-63 / 64-127 of the tile, wgmma.m64n(BN+EXT)k16 straight from the swizzled stages,
//                  then the epilogue from the accumulator registers (bias, per-image row bias, residual, LoRA, store).
//   warp 8         TMA producer (one elected thread): A tile 128 x BK, B tile BN x BK [+16 LoRA-down rows],
//                  128B (BK = 64) or 64B (BK = 32) swizzle, mbarrier ring of up to 8 stages
// Occupancy OCC = 1 or 2 CTAs per SM is a template parameter: it sets the register cap (224 or 96 per thread; no
// setmaxnreg, so the producer warp holds as many as a consumer) and the shared memory a launch may use.  With two CTAs on
// an SM, one CTA's prologue, pipeline fill and register epilogue run while the other's MMAs do, which is what short-K
// tiles (a few k-blocks each) need; deep-K tiles keep one CTA per SM and the deeper ring.
// LoRA (EXT = 16): the 16 extra B rows (bf16 hi / lo halves of the rank-r down matrix) make the main loop produce
// t = x A^T in 16 extra accumulator columns; the epilogue forms t (+ t_add, -> t_out) and adds scale * t B_up^T in fp32.
// The A operand is either a plain row-major matrix or an NHWC image read as 3x3 windows (implicit GEMM: the
// "im2col" is done by TMA box loads with shifted coordinates, out-of-bounds zero fill == conv zero padding).
//
// Replaces the cuBLAS/cuDNN calls behind models.py:124-147,231-282,373-423 (attention projections + LoRA side
// path) and diffusers' FeedForward / ResnetBlock2D / Transformer2DModel projections.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "wgmma.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

static constexpr int BLOCK_M = 128;
static constexpr int NUM_THREADS = 288;
static constexpr int PRODUCER_WARP = 8;
// Dynamic shared memory per CTA: 227 KB for one CTA per SM; for two, half of the SM's 228 KB less the 1 KB the hardware
// reserves per CTA.
template <int OCC> struct GemmOcc {
    static_assert(OCC == 1 || OCC == 2, "OCC");
    static constexpr int SMEM_LIMIT = OCC == 1 ? 232448 : 115712;
    // One CTA: 65536 registers / 288 threads, rounded down to 8.  Two CTAs: 18 warps over the SM's four 16384-register
    // quarters put 5 warps on one quarter, so 16384 / (5 * 32) = 102, rounded down to 8.
    static constexpr int MAX_REGS = OCC == 1 ? 224 : 96;
};

struct GemmParams {
    int M, N, K;
    int num_k_blocks;
    int a_mode;
    // conv geometry (output space)
    int n_img, Ho, Wo, C, cblocks, pad_lo;
    int bw, bh, bn, tiles_w, tiles_h, tiles_n;
    int num_m_blocks, num_n_blocks;
    // epilogue
    const float* bias;
    const float* row_bias;
    int rows_per_group;
    long long ld_rb;
    const __nv_bfloat16* residual;
    long long ldr;
    const float* lora_up;
    int lora_rp;
    float lora_scale;
    const float* t_add;
    float* t_out;
    void* out;
    long long ldd;
    int out_fp32;
    // split-K: tile space is (m, n, split); split s covers k-blocks [s*kb_per_split, ...) and stores its fp32 partial tile
    // to split_ws[s][M][N]; splitk_finish_kernel sums the partials and applies the epilogue.
    int splits, kb_per_split;
    float* split_ws;
};

template <int BN, int EXT, int BK>
struct GemmCfg {
    static constexpr int NT = BN + EXT;                       // N of one wgmma
    static constexpr int ROW_BYTES = BK * 2;
    static constexpr int A_BYTES = BLOCK_M * ROW_BYTES;
    static constexpr int B_BYTES = NT * ROW_BYTES;
    static constexpr int STAGE_BYTES = (A_BYTES + B_BYTES + 1023) / 1024 * 1024;
    static constexpr int SBO = 8 * ROW_BYTES;                 // 8-row swizzle atom
    static constexpr uint32_t SWZ = (BK == 64) ? SWZ_128B : SWZ_64B;
    static constexpr int ACC = NT / 2;                        // fp32 accumulators per consumer thread
    static_assert(BK == 64 || BK == 32, "BK");
    static_assert(NT % 16 == 0 && NT <= 256, "wgmma N");
    static_assert(BN % 32 == 0, "BN");
};

// Decode tile-local row r (0..127) into the global output row (or -1 if masked) and its row_bias group.
__device__ __forceinline__ void decode_row(const GemmParams& p, int m_blk, int r, int& m, int& grp) {
    if (p.a_mode == 0) {
        m = m_blk * BLOCK_M + r;
        if (m >= p.M) m = -1;
        grp = (m >= 0 && p.rows_per_group > 0) ? m / p.rows_per_group : 0;
    } else {
        int tw = m_blk % p.tiles_w;
        int th = (m_blk / p.tiles_w) % p.tiles_h;
        int tn = m_blk / (p.tiles_w * p.tiles_h);
        int dw = r % p.bw, dh = (r / p.bw) % p.bh, dn = r / (p.bw * p.bh);
        int n = tn * p.bn + dn, h = th * p.bh + dh, w = tw * p.bw + dw;
        if (n < p.n_img && h < p.Ho && w < p.Wo) {
            m = (n * p.Ho + h) * p.Wo + w;
            grp = (p.rows_per_group > 0) ? m / p.rows_per_group : 0;
        } else {
            m = -1;
            grp = 0;
        }
    }
}

template <int BN, int EXT, int BK, int OCC>
__global__ void __maxnreg__(GemmOcc<OCC>::MAX_REGS)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmE, const GemmParams p, const int num_stages) {
    pdl_launch_dependents();
    using Cfg = GemmCfg<BN, EXT, BK>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + num_stages * Cfg::STAGE_BYTES);
    uint64_t* empty_bar = full_bar + num_stages;
    const int warp_idx = uniform_warp_idx();
    const int lane = threadIdx.x & 31;
    const int wg = warp_idx >> 2;

    // tile = (m_blk * num_n + n_blk) * splits + split
    int t2 = blockIdx.x;
    const int split = t2 % p.splits; t2 /= p.splits;
    const int n_blk = t2 % p.num_n_blocks;
    const int m_blk = t2 / p.num_n_blocks;
    const int kb0 = split * p.kb_per_split;
    const int kb1 = min(p.num_k_blocks, kb0 + p.kb_per_split);

    if (warp_idx == PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (EXT) tma_prefetch_desc(&tmE);
        for (int i = 0; i < num_stages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 2);     // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();   // everything above touched only shared memory and kernel parameters

    if (warp_idx == PRODUCER_WARP) {
        if (elect_one_sync()) {
            int tw = 0, th = 0, tn = 0;
            if (p.a_mode != 0) {
                tw = m_blk % p.tiles_w;
                th = (m_blk / p.tiles_w) % p.tiles_h;
                tn = m_blk / (p.tiles_w * p.tiles_h);
            }
            int stage = 0;
            uint32_t phase = 0;
            int tap = 0, cb = 0;
            if (p.a_mode != 0) { tap = kb0 / p.cblocks; cb = kb0 - tap * p.cblocks; }
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], Cfg::A_BYTES + Cfg::B_BYTES);
                uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
                uint8_t* sb = sa + Cfg::A_BYTES;
                if (p.a_mode == 0) {
                    tma_load_2d(&tmA, &full_bar[stage], sa, kb * BK, m_blk * BLOCK_M);
                } else {
                    const int ky = tap / 3, kx = tap - ky * 3;
                    if (p.a_mode == 1) {
                        tma_load_4d(&tmA, &full_bar[stage], sa, cb * BK, tw * p.bw + kx - 1, th * p.bh + ky - 1, tn * p.bn);
                    } else {
                        const int iy = ky - p.pad_lo, ix = kx - p.pad_lo;
                        tma_load_5d(&tmA, &full_bar[stage], sa, (ix & 1) * p.C + cb * BK, tw * p.bw + (ix >> 1), iy & 1,
                                    th * p.bh + (iy >> 1), tn * p.bn);
                    }
                    if (++cb == p.cblocks) { cb = 0; ++tap; }
                }
                tma_load_2d(&tmB, &full_bar[stage], sb, kb * BK, n_blk * BN);
                if (EXT) tma_load_2d(&tmE, &full_bar[stage], sb + BN * Cfg::ROW_BYTES, kb * BK, 0);
                if (++stage == num_stages) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    // ===================================================== consumers: main loop
    float acc[Cfg::ACC];
#pragma unroll
    for (int i = 0; i < Cfg::ACC; ++i) acc[i] = 0.f;
    const uint32_t a_off = uint32_t(wg) * 64 * Cfg::ROW_BYTES;
    {
        int stage = 0, prev = -1;
        uint32_t phase = 0;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
            const uint32_t sb = sa + Cfg::A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k)
                Wgmma<Cfg::NT, 0, 0>::mma(acc, make_smem_desc(sa + a_off + k * 32, 16, Cfg::SBO, Cfg::SWZ),
                                          make_smem_desc(sb + k * 32, 16, Cfg::SBO, Cfg::SWZ), (kb > kb0 || k > 0) ? 1 : 0);
            wgmma_commit();
            wgmma_wait<1>();          // the previous k-block's MMAs are done: release its stage
            if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == num_stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
    }

    // ===================================================== epilogue from registers
    // accumulator layout of wgmma m64nNk16: acc[j*4 + i*2 + c] = D[row w*16 + lane/4 + 8i][col 8j + 2*(lane%4) + c]
    const int w4 = warp_idx & 3, q = lane & 3;
    // Both rows of this lane first (row index, row_bias group, LoRA t), then the columns: each column's lora_up values are
    // loaded once for the two rows.
    int m[2], grp[2];
    float t[2][8];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        decode_row(p, m_blk, wg * 64 + w4 * 16 + (lane >> 2) + 8 * i, m[i], grp[i]);
        if (EXT) {
            // t[j] = e[j] + e[j + 8]: this lane holds columns 2q, 2q+1 of both halves; gather the quad's 8 values
            const float t0 = acc[(BN / 8) * 4 + i * 2] + acc[(BN / 8 + 1) * 4 + i * 2];
            const float t1 = acc[(BN / 8) * 4 + i * 2 + 1] + acc[(BN / 8 + 1) * 4 + i * 2 + 1];
#pragma unroll
            for (int qq = 0; qq < 4; ++qq) {
                t[i][2 * qq] = __shfl_sync(0xffffffffu, t0, (lane & ~3) | qq);
                t[i][2 * qq + 1] = __shfl_sync(0xffffffffu, t1, (lane & ~3) | qq);
            }
            const int rp = p.lora_rp;
            if (m[i] >= 0) {
                const long long tb = (long long)m[i] * rp;
                float o0 = t0, o1 = t1;   // this lane's own columns 2q, 2q+1, so t is never indexed by the lane
                if (p.t_add != nullptr) {
                    if (2 * q < rp) { o0 += p.t_add[tb + 2 * q]; o1 += p.t_add[tb + 2 * q + 1]; }   // rp is even
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj)
                        if (jj < rp) t[i][jj] += p.t_add[tb + jj];
                }
                if (p.t_out != nullptr && n_blk == 0 && 2 * q < rp) { p.t_out[tb + 2 * q] = o0; p.t_out[tb + 2 * q + 1] = o1; }
            }
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) t[i][jj] = (jj < rp) ? t[i][jj] * p.lora_scale : 0.f;
        }
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int n = n_blk * BN + 8 * j + 2 * q;
        if (n >= p.N) continue;          // N % 4 == 0: n < N implies n + 1 < N
        float u0[8], u1[8];
        if (EXT) {
            const float* up = p.lora_up + (long long)n * p.lora_rp;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                u0[jj] = jj < p.lora_rp ? __ldg(up + jj) : 0.f;
                u1[jj] = jj < p.lora_rp ? __ldg(up + p.lora_rp + jj) : 0.f;
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (m[i] < 0) continue;
            float v0 = acc[j * 4 + i * 2], v1 = acc[j * 4 + i * 2 + 1];
            if (EXT) {
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    if (jj < p.lora_rp) { v0 = fmaf(t[i][jj], u0[jj], v0); v1 = fmaf(t[i][jj], u1[jj], v1); }
                }
            }
            if (p.splits > 1) {     // host cleared bias / row_bias / residual: the finishing kernel applies them
                *reinterpret_cast<float2*>(p.split_ws + (long long)split * p.M * p.N + (long long)m[i] * p.N + n) = make_float2(v0, v1);
                continue;
            }
            if (p.bias != nullptr) { v0 += __ldg(p.bias + n); v1 += __ldg(p.bias + n + 1); }
            if (p.row_bias != nullptr) {
                const float2 rb = *reinterpret_cast<const float2*>(p.row_bias + (long long)grp[i] * p.ld_rb + n);
                v0 += rb.x; v1 += rb.y;
            }
            if (p.residual != nullptr) {
                const float2 rr = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.residual + (long long)m[i] * p.ldr + n));
                v0 += rr.x; v1 += rr.y;
            }
            if (p.out_fp32) {
                *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + (long long)m[i] * p.ldd + n) = make_float2(v0, v1);
            } else {
                *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + (long long)m[i] * p.ldd + n) = pack_bf16x2(v0, v1);
            }
        }
    }
}

// out = epilogue(sum_s ws[s]) for the split-K path: one thread per 4 output columns.
__global__ void __launch_bounds__(256)
splitk_finish_kernel(const float* __restrict__ ws, int splits, int M, int N, const float* __restrict__ bias,
                     const float* __restrict__ row_bias, int rows_per_group, long long ld_rb,
                     const __nv_bfloat16* __restrict__ residual, long long ldr, void* __restrict__ out, long long ldd,
                     int out_fp32) {
    pdl_launch_dependents();
    pdl_wait();
    const int nq = N >> 2;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)M * nq) return;
    const int m = (int)(idx / nq);
    const int n0 = (int)(idx - (long long)m * nq) * 4;
    const long long MN = (long long)M * N;
    const float* src = ws + (long long)m * N + n0;
    float4 acc = *reinterpret_cast<const float4*>(src);
    for (int s = 1; s < splits; ++s) {
        const float4 v = *reinterpret_cast<const float4*>(src + s * MN);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (row_bias != nullptr) {
        const float4 v = *reinterpret_cast<const float4*>(row_bias + (long long)(m / rows_per_group) * ld_rb + n0);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (residual != nullptr) {
        const uint2 rr = *reinterpret_cast<const uint2*>(residual + (long long)m * ldr + n0);
        const float2 a = unpack_bf16x2(rr.x), b = unpack_bf16x2(rr.y);
        acc.x += a.x; acc.y += a.y; acc.z += b.x; acc.w += b.y;
    }
    if (bias != nullptr) {
        const float4 v = *reinterpret_cast<const float4*>(bias + n0);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (out_fp32) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + (long long)m * ldd + n0) = acc;
    } else {
        uint2 o;
        o.x = pack_bf16x2(acc.x, acc.y);
        o.y = pack_bf16x2(acc.z, acc.w);
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + (long long)m * ldd + n0) = o;
    }
}

// =====================================================================================================
// host side
// =====================================================================================================

// Launches the GEMM; with `resident` set, launches nothing and stores how many CTAs of this instantiation the device keeps
// resident per SM at the shared-memory size the launch would use.
template <int BN, int EXT, int BK, int OCC>
static int launch_gemm(const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tE, const GemmParams& p_in,
                       cudaStream_t stream, int* resident) {
    using Cfg = GemmCfg<BN, EXT, BK>;
    constexpr int SMEM_LIMIT = GemmOcc<OCC>::SMEM_LIMIT;
    GemmParams p = p_in;
    const int fixed = 1024 /*align slack*/ + 256 /*barriers*/;
    int stages = (SMEM_LIMIT - fixed) / Cfg::STAGE_BYTES;
    if (stages > 8) stages = 8;
    if (stages < 2) return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: not enough shared memory for 2 stages");
    const int smem_bytes = fixed + stages * Cfg::STAGE_BYTES;
    const long long grid = (long long)p.num_m_blocks * p.num_n_blocks * p.splits;
    if (grid > 0x7fffffffLL) return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: too many tiles");
    const GemmParams full = p;
    if (p.splits > 1) { p.bias = nullptr; p.row_bias = nullptr; p.residual = nullptr; }
    static bool attr_done = false;
    if (!attr_done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(gemm_wgmma_kernel<BN, EXT, BK, OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
        attr_done = true;
    }
    if (resident != nullptr) {
        CL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(resident, gemm_wgmma_kernel<BN, EXT, BK, OCC>, NUM_THREADS, smem_bytes));
        return CL_OK;
    }
    launch_k_pdl(gemm_wgmma_kernel<BN, EXT, BK, OCC>, (unsigned)grid, NUM_THREADS, smem_bytes, stream, tA, tB, tE, p, stages);
    count_launch();
    if (p.splits > 1) {
        const long long quads = (long long)p.M * (p.N / 4);
        launch_k_pdl(splitk_finish_kernel, (unsigned)((quads + 255) / 256), 256, 0, stream,
            p.split_ws, p.splits, p.M, p.N, full.bias, full.row_bias, full.rows_per_group, full.ld_rb, full.residual,
            full.ldr, full.out, full.ldd, full.out_fp32);
        count_launch();
    }
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

}  // namespace clb

using namespace clb;

// Output-tile plan: block_n, the number of K splits and CTAs per SM (rule at the end of plan_tiles).  Cost model: a CTA streams (128 + bn) operand rows per k-block
// and the kernel runs `waves` rounds of tiles, so
//   cost = waves(tiles * splits) * (128 + bn + 32) * ceil(nkb / splits)          (+32: per-tile epilogue / ramp)
// Splitting K is only considered when the (m, n) tiles leave more than half of the SMs idle and every split keeps
// >= 8 k-blocks.  The caller provides split_ws = splits * M * N floats (cl_gemm_split_hint tells how many).
struct TilePlan { int bn, splits, occ; };

static inline int gemm_block_k(const cl_gemm_args* a) { return (a->a_mode != 0 && a->C % 64 != 0) ? 32 : 64; }

// The instantiations that compile within GemmOcc<2>::MAX_REGS registers without spilling.
static inline bool gemm_fits_two_ctas(int bn, bool lora, int BK) { return !lora && (BK == 32 ? bn <= 128 : bn == 128); }

static TilePlan plan_tiles(const cl_gemm_args* a, int BK, int num_m_blocks, bool allow_split) {
    const bool lora = a->lora_up != nullptr;
    const int nkb = (a->K + BK - 1) / BK;
    const int sms = num_sms();
    TilePlan best = {0, 1, 1};
    long long best_cost = -1;
    static const int cands[5] = {256, 160, 128, 64, 32};
    for (int ci = 0; ci < 5; ++ci) {
        const int bn = cands[ci];
        if (a->block_n != 0 && bn != a->block_n) continue;
        if (a->N % bn != 0 && a->block_n == 0) continue;
        if (BK == 32 ? (bn > 128 || bn == 160) : (bn < 64)) continue;   // instantiated variants
        if (lora && (bn > 160 || bn < 64)) continue;
        const int tiles = num_m_blocks * ((a->N + bn - 1) / bn);
        int splits = 1;
        if (allow_split && !lora && tiles * 2 <= sms) {
            splits = sms / tiles;
            if (splits > nkb / 8) splits = nkb / 8;
            if (splits > 16) splits = 16;
            if (splits < 2) splits = 1;
        }
        const int kbps = (nkb + splits - 1) / splits;
        splits = (nkb + kbps - 1) / kbps;
        const long long waves = ((long long)tiles * splits + sms - 1) / sms;
        const long long cost = waves * (128 + bn + 32) * kbps;
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = {bn, splits, 1}; }
    }
    if (best_cost < 0) {   // no candidate divides N: tail tiles
        if (lora) best.bn = (a->N % 128 == 0) ? 128 : 160;
        else if (a->N <= 32 && BK == 32) best.bn = 32;
        else if (a->N <= 64) best.bn = 64;
        else if (a->N <= 128 || BK == 32) best.bn = 128;
        else best.bn = 160;
        best.splits = 1;
    }
    // Two CTAs per SM for unsplit short-K launches (<= 20 k-blocks per tile) whose tiles fill every one of the 2 * sms
    // CTA slots: then one CTA's prologue, pipeline fill and epilogue overlap the other's MMAs.  Measured on the bench step
    // (H100 SXM): the 9-18 k-block launches with >= 1024 tiles ran 0.79-0.85x the one-CTA time at BK 64 and BN 128;
    // launches of 80-240 tiles were slower at two CTAs per SM (pairs share SMs while others idle), deep-K ones were too.
    if (best.splits == 1 && nkb <= 20 && gemm_fits_two_ctas(best.bn, lora, BK)) {
        const long long tiles = (long long)num_m_blocks * ((a->N + best.bn - 1) / best.bn);
        if (tiles >= 2LL * sms) best.occ = 2;
    }
    return best;
}

extern "C" int cl_gemm_split_hint(const cl_gemm_args* a) {
    if (a == nullptr || a->lora_up != nullptr || a->M <= 0 || a->N <= 0 || a->K <= 0) return 1;
    // conv tiles may pad M when the image does not tile evenly; cl_gemm re-plans with the exact count and clamps
    return plan_tiles(a, gemm_block_k(a), (a->M + BLOCK_M - 1) / BLOCK_M, true).splits;
}

static int dispatch_gemm(const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tE, const GemmParams& p,
                         cudaStream_t stream, int* q, int bn_sel, bool two, bool lora, int BK) {
    if (BK == 32) {
        if (lora) return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: LoRA epilogue is not instantiated for 32-channel convs");
        switch (bn_sel) {
            case 32: return two ? launch_gemm<32, 0, 32, 2>(tA, tB, tE, p, stream, q) : launch_gemm<32, 0, 32, 1>(tA, tB, tE, p, stream, q);
            case 64: return two ? launch_gemm<64, 0, 32, 2>(tA, tB, tE, p, stream, q) : launch_gemm<64, 0, 32, 1>(tA, tB, tE, p, stream, q);
            case 128: return two ? launch_gemm<128, 0, 32, 2>(tA, tB, tE, p, stream, q) : launch_gemm<128, 0, 32, 1>(tA, tB, tE, p, stream, q);
            default: return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: block_n for 32-channel convs must be 32/64/128");
        }
    }
    if (lora) {
        switch (bn_sel) {
            case 64: return launch_gemm<64, 16, 64, 1>(tA, tB, tE, p, stream, q);
            case 128: return launch_gemm<128, 16, 64, 1>(tA, tB, tE, p, stream, q);
            case 160: return launch_gemm<160, 16, 64, 1>(tA, tB, tE, p, stream, q);
            default: return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: block_n for LoRA must be 64/128/160");
        }
    }
    switch (bn_sel) {
        case 64: return launch_gemm<64, 0, 64, 1>(tA, tB, tE, p, stream, q);
        case 128: return two ? launch_gemm<128, 0, 64, 2>(tA, tB, tE, p, stream, q) : launch_gemm<128, 0, 64, 1>(tA, tB, tE, p, stream, q);
        case 160: return launch_gemm<160, 0, 64, 1>(tA, tB, tE, p, stream, q);
        case 256: return launch_gemm<256, 0, 64, 1>(tA, tB, tE, p, stream, q);
        default: return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: block_n must be 64/128/160/256");
    }
}

// cl_gemm, or with `info` set, cl_gemm_plan: info = {block_n, splits, ctas_per_sm, resident_per_sm} and no launch.
static int run_gemm(const cl_gemm_args* a, cudaStream_t stream, int32_t* info) {
    if (a == nullptr || a->a == nullptr || a->b == nullptr || a->out == nullptr)
        return set_error(CL_ERR_INVALID, "cl_gemm: null pointer");
    if (a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error(CL_ERR_INVALID, "cl_gemm: non-positive dims");
    if (a->N % 4 != 0) return set_error(CL_ERR_INVALID, "cl_gemm: N must be a multiple of 4");
    if (a->K % 8 != 0 || a->ldb % 8 != 0) return set_error(CL_ERR_INVALID, "cl_gemm: K/ldb must be multiples of 8");
    const bool lora = a->lora_up != nullptr;
    if (lora && (a->ext == nullptr || (a->lora_rp != 4 && a->lora_rp != 8)))
        return set_error(CL_ERR_INVALID, "cl_gemm: LoRA epilogue needs ext and lora_rp in {4,8}");
    if ((a->t_add || a->t_out) && !lora) return set_error(CL_ERR_INVALID, "cl_gemm: t_add/t_out need the LoRA epilogue");

    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.M = a->M; p.N = a->N; p.K = a->K;
    p.a_mode = a->a_mode;
    // K-block: 64 (128B swizzle) unless this is a conv whose channel count only allows 32-element K runs
    const int BK = gemm_block_k(a);
    const int swz = (BK == 64) ? 128 : 64;
    p.num_k_blocks = (a->K + BK - 1) / BK;
    CUtensorMap tA, tB, tE;
    memset(&tE, 0, sizeof(tE));

    if (a->a_mode == 0) {
        if (a->lda % 8 != 0) return set_error(CL_ERR_INVALID, "cl_gemm: lda must be a multiple of 8");
        p.num_m_blocks = (a->M + BLOCK_M - 1) / BLOCK_M;
        uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->M};
        uint64_t strides[1] = {(uint64_t)a->lda * 2};
        uint32_t box[2] = {(uint32_t)BK, BLOCK_M};
        CL_CHECK(get_tensor_map(&tA, a->a, 2, dims, strides, box, swz));
    } else if (a->a_mode == 1 || a->a_mode == 2) {
        if (a->C % 32 != 0) return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: conv C must be a multiple of 32");
        if (a->K != 9 * a->C) return set_error(CL_ERR_INVALID, "cl_gemm: conv K must be 9*C");
        const int s = (a->a_mode == 2) ? 2 : 1;
        if (a->H % s || a->W % s) return set_error(CL_ERR_INVALID, "cl_gemm: stride-2 conv needs even H, W");
        p.n_img = a->n_img; p.Ho = a->H / s; p.Wo = a->W / s; p.C = a->C; p.cblocks = a->C / BK;
        p.pad_lo = a->pad_lo;
        if (a->M != p.n_img * p.Ho * p.Wo) return set_error(CL_ERR_INVALID, "cl_gemm: conv M != n*Ho*Wo");
        int bw = 128;
        while (bw > 1 && (p.Wo % bw) != 0) bw >>= 1;
        int bh = 128 / bw;
        while (bh > 1 && (p.Ho % bh) != 0) bh >>= 1;
        int bn = 128 / (bw * bh);
        if (bw > 256 || bh > 256 || bn > 256) return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: conv tile");
        p.bw = bw; p.bh = bh; p.bn = bn;
        p.tiles_w = p.Wo / bw; p.tiles_h = p.Ho / bh; p.tiles_n = (p.n_img + bn - 1) / bn;
        p.num_m_blocks = p.tiles_w * p.tiles_h * p.tiles_n;
        const uint64_t C = a->C, W = a->W, H = a->H, NI = a->n_img;
        if (a->a_mode == 1) {
            uint64_t dims[4] = {C, W, H, NI};
            uint64_t strides[3] = {C * 2, W * C * 2, H * W * C * 2};
            uint32_t box[4] = {(uint32_t)BK, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
            CL_CHECK(get_tensor_map(&tA, a->a, 4, dims, strides, box, swz));
        } else {
            uint64_t dims[5] = {2 * C, W / 2, 2, H / 2, NI};
            uint64_t strides[4] = {2 * C * 2, W * C * 2, 2 * W * C * 2, H * W * C * 2};
            uint32_t box[5] = {(uint32_t)BK, (uint32_t)bw, 1, (uint32_t)bh, (uint32_t)bn};
            CL_CHECK(get_tensor_map(&tA, a->a, 5, dims, strides, box, swz));
        }
    } else {
        return set_error(CL_ERR_INVALID, "cl_gemm: bad a_mode");
    }

    // block_n / split choice: LoRA needs BN + 16 <= 256 (wgmma N).
    if (a->split_k > 1 && lora) return set_error(CL_ERR_INVALID, "cl_gemm: split_k cannot be combined with the LoRA epilogue");
    if (a->split_k > 1 && a->split_ws == nullptr) return set_error(CL_ERR_INVALID, "cl_gemm: split_k needs split_ws");
    const TilePlan plan = plan_tiles(a, BK, p.num_m_blocks, a->split_k > 1);
    const int bn_sel = plan.bn;
    {
        static const int dbg = [] { const char* e = getenv("CLB_GEMM_DEBUG"); return (e && e[0] == '1') ? 1 : 0; }();
        if (dbg) fprintf(stderr, "cl_gemm M=%d N=%d K=%d mode=%d lora=%d -> bn=%d splits=%d occ=%d (asked bn=%d split_k=%d)\n", a->M, a->N,
                         a->K, a->a_mode, lora ? 1 : 0, bn_sel, plan.splits, plan.occ, a->block_n, a->split_k);
    }
    p.num_n_blocks = (a->N + bn_sel - 1) / bn_sel;
    p.splits = 1;
    p.kb_per_split = p.num_k_blocks;
    if (plan.splits > 1) {
        const int want = plan.splits < a->split_k ? plan.splits : a->split_k;   // split_ws holds a->split_k partials
        p.kb_per_split = (p.num_k_blocks + want - 1) / want;
        p.splits = (p.num_k_blocks + p.kb_per_split - 1) / p.kb_per_split;     // no empty split
        p.split_ws = reinterpret_cast<float*>(a->split_ws);
    }
    {
        uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->N};
        uint64_t strides[1] = {(uint64_t)a->ldb * 2};
        uint32_t box[2] = {(uint32_t)BK, (uint32_t)bn_sel};
        CL_CHECK(get_tensor_map(&tB, a->b, 2, dims, strides, box, swz));
    }
    if (lora) {
        if (a->ldb_ext % 8 != 0) return set_error(CL_ERR_INVALID, "cl_gemm: ldb_ext must be a multiple of 8");
        uint64_t dims[2] = {(uint64_t)a->K, 16};
        uint64_t strides[1] = {(uint64_t)a->ldb_ext * 2};
        uint32_t box[2] = {(uint32_t)BK, 16};
        CL_CHECK(get_tensor_map(&tE, a->ext, 2, dims, strides, box, swz));
    }

    p.bias = a->bias; p.row_bias = a->row_bias; p.rows_per_group = a->rows_per_group;
    p.ld_rb = a->ld_row_bias > 0 ? a->ld_row_bias : a->N;
    if (p.row_bias && (p.ld_rb % 4)) return set_error(CL_ERR_INVALID, "cl_gemm: ld_row_bias must be a multiple of 4");
    p.residual = reinterpret_cast<const __nv_bfloat16*>(a->residual); p.ldr = a->ldr;
    p.lora_up = a->lora_up; p.lora_rp = lora ? a->lora_rp : 4; p.lora_scale = a->lora_scale;
    p.t_add = a->t_add; p.t_out = a->t_out;
    p.out = a->out; p.ldd = a->ldd; p.out_fp32 = a->out_fp32;
    if (p.row_bias && p.rows_per_group <= 0) return set_error(CL_ERR_INVALID, "cl_gemm: rows_per_group");
    if ((p.ldd % 4) || (p.residual && (p.ldr % 4))) return set_error(CL_ERR_INVALID, "cl_gemm: ldd/ldr % 4");

    const bool two = plan.occ == 2;
    int resident = 0;
    int* const q = info != nullptr ? &resident : nullptr;
    const int st = dispatch_gemm(tA, tB, tE, p, stream, q, bn_sel, two, lora, BK);
    if (info != nullptr && st == CL_OK) { info[0] = bn_sel; info[1] = p.splits; info[2] = plan.occ; info[3] = resident; }
    return st;
}

extern "C" int cl_gemm(const cl_gemm_args* a, void* stream) { return run_gemm(a, reinterpret_cast<cudaStream_t>(stream), nullptr); }

extern "C" int cl_gemm_plan(const cl_gemm_args* a, int32_t* info) {
    if (info == nullptr) return set_error(CL_ERR_INVALID, "cl_gemm_plan: null info");
    return run_gemm(a, nullptr, info);
}
