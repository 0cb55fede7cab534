// K1/K4 — warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = epilogue( A[M,K] * B[N,K]^T ),  bf16 operands, fp32 accumulation in registers.
//
// One CTA per 128 x BN output tile (x one K range under split-K):
//   warpgroups 0-1 consumers: rows 0-63 / 64-127 of the tile, wgmma.m64n(BN+EXT)k16 straight from the swizzled stages,
//                  then the epilogue: bias, per-image row bias and residual added to the accumulators, the tile staged
//                  in the drained ring and written by TMA stores (epilogue_tma).
//   TMA loads (one thread): A tile 128 x BK, B tile BN x BK [+16 LoRA-down rows], 128B (BK = 64) or 64B (BK = 32)
//                  swizzle, mbarrier ring of up to 8 stages.
// Occupancy OCC = 1 or 2 CTAs per SM is a template parameter; with two CTAs on an SM, one CTA's prologue, pipeline fill
// and epilogue run while the other's MMAs do, which is what short-K tiles (a few k-blocks each) need.  Two thread
// layouts (GemmLayout):
//   producer warp: 288 threads, the loads come from warp 8, which runs ahead through the whole ring; cap 224 registers
//                  at one CTA per SM, 96 at two (18 warps put five on one register-file quarter).
//   no producer:   256 threads, thread 0 of warpgroup 0 fills the ring at tile start and refills each stage once both
//                  warpgroups have released it; cap 128 at two CTAs per SM.  Used only by the two-CTA tiles that do not
//                  fit 96 registers (BN 160, LoRA).  Each warpgroup retires a k-block's four MMAs (one commit group)
//                  before it releases the stage and thread 0 refills it: a single-thread path run while a group is in
//                  flight makes ptxas serialise every wgmma of the kernel (C7518).  The other CTA on the SM keeps the
//                  tensor cores busy across that drain.
// Both layouts issue the same MMA sequence.
// LoRA (EXT = 16): the 16 extra B rows (bf16 hi / lo halves of the rank-r down matrix) make the main loop produce
// t = x A^T in 16 extra accumulator columns.  After the main loop, t (+ t_add, -> t_out) is scaled, split exactly into
// three bf16 parts t1 + t2 + t3 (as is B_up = b1 + b2 + b3) and added to the BN output columns on the tensor cores: three
// register-A wgmma k16 steps [t1 | t2] * [b1 ; b1] + [t1 | t2] * [b2 ; b2] + [t1 | t3] * [b3 ; b1], which keep every
// product down to 2^-16 relative; B_up's parts are staged in shared memory in the prologue.
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
static constexpr int PRODUCER_WARP = 8;
static constexpr int CONSUMER_THREADS = 256;
// Dynamic shared memory per CTA: 227 KB for one CTA per SM; for two, half of the SM's 228 KB less the 1 KB the hardware
// reserves per CTA.
template <int OCC> struct GemmOcc {
    static_assert(OCC == 1 || OCC == 2, "OCC");
    static constexpr int SMEM_LIMIT = OCC == 1 ? 232448 : 115712;
};
template <int BN, int EXT, int BK, int OCC> struct GemmLayout {
    // the producer-warp layout unless two CTAs per SM need more than 96 registers (BN 160 or the LoRA tiles)
    static constexpr bool PRODUCER = OCC == 1 || (EXT == 0 && BN <= 128);
    static constexpr int NUM_THREADS = PRODUCER ? CONSUMER_THREADS + 32 : CONSUMER_THREADS;
    // One CTA: 65536 registers / 288 threads, rounded down to 8.  Two CTAs of 288 threads: 18 warps over the SM's four
    // 16384-register quarters put 5 warps on one, so 16384 / (5 * 32) = 102, rounded down to 8; of 256 threads: 4 warps
    // on each quarter, 16384 / (4 * 32) = 128.
    static constexpr int MAX_REGS = OCC == 1 ? 224 : PRODUCER ? 96 : 128;
    // the thread that initialises the barriers and issues the TMA loads
    static constexpr int TMA_THREAD = PRODUCER ? PRODUCER_WARP * 32 : 0;
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
    // 1: the output tile (or split-K partial) is staged in shared memory and written by TMA stores (tmD), the residual
    // read by TMA (tmR)
    int tma_epilogue;
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
    // LoRA rank-update B operand (B_up of the tile's BN columns): three k16 steps of BN x 16 bf16, K-major, no swizzle
    static constexpr int UP_STEP_BYTES = BN * 32;
    static constexpr int UP_BYTES = EXT ? 3 * UP_STEP_BYTES : 0;
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

// (a, b) -> three bf16x2 parts whose sum is exactly (a, b): each residual is exact in fp32 and 8 + 8 + 8 bits cover
// fp32's 24-bit significand (short of bf16's underflow range).
__device__ __forceinline__ void split3_bf16x2(float a, float b, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
    p1 = pack_bf16x2(a, b);
    const float2 f1 = unpack_bf16x2(p1);
    const float ra = a - f1.x, rb = b - f1.y;
    p2 = pack_bf16x2(ra, rb);
    const float2 f2 = unpack_bf16x2(p2);
    p3 = pack_bf16x2(ra - f2.x, rb - f2.y);
}

// Loads k-block kb of the tile into ring stage `stage` (A tile, B tile and the LoRA-down rows) on its full barrier.
// Convs: (tw, th, tn) is the tile's position and (tap, cb) = (kb / cblocks, kb % cblocks), which the caller steps along.
template <int BN, int EXT, int BK>
__device__ __forceinline__ void load_stage(const CUtensorMap* tmA, const CUtensorMap* tmB, const CUtensorMap* tmE,
                                           const GemmParams& p, uint8_t* smem, uint64_t* full_bar, int stage, int kb,
                                           int m_blk, int n_blk, int tw, int th, int tn, int tap, int cb) {
    using Cfg = GemmCfg<BN, EXT, BK>;
    mbar_arrive_expect_tx(&full_bar[stage], Cfg::A_BYTES + Cfg::B_BYTES);
    uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
    uint8_t* sb = sa + Cfg::A_BYTES;
    if (p.a_mode == 0) {
        tma_load_2d(tmA, &full_bar[stage], sa, kb * BK, m_blk * BLOCK_M);
    } else {
        const int ky = tap / 3, kx = tap - ky * 3;
        if (p.a_mode == 1) {
            tma_load_4d(tmA, &full_bar[stage], sa, cb * BK, tw * p.bw + kx - 1, th * p.bh + ky - 1, tn * p.bn);
        } else {
            const int iy = ky - p.pad_lo, ix = kx - p.pad_lo;
            tma_load_5d(tmA, &full_bar[stage], sa, (ix & 1) * p.C + cb * BK, tw * p.bw + (ix >> 1), iy & 1,
                        th * p.bh + (iy >> 1), tn * p.bn);
        }
    }
    tma_load_2d(tmB, &full_bar[stage], sb, kb * BK, n_blk * BN);
    if (EXT) tma_load_2d(tmE, &full_bar[stage], sb + BN * Cfg::ROW_BYTES, kb * BK, 0);
}

// TMA epilogue: the output tile is staged in the drained ring as 64-byte-wide column chunks of 128 rows (bf16: 32 columns,
// fp32: 16), 64B-swizzled like the boxes of tmD / tmR, so that a warp's 8 rows x 16 bytes of one accumulator column pair
// fall into 32 different banks.  Byte (row, c) sits at chunk c / 64, row * 64, 16-byte unit ((c / 16) % 4) ^ ((row / 2) % 4).
// The residual tile (bf16 output only) comes in by TMA into the staging chunks; the consumers add bias, row bias and
// residual to their accumulators in the register epilogue's order and overwrite their own slots; the chunks leave by TMA
// stores, whose bounds drop rows past M (or past the images) and columns past N.  One thread issues the TMA operations:
// a producer-warp lane, which holds no accumulators, or thread 0 where there is no producer warp.  Named barrier 2: every
// MMA has read the ring (and s_up); barrier 3: the staged tile is complete.
__device__ __forceinline__ void epi_conv_pos(const GemmParams& p, int m_blk, int& x, int& y, int& z) {
    x = m_blk % p.tiles_w * p.bw;
    y = (m_blk / p.tiles_w) % p.tiles_h * p.bh;
    z = m_blk / (p.tiles_w * p.tiles_h) * p.bn;
}

template <int BN>
__device__ __forceinline__ void epi_load_residual(const CUtensorMap* tmR, const GemmParams& p, uint8_t* stile,
                                                  uint64_t* res_bar, int m_blk, int n_blk) {
    mbar_arrive_expect_tx(res_bar, BLOCK_M * BN * 2);
    int x = 0, y = 0, z = 0;
    if (p.a_mode != 0) epi_conv_pos(p, m_blk, x, y, z);
#pragma unroll 1
    for (int k = 0; k < BN / 32; ++k) {
        uint8_t* dst = stile + k * BLOCK_M * 64;
        if (p.a_mode == 0) tma_load_2d(tmR, res_bar, dst, n_blk * BN + 32 * k, m_blk * BLOCK_M);
        else tma_load_4d(tmR, res_bar, dst, n_blk * BN + 32 * k, x, y, z);
    }
}

// split-K partials go to split_ws[split] through a map with the split as its outermost dimension
template <int BN>
__device__ __forceinline__ void epi_store(const CUtensorMap* tmD, const GemmParams& p, uint8_t* stile, int m_blk, int n_blk,
                                          int split) {
    const int esz = (p.out_fp32 || p.splits > 1) ? 4 : 2;
    int x = 0, y = 0, z = 0;
    if (p.a_mode != 0) epi_conv_pos(p, m_blk, x, y, z);
    const uint32_t base = smem_u32(stile);
#pragma unroll 1
    for (int k = 0; k < BN * esz / 64; ++k) {
        const int c0 = n_blk * BN * esz / 2 + 32 * k;   // the maps count 2-byte elements
        const uint32_t src = base + k * BLOCK_M * 64;
        if (p.splits > 1) {
            if (p.a_mode == 0) tma_store_3d(tmD, src, c0, m_blk * BLOCK_M, split);
            else tma_store_5d(tmD, src, c0, x, y, z, split);
        } else {
            if (p.a_mode == 0) tma_store_2d(tmD, src, c0, m_blk * BLOCK_M);
            else tma_store_4d(tmD, src, c0, x, y, z);
        }
    }
    bulk_commit_group();
    bulk_wait_group_read<0>();             // shared memory stays valid until the stores have read it
}

// the consumers' half; ISSUE: this kernel has no producer warp, so thread 0 issues the TMA operations
template <int BN, int ESZ, bool ISSUE, int NACC>
__device__ __forceinline__ void epilogue_tma(const CUtensorMap* tmD, const CUtensorMap* tmR, const GemmParams& p,
                                             const float (&acc)[NACC], uint8_t* stile, uint64_t* res_bar, int m_blk,
                                             int n_blk, int split, const float* const (&rbp)[2], int row0, int q,
                                             int bar_threads) {
    const bool res = p.residual != nullptr;
    named_bar_sync(2, bar_threads);
    if (res) {
        if (ISSUE && threadIdx.x == 0) epi_load_residual<BN>(tmR, p, stile, res_bar, m_blk, n_blk);
        mbar_wait(res_bar, 0);
    }
    // this thread's byte columns are 8 j ESZ + 2 q ESZ: the q part, the row's swizzle and the row go into one address per
    // row, the j part is a constant unit XOR and chunk offset (no carries: 2 q ESZ stays within its 16- or 32-byte group)
    const uint32_t base = smem_u32(stile);
    uint32_t addr[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int row = row0 + 8 * i, cq = 2 * q * ESZ;
        addr[i] = base + row * 64 + ((((cq >> 4) ^ (row >> 1)) & 3) << 4) + (cq & 15);
    }
    const int n0 = n_blk * BN + 2 * q, n_left = p.N - n0;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j;
        const bool n_in = 8 * j < n_left;  // N % 4 == 0: n < N implies n + 1 < N
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float v0 = acc[j * 4 + i * 2], v1 = acc[j * 4 + i * 2 + 1];
            if (p.bias != nullptr && n_in) { v0 += __ldg(p.bias + n); v1 += __ldg(p.bias + n + 1); }
            if (rbp[i] != nullptr && n_in) {
                const float2 rb = *reinterpret_cast<const float2*>(rbp[i] + n);
                v0 += rb.x; v1 += rb.y;
            }
            const uint32_t a = (addr[i] ^ ((((8 * j * ESZ) >> 4) & 3) << 4)) + ((8 * j * ESZ) >> 6) * (BLOCK_M * 64);
            if (ESZ == 4) {
                st_shared_f2(a, v0, v1);
            } else {
                if (res) {
                    const float2 rr = unpack_bf16x2(ld_shared_u32(a));
                    v0 += rr.x; v1 += rr.y;
                }
                st_shared_u32(a, pack_bf16x2(v0, v1));
            }
        }
    }
    fence_proxy_async_smem();              // generic-proxy stores -> TMA reads
    if (ISSUE) {
        named_bar_sync(3, bar_threads);
        if (threadIdx.x == 0) epi_store<BN>(tmD, p, stile, m_blk, n_blk, split);
    } else {
        named_bar_arrive(3, bar_threads);
    }
}

template <int BN, int EXT, int BK, int OCC>
__global__ void __maxnreg__((GemmLayout<BN, EXT, BK, OCC>::MAX_REGS))
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmE, const __grid_constant__ CUtensorMap tmD,
                  const __grid_constant__ CUtensorMap tmR, const GemmParams p, const int num_stages) {
    pdl_launch_dependents();
    using Cfg = GemmCfg<BN, EXT, BK>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* s_up = smem + num_stages * Cfg::STAGE_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_up + Cfg::UP_BYTES);
    uint64_t* empty_bar = full_bar + num_stages;
    uint64_t* res_bar = empty_bar + num_stages;    // residual tile of the TMA epilogue
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

    using Layout = GemmLayout<BN, EXT, BK, OCC>;
    int tw = 0, th = 0, tn = 0;   // conv tile position (TMA issue only)
    if (p.a_mode != 0) {
        tw = m_blk % p.tiles_w;
        th = (m_blk / p.tiles_w) % p.tiles_h;
        tn = m_blk / (p.tiles_w * p.tiles_h);
    }
    if (threadIdx.x == Layout::TMA_THREAD) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (EXT) tma_prefetch_desc(&tmE);
        for (int i = 0; i < num_stages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 2);     // one arrival per consumer warpgroup
        }
        mbar_init(res_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();   // everything above touched only shared memory and kernel parameters

    if (Layout::PRODUCER && warp_idx == PRODUCER_WARP) {
        if (elect_one_sync()) {
            int stage = 0;
            uint32_t phase = 0;
            int tap = 0, cb = 0;
            if (p.a_mode != 0) { tap = kb0 / p.cblocks; cb = kb0 - tap * p.cblocks; }
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                load_stage<BN, EXT, BK>(&tmA, &tmB, &tmE, p, smem, full_bar, stage, kb, m_blk, n_blk, tw, th, tn, tap, cb);
                if (p.a_mode != 0 && ++cb == p.cblocks) { cb = 0; ++tap; }
                if (++stage == num_stages) { stage = 0; phase ^= 1; }
            }
        }
        __syncwarp();
        if (p.tma_epilogue) {   // the TMA epilogue's loads and stores, issued for the consumers
            named_bar_sync(2, Layout::NUM_THREADS);
            if (lane == 0 && p.residual != nullptr) epi_load_residual<BN>(&tmR, p, smem, res_bar, m_blk, n_blk);
            named_bar_sync(3, Layout::NUM_THREADS);
            if (lane == 0) epi_store<BN>(&tmD, p, smem, m_blk, n_blk, split);
        }
        return;
    }
    const bool tma_thread = !Layout::PRODUCER && threadIdx.x == Layout::TMA_THREAD;
    if (tma_thread) {   // fill the ring; the main loop refills it
        for (int kb = kb0; kb < kb1 && kb - kb0 < num_stages; ++kb)
            load_stage<BN, EXT, BK>(&tmA, &tmB, &tmE, p, smem, full_bar, kb - kb0, kb, m_blk, n_blk, tw, th, tn,
                                    kb / p.cblocks, kb % p.cblocks);
    }

    if (EXT) {
        // B operand of the rank update while the ring fills: B_up rows of this tile's columns (zero past N and past the
        // rank), split into bf16 b1 + b2 + b3.  Core matrices of 8 rows x 16 bytes, (row group g, k half h) at
        // g * 256 + h * 128; the steps hold k = [b1 | b1], [b2 | b2], [b3 | b1] (k = rank index j in each half).
        for (int n = threadIdx.x; n < BN; n += CONSUMER_THREADS) {
            const int gn = n_blk * BN + n;
            float u[8];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
                u[jj] = (gn < p.N && jj < p.lora_rp) ? __ldg(p.lora_up + (long long)gn * p.lora_rp + jj) : 0.f;
            uint4 b1, b2, b3;
            split3_bf16x2(u[0], u[1], b1.x, b2.x, b3.x);
            split3_bf16x2(u[2], u[3], b1.y, b2.y, b3.y);
            split3_bf16x2(u[4], u[5], b1.z, b2.z, b3.z);
            split3_bf16x2(u[6], u[7], b1.w, b2.w, b3.w);
            const uint32_t dst = smem_u32(s_up) + (n >> 3) * 256 + (n & 7) * 16;
            st_shared_u4(dst, b1);
            st_shared_u4(dst + 128, b1);
            st_shared_u4(dst + Cfg::UP_STEP_BYTES, b2);
            st_shared_u4(dst + Cfg::UP_STEP_BYTES + 128, b2);
            st_shared_u4(dst + 2 * Cfg::UP_STEP_BYTES, b3);
            st_shared_u4(dst + 2 * Cfg::UP_STEP_BYTES + 128, b1);
        }
        fence_proxy_async_smem();                   // generic-proxy stores -> wgmma operand reads
        named_bar_sync(1, CONSUMER_THREADS);
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
            if constexpr (Layout::PRODUCER) {
                wgmma_wait<1>();      // the previous k-block's MMAs are done: release its stage
                if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
                prev = stage;
            } else {
                // No producer warp: the release and the refill are single-thread paths, which ptxas answers by
                // serialising every wgmma of the kernel when they run with a group in flight.  So this k-block's group
                // retires first, and the other CTA on the SM keeps the tensor cores busy across the drain.
                wgmma_wait<0>();
                if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);
                // once both warpgroups have released it, the stage takes the k-block num_stages on
                if (tma_thread && kb + num_stages < kb1) {
                    mbar_wait(&empty_bar[stage], phase);
                    const int kn = kb + num_stages;
                    load_stage<BN, EXT, BK>(&tmA, &tmB, &tmE, p, smem, full_bar, stage, kn, m_blk, n_blk, tw, th, tn,
                                            kn / p.cblocks, kn % p.cblocks);
                }
            }
            if (++stage == num_stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
    }

    // ===================================================== LoRA rank update, then the epilogue
    // accumulator layout of wgmma m64nNk16: acc[j*4 + i*2 + c] = D[row w*16 + lane/4 + 8i][col 8j + 2*(lane%4) + c]
    const int w4 = warp_idx & 3, q = lane & 3;
    int m[2], grp[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) decode_row(p, m_blk, wg * 64 + w4 * 16 + (lane >> 2) + 8 * i, m[i], grp[i]);
    if constexpr (EXT != 0) {
        // t[j] = e[j] + e[j + 8]: this lane holds t columns 2q, 2q+1 of rows i = 0, 1, which is where the register-A
        // fragment of a k16 step wants k = 2q, 2q+1 (a0 / a1) and k = 8 + 2q, 9 + 2q (a2 / a3).
        const int rp = p.lora_rp;
        uint32_t tp1[2], tp2[2], tp3[2];   // s t = tp1 + tp2 + tp3
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float t0 = acc[(BN / 8) * 4 + i * 2] + acc[(BN / 8 + 1) * 4 + i * 2];
            float t1 = acc[(BN / 8) * 4 + i * 2 + 1] + acc[(BN / 8 + 1) * 4 + i * 2 + 1];
            if (m[i] >= 0 && 2 * q < rp) {   // rp is even
                const long long tb = (long long)m[i] * rp;
                if (p.t_add != nullptr) { t0 += p.t_add[tb + 2 * q]; t1 += p.t_add[tb + 2 * q + 1]; }
                if (p.t_out != nullptr && n_blk == 0) { p.t_out[tb + 2 * q] = t0; p.t_out[tb + 2 * q + 1] = t1; }
            }
            const float s0 = 2 * q < rp ? t0 * p.lora_scale : 0.f, s1 = 2 * q < rp ? t1 * p.lora_scale : 0.f;
            split3_bf16x2(s0, s1, tp1[i], tp2[i], tp3[i]);
        }
        const uint32_t a12[4] = {tp1[0], tp1[1], tp2[0], tp2[1]};
        const uint32_t a13[4] = {tp1[0], tp1[1], tp3[0], tp3[1]};
        const uint32_t su = smem_u32(s_up);
        wgmma_fence();
        WgmmaRs<BN, 0>::mma(acc, a12, make_smem_desc(su, 128, 256, 0), 1);
        WgmmaRs<BN, 0>::mma(acc, a12, make_smem_desc(su + Cfg::UP_STEP_BYTES, 128, 256, 0), 1);
        WgmmaRs<BN, 0>::mma(acc, a13, make_smem_desc(su + 2 * Cfg::UP_STEP_BYTES, 128, 256, 0), 1);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
    }
    if (p.tma_epilogue) {
        const int row0 = wg * 64 + w4 * 16 + (lane >> 2);
        // row bias of each of this thread's two rows (none past M or past the images)
        const float* rbp[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) rbp[i] = (p.row_bias != nullptr && m[i] >= 0) ? p.row_bias + (long long)grp[i] * p.ld_rb : nullptr;
        constexpr bool ISSUE = !Layout::PRODUCER;
        if (p.out_fp32 || p.splits > 1)   // split-K partials are fp32, with no epilogue inputs (the finishing kernel adds them)
            epilogue_tma<BN, 4, ISSUE>(&tmD, &tmR, p, acc, smem, res_bar, m_blk, n_blk, split, rbp, row0, q, Layout::NUM_THREADS);
        else
            epilogue_tma<BN, 2, ISSUE>(&tmD, &tmR, p, acc, smem, res_bar, m_blk, n_blk, split, rbp, row0, q, Layout::NUM_THREADS);
        return;
    }
    // register epilogue: outputs, residuals or split-K workspaces a TMA map cannot address (not 16-byte aligned), fp32
    // outputs with a residual
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int n = n_blk * BN + 8 * j + 2 * q;
        if (n >= p.N) continue;          // N % 4 == 0: n < N implies n + 1 < N
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (m[i] < 0) continue;
            float v0 = acc[j * 4 + i * 2], v1 = acc[j * 4 + i * 2 + 1];
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

// Launches the GEMM; with `plan` set, launches nothing and stores plan[0] = how many CTAs of this instantiation the device
// keeps resident per SM at the shared-memory size the launch would use, plan[1] = the epilogue's store path (1: TMA,
// 0: register stores).
template <int BN, int EXT, int BK, int OCC>
static int launch_gemm(const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tE, const CUtensorMap& tD,
                       const CUtensorMap& tR, const GemmParams& p_in, cudaStream_t stream, int* plan) {
    using Cfg = GemmCfg<BN, EXT, BK>;
    constexpr int SMEM_LIMIT = GemmOcc<OCC>::SMEM_LIMIT;
    GemmParams p = p_in;
    constexpr int NUM_THREADS = GemmLayout<BN, EXT, BK, OCC>::NUM_THREADS;
    const int fixed = 1024 /*align slack*/ + Cfg::UP_BYTES + 256 /*barriers*/;
    int stages = (SMEM_LIMIT - fixed) / Cfg::STAGE_BYTES;
    if (stages > 8) stages = 8;
    if (stages < 2) return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: not enough shared memory for 2 stages");
    const int smem_bytes = fixed + stages * Cfg::STAGE_BYTES;
    const long long grid = (long long)p.num_m_blocks * p.num_n_blocks * p.splits;
    if (grid > 0x7fffffffLL) return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: too many tiles");
    // the staged output tile has to fit the ring (and s_up behind it)
    if ((long long)BLOCK_M * BN * ((p.out_fp32 || p.splits > 1) ? 4 : 2) > (long long)stages * Cfg::STAGE_BYTES + Cfg::UP_BYTES)
        p.tma_epilogue = 0;
    const GemmParams full = p;
    if (p.splits > 1) { p.bias = nullptr; p.row_bias = nullptr; p.residual = nullptr; }
    static bool attr_done = false;
    if (!attr_done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(gemm_wgmma_kernel<BN, EXT, BK, OCC>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
        attr_done = true;
    }
    if (plan != nullptr) {
        CL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&plan[0], gemm_wgmma_kernel<BN, EXT, BK, OCC>, NUM_THREADS, smem_bytes));
        plan[1] = p.tma_epilogue ? 1 : 0;
        return CL_OK;
    }
    launch_k_pdl(gemm_wgmma_kernel<BN, EXT, BK, OCC>, (unsigned)grid, NUM_THREADS, smem_bytes, stream, tA, tB, tE, tD, tR, p,
                 stages);
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
static inline bool gemm_fits_two_ctas(int bn, bool lora, int BK) {
    if (BK == 32) return !lora && bn <= 128;
    return lora ? (bn == 64 || bn == 128 || bn == 160) : (bn == 128 || bn == 160);
}

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
    // At BN 160 the 5-20 k-block launches of 384-1536 tiles ran 0.72-0.97x (plain) of their one-CTA step time, and the
    // LoRA ones 0.57-0.91x (together with the rank update moving onto the tensor cores).
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

static int dispatch_gemm(const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tE, const CUtensorMap& tD,
                         const CUtensorMap& tR, const GemmParams& p, cudaStream_t stream, int* q, int bn_sel, bool two,
                         bool lora, int BK) {
    if (BK == 32) {
        if (lora) return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: LoRA epilogue is not instantiated for 32-channel convs");
        switch (bn_sel) {
            case 32: return two ? launch_gemm<32, 0, 32, 2>(tA, tB, tE, tD, tR, p, stream, q) : launch_gemm<32, 0, 32, 1>(tA, tB, tE, tD, tR, p, stream, q);
            case 64: return two ? launch_gemm<64, 0, 32, 2>(tA, tB, tE, tD, tR, p, stream, q) : launch_gemm<64, 0, 32, 1>(tA, tB, tE, tD, tR, p, stream, q);
            case 128: return two ? launch_gemm<128, 0, 32, 2>(tA, tB, tE, tD, tR, p, stream, q) : launch_gemm<128, 0, 32, 1>(tA, tB, tE, tD, tR, p, stream, q);
            default: return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: block_n for 32-channel convs must be 32/64/128");
        }
    }
    if (lora) {
        switch (bn_sel) {
            case 64: return two ? launch_gemm<64, 16, 64, 2>(tA, tB, tE, tD, tR, p, stream, q) : launch_gemm<64, 16, 64, 1>(tA, tB, tE, tD, tR, p, stream, q);
            case 128: return two ? launch_gemm<128, 16, 64, 2>(tA, tB, tE, tD, tR, p, stream, q) : launch_gemm<128, 16, 64, 1>(tA, tB, tE, tD, tR, p, stream, q);
            case 160: return two ? launch_gemm<160, 16, 64, 2>(tA, tB, tE, tD, tR, p, stream, q) : launch_gemm<160, 16, 64, 1>(tA, tB, tE, tD, tR, p, stream, q);
            default: return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: block_n for LoRA must be 64/128/160");
        }
    }
    switch (bn_sel) {
        case 64: return launch_gemm<64, 0, 64, 1>(tA, tB, tE, tD, tR, p, stream, q);
        case 128: return two ? launch_gemm<128, 0, 64, 2>(tA, tB, tE, tD, tR, p, stream, q) : launch_gemm<128, 0, 64, 1>(tA, tB, tE, tD, tR, p, stream, q);
        case 160: return two ? launch_gemm<160, 0, 64, 2>(tA, tB, tE, tD, tR, p, stream, q) : launch_gemm<160, 0, 64, 1>(tA, tB, tE, tD, tR, p, stream, q);
        case 256: return launch_gemm<256, 0, 64, 1>(tA, tB, tE, tD, tR, p, stream, q);
        default: return set_error(CL_ERR_UNSUPPORTED, "cl_gemm: block_n must be 64/128/160/256");
    }
}

// cl_gemm, or with `info` set, cl_gemm_plan: info = {block_n, splits, ctas_per_sm, resident_per_sm, tma_store} and no launch.
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
        // the finishing kernel moves 4 columns per thread: 16-byte loads of the partials and the bias, 8 bytes of a bf16
        // output or residual, 16 of an fp32 output
        const uintptr_t ws = reinterpret_cast<uintptr_t>(a->split_ws), bi = reinterpret_cast<uintptr_t>(a->bias),
                        rb = reinterpret_cast<uintptr_t>(a->row_bias), rs = reinterpret_cast<uintptr_t>(a->residual),
                        out = reinterpret_cast<uintptr_t>(a->out);
        if ((ws & 15) || (bi & 15) || (rb & 15) || (rs & 7) || (out & (a->out_fp32 ? 15 : 7)))
            return set_error(CL_ERR_INVALID, "cl_gemm: split-K needs 16-byte aligned split_ws, bias, row_bias and fp32 out, "
                                             "8-byte aligned bf16 out and residual");
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

    // TMA epilogue: output (and residual) as 2-D maps, or for convs 4-D maps over the output image, in 64-byte column boxes
    // of 128 rows (the conv tile's bw x bh x bn box); an fp32 output is addressed as pairs of 2-byte elements.  Split-K
    // partials: the same over split_ws ([splits][M][N] fp32) with the split as one more, outermost dimension.
    CUtensorMap tD, tR;
    memset(&tD, 0, sizeof(tD));
    memset(&tR, 0, sizeof(tR));
    const bool split = p.splits > 1;
    const int esz = (p.out_fp32 || split) ? 4 : 2;
    void* const dst = split ? static_cast<void*>(p.split_ws) : p.out;
    const uint64_t ldd = (split ? (uint64_t)p.N : (uint64_t)p.ldd) * esz, ldr = p.ldr * 2;
    const bool res = !split && p.residual != nullptr;
    p.tma_epilogue = (reinterpret_cast<uintptr_t>(dst) & 15) == 0 && ldd % 16 == 0 &&
                     (!res || (!p.out_fp32 && (reinterpret_cast<uintptr_t>(p.residual) & 15) == 0 && ldr % 16 == 0));
    if (p.tma_epilogue) {
        const uint64_t M = a->M, NE = (uint64_t)a->N * esz / 2, S = p.splits;
        if (a->a_mode == 0) {
            uint64_t dims[3] = {NE, M, S}, strides[2] = {ldd, M * ldd};
            uint32_t box[3] = {32, BLOCK_M, 1};
            CL_CHECK(get_tensor_map(&tD, dst, split ? 3 : 2, dims, strides, box, 64));
            if (res) {
                dims[0] = a->N;
                CL_CHECK(get_tensor_map(&tR, p.residual, 2, dims, &ldr, box, 64));
            }
        } else {
            const uint64_t Wo = p.Wo, Ho = p.Ho;
            uint64_t dims[5] = {NE, Wo, Ho, (uint64_t)p.n_img, S};
            uint32_t box[5] = {32, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn, 1};
            uint64_t strides[4] = {ldd, Wo * ldd, Ho * Wo * ldd, M * ldd};
            CL_CHECK(get_tensor_map(&tD, dst, split ? 5 : 4, dims, strides, box, 64));
            if (res) {
                dims[0] = a->N;
                uint64_t rs[3] = {ldr, Wo * ldr, Ho * Wo * ldr};
                CL_CHECK(get_tensor_map(&tR, p.residual, 4, dims, rs, box, 64));
            }
        }
    }

    const bool two = plan.occ == 2;
    int launch_plan[2] = {0, 0};   // resident CTAs per SM, store path
    int* const q = info != nullptr ? launch_plan : nullptr;
    const int st = dispatch_gemm(tA, tB, tE, tD, tR, p, stream, q, bn_sel, two, lora, BK);
    if (info != nullptr && st == CL_OK) {
        info[0] = bn_sel; info[1] = p.splits; info[2] = plan.occ; info[3] = launch_plan[0]; info[4] = launch_plan[1];
    }
    return st;
}

extern "C" int cl_gemm(const cl_gemm_args* a, void* stream) { return run_gemm(a, reinterpret_cast<cudaStream_t>(stream), nullptr); }

extern "C" int cl_gemm_plan(const cl_gemm_args* a, int32_t* info) {
    if (info == nullptr) return set_error(CL_ERR_INVALID, "cl_gemm_plan: null info");
    return run_gemm(a, nullptr, info);
}
