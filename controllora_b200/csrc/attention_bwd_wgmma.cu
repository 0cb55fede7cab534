// K2 (backward) — flash-attention backward for sm_90a on wgmma, what torch autograd derives for the reference's baddbmm /
// softmax / bmm (models.py:140-141, 270-271, 407-408).  P is recomputed from Q, K and the forward's log2-domain LSE;
// delta = rowsum(dO * O) comes from a small kernel first.  Both kernels use three warpgroups: a TMA producer (one elected
// thread: the CTA's own tiles once, then a three-stage mbarrier ring of the streamed tiles; in the dKV kernel a second
// warp stages each streamed query tile's lse and delta into the same ring) and two consumer warpgroups of
// 64 rows each, whose products run on wgmma with the accumulators in registers and P / dS fed back as register A operands.
//
//   dKV kernel: one CTA = 128 keys of one (batch, head); it streams Q / dO tiles of 64 queries (32 for heads wider than 64):
//               S^T = K Q^T -> P^T,  dV += P^T dO,  dP^T = V dO^T,  dS^T = P^T (dP^T - delta),  dK += dS^T Q
//               (heads wider than 128 split the dK / dV columns over two CTAs to bound the accumulator registers)
//   dQ kernel:  one CTA = 128 queries; it streams K / V tiles of 64 keys (32 for heads wider than 64):
//               S = Q K^T -> P,  dP = dO V^T,  dS = P (dP - delta),  dQ += dS K
// Per streamed tile a consumer issues S and dP back to back as two commit groups and waits for S only; P is computed while
// dP runs, and the gradient products (dV / dK, or dQ) stay in flight until after the next tile's S and dP are issued.  A
// ring stage is released once every product that reads it has retired.  The MMAs are sized to the head dim (D16 =
// ceil(d / 16), attention_tile.cuh).
// No atomics: every output element is written by exactly one thread.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "attention_tile.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

struct AttnBwdParams {
    int B, H, Nq, Nk, d;
    const float* lse;
    const float* delta;
    __nv_bfloat16* dq; long long lddq;
    __nv_bfloat16* dk; long long lddk;
    __nv_bfloat16* dv; long long lddv;
    float scale, scale_log2;
    int num_blocks;
};

template <int D16>
struct BwdCfg {
    static constexpr int DCH = head_chunks<D16>();
    static constexpr int BI = (DCH == 1) ? 64 : 32;        // streamed rows per stage (queries for dKV, keys for dQ): register budget
    static constexpr int OUTC = DCH < 2 ? DCH : 2;         // dK / dV column chunks per dKV CTA
    static constexpr int FIX_BYTES = DCH * 128 * 128;      // one of the CTA's own 128-row tiles
    static constexpr int IN_BYTES = DCH * BI * 128;        // one streamed tile
    static constexpr int STAGE_BYTES = 2 * IN_BYTES;
    static constexpr int STAGES = 3;                       // a stage stays busy until the next tile's S has retired
    static constexpr int STAT_BYTES = 2 * BI * 4;          // dKV: lse and delta of a streamed tile's queries, per stage
    static constexpr int SMEM_BYTES = 1024 + 2 * FIX_BYTES + STAGES * (STAGE_BYTES + STAT_BYTES) + 256;
};

// the shared producer: fixed tiles f0 / f1 (128 rows from frow0) once, then n tiles of BI rows of s0 / s1 through the ring
// (one elected thread of warp 0)
template <int D16>
__device__ __forceinline__ void bwd_produce(const CUtensorMap* f0, const CUtensorMap* f1, int frow0, const CUtensorMap* s0,
                                            const CUtensorMap* s1, int n, uint8_t* sfix, uint8_t* sin, uint64_t* fix_bar,
                                            uint64_t* full_bar, uint64_t* empty_bar, int h, int b) {
    using Cfg = BwdCfg<D16>;
    constexpr int DCH = Cfg::DCH;
    mbar_arrive_expect_tx(fix_bar, 2 * Cfg::FIX_BYTES);
    load_head_tile<DCH, 128>(f0, fix_bar, sfix, h, frow0, b);
    load_head_tile<DCH, 128>(f1, fix_bar, sfix + Cfg::FIX_BYTES, h, frow0, b);
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < n; ++j) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
        uint8_t* st = sin + stage * Cfg::STAGE_BYTES;
        load_head_tile<DCH, Cfg::BI>(s0, &full_bar[stage], st, h, j * Cfg::BI, b);
        load_head_tile<DCH, Cfg::BI>(s1, &full_bar[stage], st + Cfg::IN_BYTES, h, j * Cfg::BI, b);
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    }
}

// dKV: warp 1 of the producer warpgroup stages lse and delta of every streamed query tile into the ring (sstat, BI of
// each per stage), with padding queries (>= Nq) set to lse = +inf (so P = 0) and delta = 0.  Each lane arrives on full_bar
// after its stores.
template <int D16>
__device__ __forceinline__ void bwd_produce_stats(const AttnBwdParams& p, int n, float* sstat, uint64_t* full_bar,
                                                  uint64_t* empty_bar, int h, int b, int lane) {
    using Cfg = BwdCfg<D16>;
    constexpr int BI = Cfg::BI;
    const float* glse = p.lse + ((long long)b * p.H + h) * p.Nq;
    const float* gdelta = p.delta + ((long long)b * p.H + h) * p.Nq;
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < n; ++j) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        float* st = sstat + stage * (2 * BI);
#pragma unroll 1
        for (int i = lane; i < BI; i += 32) {
            const int qq = j * BI + i;
            st[i] = (qq < p.Nq) ? __ldg(glse + qq) : INFINITY;
            st[BI + i] = (qq < p.Nq) ? __ldg(gdelta + qq) : 0.f;
        }
        mbar_arrive(&full_bar[stage]);
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    }
}

// FULL_COUNT: arrivals that complete a ring stage besides the TMA bytes (the TMA thread, plus 32 lanes staging lse / delta)
#define BWD_PROLOGUE(FULL_COUNT)                                                                                         \
    extern __shared__ __align__(1024) uint8_t smem_raw[];                                                                \
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));      \
    uint8_t* sfix = smem;                                                                                                \
    uint8_t* sin = sfix + 2 * Cfg::FIX_BYTES;                                                                            \
    float* sstat = reinterpret_cast<float*>(sin + Cfg::STAGES * Cfg::STAGE_BYTES);                                       \
    uint64_t* fix_bar = reinterpret_cast<uint64_t*>(sstat + Cfg::STAGES * 2 * Cfg::BI);                                  \
    uint64_t* full_bar = fix_bar + 1;                                                                                    \
    uint64_t* empty_bar = full_bar + Cfg::STAGES;                                                                        \
    const int warp_idx = uniform_warp_idx(), lane = threadIdx.x & 31;                                                    \
    const int wg = warp_idx >> 2;                                                                                        \
    if (threadIdx.x == 0) {                                                                                              \
        mbar_init(fix_bar, 1);                                                                                           \
        for (int i = 0; i < Cfg::STAGES; ++i) { mbar_init(&full_bar[i], FULL_COUNT); mbar_init(&empty_bar[i], 2); }     \
        fence_barrier_init();                                                                                            \
    }                                                                                                                    \
    __syncthreads();                                                                                                     \
    pdl_wait();

// one dKV consumer warpgroup (keys row0 .. row0 + 63 of the CTA's 128) for output chunks [C0, C0 + NC), the last NL wide
template <int D16, int C0, int NC, int NL>
__device__ __forceinline__ void dkv_consume(const AttnBwdParams& p, uint8_t* sfix, uint8_t* sin, const float* sstat,
                                            uint64_t* fix_bar, uint64_t* full_bar, uint64_t* empty_bar, int h, int b, int k0,
                                            int nqb, int row0, int lane, int w4) {
    using Cfg = BwdCfg<D16>;
    constexpr int BI = Cfg::BI, ACC = 32 * (NC - 1) + NL / 2;   // accumulator registers per thread of dK (and of dV)
    float dk[NC][32], dv[NC][32];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) dk[c][i] = dv[c][i] = 0.f;
    uint32_t pa[BI / 16][4], dsa[BI / 16][4];                   // P^T / dS^T operands of the dV / dK products in flight
    mbar_wait(fix_bar, 0);
    const uint32_t k_addr = smem_u32(sfix), v_addr = k_addr + Cfg::FIX_BYTES;
    int stage = 0, prev = 0; uint32_t phase = 0;
    int j = 0;
    do {   // nqb >= 1: a path that skips the loop would redefine dk / dv before the final wait, and ptxas serialises (C7515)
        mbar_wait(&full_bar[stage], phase);
        const uint32_t q_addr = smem_u32(sin + stage * Cfg::STAGE_BYTES), do_addr = q_addr + Cfg::IN_BYTES;
        float s[BI / 2], dp[BI / 2];
        wgmma_fence();
        att_abt_issue<D16, 128, BI>(s, k_addr, row0, q_addr);     // S^T[64 keys][BI queries]
        att_abt_issue<D16, 128, BI>(dp, v_addr, row0, do_addr);   // dP^T = V dO^T
        // this lane's query columns 8nt + 2(lane%4) + {0,1} of the tile's lse and delta, as float2 pairs
        const uint32_t stat_addr = smem_u32(sstat + stage * (2 * BI)) + 8 * (lane & 3);
        wgmma_wait<1>();                                          // S^T, and the previous tile's dK, have retired
        wgmma_fence_acc(s);
        if (j > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
#pragma unroll
        for (int nt = 0; nt < BI / 8; ++nt) {
            const float2 l2 = ld_shared_f2(stat_addr + nt * 32);
#pragma unroll
            for (int c = 0; c < 4; ++c) s[nt * 4 + c] = fast_exp2(s[nt * 4 + c] * p.scale_log2 - ((c & 1) ? l2.y : l2.x));
        }
        acc_to_a<BI / 8>(s, pa);
        att_pv_issue<NC, NL, BI, BI / 16>(dv, pa, do_addr, C0);  // dV += P^T dO
        wgmma_wait<1>();                                          // dP^T has retired
        wgmma_fence_acc(dp);
#pragma unroll
        for (int nt = 0; nt < BI / 8; ++nt) {
            const float2 d2 = ld_shared_f2(stat_addr + BI * 4 + nt * 32);
#pragma unroll
            for (int c = 0; c < 4; ++c) dp[nt * 4 + c] = s[nt * 4 + c] * (dp[nt * 4 + c] - ((c & 1) ? d2.y : d2.x));
        }
        acc_to_a<BI / 8>(dp, dsa);
        att_pv_issue<NC, NL, BI, BI / 16>(dk, dsa, q_addr, C0);  // dK += dS^T Q
        // dV retires.  dK stays in flight into the next tile where its accumulators are small enough (ptxas -v: with
        // both in flight, or with dK at 32 x 64-row columns per 64-query tile or more, the MMAs serialise (C7512) or spill)
        if (ACC * BI <= 48 * 32) wgmma_wait<1>();
        else wgmma_wait<0>();
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    } while (++j < nqb);
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NC; ++c) { wgmma_fence_acc(dk[c]); wgmma_fence_acc(dv[c]); }
    store_rows<NC>(dk, p.scale, p.dk + (long long)b * p.Nk * p.lddk + h * p.d, p.lddk, k0 + row0, p.Nk, p.d, C0, lane, w4);
    store_rows<NC>(dv, 1.f, p.dv + (long long)b * p.Nk * p.lddv + h * p.d, p.lddv, k0 + row0, p.Nk, p.d, C0, lane, w4);
}

template <int D16>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO, const AttnBwdParams p) {
    pdl_launch_dependents();
    using Cfg = BwdCfg<D16>;
    constexpr int DCH = Cfg::DCH, BI = Cfg::BI;
    BWD_PROLOGUE(33)
    int bid = blockIdx.x;
    const int kb = bid % p.num_blocks; bid /= p.num_blocks;
    const int h = bid % p.H, b = bid / p.H;
    const int k0 = kb * 128;
    const int nqb = (p.Nq + BI - 1) / BI;
    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (warp_idx == 0 && elect_one_sync())
            bwd_produce<D16>(&tmK, &tmV, k0, &tmQ, &tmDO, nqb, sfix, sin, fix_bar, full_bar, empty_bar, h, b);
        else if (warp_idx == 1)
            bwd_produce_stats<D16>(p, nqb, sstat, full_bar, empty_bar, h, b, lane);
        return;
    }
    setmaxnreg_inc<232>();
    const int row0 = (wg - 1) * 64, w4 = warp_idx & 3;
    // the column split is per CTA and uniform, so each side is its own fully unrolled instance
    if (DCH <= 2)
        dkv_consume<D16, 0, DCH, head_last_n<D16>()>(p, sfix, sin, sstat, fix_bar, full_bar, empty_bar, h, b, k0, nqb, row0, lane, w4);
    else if (blockIdx.y == 0)
        dkv_consume<D16, 0, 2, 64>(p, sfix, sin, sstat, fix_bar, full_bar, empty_bar, h, b, k0, nqb, row0, lane, w4);
    else
        dkv_consume<D16, 2, 1, head_last_n<D16>()>(p, sfix, sin, sstat, fix_bar, full_bar, empty_bar, h, b, k0, nqb, row0, lane, w4);
}

template <int D16>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO, const AttnBwdParams p) {
    pdl_launch_dependents();
    using Cfg = BwdCfg<D16>;
    constexpr int BI = Cfg::BI, DCH = Cfg::DCH;
    BWD_PROLOGUE(1)
    int bid = blockIdx.x;
    const int qb = bid % p.num_blocks; bid /= p.num_blocks;
    const int h = bid % p.H, b = bid / p.H;
    const int q0 = qb * 128;
    const int nkb = (p.Nk + BI - 1) / BI;
    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (warp_idx == 0 && elect_one_sync())
            bwd_produce<D16>(&tmQ, &tmDO, q0, &tmK, &tmV, nkb, sfix, sin, fix_bar, full_bar, empty_bar, h, b);
        return;
    }
    setmaxnreg_inc<232>();
    const int row0 = (wg - 1) * 64, w4 = warp_idx & 3;
    float lse[2], delta[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int qq = q0 + row0 + w4 * 16 + (lane >> 2) + 8 * i;
        const long long si = ((long long)b * p.H + h) * p.Nq + qq;
        lse[i] = (qq < p.Nq) ? p.lse[si] : INFINITY;
        delta[i] = (qq < p.Nq) ? p.delta[si] : 0.f;
    }
    float dq[DCH][32];
#pragma unroll
    for (int c = 0; c < DCH; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) dq[c][i] = 0.f;
    uint32_t dsa[BI / 16][4];                                     // dS operand of the dQ product in flight
    const bool ragged = (p.Nk % BI) != 0;
    mbar_wait(fix_bar, 0);
    const uint32_t q_addr = smem_u32(sfix), do_addr = q_addr + Cfg::FIX_BYTES;
    int stage = 0, prev = 0; uint32_t phase = 0;
    int j = 0;
    do {   // nkb >= 1 (see dkv_consume)
        mbar_wait(&full_bar[stage], phase);
        const uint32_t k_addr = smem_u32(sin + stage * Cfg::STAGE_BYTES), v_addr = k_addr + Cfg::IN_BYTES;
        float s[BI / 2], dp[BI / 2];
        wgmma_fence();
        att_abt_issue<D16, 128, BI>(s, q_addr, row0, k_addr);     // S[64 queries][BI keys]
        att_abt_issue<D16, 128, BI>(dp, do_addr, row0, v_addr);   // dP = dO V^T
        wgmma_wait<1>();                                          // S, and the previous tile's dQ, have retired
        wgmma_fence_acc(s);
        if (j > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
#pragma unroll
        for (int i = 0; i < BI / 2; ++i) s[i] = fast_exp2(s[i] * p.scale_log2 - lse[(i >> 1) & 1]);
        if (ragged && j == nkb - 1) {                             // keys beyond Nk occur in the last tile only
#pragma unroll
            for (int nt = 0; nt < BI / 8; ++nt)
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (j * BI + nt * 8 + 2 * (lane & 3) + (c & 1) >= p.Nk) s[nt * 4 + c] = 0.f;
        }
        wgmma_wait<0>();                                          // dP has retired
        wgmma_fence_acc(dp);
#pragma unroll
        for (int nt = 0; nt < BI / 8; ++nt)
#pragma unroll
            for (int c = 0; c < 4; ++c) dp[nt * 4 + c] = s[nt * 4 + c] * (dp[nt * 4 + c] - delta[c >> 1]);
        acc_to_a<BI / 8>(dp, dsa);
        att_pv_issue<DCH, head_last_n<D16>(), BI, BI / 16>(dq, dsa, k_addr, 0);   // dQ += dS K
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    } while (++j < nkb);
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < DCH; ++c) wgmma_fence_acc(dq[c]);
    store_rows<DCH>(dq, p.scale, p.dq + (long long)b * p.Nq * p.lddq + h * p.d, p.lddq, q0 + row0, p.Nq, p.d, 0, lane, w4);
}

// ===================================================================================================== delta
// delta[b, h, q] = sum_d dO[b, q, h*d + :] * O[b, q, h*d + :]
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ o, long long ldo, const __nv_bfloat16* __restrict__ d_o,
                                  long long lddo, float* __restrict__ delta, int B, int H, int Nq, int d) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)B * Nq * H;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int h = (int)(i % H);
        const long long bq = i / H;
        const int q = (int)(bq % Nq);
        const int b = (int)(bq / Nq);
        const __nv_bfloat16* po = o + bq * ldo + h * d;
        const __nv_bfloat16* pd = d_o + bq * lddo + h * d;
        float s = 0.f;
        for (int c = 0; c < d; c += 8) {
            const uint4 a = *reinterpret_cast<const uint4*>(po + c);
            const uint4 g = *reinterpret_cast<const uint4*>(pd + c);
            const float2 a0 = unpack_bf16x2(a.x), a1 = unpack_bf16x2(a.y), a2 = unpack_bf16x2(a.z), a3 = unpack_bf16x2(a.w);
            const float2 g0 = unpack_bf16x2(g.x), g1 = unpack_bf16x2(g.y), g2 = unpack_bf16x2(g.z), g3 = unpack_bf16x2(g.w);
            s += a0.x * g0.x + a0.y * g0.y + a1.x * g1.x + a1.y * g1.y + a2.x * g2.x + a2.y * g2.y + a3.x * g3.x + a3.y * g3.y;
        }
        delta[((long long)b * H + h) * Nq + q] = s;
    }
}

template <int D16>
static int launch_attn_bwd(const cl_attn_bwd_args* a, cudaStream_t stream) {
    using Cfg = BwdCfg<D16>;
    constexpr int DCH = Cfg::DCH;
    AttnBwdParams p;
    p.B = a->B; p.H = a->H; p.Nq = a->Nq; p.Nk = a->Nk; p.d = a->d;
    p.lse = a->lse; p.delta = a->delta;
    p.dq = reinterpret_cast<__nv_bfloat16*>(a->dq); p.lddq = a->lddq;
    p.dk = reinterpret_cast<__nv_bfloat16*>(a->dk); p.lddk = a->lddk;
    p.dv = reinterpret_cast<__nv_bfloat16*>(a->dv); p.lddv = a->lddv;
    p.scale = a->scale; p.scale_log2 = a->scale * 1.4426950408889634f;
    {
        const long long total = (long long)a->B * a->Nq * a->H;
        int blocks = (int)((total + 255) / 256);
        if (blocks > num_sms() * 8) blocks = num_sms() * 8;
        launch_k(attn_delta_kernel, blocks, 256, 0, stream, reinterpret_cast<const __nv_bfloat16*>(a->o), a->ldo,
                                                      reinterpret_cast<const __nv_bfloat16*>(a->d_o), a->lddo, a->delta,
                                                      a->B, a->H, a->Nq, a->d);
        count_launch();
    }
    static bool attr_done = false;
    if (!attr_done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dkv_kernel<D16>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        CL_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dq_kernel<D16>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        attr_done = true;
    }
    if (a->dk != nullptr) {
        CUtensorMap tq, tk, tv, tdo;
        CL_CHECK(make_head_map(&tq, a->q, a->B, a->H, a->Nq, a->d, a->ldq, Cfg::BI));
        CL_CHECK(make_head_map(&tdo, a->d_o, a->B, a->H, a->Nq, a->d, a->lddo, Cfg::BI));
        CL_CHECK(make_head_map(&tk, a->k, a->B, a->H, a->Nk, a->d, a->ldk, 128));
        CL_CHECK(make_head_map(&tv, a->v, a->B, a->H, a->Nk, a->d, a->ldv, 128));
        p.num_blocks = (a->Nk + 127) / 128;
        const long long grid = (long long)a->B * a->H * p.num_blocks;
        if (grid > 0x7fffffffLL) return set_error(CL_ERR_UNSUPPORTED, "cl_attn_bwd: too many blocks");
        launch_k(attn_bwd_dkv_kernel<D16>, dim3((unsigned)grid, (DCH + Cfg::OUTC - 1) / Cfg::OUTC), ATT_THREADS, Cfg::SMEM_BYTES,
                 stream, tq, tk, tv, tdo, p);
        count_launch();
    }
    if (a->dq != nullptr) {
        CUtensorMap tq, tk, tv, tdo;
        CL_CHECK(make_head_map(&tq, a->q, a->B, a->H, a->Nq, a->d, a->ldq, 128));
        CL_CHECK(make_head_map(&tdo, a->d_o, a->B, a->H, a->Nq, a->d, a->lddo, 128));
        CL_CHECK(make_head_map(&tk, a->k, a->B, a->H, a->Nk, a->d, a->ldk, Cfg::BI));
        CL_CHECK(make_head_map(&tv, a->v, a->B, a->H, a->Nk, a->d, a->ldv, Cfg::BI));
        p.num_blocks = (a->Nq + 127) / 128;
        const long long grid = (long long)a->B * a->H * p.num_blocks;
        if (grid > 0x7fffffffLL) return set_error(CL_ERR_UNSUPPORTED, "cl_attn_bwd: too many blocks");
        launch_k(attn_bwd_dq_kernel<D16>, (unsigned)grid, ATT_THREADS, Cfg::SMEM_BYTES, stream, tq, tk, tv, tdo, p);
        count_launch();
    }
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

}  // namespace clb

using namespace clb;

extern "C" int cl_attn_bwd(const cl_attn_bwd_args* a, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || !a->q || !a->k || !a->v || !a->o || !a->d_o || !a->lse || !a->delta)
        return set_error(CL_ERR_INVALID, "cl_attn_bwd: null pointer");
    if ((a->dk == nullptr) != (a->dv == nullptr)) return set_error(CL_ERR_INVALID, "cl_attn_bwd: dk and dv go together");
    if (a->d % 8 != 0 || a->d <= 0 || a->d > 192) return set_error(CL_ERR_UNSUPPORTED, "cl_attn_bwd: head dim must be a multiple of 8, <= 192");
    if ((a->ldq % 8) || (a->ldk % 8) || (a->ldv % 8) || (a->ldo % 8) || (a->lddo % 8) || (a->dq && a->lddq % 8) ||
        (a->dk && ((a->lddk % 8) || (a->lddv % 8))))
        return set_error(CL_ERR_INVALID, "cl_attn_bwd: row strides must be multiples of 8");
    if (a->B <= 0 || a->H <= 0 || a->Nq <= 0 || a->Nk <= 0) return set_error(CL_ERR_INVALID, "cl_attn_bwd: dims");
    return with_head_d16(a->d, [&](auto d16) { return launch_attn_bwd<decltype(d16)::value>(a, stream); });
}
