// K2 (forward) — fused scaled-dot-product attention for sm_90a (flash attention on wgmma).
//
//   O = softmax(Q K^T * scale) V,   per (batch, head);  Q/K/V/O are bf16 token matrices [B, N, H*d] (row stride ld*),
//   head h = columns [h*d, (h+1)*d).  The N x N probability matrix is never written to HBM (the reference
//   materialises it: attn.get_attention_scores + torch.bmm, models.py:140-141, 270-271, 407-408).
//
// One CTA = one (batch, head, 128-query block), three warpgroups:
//   warpgroup 0    TMA producer (one elected thread): Q once, then a two-stage mbarrier ring of K / V tiles of BN keys
//                  (4-D tensor maps {d, H, N, B}; the head dim is padded to a multiple of 64 by TMA zero fill, and
//                  S = Q K^T runs over ceil(d / 16) K16 steps only, and O += P V over ceil(d / 16) * 16 columns)
//   warpgroups 1-2 64 query rows each: S = Q K^T with wgmma from shared memory, online softmax in the exp2 domain on the
//                  accumulator registers (one row's statistics shared by the 4 lanes of a quad), O += P V with P as the
//                  register A operand and V read MN-major, O kept in registers.  The warpgroups take turns (named
//                  barriers 1 and 2) to issue S, so one warpgroup's softmax runs while the other's MMAs do.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "attention_tile.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

struct AttnFwdParams {
    int B, H, Nq, Nk, d;
    __nv_bfloat16* o; long long ldo;
    float* lse;
    float scale_log2;
    int num_q_blocks;
};

template <int D16>
struct AttnFwdCfg {
    static constexpr int DCH = head_chunks<D16>();
    static constexpr int BN = (DCH <= 2) ? 128 : 64;          // keys per stage (register budget of S + O)
    static constexpr int Q_BYTES = DCH * 128 * 128;
    static constexpr int KV_BYTES = DCH * BN * 128;
    static constexpr int STAGE_BYTES = 2 * KV_BYTES;
    static constexpr int STAGES = 2;
    static constexpr int SMEM_BYTES = 1024 + Q_BYTES + STAGES * STAGE_BYTES + 256;
};

template <int D16>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p) {
    pdl_launch_dependents();
    using Cfg = AttnFwdCfg<D16>;
    constexpr int BN = Cfg::BN, DCH = Cfg::DCH;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sq = smem;
    uint8_t* skv = sq + Cfg::Q_BYTES;
    uint64_t* q_bar = reinterpret_cast<uint64_t*>(skv + Cfg::STAGES * Cfg::STAGE_BYTES);
    uint64_t* full_bar = q_bar + 1;
    uint64_t* empty_bar = full_bar + Cfg::STAGES;
    const int warp_idx = uniform_warp_idx(), lane = threadIdx.x & 31;
    const int wg = warp_idx >> 2;
    int bid = blockIdx.x;
    const int qb = bid % p.num_q_blocks; bid /= p.num_q_blocks;
    const int h = bid % p.H, b = bid / p.H;
    const int q0 = qb * 128;
    const int nkb = (p.Nk + BN - 1) / BN;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
        mbar_init(q_bar, 1);
        for (int i = 0; i < Cfg::STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();   // everything above touched only shared memory and kernel parameters

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (warp_idx == 0 && elect_one_sync()) {
            mbar_arrive_expect_tx(q_bar, Cfg::Q_BYTES);
            load_head_tile<DCH, 128>(&tmQ, q_bar, sq, h, q0, b);
            int stage = 0; uint32_t phase = 0;
            for (int j = 0; j < nkb; ++j) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                uint8_t* st = skv + stage * Cfg::STAGE_BYTES;
                load_head_tile<DCH, BN>(&tmK, &full_bar[stage], st, h, j * BN, b);
                load_head_tile<DCH, BN>(&tmV, &full_bar[stage], st + Cfg::KV_BYTES, h, j * BN, b);
                if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }

    setmaxnreg_inc<232>();
    const int row0 = (wg - 1) * 64, w4 = warp_idx & 3;
    // Ping-pong: the two warpgroups take turns to issue S = Q K^T, so that one warpgroup's softmax runs while the other's
    // MMAs do.  Named barrier wg (1 or 2) opens this warpgroup's turn: it completes with this warpgroup's sync and the other
    // warpgroup's arrive at the end of its own turn.
    const int bar_me = wg, bar_other = 3 - wg;
    float o[DCH][32];
#pragma unroll
    for (int c = 0; c < DCH; ++c)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    if (wg == 2) named_bar_arrive(1, 256);                   // warpgroup 1 takes the first turn
    mbar_wait(q_bar, 0);
    const uint32_t q_addr = smem_u32(sq);
    const bool ragged = (p.Nk % BN) != 0;
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < nkb; ++j) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t k_addr = smem_u32(skv + stage * Cfg::STAGE_BYTES), v_addr = k_addr + Cfg::KV_BYTES;
        float s[BN / 2];
        // this warpgroup's turn to issue S (see above)
        named_bar_sync(bar_me, 256);
        wgmma_fence();
        att_abt_issue<D16, 128, BN>(s, q_addr, row0, k_addr);
        named_bar_arrive(bar_other, 256);
        wgmma_wait<0>();
        wgmma_fence_acc(s);
        // scaled scores in the log2 domain; s[nt*4 + c]: row lane/4 + 8(c/2), key 8nt + 2(lane%4) + c%2.  Keys beyond Nk
        // occur in the last tile only and are masked there.
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) s[i] *= p.scale_log2;
        if (ragged && j == nkb - 1) {
#pragma unroll
            for (int nt = 0; nt < BN / 8; ++nt)
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (j * BN + nt * 8 + 2 * (lane & 3) + (c & 1) >= p.Nk) s[nt * 4 + c] = -INFINITY;
        }
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
        float corr[2], m_use[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
            mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
            const float m_new = fmaxf(m_run[i], mx[i]);
            m_use[i] = (m_new == -INFINITY) ? 0.f : m_new;
            corr[i] = fast_exp2(m_run[i] - m_use[i]);
            m_run[i] = m_new;
            l_run[i] *= corr[i];
        }
#pragma unroll
        for (int nt = 0; nt < BN / 8; ++nt)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                s[nt * 4 + c] = fast_exp2(s[nt * 4 + c] - m_use[c >> 1]);
                l_run[c >> 1] += s[nt * 4 + c];
            }
        uint32_t pa[BN / 16][4];
        acc_to_a<BN / 8>(s, pa);
#pragma unroll
        for (int c = 0; c < DCH; ++c)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                o[c][jj * 4] *= corr[0]; o[c][jj * 4 + 1] *= corr[0];
                o[c][jj * 4 + 2] *= corr[1]; o[c][jj * 4 + 3] *= corr[1];
            }
        att_pv<DCH, head_last_n<D16>(), BN, BN / 16>(o, pa, v_addr, 0);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
    }
    if (wg == 1) named_bar_sync(1, 256);                     // the sync that matches warpgroup 2's last arrive
    // epilogue: O / l, bf16 store, log2-domain LSE
    float inv[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 1);
        l_run[i] += __shfl_xor_sync(0xffffffffu, l_run[i], 2);
        inv[i] = 1.f / l_run[i];
        const int qrow = q0 + row0 + w4 * 16 + (lane >> 2) + 8 * i;
        if (qrow < p.Nq && p.lse != nullptr && (lane & 3) == 0) p.lse[((long long)b * p.H + h) * p.Nq + qrow] = m_run[i] + log2f(l_run[i]);
    }
#pragma unroll
    for (int c = 0; c < DCH; ++c)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            o[c][jj * 4] *= inv[0]; o[c][jj * 4 + 1] *= inv[0];
            o[c][jj * 4 + 2] *= inv[1]; o[c][jj * 4 + 3] *= inv[1];
        }
    store_rows<DCH>(o, 1.f, p.o + (long long)b * p.Nq * p.ldo + h * p.d, p.ldo, q0 + row0, p.Nq, p.d, 0, lane, w4);
}

template <int D16>
static int launch_attn_fwd(const cl_attn_fwd_args* a, cudaStream_t stream) {
    using Cfg = AttnFwdCfg<D16>;
    CUtensorMap tq, tk, tv;
    CL_CHECK(make_head_map(&tq, a->q, a->B, a->H, a->Nq, a->d, a->ldq, 128));
    CL_CHECK(make_head_map(&tk, a->k, a->B, a->H, a->Nk, a->d, a->ldk, Cfg::BN));
    CL_CHECK(make_head_map(&tv, a->v, a->B, a->H, a->Nk, a->d, a->ldv, Cfg::BN));
    AttnFwdParams p;
    p.B = a->B; p.H = a->H; p.Nq = a->Nq; p.Nk = a->Nk; p.d = a->d;
    p.o = reinterpret_cast<__nv_bfloat16*>(a->o); p.ldo = a->ldo; p.lse = a->lse;
    p.scale_log2 = a->scale * 1.4426950408889634f;
    p.num_q_blocks = (a->Nq + 127) / 128;
    static bool attr_done = false;
    if (!attr_done) {
        CL_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_wgmma_kernel<D16>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        attr_done = true;
    }
    const long long grid = (long long)a->B * a->H * p.num_q_blocks;
    if (grid > 0x7fffffffLL) return set_error(CL_ERR_UNSUPPORTED, "cl_attn_fwd: too many blocks");
    launch_k(attn_fwd_wgmma_kernel<D16>, (unsigned)grid, ATT_THREADS, Cfg::SMEM_BYTES, stream, tq, tk, tv, p);
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

}  // namespace clb

using namespace clb;

extern "C" int cl_attn_fwd(const cl_attn_fwd_args* a, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!a || !a->q || !a->k || !a->v || !a->o) return set_error(CL_ERR_INVALID, "cl_attn_fwd: null pointer");
    if (a->d % 8 != 0 || a->d <= 0 || a->d > 192) return set_error(CL_ERR_UNSUPPORTED, "cl_attn_fwd: head dim must be a multiple of 8, <= 192");
    if ((a->ldq % 8) || (a->ldk % 8) || (a->ldv % 8) || (a->ldo % 8)) return set_error(CL_ERR_INVALID, "cl_attn_fwd: row strides must be multiples of 8");
    if (a->B <= 0 || a->H <= 0 || a->Nq <= 0 || a->Nk <= 0) return set_error(CL_ERR_INVALID, "cl_attn_fwd: dims");
    return with_head_d16(a->d, [&](auto d16) { return launch_attn_fwd<decltype(d16)::value>(a, stream); });
}
