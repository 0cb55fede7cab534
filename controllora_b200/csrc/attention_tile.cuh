// Building blocks of the sm_90a attention kernels: TMA loads of head-slice tiles into 128B-swizzled shared memory, the
// wgmma descriptors over them, and the two warpgroup products every kernel is made of.
//
// A tile of R rows of one (batch, head) slice is stored as DCH chunks of 64 head-dim columns, each chunk R rows x 128 bytes
// (what a TMA box {64, 1, R, 1} with the 128B swizzle writes); columns beyond d and rows beyond N arrive as zeros.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"
#include "host_common.h"

namespace clb {

static constexpr int ATT_THREADS = 384;   // producer warpgroup + two consumer warpgroups of 64 rows each

// tensor map of the head slices of a [B, N, H*d] token matrix (row stride ld elements): dims {d, H, N, B}, box {64, 1, rows, 1}
static inline int make_head_map(CUtensorMap* tm, const void* ptr, int B, int H, int N, int d, long long ld, int box_rows) {
    uint64_t dims[4] = {(uint64_t)d, (uint64_t)H, (uint64_t)N, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)d * 2, (uint64_t)ld * 2, (uint64_t)N * ld * 2};
    uint32_t box[4] = {64, 1, (uint32_t)box_rows, 1};
    return get_tensor_map(tm, ptr, 4, dims, strides, box, 128);
}

// rows [r0, r0 + ROWS) of head (h, b) -> DCH chunks at dst, completion counted on `bar` (DCH * ROWS * 128 bytes)
template <int DCH, int ROWS>
__device__ __forceinline__ void load_head_tile(const CUtensorMap* m, uint64_t* bar, uint8_t* dst, int h, int r0, int b) {
#pragma unroll
    for (int c = 0; c < DCH; ++c) tma_load_4d(m, bar, dst + c * ROWS * 128, c * 64, h, r0, b);
}

// Head dims are handled in 16-column units: D16 = ceil(d / 16).  A tile keeps DCH = ceil(D16 / 4) chunks of 64 columns, and
// the MMAs cover only the D16 * 16 columns that hold data: the last chunk is head_last_n<D16>() columns wide.  Columns from
// d up to D16 * 16 are TMA zero fill and contribute exact zeros.  D16 is a template parameter because a run-time guard or
// width switch around a wgmma makes ptxas serialise the warpgroup (C7519, an injected warpgroup.arrive).
template <int D16> constexpr int head_chunks() { return (D16 + 3) / 4; }
template <int D16> constexpr int head_last_n() { return 16 * (D16 - 4 * (head_chunks<D16>() - 1)); }

// calls f(std::integral_constant<int, D16>) for the head dim d (1 <= d <= 192)
template <class F>
static inline int with_head_d16(int d, F&& f) {
    switch ((d + 15) / 16) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    case 3: return f(std::integral_constant<int, 3>());
    case 4: return f(std::integral_constant<int, 4>());
    case 5: return f(std::integral_constant<int, 5>());
    case 6: return f(std::integral_constant<int, 6>());
    case 7: return f(std::integral_constant<int, 7>());
    case 8: return f(std::integral_constant<int, 8>());
    case 9: return f(std::integral_constant<int, 9>());
    case 10: return f(std::integral_constant<int, 10>());
    case 11: return f(std::integral_constant<int, 11>());
    default: return f(std::integral_constant<int, 12>());
    }
}

// K-major operand (rows = M or N, the head dim is K): 64 rows from `row0` of a ROWS-row tile, K16 step k16 of D16
template <int ROWS>
__device__ __forceinline__ uint64_t desc_kmaj(uint32_t base, int row0, int k16) {
    return make_smem_desc(base + (k16 >> 2) * ROWS * 128 + row0 * 128 + (k16 & 3) * 32, 16, 1024, SWZ_128B);
}
// MN-major operand (rows = K, the head dim is N): rows [k0, k0 + 16) of a ROWS-row tile, head-dim chunk c (64 columns)
template <int ROWS>
__device__ __forceinline__ uint64_t desc_mnmaj(uint32_t base, int c, int k0) {
    return make_smem_desc(base + c * ROWS * 128 + k0 * 128, ROWS * 128, 1024, SWZ_128B);
}

// issue (one commit group, no wait) s[64 x N] = A B^T over the D16 * 16 head-dim columns: A = 64 rows from a_row0 of an
// AR-row tile, B = the N rows of a tile.  The caller fences before and waits after.
template <int D16, int AR, int N>
__device__ __forceinline__ void att_abt_issue(float (&s)[N / 2], uint32_t a_base, int a_row0, uint32_t b_base) {
    Wgmma<N, 0, 0>::mma_zero(s, desc_kmaj<AR>(a_base, a_row0, 0), desc_kmaj<N>(b_base, 0, 0));
#pragma unroll
    for (int k16 = 1; k16 < D16; ++k16) Wgmma<N, 0, 0>::mma(s, desc_kmaj<AR>(a_base, a_row0, k16), desc_kmaj<N>(b_base, 0, k16), 1);
    wgmma_commit();
}

// issue (fence, one commit group, no wait) o[oc] += P V[:, chunk c0 + oc] for NC output chunks, the last one NL columns
// wide: P = KC*16 columns of bf16 A fragments in registers (k = rows of the VR-row tile v), v read MN-major.  pa and o
// must not be touched until the group has retired.
template <int NC, int NL, int VR, int KC>
__device__ __forceinline__ void att_pv_issue(float (&o)[NC][32], const uint32_t (&pa)[KC][4], uint32_t v_base, int c0) {
    wgmma_fence();
#pragma unroll
    for (int oc = 0; oc < NC; ++oc) {
#pragma unroll
        for (int kc = 0; kc < KC; ++kc) {
            const uint64_t db = desc_mnmaj<VR>(v_base, c0 + oc, kc * 16);
            if (oc < NC - 1) WgmmaRs<64, 1>::mma(o[oc], pa[kc], db, 1);
            else WgmmaRs<NL, 1>::mma(o[oc], pa[kc], db, 1);
        }
    }
    wgmma_commit();
}

template <int NC, int NL, int VR, int KC>
__device__ __forceinline__ void att_pv(float (&o)[NC][32], const uint32_t (&pa)[KC][4], uint32_t v_base, int c0) {
    att_pv_issue<NC, NL, VR, KC>(o, pa, v_base, c0);
    wgmma_wait<0>();
#pragma unroll
    for (int oc = 0; oc < NC; ++oc) wgmma_fence_acc(o[oc]);
}

__device__ __forceinline__ float2 ld_shared_f2(uint32_t addr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
    return v;
}

// bf16 A fragments (K16 chunks) of a 64 x (NT*8) accumulator block: accumulator column block nt holds k = 8nt .. 8nt + 7
template <int NT>
__device__ __forceinline__ void acc_to_a(const float (&s)[NT * 4], uint32_t (&a)[NT / 2][4]) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        a[nt >> 1][(nt & 1) * 2] = pack_bf16x2(s[nt * 4], s[nt * 4 + 1]);
        a[nt >> 1][(nt & 1) * 2 + 1] = pack_bf16x2(s[nt * 4 + 2], s[nt * 4 + 3]);
    }
}

// bf16 store of output chunks [c0, c0 + NC) of 64-row accumulator blocks: rows row0 + w*16 + lane/4 (+8), scaled by mul
template <int NC>
__device__ __forceinline__ void store_rows(const float (&acc)[NC][32], float mul, __nv_bfloat16* base, long long ld, int row0, int n,
                                           int d, int c0, int lane, int w4) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int r = row0 + w4 * 16 + (lane >> 2) + 8 * i;
        if (r >= n) continue;
        __nv_bfloat16* row = base + (long long)r * ld;
#pragma unroll
        for (int oc = 0; oc < NC; ++oc)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int col = (c0 + oc) * 64 + j * 8 + 2 * (lane & 3);
                if (col < d) *reinterpret_cast<uint32_t*>(row + col) = pack_bf16x2(acc[oc][j * 4 + i * 2] * mul, acc[oc][j * 4 + i * 2 + 1] * mul);
            }
    }
}

}  // namespace clb
