// Host-side helpers shared by the C-ABI translation units: error reporting, launch counting, TMA descriptor cache.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/controllora_b200.h"

namespace clb {

int set_error(int code, const char* fmt, ...);
void count_launch(int n = 1);
int num_sms();

// Encode (or fetch from the cache) a tiled bf16 tensor map.  dims/box are innermost-first, strides are the byte
// strides of dims 1..rank-1.  Returns CL_OK or a negative status.
int get_tensor_map(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int swizzle_bytes /* 0, 64 or 128 */);

// Launch `kernel` on `stream`.  A launch error is left in cudaGetLastError() for the caller's check.
template <typename... KArgs, typename... Args>
static inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    kernel<<<grid, block, smem, stream>>>(static_cast<KArgs>(args)...);
}

// As launch_k, with the programmatic-stream-serialization attribute: inside a stream (or a captured CUDA graph) the grid
// may start while the previous kernel drains; every kernel of this library executes griddepcontrol.wait (pdl_wait in
// common.cuh) before its first global-memory access.  Only the GEMM launches use it, including those planned at two CTAs
// per SM: an early-started grid lands on the SMs that free up first, which can unbalance a kernel running several CTAs per
// SM, but on the bench step (H100 SXM, 700 W) turning PDL off for the two-CTA launches changed throughput by less than
// the run-to-run spread of about 0.2 images/s, so every GEMM keeps it.  What the
// early start hides is the prologue (barrier init, descriptor prefetch).
template <typename... KArgs, typename... Args>
static inline void launch_k_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    (void)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace clb

#define CL_CHECK(expr)                   \
    do {                                 \
        int _st = (expr);                \
        if (_st != CL_OK) return _st;    \
    } while (0)

#define CL_CUDA_CHECK(expr)                                                                              \
    do {                                                                                                 \
        cudaError_t _e = (expr);                                                                         \
        if (_e != cudaSuccess)                                                                           \
            return clb::set_error(CL_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    } while (0)
