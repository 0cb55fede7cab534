// What Stable Diffusion 2.x checkpoints need on top of the SD-1.5 kernels:
//
// * cl_gelu: the exact erf GELU of SD-2's OpenCLIP-H text tower in transformers format (`hidden_act: gelu`,
//   torch.nn.functional.gelu, not the tanh form), in place on bf16, with the blocking of cl_quick_gelu.
// * v-prediction forms of the graph-replayable denoise steps (diffusers 0.13 schedulers with prediction_type
//   "v_prediction", the SD-2.1 768 scheduler config).  Guidance combines the model outputs v = [uncond | cond] first, as the
//   pipelines do; every per-step scalar comes from the same host-built tables as the epsilon steps, indexed by a device step
//   counter that advances in the same launch (sampler_step_read / sampler_step_arrive in common.cuh, as in plms.cu).
#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

__global__ void __launch_bounds__(256)
gelu_kernel(__nv_bfloat16* __restrict__ x, long long total_chunks) {
    pdl_launch_dependents();
    pdl_wait();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total_chunks; i += (long long)gridDim.x * blockDim.x) {
        uint4 u = *reinterpret_cast<const uint4*>(x + i * 8);
        uint32_t* w = reinterpret_cast<uint32_t*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = unpack_bf16x2(w[j]);
            w[j] = pack_bf16x2(gelu_f(f.x), gelu_f(f.y));
        }
        *reinterpret_cast<uint4*>(x + i * 8) = u;
    }
}

// coef rows of cl_cfg_solver_step_dev ([num_steps][8]):
//   kind 0, DDIM (sqrt_at, sqrt_1m_at, sqrt_aprev, sqrt_1m_aprev):  x0 = c0 x - c1 v;  eps = c0 v + c1 x;  x <- c2 x0 + c3 eps
//   kind 1, DPM-Solver++(2M) (alpha_s, sigma_s, c_x, c_m0, c_m1):   x0 = c0 x - c1 v;  x <- c2 x + c3 x0 + c4 x0_prev;
//                                                                   x0_prev <- x0
__global__ void __launch_bounds__(256)
cfg_solver_v_dev_kernel(const float* __restrict__ v2, float* __restrict__ x, float* __restrict__ x0_prev,
                        const float* __restrict__ coef, unsigned long long* step_ctr, long long n_half, float g, int kind) {
    pdl_launch_dependents();
    pdl_wait();
    const float* c = coef + 8 * sampler_step_read(step_ctr);
    const float c0 = c[0], c1 = c[1], c2 = c[2], c3 = c[3], c4 = c[4];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_half; i += (long long)gridDim.x * blockDim.x) {
        const float vu = v2[i], vc = v2[n_half + i];
        const float v = vu + g * (vc - vu);
        const float xv = x[i];
        const float x0 = c0 * xv - c1 * v;
        if (kind == 0) {
            const float e = c0 * v + c1 * xv;
            x[i] = c2 * x0 + c3 * e;
        } else {
            x[i] = c2 * xv + c3 * x0 + c4 * x0_prev[i];
            x0_prev[i] = x0;
        }
    }
    __syncthreads();
    sampler_step_arrive(step_ctr);
}

// PNDM (PLMS, skip_prk_steps): the ring holds the guided v outputs unchanged and the v -> eps conversion follows the PLMS
// combination, where diffusers' PNDMScheduler._get_prev_sample makes it: at the alpha_bar a of the transfer's source timestep
// (t + ratio on the restart row) and with the sample s the row uses.  Converting each v at its own timestep before it enters
// the ring would give different numbers.  Rows are [num_calls][10]: the 8 columns of cl_cfg_plms_step_dev, then sqrt(a) and
// sqrt(1 - a).  Per element:  v = v_u + g (v_c - v_u);  v' = w0 v + w1 r1 + w2 r2 + w3 r3;  s = restart ? saved : x;
// saved <- s if save;  e' = sqrt(a) v' + sqrt(1 - a) s;  x <- sample_coeff s + eps_coeff e';  (r3, r2, r1) <- (r2, r1, v) if push.
__global__ void __launch_bounds__(256)
cfg_plms_v_dev_kernel(const float* __restrict__ v2, float* __restrict__ x, float* __restrict__ ring, float* __restrict__ saved,
                      const float* __restrict__ rows, unsigned long long* step_ctr, long long n_half, float g) {
    pdl_launch_dependents();
    pdl_wait();
    const float* row = rows + 10 * sampler_step_read(step_ctr);
    const float sc = row[1], ec = row[2], w0 = row[3], w1 = row[4], w2 = row[5], w3 = row[6];
    const int flags = (int)row[7];
    const float sa = row[8], s1a = row[9];
    const bool push = flags & 1, save = flags & 2, restart = flags & 4;
    float* __restrict__ r1 = ring;
    float* __restrict__ r2 = ring + n_half;
    float* __restrict__ r3 = ring + 2 * n_half;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_half; i += (long long)gridDim.x * blockDim.x) {
        const float vu = v2[i], vc = v2[n_half + i];
        const float v = vu + g * (vc - vu);
        const float p1 = r1[i], p2 = r2[i], p3 = r3[i];
        const float vp = w0 * v + w1 * p1 + w2 * p2 + w3 * p3;
        const float s = restart ? saved[i] : x[i];
        if (save) saved[i] = s;
        const float ep = sa * vp + s1a * s;
        x[i] = sc * s + ec * ep;
        if (push) {
            r3[i] = p2;
            r2[i] = p1;
            r1[i] = v;
        }
    }
    __syncthreads();
    sampler_step_arrive(step_ctr);
}

}  // namespace clb

using namespace clb;

static int step_blocks(int64_t n_half) {
    int blocks = (int)((n_half + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    return blocks;
}

extern "C" int cl_gelu(void* x, int64_t n, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || n <= 0 || n % 8 != 0) return set_error(CL_ERR_INVALID, "cl_gelu: n must be a positive multiple of 8");
    long long blocks = (n / 8 + 255) / 256;
    if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
    launch_k(clb::gelu_kernel, (int)blocks, 256, 0, stream, reinterpret_cast<__nv_bfloat16*>(x), (long long)(n / 8));
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

extern "C" int cl_cfg_solver_step_v_dev(const float* v2, float* latents, float* x0_prev, const float* coef,
                                        unsigned long long* step_ctr, int64_t n_half, float guidance, int kind, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!v2 || !latents || !coef || !step_ctr) return set_error(CL_ERR_INVALID, "cl_cfg_solver_step_v_dev: null pointer");
    if (kind != 0 && kind != 1) return set_error(CL_ERR_INVALID, "cl_cfg_solver_step_v_dev: kind must be 0 (DDIM) or 1 (DPM-Solver++)");
    if (kind == 1 && !x0_prev) return set_error(CL_ERR_INVALID, "cl_cfg_solver_step_v_dev: null x0_prev for DPM-Solver++");
    if (n_half <= 0) return set_error(CL_ERR_INVALID, "cl_cfg_solver_step_v_dev: n_half must be positive");
    launch_k(clb::cfg_solver_v_dev_kernel, step_blocks(n_half), 256, 0, stream, v2, latents, x0_prev, coef, step_ctr,
             (long long)n_half, guidance, kind);
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

extern "C" int cl_cfg_plms_step_v_dev(const float* v2, float* latents, float* ring, float* saved, const float* rows,
                                      unsigned long long* step_ctr, int64_t n_half, float guidance, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!v2 || !latents || !ring || !saved || !rows || !step_ctr)
        return set_error(CL_ERR_INVALID, "cl_cfg_plms_step_v_dev: null pointer");
    if (n_half <= 0) return set_error(CL_ERR_INVALID, "cl_cfg_plms_step_v_dev: n_half must be positive");
    launch_k(clb::cfg_plms_v_dev_kernel, step_blocks(n_half), 256, 0, stream, v2, latents, ring, saved, rows, step_ctr,
             (long long)n_half, guidance);
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
