// CFG + PNDM (pseudo linear multistep, skip_prk_steps) update of the denoise loop, graph-replayable: diffusers'
// PNDMScheduler.step_plms, the scheduler of an SD-1.5 pipeline whose scheduler was not replaced (the class-image loop of
// train_dreambooth_lora.py:586-620).  The scheduler's state - the history `ets` of past noise predictions, the sample saved
// for the restart at the repeated timestep, the step counter - lives in device memory, and every per-step scalar comes
// from a host-built table row, so one captured step replays unchanged for all N + 1 model calls.
//
// Row r of `rows` ([num_calls][8] fp32, built by controllora_b200/sampler.py:pndm_rows):
//   0 UNet timestep (read by cl_sampler_prep, not here)   1 sample_coeff = sqrt(a_prev / a_t)
//   2 eps_coeff = -(a_prev - a_t) / (a_t sqrt(1 - a_prev) + sqrt(a_t (1 - a_t) a_prev))
//   3..6 weights on the new eps and on ring slots 1, 2, 3 (the 1, 2, 3 most recent pushed eps)
//   7 flags: bit 0 push the new eps into the ring, bit 1 save the sample, bit 2 restart from the saved sample
// Per element:  e = e_u + g (e_c - e_u);  e' = w0 e + w1 r1 + w2 r2 + w3 r3;  s = restart ? saved : x;  saved <- s if save;
//               x <- sample_coeff s + eps_coeff e';  (r3, r2, r1) <- (r2, r1, e) if push.
// Each thread owns its elements of x, the ring and the saved sample, so the in-place updates need no synchronisation.
//
// The step counter advances in the same launch (sampler_step_read / sampler_step_arrive in common.cuh).
#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

__global__ void __launch_bounds__(256)
cfg_plms_dev_kernel(const float* __restrict__ eps2, float* __restrict__ x, float* __restrict__ ring,
                    float* __restrict__ saved, const float* __restrict__ rows, unsigned long long* step_ctr,
                    long long n_half, float g) {
    pdl_launch_dependents();
    pdl_wait();
    const float* row = rows + 8 * sampler_step_read(step_ctr);
    const float sc = row[1], ec = row[2], w0 = row[3], w1 = row[4], w2 = row[5], w3 = row[6];
    const int flags = (int)row[7];
    const bool push = flags & 1, save = flags & 2, restart = flags & 4;
    float* __restrict__ r1 = ring;
    float* __restrict__ r2 = ring + n_half;
    float* __restrict__ r3 = ring + 2 * n_half;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_half; i += (long long)gridDim.x * blockDim.x) {
        const float eu = eps2[i], ec_ = eps2[n_half + i];
        const float e = eu + g * (ec_ - eu);
        const float p1 = r1[i], p2 = r2[i], p3 = r3[i];
        const float ep = w0 * e + w1 * p1 + w2 * p2 + w3 * p3;
        const float s = restart ? saved[i] : x[i];
        if (save) saved[i] = s;
        x[i] = sc * s + ec * ep;
        if (push) {
            r3[i] = p2;
            r2[i] = p1;
            r1[i] = e;
        }
    }
    __syncthreads();                                  // every thread of this CTA has read the step
    sampler_step_arrive(step_ctr);
}

}  // namespace clb

using namespace clb;

extern "C" int cl_cfg_plms_step_dev(const float* eps2, float* latents, float* ring, float* saved, const float* rows,
                                    unsigned long long* step_ctr, int64_t n_half, float guidance, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!eps2 || !latents || !ring || !saved || !rows || !step_ctr)
        return set_error(CL_ERR_INVALID, "cl_cfg_plms_step_dev: null pointer");
    if (n_half <= 0) return set_error(CL_ERR_INVALID, "cl_cfg_plms_step_dev: n_half must be positive");
    int blocks = (int)((n_half + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(clb::cfg_plms_dev_kernel, blocks, 256, 0, stream, eps2, latents, ring, saved, rows, step_ctr, (long long)n_half,
             guidance);
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
