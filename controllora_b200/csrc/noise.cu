// Step glue in front of the UNet (train_text_to_image_control_lora.py:757-765, 774-779): per training step, on the device
// and inside the captured CUDA graph,
//     noise      ~ N(0, 1)                                   (torch.randn_like(latents)                          :757)
//     timesteps  ~ U{0, ..., T-1}, one per image             (torch.randint(0, num_train_timesteps, (bsz,))      :760)
//     noisy      = sqrt(ac[t]) x0 + sqrt(1 - ac[t]) noise    (DDPMScheduler.add_noise                             :765)
//     target     = noise                    (epsilon)   or   sqrt(ac[t]) noise - sqrt(1 - ac[t]) x0  (v_prediction :774-779)
// Random numbers: Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3"), key = the 64-bit seed,
// counter = (element group, 0, stream id, step counter).  The step counter lives in device memory and is advanced by a
// one-thread kernel, so a replayed CUDA graph draws fresh numbers every step.  Normals: Box-Muller on two uniforms.
// HBM-bound elementwise pass: reads x0 once, writes noisy + target once (and the B timesteps).
#include <stdio.h>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                               uint32_t (&out)[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// uniform in (0, 1]: (x + 1) * 2^-32 computed in fp32 from the top 24 bits (never 0, so log() is finite)
__device__ __forceinline__ float u01(uint32_t x) { return ((x >> 8) + 1u) * (1.0f / 16777216.0f); }

// one thread = 4 consecutive elements of one image (per_image % 4 == 0)
__global__ void __launch_bounds__(256)
add_noise_kernel(const float* __restrict__ x0, const float* __restrict__ sqrt_ac, const float* __restrict__ sqrt_1mac,
                 const unsigned long long* __restrict__ ctr, unsigned long long seed, int num_train_timesteps, int v_prediction,
                 float* __restrict__ noisy, float* __restrict__ target, float* __restrict__ timesteps, int B, int per_image) {
    pdl_launch_dependents();
    pdl_wait();
    const unsigned long long step = *ctr;
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    const long long groups = (long long)B * (per_image / 4);
    for (long long gi = (long long)blockIdx.x * blockDim.x + threadIdx.x; gi < groups; gi += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(gi / (per_image / 4));
        // timestep of image b: stream 1, counter word 0 = b  (multiply-shift maps 32 random bits onto [0, T))
        uint32_t r[4];
        philox4x32_10((uint32_t)b, 0u, 1u + (((uint32_t)(step >> 32)) << 8), (uint32_t)step, k0, k1, r);
        const int t = (int)(((unsigned long long)r[0] * (unsigned long long)num_train_timesteps) >> 32);
        const float sa = sqrt_ac[t], sb = sqrt_1mac[t];
        // 4 normals of this element group: stream 0
        philox4x32_10((uint32_t)gi, (uint32_t)(gi >> 32), 0u + (((uint32_t)(step >> 32)) << 8), (uint32_t)step, k0, k1, r);
        float n[4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const float rad = sqrtf(-2.0f * logf(u01(r[2 * h])));
            float s, c;
            sincospif(2.0f * u01(r[2 * h + 1]), &s, &c);
            n[2 * h] = rad * c;
            n[2 * h + 1] = rad * s;
        }
        const float4 x = *reinterpret_cast<const float4*>(x0 + gi * 4);
        float4 y, tg;
        y.x = sa * x.x + sb * n[0]; y.y = sa * x.y + sb * n[1]; y.z = sa * x.z + sb * n[2]; y.w = sa * x.w + sb * n[3];
        if (v_prediction) {
            tg.x = sa * n[0] - sb * x.x; tg.y = sa * n[1] - sb * x.y; tg.z = sa * n[2] - sb * x.z; tg.w = sa * n[3] - sb * x.w;
        } else {
            tg = make_float4(n[0], n[1], n[2], n[3]);
        }
        *reinterpret_cast<float4*>(noisy + gi * 4) = y;
        *reinterpret_cast<float4*>(target + gi * 4) = tg;
        if (gi % (per_image / 4) == 0) timesteps[b] = (float)t;
    }
}

__global__ void rng_advance_kernel(unsigned long long* ctr) {
    pdl_launch_dependents();
    pdl_wait();
    *ctr += 1ull;
}

}  // namespace clb

using namespace clb;

extern "C" int cl_add_noise(const float* x0, const float* sqrt_ac, const float* sqrt_1mac, unsigned long long* step_counter,
                            unsigned long long seed, int num_train_timesteps, int v_prediction, float* noisy, float* target,
                            float* timesteps, int B, int per_image, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x0 || !sqrt_ac || !sqrt_1mac || !step_counter || !noisy || !target || !timesteps)
        return set_error(CL_ERR_INVALID, "cl_add_noise: null pointer");
    if (B <= 0 || per_image <= 0 || per_image % 4 != 0 || num_train_timesteps <= 0)
        return set_error(CL_ERR_INVALID, "cl_add_noise: B, per_image (multiple of 4) and num_train_timesteps must be positive");
    const long long groups = (long long)B * (per_image / 4);
    int blocks = (int)((groups + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(add_noise_kernel, blocks, 256, 0, stream, x0, sqrt_ac, sqrt_1mac, (const unsigned long long*)step_counter, seed,
             num_train_timesteps, v_prediction, noisy, target, timesteps, B, per_image);
    count_launch();
    launch_k(rng_advance_kernel, 1, 1, 0, stream, step_counter);
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
