// K8 — gradient-norm, clipping and AdamW fused over the flat fp32 arenas that hold every trainable ControlLoRA
// parameter (replaces accelerator.clip_grad_norm_ + torch.optim.AdamW.step + zero_grad,
// train_text_to_image_control_lora.py:791-796).  The clip coefficient is computed on the device from the squared
// norm, so the training step has no host synchronisation.
#include <stdio.h>

#include "common.cuh"
#include "host_common.h"
#include "../../include/controllora_b200.h"

namespace clb {

__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ x, long long n, float* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    float s = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = x[i];
        s += v * v;
    }
    s = warp_sum(s);
    __shared__ float part[8];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += part[i];
        atomicAdd(out, t);
    }
}

__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n, float lr,
             float beta1, float beta2, float eps, float wd, float bc1, float bc2_sqrt, const float* __restrict__ gnorm_sq,
             float max_norm, float grad_scale, int zero_grad) {
    pdl_launch_dependents();
    pdl_wait();
    float coef = grad_scale;
    if (gnorm_sq != nullptr && max_norm > 0.f) {
        const float total = sqrtf(*gnorm_sq) * grad_scale;
        const float c = max_norm / (total + 1e-6f);
        coef *= fminf(c, 1.f);
    }
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gi = g[i] * coef;
        float pi = p[i];
        pi *= (1.f - lr * wd);
        const float mi = beta1 * m[i] + (1.f - beta1) * gi;
        const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        pi -= (lr / bc1) * (mi / denom);
        p[i] = pi;
        if (zero_grad) g[i] = 0.f;
    }
}

// start of the optimizer tail inside a captured step: clears the squared-norm accumulator and advances the device step counter
__global__ void step_begin_kernel(float* __restrict__ gnorm_sq, long long* __restrict__ step) {
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0 && blockIdx.x == 0) { *gnorm_sq = 0.f; *step += 1; }
}

// AdamW with the bias corrections taken from a device-side step counter (CUDA-graph replays advance it)
__global__ void __launch_bounds__(256)
adamw_dev_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n, float lr,
                 float beta1, float beta2, float eps, float wd, const long long* __restrict__ step_dev, const float* __restrict__ gnorm_sq,
                 float max_norm, float grad_scale, int zero_grad) {
    pdl_launch_dependents();
    pdl_wait();
    const float step = (float)(*step_dev);
    const float bc1 = 1.f - powf(beta1, step);
    const float bc2_sqrt = sqrtf(1.f - powf(beta2, step));
    float coef = grad_scale;
    if (gnorm_sq != nullptr && max_norm > 0.f) {
        const float total = sqrtf(*gnorm_sq) * grad_scale;
        const float c = max_norm / (total + 1e-6f);
        coef *= fminf(c, 1.f);
    }
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gi = g[i] * coef;
        float pi = p[i];
        pi *= (1.f - lr * wd);
        const float mi = beta1 * m[i] + (1.f - beta1) * gi;
        const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        pi -= (lr / bc1) * (mi / denom);
        p[i] = pi;
        if (zero_grad) g[i] = 0.f;
    }
}

}  // namespace clb

using namespace clb;

extern "C" int cl_sumsq(const float* x, int64_t n, float* out, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!x || !out) return set_error(CL_ERR_INVALID, "cl_sumsq: null");
    int blocks = (int)((n + 255) / 256);
    if (blocks > num_sms() * 4) blocks = num_sms() * 4;
    if (blocks < 1) blocks = 1;
    launch_k(sumsq_kernel, blocks, 256, 0, stream, x, n, out);
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

extern "C" int cl_adamw(float* p, float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                        float weight_decay, int step, const float* gnorm_sq, float max_norm, float grad_scale, int zero_grad,
                        void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!p || !g || !m || !v || step < 1) return set_error(CL_ERR_INVALID, "cl_adamw: bad args");
    const float bc1 = 1.f - powf(beta1, (float)step);
    const float bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
    int blocks = (int)((n + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(adamw_kernel, blocks, 256, 0, stream, p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2_sqrt, gnorm_sq,
                                            max_norm, grad_scale, zero_grad);
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}


extern "C" int cl_step_begin(float* gnorm_sq, int64_t* step_dev, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!gnorm_sq || !step_dev) return set_error(CL_ERR_INVALID, "cl_step_begin: null");
    launch_k(step_begin_kernel, 1, 32, 0, stream, gnorm_sq, reinterpret_cast<long long*>(step_dev));
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}

extern "C" int cl_adamw_dev(float* p, float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                            float weight_decay, const int64_t* step_dev, const float* gnorm_sq, float max_norm, float grad_scale,
                            int zero_grad, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!p || !g || !m || !v || !step_dev) return set_error(CL_ERR_INVALID, "cl_adamw_dev: bad args");
    int blocks = (int)((n + 255) / 256);
    if (blocks > num_sms() * 8) blocks = num_sms() * 8;
    launch_k(adamw_dev_kernel, blocks, 256, 0, stream, p, g, m, v, (long long)n, lr, beta1, beta2, eps, weight_decay,
             reinterpret_cast<const long long*>(step_dev), gnorm_sq, max_norm, grad_scale, zero_grad);
    count_launch();
    CL_CUDA_CHECK(cudaGetLastError());
    return CL_OK;
}
