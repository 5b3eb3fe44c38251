// g2v_cbow_common.cuh -- device helpers shared by the CBOW kernels (g2v_cbow.cu, g2v_cbow_slab.cu, g2v_cbow_rank1.cu).
#pragma once
#include "g2v_common.cuh"

namespace g2v {

constexpr int kCbowWarps = 8;

__device__ __forceinline__ float4 ldg4(const float4 *p) { return __ldg(p); }
__device__ __forceinline__ void red_add4(float *p, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ float sigmoid_stable(float x) {
    if (x >= 0.f) { const float z = expf(-x); return 1.f / (1.f + z); }
    const float z = expf(x);
    return z / (1.f + z);
}

// TF1 ApplyAdam (tensorflow/core/kernels/training_ops.cc):  m += (g-m)(1-b1); v += (g*g-v)(1-b2);
// var -= (m*alpha)/(sqrt(v)+eps), alpha = lr*sqrt(1-b2^t)/(1-b1^t).
__device__ __forceinline__ void adam1(float &w, float &m, float &v, float g, float alpha, float omb1,
                                      float omb2, float eps) {
    m += (g - m) * omb1;
    v += (g * g - v) * omb2;
    w -= (m * alpha) / (sqrtf(v) + eps);
}

// alpha of step t >= 1, with beta^t by repeated float32 multiplication, as TF1's beta1_power / beta2_power variables
inline float adam_tf1_alpha(float lr, float beta1, float beta2, int32_t t) {
    float b1p = 1.f, b2p = 1.f;
    for (int i = 0; i < t; ++i) { b1p *= beta1; b2p *= beta2; }
    return lr * sqrtf(1.f - b2p) / (1.f - b1p);
}

struct CtaAcc {   // per-CTA accumulators in shared memory
    double loss;
    unsigned long long correct;
};

// End of a forward kernel: the CTA sums its lanes' g_ho partials (TRAIN) in sh_gho [D], its warps' loss (TRAIN) and
// correct counts in sh_acc, then adds each total into global memory with one atomic per element.  ACTIVE = false
// (a slab pass that does not finish the windows) only takes part in the barrier.
template <int VEC, bool TRAIN, bool ACTIVE>
__device__ __forceinline__ void cta_epilogue(float *sh_gho, CtaAcc &sh_acc, const float4 (&gho)[VEC], float loss_acc,
                                             unsigned correct_acc, int lane, float *__restrict__ g_ho,
                                             double *__restrict__ loss_sum, unsigned long long *__restrict__ n_correct) {
    constexpr int D = 128 * VEC;
    if (TRAIN && ACTIVE) {
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
            float *p = sh_gho + (v * 32 + lane) * 4;
            atomicAdd(p + 0, gho[v].x); atomicAdd(p + 1, gho[v].y);
            atomicAdd(p + 2, gho[v].z); atomicAdd(p + 3, gho[v].w);
        }
    }
    if (ACTIVE && lane == 0) {
        if (TRAIN) atomicAdd(&sh_acc.loss, (double)loss_acc);
        atomicAdd(&sh_acc.correct, (unsigned long long)correct_acc);
    }
    __syncthreads();
    if (TRAIN && ACTIVE) for (int i = threadIdx.x; i < D; i += blockDim.x) atomicAdd(g_ho + i, sh_gho[i]);
    if (ACTIVE && threadIdx.x == 0) {
        if (TRAIN && loss_sum) atomicAdd(loss_sum, sh_acc.loss);
        if (n_correct) atomicAdd(n_correct, sh_acc.correct);
    }
}

// grid of a one-warp-per-item kernel (window, gene): whole chip resident (SMs x occupancy), never more CTAs than
// kCbowWarps items each
int rows_grid(const void *kernel, size_t smem, int64_t n_items, int *grid_out);

}  // namespace g2v
