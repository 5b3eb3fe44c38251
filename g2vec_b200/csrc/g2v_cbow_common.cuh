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

// Decoupled weight decay (DESIGN.md §4.18), TF1's DecoupledWeightDecayExtension: var -= weight_decay * var before the
// optimizer step.  Both operations are rounded on their own (never one FMA), so a kernel that decays in a register
// computes what a separate decay pass followed by the undecayed kernel computes, bit for bit.
template <bool WD>
__device__ __forceinline__ void decay1(float &w, float wd) {
    if (WD) w = __fsub_rn(w, __fmul_rn(wd, w));
}
template <bool WD>
__device__ __forceinline__ void decay4(float4 &w, float wd) {
    decay1<WD>(w.x, wd); decay1<WD>(w.y, wd); decay1<WD>(w.z, wd); decay1<WD>(w.w, wd);
}
// weight_decay as the *_wd entry points admit it: finite, 0 <= wd < 1 (NaN fails both comparisons)
inline bool weight_decay_ok(float wd) { return wd >= 0.f && wd < 1.f; }

// Class weights of the training loss (DESIGN.md §4.20): a window of label y counts with weight w_y, cw = {w0, w1}.
// Applied to fl(fl(sigmoid(o) - y) * inv_n) and to the window's loss term, each product rounded on its own (never
// one FMA), so cw = {1, 1} gives the unweighted bits.  CW = false is the unweighted kernel; cw is then unused.
template <bool CW>
__device__ __forceinline__ float class_weighted(float x, float y, float2 cw) {
    return CW ? __fmul_rn(x, y != 0.f ? cw.y : cw.x) : x;
}
// a class weight as the *_cw entry points admit it: finite and > 0 (NaN fails both comparisons)
inline bool class_weight_ok(float w) { return w > 0.f && w <= 0x1.fffffep127f; }
#define G2V_CW_CHECK(name)                                                                                             \
    G2V_REQUIRE(class_weight_ok(w0) && class_weight_ok(w1), name ": class weights must be finite and > 0 (w0=%g w1=%g)", \
                (double)w0, (double)w1)

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

// The row-gather logit of one window, genes gene[b..e), the whole warp: h = sum of the window's W_ih rows (lane owns
// VEC float4 of the row, D = 128*VEC), scaled by the window's scale (1, or 1/l for the mean), o = <h, W_ho> by a lane
// partial and warp_sum.  h and scale are left for a backward.  cbow_rows_kernel and the certified accuracy pass's
// fallback both call this, so a window's o is the same bits in both.
template <int VEC>
__device__ __forceinline__ float rows_logit(const int32_t *__restrict__ gene, const float4 *__restrict__ W4, int32_t b,
                                            int32_t e, int lane, int32_t reduce_mean, const float4 (&who)[VEC],
                                            float4 (&h)[VEC], float &scale) {
    constexpr int D4 = 32 * VEC;
    constexpr int UNR = 8 / VEC;                 // 8 float4 (128 B) in flight per lane
#pragma unroll
    for (int v = 0; v < VEC; ++v) h[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int32_t base = b; base < e; base += 32) {
        const int cnt = min(32, e - base);
        const int32_t g = (lane < cnt) ? __ldg(gene + base + lane) : 0;
        for (int k = 0; k < cnt; k += UNR) {
            float4 r[UNR][VEC];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int32_t gk = __shfl_sync(0xffffffffu, g, (k + u) & 31);
                const float4 *row = W4 + (size_t)gk * D4 + lane;
#pragma unroll
                for (int v = 0; v < VEC; ++v)
                    r[u][v] = (k + u < cnt) ? ldg4(row + v * 32) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u)
#pragma unroll
                for (int v = 0; v < VEC; ++v) {
                    h[v].x += r[u][v].x; h[v].y += r[u][v].y; h[v].z += r[u][v].z; h[v].w += r[u][v].w;
                }
        }
    }
    scale = (reduce_mean && e > b) ? 1.f / (float)(e - b) : 1.f;
    float part = 0.f;
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
        if (reduce_mean) { h[v].x *= scale; h[v].y *= scale; h[v].z *= scale; h[v].w *= scale; }
        part += h[v].x * who[v].x + h[v].y * who[v].y + h[v].z * who[v].z + h[v].w * who[v].w;
    }
    return warp_sum(part);
}

// rows_logit for any D (cbow_rows_generic_kernel): h [D] is the warp's shared-memory row, lane owns h[lane + 32k].
__device__ __forceinline__ float rows_generic_logit(const int32_t *__restrict__ gene, const float *__restrict__ W_ih,
                                                    const float *__restrict__ W_ho, int32_t b, int32_t e, int lane,
                                                    int32_t D, int32_t reduce_mean, float *h, float &scale) {
    for (int d = lane; d < D; d += 32) h[d] = 0.f;
    for (int32_t j = b; j < e; ++j) {
        const float *row = W_ih + (size_t)__ldg(gene + j) * D;
        for (int d = lane; d < D; d += 32) h[d] += __ldg(row + d);
    }
    scale = (reduce_mean && e > b) ? 1.f / (float)(e - b) : 1.f;
    float part = 0.f;
    for (int d = lane; d < D; d += 32) {
        if (reduce_mean) h[d] *= scale;
        part += h[d] * __ldg(W_ho + d);
    }
    return warp_sum(part);
}

// grid of a one-warp-per-item kernel (window, gene): whole chip resident (SMs x occupancy), never more CTAs than
// kCbowWarps items each
int rows_grid(const void *kernel, size_t smem, int64_t n_items, int *grid_out);

// r1_prepare_kernel (g2v_cbow_rank1.cu): s[g] = <W_ih[g,:], W_ho>; with_t: st[g] = {s[g], t[g]} (float2) with
// t[g] = sum_d |W_ih[g,d] * W_ho[d]|, +inf for a row with an element of magnitude > 2^64 (DESIGN.md §4.16)
int launch_r1_prepare(const float *W_ih, const float *W_ho, float *s, int32_t V, int32_t D, bool with_t,
                      cudaStream_t stream);

}  // namespace g2v
