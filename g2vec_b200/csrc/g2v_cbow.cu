// g2v_cbow.cu -- HOT PATH 2: modified CBOW (G2Vec.py:217-286) as fused sm_90a kernels.
//
// The reference builds  H = X.W_ih ; O = H.W_ho ; cost = mean(sigmoid_BCE(O, Y))  on a dense
// multi-hot X [N, V] (99.7 % zeros) and lets TF1 autodiff + ApplyAdam train W_ih, W_ho
// (G2Vec.py:239-246).  Here X is CSR (window -> gene ids) and one warp owns one window:
//
//   cbow_rows_kernel<VEC, BACKWARD, SCATTER_TMA, GATHER_TMA>
//                                         D = 128*VEC, each lane owns VEC float4 of the row; the two TMA
//                                         flags select the measured-and-not-shipped staged variants (4.4)
//     gather   h   = sum_{g in window} W_ih[g, :]          (512*VEC B coalesced per row, 8 rows in flight)
//     logit    o   = <h, W_ho>                            (warp shuffle reduction)
//     loss/acc     max(o,0) - o*y + log1p(exp(-|o|)),  (o > 0) == y
//     grad     dO  = (sigmoid(o) - y) / N                 (N known up front: no global barrier)
//     scatter  g_ih[g, :] += dO * W_ho  for g in window   (red.global.add.v4.f32, 16 B per lane)
//              g_ho       += h * dO                       (registers -> smem -> one atomic per CTA)
//   cbow_rows_kernel<VEC, true, false, false, CSC=true>   the same up to dO; then, instead of the scatter,
//                                         dO_pos[i] = dO * scale  at the window's list position i (4 B per window)
//   cbow_csc_expand_kernel                one warp per gene: c = sum of dO_pos over the gene's segment of the list's
//                                         transposed incidence (CSC), then g_ih[g, :] += c * W_ho, one plain
//                                         read-modify-write per touched row.  Exact because the model is linear:
//                                         every window adds the same row W_ho to its genes, only the scale differs.
//                                         This is the backward of a prepared full list (g2v_cbow_fwdbwd_csc): it
//                                         replaces l*D*4 bytes of L2 atomics per window by 8 bytes per incidence.
//   cbow_update_kernel                   dense epilogue over [V*D] (+[D]): TF1 Adam or SGD,
//                                         float4, zeroes the gradient for the next step
//   adam_tick_kernel                      TF1's beta1_power / beta2_power / alpha_t kept on the device so
//                                         that a whole step can be replayed as one CUDA graph
//
// No tensor cores: the 128..512-wide reduction is a memory-bound gather/scatter, not a dense
// contraction.  Algorithmic bytes per window: l*(8D+4)+5 with the scatter, l*(4D+12)+9 with the CSC backward
// (+ 8*D per touched gene row) (DESIGN.md), per step + 32*V*D (Adam).
#include <stdlib.h>

#include "g2v_cbow_common.cuh"

namespace g2v {

constexpr bool kDefaultGatherTma = false;
constexpr bool kDefaultScatterTma = false;   // G2V_CBOW_SCATTER=tma selects the bulk-reduction scatter

// SCATTER_TMA: the gradient row dO*W_ho (identical for every gene of the window) is staged once in
// shared memory and added into g_ih[gene,:] with one TMA bulk reduction per gene
// (cp.reduce.async.bulk.global.shared::cta.add.f32, D*4 bytes, SASS UBLKRED) instead of 32 lanes x
// red.global.add.v4.f32: the scatter leaves the LSU/L1TEX path, which bounds the L2-resident configs.
// GATHER_TMA: embedding rows are staged through shared memory with TMA bulk copies
// (cp.async.bulk.shared::cluster.global + mbarrier complete_tx, SASS UBLKCP), 2 stages of 2 KB per warp,
// one lane issuing one row; the lanes then sum the rows with LDS.128 instead of LDG.128.
// CSC: the backward stops at dO -- it stores dO*scale at the window's list position i (dO_pos[i]) instead of
// scattering rows into g_ih; cbow_csc_expand_kernel then sums those scalars per gene and writes each gene row once.
template <int VEC, bool BACKWARD, bool SCATTER_TMA, bool GATHER_TMA, bool CSC = false>
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_rows_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                 const uint8_t *__restrict__ label, const int32_t *__restrict__ win,
                 int64_t win_begin, int64_t n_win, float inv_n, const float *__restrict__ W_ih,
                 const float *__restrict__ W_ho, float *__restrict__ g_ih, float *__restrict__ g_ho,
                 double *__restrict__ loss_sum, unsigned long long *__restrict__ n_correct,
                 int32_t reduce_mean, const int32_t *__restrict__ skip, float *__restrict__ dO_pos) {
    static_assert(!CSC || (BACKWARD && !SCATTER_TMA), "the CSC backward replaces the scatter");
    G2V_SKIP_IF_STOPPED(skip);
    constexpr int D = 128 * VEC;
    constexpr int D4 = D / 4;
    constexpr int UNR = 8 / VEC;                 // 8 float4 (128 B) in flight per lane
    __shared__ float sh_gho[BACKWARD ? D : 1];
    // scatter staging row: its own buffer, or (both TMA paths on) stage 0 of the gather tile
    __shared__ __align__(128) float sh_row[(BACKWARD && SCATTER_TMA && !GATHER_TMA) ? kCbowWarps * D : 4];
    __shared__ CtaAcc sh_acc;
    constexpr int R = 4 / VEC;                   // rows per TMA stage (2 KB per warp per stage)
    __shared__ __align__(128) float sh_tile[GATHER_TMA ? kCbowWarps * 2 * R * D : 4];
    __shared__ __align__(8) unsigned long long sh_bar[GATHER_TMA ? kCbowWarps * 2 : 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (BACKWARD) for (int i = threadIdx.x; i < D; i += blockDim.x) sh_gho[i] = 0.f;
    if (threadIdx.x == 0) { sh_acc.loss = 0.0; sh_acc.correct = 0ull; }
    if (GATHER_TMA) {
        if (lane < 2) {
            const uint32_t a = (uint32_t)__cvta_generic_to_shared(&sh_bar[warp * 2 + lane]);
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(a) : "memory");
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    uint32_t tma_phase = 0;                      // bit s = parity of stage s

    const float4 *__restrict__ W4 = reinterpret_cast<const float4 *>(W_ih);
    float4 who[VEC], gho[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
        who[v] = ldg4(reinterpret_cast<const float4 *>(W_ho) + v * 32 + lane);
        gho[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float loss_acc = 0.f;
    unsigned correct_acc = 0;

    const int64_t warps_total = (int64_t)gridDim.x * kCbowWarps;
    for (int64_t i = (int64_t)blockIdx.x * kCbowWarps + warp; i < n_win; i += warps_total) {
        const int64_t n = win ? (int64_t)__ldg(win + win_begin + i) : win_begin + i;
        const int32_t b = __ldg(rowptr + n), e = __ldg(rowptr + n + 1);
        const float y = (float)__ldg(label + n);
        float4 h[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) h[v] = make_float4(0.f, 0.f, 0.f, 0.f);

        // ---- gather + segmented sum
        if (GATHER_TMA) {
            float *tile = sh_tile + (size_t)warp * 2 * R * D;
            if (BACKWARD && SCATTER_TMA) {        // stage 0 doubles as the scatter staging row: drain its readers
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                __syncwarp();
            }
            const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(&sh_bar[warp * 2]);
            const int nchunk = (e - b + R - 1) / R;
            auto issue = [&](int c) {             // chunk c -> stage c & 1: lane r copies row r
                const int st = c & 1;
                const int32_t j = b + c * R + lane;
                const int cnt = min(R, e - (b + c * R));
                if (lane == 0)
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar0 + st * 8),
                                 "r"(cnt * D * 4)
                                 : "memory");
                if (lane < cnt) {
                    const float *src = W_ih + (size_t)__ldg(gene + j) * D;
                    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(tile + (size_t)(st * R + lane) * D);
                    asm volatile(
                        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                        "l"(src), "n"(D * 4), "r"(bar0 + st * 8)
                        : "memory");
                }
            };
            if (nchunk > 0) issue(0);
            for (int c = 0; c < nchunk; ++c) {
                const int st = c & 1;
                if (c + 1 < nchunk) issue(c + 1);
                const uint32_t par = (tma_phase >> st) & 1u;
                uint32_t ok = 0;
                while (!ok)
                    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                 : "=r"(ok)
                                 : "r"(bar0 + st * 8), "r"(par)
                                 : "memory");
                tma_phase ^= (1u << st);
                const int cnt = min(R, e - (b + c * R));
                const float4 *t4 = reinterpret_cast<const float4 *>(tile + (size_t)st * R * D);
#pragma unroll
                for (int r = 0; r < R; ++r)
                    if (r < cnt) {
#pragma unroll
                        for (int v = 0; v < VEC; ++v) {
                            const float4 x = t4[r * D4 + v * 32 + lane];
                            h[v].x += x.x; h[v].y += x.y; h[v].z += x.z; h[v].w += x.w;
                        }
                    }
                __syncwarp();                     // stage st is free for chunk c + 2
            }
        } else
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
        const float scale = (reduce_mean && e > b) ? 1.f / (float)(e - b) : 1.f;
        float part = 0.f;
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
            if (reduce_mean) { h[v].x *= scale; h[v].y *= scale; h[v].z *= scale; h[v].w *= scale; }
            part += h[v].x * who[v].x + h[v].y * who[v].y + h[v].z * who[v].z + h[v].w * who[v].w;
        }
        const float o = warp_sum(part);
        if (lane == 0) {
            correct_acc += ((o > 0.f) == (y != 0.f)) ? 1u : 0u;
            if (BACKWARD) loss_acc += fmaxf(o, 0.f) - o * y + log1pf(expf(-fabsf(o)));
        }
        if (CSC) {
            const float dO = (sigmoid_stable(o) - y) * inv_n;
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
                gho[v].x += h[v].x * dO; gho[v].y += h[v].y * dO; gho[v].z += h[v].z * dO; gho[v].w += h[v].w * dO;
            }
            if (lane == 0) dO_pos[i] = dO * scale;
        } else if (BACKWARD) {
            const float dO = (sigmoid_stable(o) - y) * inv_n;
            float4 gv[VEC];
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
                gho[v].x += h[v].x * dO; gho[v].y += h[v].y * dO; gho[v].z += h[v].z * dO; gho[v].w += h[v].w * dO;
                const float s = dO * scale;
                gv[v] = make_float4(who[v].x * s, who[v].y * s, who[v].z * s, who[v].w * s);
            }
            // ---- scatter-add the gradient rows
            if (SCATTER_TMA) {
                float *stage = GATHER_TMA ? sh_tile + (size_t)warp * 2 * R * D : sh_row + warp * D;
                // the previous window's bulk reductions must have finished READING the staging row
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                __syncwarp();
#pragma unroll
                for (int v = 0; v < VEC; ++v) reinterpret_cast<float4 *>(stage)[v * 32 + lane] = gv[v];
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> async proxy
                __syncwarp();
                const uint32_t src = (uint32_t)__cvta_generic_to_shared(stage);
                for (int32_t j = b + lane; j < e; j += 32) {
                    float *dst = g_ih + (size_t)__ldg(gene + j) * D;
                    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;"
                                 ::"l"(dst), "r"(src), "n"(D * 4)
                                 : "memory");
                }
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            } else
            for (int32_t base = b; base < e; base += 32) {
                const int cnt = min(32, e - base);
                const int32_t g = (lane < cnt) ? __ldg(gene + base + lane) : 0;
                for (int k = 0; k < cnt; ++k) {
                    const int32_t gk = __shfl_sync(0xffffffffu, g, k);
                    float *dst = g_ih + (size_t)gk * D + lane * 4;
#pragma unroll
                    for (int v = 0; v < VEC; ++v) red_add4(dst + v * 128, gv[v]);
                }
            }
        }
    }

    if (BACKWARD && SCATTER_TMA) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");

    // ---- CTA-level reduction of g_ho / loss / correct, then one global atomic each
    if (BACKWARD) {
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
            float *p = sh_gho + (v * 32 + lane) * 4;
            atomicAdd(p + 0, gho[v].x); atomicAdd(p + 1, gho[v].y);
            atomicAdd(p + 2, gho[v].z); atomicAdd(p + 3, gho[v].w);
        }
    }
    if (lane == 0) {
        if (BACKWARD) atomicAdd(&sh_acc.loss, (double)loss_acc);
        atomicAdd(&sh_acc.correct, (unsigned long long)correct_acc);
    }
    __syncthreads();
    if (BACKWARD) for (int i = threadIdx.x; i < D; i += blockDim.x) atomicAdd(g_ho + i, sh_gho[i]);
    if (threadIdx.x == 0) {
        if (BACKWARD && loss_sum) atomicAdd(loss_sum, sh_acc.loss);
        if (n_correct) atomicAdd(n_correct, sh_acc.correct);
    }
}

// Any D (not a multiple of 128): h and the g_ho partial live in shared memory per warp.
// dO_pos != NULL: the CSC backward of cbow_rows_kernel (dO*scale stored per list position, no scatter).
template <bool BACKWARD>
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_rows_generic_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                         const uint8_t *__restrict__ label, const int32_t *__restrict__ win,
                         int64_t win_begin, int64_t n_win, float inv_n, const float *__restrict__ W_ih,
                         const float *__restrict__ W_ho, float *__restrict__ g_ih,
                         float *__restrict__ g_ho, double *__restrict__ loss_sum,
                         unsigned long long *__restrict__ n_correct, int32_t D, int32_t reduce_mean,
                         const int32_t *__restrict__ skip, float *__restrict__ dO_pos) {
    G2V_SKIP_IF_STOPPED(skip);
    extern __shared__ float shf[];
    __shared__ CtaAcc sh_acc;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *h = shf + (size_t)warp * 2 * D;
    float *gho = h + D;
    for (int d = lane; d < D; d += 32) gho[d] = 0.f;
    if (threadIdx.x == 0) { sh_acc.loss = 0.0; sh_acc.correct = 0ull; }
    __syncthreads();
    float loss_acc = 0.f;
    unsigned correct_acc = 0;
    const int64_t warps_total = (int64_t)gridDim.x * kCbowWarps;
    for (int64_t i = (int64_t)blockIdx.x * kCbowWarps + warp; i < n_win; i += warps_total) {
        const int64_t n = win ? (int64_t)__ldg(win + win_begin + i) : win_begin + i;
        const int32_t b = __ldg(rowptr + n), e = __ldg(rowptr + n + 1);
        const float y = (float)__ldg(label + n);
        for (int d = lane; d < D; d += 32) h[d] = 0.f;
        for (int32_t j = b; j < e; ++j) {
            const float *row = W_ih + (size_t)__ldg(gene + j) * D;
            for (int d = lane; d < D; d += 32) h[d] += __ldg(row + d);
        }
        const float scale = (reduce_mean && e > b) ? 1.f / (float)(e - b) : 1.f;
        float part = 0.f;
        for (int d = lane; d < D; d += 32) {
            if (reduce_mean) h[d] *= scale;
            part += h[d] * __ldg(W_ho + d);
        }
        const float o = warp_sum(part);
        if (lane == 0) {
            correct_acc += ((o > 0.f) == (y != 0.f)) ? 1u : 0u;
            if (BACKWARD) loss_acc += fmaxf(o, 0.f) - o * y + log1pf(expf(-fabsf(o)));
        }
        if (BACKWARD) {
            const float dO = (sigmoid_stable(o) - y) * inv_n;
            for (int d = lane; d < D; d += 32) gho[d] += h[d] * dO;
            const float s = dO * scale;
            if (dO_pos) {
                if (lane == 0) dO_pos[i] = s;
                continue;
            }
            for (int32_t j = b; j < e; ++j) {
                float *dst = g_ih + (size_t)__ldg(gene + j) * D;
                for (int d = lane; d < D; d += 32) atomicAdd(dst + d, __ldg(W_ho + d) * s);
            }
        }
    }
    if (BACKWARD) for (int d = lane; d < D; d += 32) atomicAdd(g_ho + d, gho[d]);
    if (lane == 0) {
        if (BACKWARD) atomicAdd(&sh_acc.loss, (double)loss_acc);
        atomicAdd(&sh_acc.correct, (unsigned long long)correct_acc);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (BACKWARD && loss_sum) atomicAdd(loss_sum, sh_acc.loss);
        if (n_correct) atomicAdd(n_correct, sh_acc.correct);
    }
}

// Second half of the CSC backward.  The model is linear, so every window adds the same row W_ho to its genes,
// scaled by its dO*scale:  g_ih[g,:] += c[g] * W_ho  with  c[g] = sum of dO_pos over the list positions of the
// windows that contain g (the gene's CSC segment).  One warp per gene owns the row: a coalesced read-modify-write,
// no atomics.  Genes in no listed window are not touched.
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_csc_expand_kernel(const int32_t *__restrict__ cscptr, const int32_t *__restrict__ csc_pos,
                       const float *__restrict__ dO_pos, const float *__restrict__ W_ho, float *__restrict__ g_ih,
                       int32_t V, int32_t D, const int32_t *__restrict__ skip) {
    G2V_SKIP_IF_STOPPED(skip);
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * kCbowWarps + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * kCbowWarps;
    for (int64_t g = warp; g < V; g += nwarps) {
        const int32_t b = __ldg(cscptr + g), e = __ldg(cscptr + g + 1);
        if (b == e) continue;
        const float c = csc_segment_sum(csc_pos, dO_pos, b, e, lane);
        float *row = g_ih + (size_t)g * D;
        if ((D & 3) == 0) {
            float4 *r4 = reinterpret_cast<float4 *>(row);
            for (int k = lane; k < (D >> 2); k += 32) {
                const float4 w = ldg4(reinterpret_cast<const float4 *>(W_ho) + k);
                float4 a = r4[k];
                a.x += c * w.x; a.y += c * w.y; a.z += c * w.z; a.w += c * w.w;
                r4[k] = a;
            }
        } else {
            for (int d = lane; d < D; d += 32) row[d] += c * __ldg(W_ho + d);
        }
    }
}

// ---- optimizer epilogue --------------------------------------------------------------------
// TF1 ApplyAdam (tensorflow/core/kernels/training_ops.cc):  m += (g-m)(1-b1); v += (g*g-v)(1-b2);
// var -= (m*alpha)/(sqrt(v)+eps), alpha = lr*sqrt(1-b2^t)/(1-b1^t).
__device__ __forceinline__ void adam1(float &w, float &m, float &v, float g, float alpha, float omb1,
                                      float omb2, float eps) {
    m += (g - m) * omb1;
    v += (g * g - v) * omb2;
    w -= (m * alpha) / (sqrtf(v) + eps);
}

template <int OPT>
__global__ void __launch_bounds__(256)
cbow_update_kernel(float *__restrict__ W, float *__restrict__ M, float *__restrict__ Vv,
                   float *__restrict__ G, int64_t n, float *__restrict__ W2, float *__restrict__ M2,
                   float *__restrict__ V2, float *__restrict__ G2, int64_t n2, float alpha_host, float omb1,
                   float omb2, float eps, const float *__restrict__ alpha_dev, const int32_t *__restrict__ skip) {
    G2V_SKIP_IF_STOPPED(skip);
    // alpha_dev != NULL: the step size lives on the device (g2v_cbow_adam_tick), so the launch can be replayed
    const float alpha = alpha_dev ? __ldg(alpha_dev + 2) : alpha_host;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t nthreads = (int64_t)gridDim.x * blockDim.x;
    const int64_t n4 = n >> 2;
    float4 *W4 = reinterpret_cast<float4 *>(W), *G4 = reinterpret_cast<float4 *>(G);
    float4 *M4 = reinterpret_cast<float4 *>(M), *V4 = reinterpret_cast<float4 *>(Vv);
    for (int64_t i = tid; i < n4; i += nthreads) {
        float4 w = W4[i];
        const float4 g = G4[i];
        if (OPT == G2V_OPT_ADAM_TF1) {
            float4 m = M4[i], v = V4[i];
            adam1(w.x, m.x, v.x, g.x, alpha, omb1, omb2, eps);
            adam1(w.y, m.y, v.y, g.y, alpha, omb1, omb2, eps);
            adam1(w.z, m.z, v.z, g.z, alpha, omb1, omb2, eps);
            adam1(w.w, m.w, v.w, g.w, alpha, omb1, omb2, eps);
            M4[i] = m; V4[i] = v;
        } else {
            w.x -= alpha * g.x; w.y -= alpha * g.y; w.z -= alpha * g.z; w.w -= alpha * g.w;
        }
        W4[i] = w;
        G4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // scalar tail of W_ih, then the [D] output layer
    for (int64_t i = (n4 << 2) + tid; i < n + n2; i += nthreads) {
        float *w, *m, *v, *g;
        if (i < n) { w = W + i; m = M + i; v = Vv + i; g = G + i; }
        else { const int64_t j = i - n; w = W2 + j; m = M2 + j; v = V2 + j; g = G2 + j; }
        if (OPT == G2V_OPT_ADAM_TF1) adam1(*w, *m, *v, *g, alpha, omb1, omb2, eps);
        else *w -= alpha * *g;
        *g = 0.f;
    }
}

// ---- optimizer epilogue fused with the gradient exchange over NVLink / NVSwitch ---------------------------
// Multi-GPU form of cbow_update_kernel: instead of ncclAllReduce(gradient) followed by the same dense update on
// every rank, rank r owns the slice [r*chunk, (r+1)*chunk) of the flat parameter vector [W_ih | W_ho]:
//   reduce-scatter   g = sum over ranks of their gradient slice -- ONE multimem.ld_reduce per 16 bytes when the
//                    buffers are bound to an NVLS multicast object (the NVSwitch adds), else peer loads (P2P)
//   zero             the slice of every rank's gradient buffer (multimem.st / peer stores): ready for the next step
//   Adam / SGD       on the owned slice only -- m and v are touched for 1/world of the parameters per rank
//   all-gather       the updated weights are stored into every rank's parameter buffer (multimem.st / peer stores)
// so the transfer overlaps the arithmetic 16 bytes at a time and the dense update work is divided by `world`.
// The caller brackets the launch with two cross-GPU barriers (all gradients complete before; all weights
// delivered after).  Buffers are symmetric-memory allocations (same offset on every rank).
__device__ __forceinline__ float4 mm_ld_reduce4(const float *mc) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ void mm_st4(float *mc, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
                 ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 ld_peer4(const float *p) {
    float4 v;
    asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_peer4(float *p, float4 v) {
    asm volatile("st.volatile.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}

template <int OPT, bool MC>
__global__ void __launch_bounds__(256)
cbow_update_nvl_kernel(float *const *__restrict__ g_ptrs, float *const *__restrict__ w_ptrs, float *__restrict__ g_mc,
                       float *__restrict__ w_mc, float *__restrict__ M, float *__restrict__ Vv, int64_t n, int32_t rank,
                       int32_t world, float alpha_host, float omb1, float omb2, float eps,
                       const float *__restrict__ alpha_dev, const int32_t *__restrict__ skip) {
    G2V_SKIP_IF_STOPPED(skip);
    const float alpha = alpha_dev ? __ldg(alpha_dev + 2) : alpha_host;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
    const int64_t n4 = n >> 2, chunk = (n4 + world - 1) / world;
    const int64_t lo = (int64_t)rank * chunk, hi = min(n4, lo + chunk);
    float *Wl = w_ptrs[rank];
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t i = lo + tid; i < hi; i += nth) {
        float4 g;
        if (MC) {
            g = mm_ld_reduce4(g_mc + 4 * i);
            mm_st4(g_mc + 4 * i, zero);
        } else {
            g = zero;
            for (int p = 0; p < world; ++p) {
                float *gp = g_ptrs[(rank + p) % world] + 4 * i;
                const float4 x = ld_peer4(gp);
                g.x += x.x; g.y += x.y; g.z += x.z; g.w += x.w;
                st_peer4(gp, zero);
            }
        }
        float4 w = reinterpret_cast<const float4 *>(Wl)[i];
        if (OPT == G2V_OPT_ADAM_TF1) {
            float4 m = reinterpret_cast<float4 *>(M)[i], v = reinterpret_cast<float4 *>(Vv)[i];
            adam1(w.x, m.x, v.x, g.x, alpha, omb1, omb2, eps);
            adam1(w.y, m.y, v.y, g.y, alpha, omb1, omb2, eps);
            adam1(w.z, m.z, v.z, g.z, alpha, omb1, omb2, eps);
            adam1(w.w, m.w, v.w, g.w, alpha, omb1, omb2, eps);
            reinterpret_cast<float4 *>(M)[i] = m; reinterpret_cast<float4 *>(Vv)[i] = v;
        } else {
            w.x -= alpha * g.x; w.y -= alpha * g.y; w.z -= alpha * g.z; w.w -= alpha * g.w;
        }
        if (MC) {
            mm_st4(w_mc + 4 * i, w);
        } else {
            for (int p = 0; p < world; ++p) st_peer4(w_ptrs[(rank + p) % world] + 4 * i, w);
        }
    }
    // scalar tail (n not a multiple of 4): the last rank, peer loads/stores
    if (rank == world - 1)
        for (int64_t i = (n4 << 2) + tid; i < n; i += nth) {
            float g = 0.f;
            for (int p = 0; p < world; ++p) {
                volatile float *gp = g_ptrs[p] + i;
                g += *gp; *gp = 0.f;
            }
            float w = Wl[i];
            if (OPT == G2V_OPT_ADAM_TF1) adam1(w, M[i], Vv[i], g, alpha, omb1, omb2, eps);
            else w -= alpha * g;
            for (int p = 0; p < world; ++p) { volatile float *wp = w_ptrs[p] + i; *wp = w; }
        }
}

int rows_grid(const void *kernel, size_t smem, int64_t n_win, int *grid_out) {
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    if (dp.cc_major != 9) { set_error("needs an sm_90 device (found sm_%d%d); no CPU fallback", dp.cc_major, dp.cc_minor); return 2; }
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kCbowWarps * 32, smem);
    if (e != cudaSuccess || per_sm <= 0) { set_error("occupancy query failed: %s", cudaGetErrorString(e)); return 1; }
    int64_t grid = (int64_t)dp.sm_count * per_sm;
    const int64_t need = (n_win + kCbowWarps - 1) / kCbowWarps;
    if (grid > need) grid = need;
    *grid_out = (int)(grid > 0 ? grid : 1);
    return 0;
}

// dO_pos != NULL (backward only): the CSC backward -- dO*scale per list position instead of the scatter into g_ih
template <bool BACKWARD>
static int launch_rows(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                       int64_t win_begin, int64_t n_win, float inv_n, const float *W_ih, const float *W_ho,
                       float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t D,
                       int32_t reduce, cudaStream_t st, float *dO_pos = nullptr) {
    unsigned long long *nc = reinterpret_cast<unsigned long long *>(n_correct);
    int grid = 0, rc;
    // scatter path of the backward kernel: "red" (red.global.add.v4.f32 per lane) or "tma"
    // (cp.reduce.async.bulk per gene row); G2V_CBOW_SCATTER overrides the default
    const char *sc = getenv("G2V_CBOW_SCATTER");
    const bool tma = BACKWARD && (sc ? sc[0] == 't' : kDefaultScatterTma);
    const char *gc = getenv("G2V_CBOW_GATHER");       // "ldg" (LDG.128 per lane) or "tma" (bulk copies via smem)
    const bool gtma = gc ? gc[0] == 't' : kDefaultGatherTma;
#define G2V_LAUNCH_VEC(VEC)                                                                          \
    {                                                                                                \
        auto kern = tma ? (gtma ? cbow_rows_kernel<VEC, BACKWARD, BACKWARD, true>                    \
                                : cbow_rows_kernel<VEC, BACKWARD, BACKWARD, false>)                  \
                        : (gtma ? cbow_rows_kernel<VEC, BACKWARD, false, true>                       \
                                : cbow_rows_kernel<VEC, BACKWARD, false, false>);                    \
        if (dO_pos) kern = cbow_rows_kernel<VEC, BACKWARD, false, false, BACKWARD>;                  \
        if ((rc = rows_grid((const void *)kern, 0, n_win, &grid))) return rc;                        \
        kern<<<grid, kCbowWarps * 32, 0, st>>>(rowptr, gene, label, win, win_begin, n_win, inv_n, W_ih, W_ho, g_ih, \
                                               g_ho, loss_sum, nc, reduce, loop_skip_flag(), dO_pos); \
    }
    if (D == 128) G2V_LAUNCH_VEC(1)
    else if (D == 256) G2V_LAUNCH_VEC(2)
    else if (D == 512) G2V_LAUNCH_VEC(4)
    else {
        const size_t smem = (size_t)kCbowWarps * 2 * D * sizeof(float);
        DeviceProps dp;
        if (device_props(&dp)) return 1;
        G2V_REQUIRE(smem <= (size_t)dp.max_smem_optin, "sizeHiddenlayer %d too large for the generic kernel", D);
        G2V_CUDA_OK(cudaFuncSetAttribute(cbow_rows_generic_kernel<BACKWARD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if ((rc = rows_grid((const void *)cbow_rows_generic_kernel<BACKWARD>, smem, n_win, &grid))) return rc;
        cbow_rows_generic_kernel<BACKWARD><<<grid, kCbowWarps * 32, smem, st>>>(
            rowptr, gene, label, win, win_begin, n_win, inv_n, W_ih, W_ho, g_ih, g_ho, loss_sum, nc, D, reduce, loop_skip_flag(),
            dO_pos);
    }
#undef G2V_LAUNCH_VEC
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}


// ---- device-side training loop control (SURVEY 8f-4; G2Vec.py:262-283) ------------------------------------
// ctl (int64 x 8 in device memory):
//   [0] stopped      1 once the loop is over: the validation accuracy dropped (strict <, :276) or max_steps ran
//   [1] step         optimizer steps decided so far
//   [2] stop_step    step whose validation accuracy dropped, -1 if none (the reference breaks there, :279)
//   [3] before_val   correct validation windows of the last passed step (before_acc_val, :280; -1 = the -1. of :261)
//   [4] max_steps    cap on optimizer steps (--epoch)       [5] early_stop   0 = never stop early
// loop_begin:  if not stopped, copy the weights into `snapshot` (they are the result if THIS step's validation
//   accuracy drops: the reference returns the W_ih read at :283 after the previous step) and zero the 4 counters.
// loop_decide: if not stopped, record the step's counters in hist[step][0..3], apply the early-stop rule on the
//   validation count (same ordering as the float32 ratios the reference compares while n_val < 2^24), advance.
__global__ void __launch_bounds__(256)
loop_begin_kernel(const long long *__restrict__ ctl, long long *__restrict__ acc, const float4 *__restrict__ W4,
                  float4 *__restrict__ S4, int64_t n4, const float *__restrict__ W, float *__restrict__ S, int64_t n) {
    if (ctl[0] != 0) return;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
    if (tid < 4) acc[tid] = 0;
    if (S == nullptr) return;
    for (int64_t i = tid; i < n4; i += nth) S4[i] = W4[i];
    for (int64_t i = (n4 << 2) + tid; i < n; i += nth) S[i] = W[i];
}

// acc == NULL: the step's counters were already summed over the ranks into hist[step] (loop_counters_nvl_kernel)
__global__ void loop_decide_kernel(long long *__restrict__ ctl, const long long *__restrict__ acc,
                                   long long *__restrict__ hist) {
    if (ctl[0] != 0) return;
    const long long step = ctl[1];
    if (acc)
        for (int k = 0; k < 4; ++k) hist[step * 4 + k] = acc[k];
    const long long val = hist[step * 4 + 2];
    if (ctl[5] != 0 && val < ctl[3]) {
        ctl[0] = 1; ctl[2] = step;                  // dropped: the snapshot taken by loop_begin is the result
    } else {
        ctl[3] = val;
        if (step + 1 >= ctl[4]) ctl[0] = 1;          // ran --epoch steps without a drop
    }
    ctl[1] = step + 1;
}

// Multi-GPU: add this rank's three accuracy counters of the current step into hist[step][1..3] of EVERY rank's
// (symmetric-memory) history -- one multimem.red per counter when the buffer has an NVLS multicast address (the
// switch applies the add to all replicas), else one system-scope atomic per peer.  Every step has its own slot of
// the zero-initialised history, so no buffer is ever reset while a peer may still add to or read it.  The caller
// puts a cross-GPU barrier between this kernel and loop_decide_kernel.
__global__ void loop_counters_nvl_kernel(const long long *__restrict__ ctl, const long long *__restrict__ acc,
                                         long long *const *__restrict__ hist_ptrs, long long *__restrict__ hist_mc,
                                         int32_t world) {
    if (ctl[0] != 0) return;
    const int k = 1 + (int)threadIdx.x;              // 3 threads: pre-update train, validation, train counts
    if (k > 3) return;
    const long long step = ctl[1], v = acc[k];
    if (hist_mc) {
        asm volatile("multimem.red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(hist_mc + step * 4 + k), "l"(v) : "memory");
    } else {
        for (int p = 0; p < world; ++p)
            atomicAdd_system(reinterpret_cast<unsigned long long *>(hist_ptrs[p] + step * 4 + k), (unsigned long long)v);
    }
    __threadfence_system();
}

}  // namespace g2v

using namespace g2v;

extern "C" int g2v_cbow_loop_init(int64_t *ctl, int64_t max_steps, int32_t early_stop, void *stream) {
    G2V_REQUIRE(ctl && max_steps >= 1, "g2v_cbow_loop_init: bad arguments");
    const long long h[8] = {0, 0, -1, -1, (long long)max_steps, early_stop ? 1 : 0, 0, 0};
    G2V_CUDA_OK(cudaMemcpyAsync(ctl, h, sizeof(h), cudaMemcpyHostToDevice, (cudaStream_t)stream));
    G2V_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));        // h is on this call's stack
    return 0;
}

extern "C" int g2v_cbow_loop_attach(const int64_t *ctl) {
    // the low 32 bits of ctl[0] (little endian) are the `stopped` word every step kernel tests
    set_loop_skip_flag(reinterpret_cast<const int32_t *>(ctl));
    return 0;
}

extern "C" int g2v_cbow_loop_begin(const int64_t *ctl, int64_t *acc, const float *W_ih, float *snapshot, int64_t n,
                                   void *stream) {
    G2V_REQUIRE(ctl && acc && n >= 0 && (snapshot == nullptr || W_ih), "g2v_cbow_loop_begin: bad arguments");
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    int64_t blocks = snapshot ? (n / 4 + 255) / 256 : 1;
    if (blocks > (int64_t)dp.sm_count * 8) blocks = (int64_t)dp.sm_count * 8;
    if (blocks < 1) blocks = 1;
    loop_begin_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const long long *>(ctl), reinterpret_cast<long long *>(acc),
        reinterpret_cast<const float4 *>(W_ih), reinterpret_cast<float4 *>(snapshot), n >> 2, W_ih, snapshot, n);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_loop_counters_nvl(const int64_t *ctl, const int64_t *acc, int64_t *const *hist_ptrs_dev,
                                          int64_t *hist_multicast, int32_t world, void *stream) {
    G2V_REQUIRE(ctl && acc && hist_ptrs_dev && world >= 1, "g2v_cbow_loop_counters_nvl: bad arguments");
    loop_counters_nvl_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const long long *>(ctl), reinterpret_cast<const long long *>(acc),
        reinterpret_cast<long long *const *>(hist_ptrs_dev), reinterpret_cast<long long *>(hist_multicast), world);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_loop_decide(int64_t *ctl, const int64_t *acc, int64_t *hist, void *stream) {
    G2V_REQUIRE(ctl && hist, "g2v_cbow_loop_decide: null pointer");
    loop_decide_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<long long *>(ctl),
                                                          reinterpret_cast<const long long *>(acc),
                                                          reinterpret_cast<long long *>(hist));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_fwdbwd(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                               const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total,
                               const float *W_ih, const float *W_ho, float *g_ih, float *g_ho,
                               double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                               void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_win >= 0 && win_begin >= 0, "g2v_cbow_fwdbwd: bad sizes (V=%d D=%d n_win=%lld)", V, D, (long long)n_win);
    G2V_REQUIRE(rowptr && label && W_ih && W_ho && g_ih && g_ho, "g2v_cbow_fwdbwd: null pointer");
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "g2v_cbow_fwdbwd: unknown reduce %d", reduce);
    if (n_win == 0) return 0;
    return launch_rows<true>(rowptr, gene, label, win, win_begin, n_win, inv_n_total, W_ih, W_ho, g_ih, g_ho,
                             loss_sum, n_correct, D, reduce, (cudaStream_t)stream);
}

extern "C" int g2v_cbow_fwdbwd_csc(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                   const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                   const float *W_ho, const int32_t *cscptr, const int32_t *csc_pos, float *dO,
                                   float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V,
                                   int32_t D, int32_t reduce, void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_win >= 0, "g2v_cbow_fwdbwd_csc: bad sizes (V=%d D=%d n_win=%lld)", V, D, (long long)n_win);
    G2V_REQUIRE(rowptr && label && W_ih && W_ho && cscptr && dO && g_ih && g_ho, "g2v_cbow_fwdbwd_csc: null pointer");
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "g2v_cbow_fwdbwd_csc: unknown reduce %d", reduce);
    if (n_win == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = launch_rows<true>(rowptr, gene, label, win, 0, n_win, inv_n_total, W_ih, W_ho, g_ih, g_ho, loss_sum,
                               n_correct, D, reduce, st, dO);
    if (rc) return rc;
    int grid = 0;
    if ((rc = rows_grid((const void *)cbow_csc_expand_kernel, 0, V, &grid))) return rc;
    cbow_csc_expand_kernel<<<grid, kCbowWarps * 32, 0, st>>>(cscptr, csc_pos, dO, W_ho, g_ih, V, D, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_eval(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                             const int32_t *win, int64_t win_begin, int64_t n_win, const float *W_ih,
                             const float *W_ho, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                             void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_win >= 0 && win_begin >= 0, "g2v_cbow_eval: bad sizes");
    G2V_REQUIRE(rowptr && label && W_ih && W_ho && n_correct, "g2v_cbow_eval: null pointer");
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "g2v_cbow_eval: unknown reduce %d", reduce);
    if (n_win == 0) return 0;
    return launch_rows<false>(rowptr, gene, label, win, win_begin, n_win, 0.f, W_ih, W_ho, nullptr, nullptr,
                              nullptr, n_correct, D, reduce, (cudaStream_t)stream);
}

__global__ void adam_tick_kernel(float *state, float lr, float beta1, float beta2, const int32_t *skip) {
    G2V_SKIP_IF_STOPPED(skip);
    // TF1's beta1_power / beta2_power variables, advanced once per optimizer step on the device
    const float b1p = state[0] * beta1, b2p = state[1] * beta2;
    state[0] = b1p; state[1] = b2p;
    state[2] = lr * sqrtf(1.f - b2p) / (1.f - b1p);
}

extern "C" int g2v_cbow_adam_tick(float *state, float lr, float beta1, float beta2, void *stream) {
    G2V_REQUIRE(state != nullptr, "g2v_cbow_adam_tick: null pointer");
    adam_tick_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state, lr, beta1, beta2, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_update(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                               float *g_ih, float *g_ho, int32_t V, int32_t D, int32_t optimizer, float lr,
                               float beta1, float beta2, float eps, int32_t t, const float *alpha_dev,
                               void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && (t >= 1 || alpha_dev), "g2v_cbow_update: bad sizes (V=%d D=%d t=%d)", V, D, t);
    G2V_REQUIRE(W_ih && W_ho && g_ih && g_ho, "g2v_cbow_update: null pointer");
    G2V_REQUIRE(optimizer == G2V_OPT_ADAM_TF1 || optimizer == G2V_OPT_SGD, "g2v_cbow_update: unknown optimizer %d", optimizer);
    G2V_REQUIRE(optimizer == G2V_OPT_SGD || (m_ih && v_ih && m_ho && v_ho), "g2v_cbow_update: Adam needs m/v buffers");
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    const int64_t n = (int64_t)V * D;
    int64_t blocks = (n / 4 + 255) / 256;
    const int64_t cap = (int64_t)dp.sm_count * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (optimizer == G2V_OPT_ADAM_TF1) {
        // beta^t by repeated float32 multiplication, as TF1's beta1_power / beta2_power variables
        float b1p = 1.f, b2p = 1.f;
        for (int i = 0; i < t; ++i) { b1p *= beta1; b2p *= beta2; }
        const float alpha = alpha_dev ? 0.f : lr * sqrtf(1.f - b2p) / (1.f - b1p);
        cbow_update_kernel<G2V_OPT_ADAM_TF1><<<(unsigned)blocks, 256, 0, st>>>(
            W_ih, m_ih, v_ih, g_ih, n, W_ho, m_ho, v_ho, g_ho, (int64_t)D, alpha, 1.f - beta1, 1.f - beta2, eps,
            alpha_dev, loop_skip_flag());
    } else {
        cbow_update_kernel<G2V_OPT_SGD><<<(unsigned)blocks, 256, 0, st>>>(
            W_ih, nullptr, nullptr, g_ih, n, W_ho, nullptr, nullptr, g_ho, (int64_t)D, lr, 0.f, 0.f, 0.f, nullptr, loop_skip_flag());
    }
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_update_nvl(float *const *g_ptrs_dev, float *const *w_ptrs_dev, float *g_multicast,
                                   float *w_multicast, float *m_flat, float *v_flat, int64_t n, int32_t rank,
                                   int32_t world, int32_t optimizer, float lr, float beta1, float beta2, float eps,
                                   int32_t t, const float *alpha_dev, void *stream) {
    G2V_REQUIRE(n > 0 && world >= 1 && rank >= 0 && rank < world && (t >= 1 || alpha_dev), "g2v_cbow_update_nvl: bad sizes");
    G2V_REQUIRE(g_ptrs_dev && w_ptrs_dev, "g2v_cbow_update_nvl: null pointer tables");
    G2V_REQUIRE((g_multicast == nullptr) == (w_multicast == nullptr), "g2v_cbow_update_nvl: both or neither multicast pointer");
    G2V_REQUIRE(optimizer == G2V_OPT_ADAM_TF1 || optimizer == G2V_OPT_SGD, "g2v_cbow_update_nvl: unknown optimizer %d", optimizer);
    G2V_REQUIRE(optimizer == G2V_OPT_SGD || (m_flat && v_flat), "g2v_cbow_update_nvl: Adam needs m/v buffers");
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    const int64_t own = ((n >> 2) + world - 1) / world;
    int64_t blocks = (own + 255) / 256;
    const int64_t cap = (int64_t)dp.sm_count * 4;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    cudaStream_t st = (cudaStream_t)stream;
    const bool mc = g_multicast != nullptr;
    float alpha = lr, omb1 = 0.f, omb2 = 0.f;
    if (optimizer == G2V_OPT_ADAM_TF1) {
        float b1p = 1.f, b2p = 1.f;
        for (int i = 0; i < t; ++i) { b1p *= beta1; b2p *= beta2; }
        alpha = alpha_dev ? 0.f : lr * sqrtf(1.f - b2p) / (1.f - b1p);
        omb1 = 1.f - beta1; omb2 = 1.f - beta2;
    } else {
        alpha_dev = nullptr;
    }
#define G2V_NVL(OPT, MC)                                                                                              \
    cbow_update_nvl_kernel<OPT, MC><<<(unsigned)blocks, 256, 0, st>>>(g_ptrs_dev, w_ptrs_dev, g_multicast, w_multicast, \
                                                                      m_flat, v_flat, n, rank, world, alpha, omb1, omb2, \
                                                                      eps, alpha_dev, loop_skip_flag())
    if (optimizer == G2V_OPT_ADAM_TF1) { if (mc) G2V_NVL(G2V_OPT_ADAM_TF1, true); else G2V_NVL(G2V_OPT_ADAM_TF1, false); }
    else { if (mc) G2V_NVL(G2V_OPT_SGD, true); else G2V_NVL(G2V_OPT_SGD, false); }
#undef G2V_NVL
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_step_host(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                  int64_t n_win, int64_t nnz, float *W_ih, float *W_ho, float *m_ih,
                                  float *v_ih, float *m_ho, float *v_ho, int32_t V, int32_t D,
                                  int32_t optimizer, int32_t reduce, float lr, float beta1, float beta2,
                                  float eps, int32_t t, double *loss_sum, int64_t *n_correct) {
    G2V_REQUIRE(V > 0 && D > 0 && n_win > 0 && nnz >= 0, "g2v_cbow_step_host: bad sizes");
    G2V_REQUIRE(optimizer == G2V_OPT_SGD || (m_ih && v_ih && m_ho && v_ho), "g2v_cbow_step_host: Adam needs m/v");
    const size_t nW = (size_t)V * D * sizeof(float), nD = (size_t)D * sizeof(float);
    const bool adam = optimizer == G2V_OPT_ADAM_TF1;
    // one slab: rowptr | gene | label | W | Wo | m | v | mo | vo | g | go | loss | correct
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    const size_t o_rp = take(sizeof(int32_t) * (size_t)(n_win + 1)), o_ge = take(sizeof(int32_t) * (size_t)(nnz ? nnz : 1)),
                 o_la = take((size_t)n_win), o_W = take(nW), o_Wo = take(nD), o_m = take(nW), o_v = take(nW),
                 o_mo = take(nD), o_vo = take(nD), o_g = take(nW), o_go = take(nD), o_ls = take(8), o_nc = take(8);
    char *d = nullptr;
    cudaStream_t st = nullptr;
    int rc = 1;
    do {
        if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) break;
        if (cudaMalloc(&d, off) != cudaSuccess) break;
#define H2D(dst, src, bytes) if (cudaMemcpyAsync(d + (dst), (src), (bytes), cudaMemcpyHostToDevice, st) != cudaSuccess) break
#define D2H(dst, src, bytes) if (cudaMemcpyAsync((dst), d + (src), (bytes), cudaMemcpyDeviceToHost, st) != cudaSuccess) break
        H2D(o_rp, rowptr, sizeof(int32_t) * (size_t)(n_win + 1));
        if (nnz) { H2D(o_ge, gene, sizeof(int32_t) * (size_t)nnz); }
        H2D(o_la, label, (size_t)n_win);
        H2D(o_W, W_ih, nW); H2D(o_Wo, W_ho, nD);
        if (adam) { H2D(o_m, m_ih, nW); H2D(o_v, v_ih, nW); H2D(o_mo, m_ho, nD); H2D(o_vo, v_ho, nD); }
        if (cudaMemsetAsync(d + o_g, 0, off - o_g, st) != cudaSuccess) break;
        rc = g2v_cbow_fwdbwd((int32_t *)(d + o_rp), (int32_t *)(d + o_ge), (uint8_t *)(d + o_la), nullptr, 0, n_win,
                             1.0f / (float)n_win, (float *)(d + o_W), (float *)(d + o_Wo), (float *)(d + o_g),
                             (float *)(d + o_go), (double *)(d + o_ls), (int64_t *)(d + o_nc), V, D, reduce, st);
        if (rc) break;
        rc = g2v_cbow_update((float *)(d + o_W), (float *)(d + o_Wo), (float *)(d + o_m), (float *)(d + o_v),
                             (float *)(d + o_mo), (float *)(d + o_vo), (float *)(d + o_g), (float *)(d + o_go), V, D,
                             optimizer, lr, beta1, beta2, eps, t, nullptr, st);
        if (rc) break;
        rc = 1;
        D2H(W_ih, o_W, nW); D2H(W_ho, o_Wo, nD);
        if (adam) { D2H(m_ih, o_m, nW); D2H(v_ih, o_v, nW); D2H(m_ho, o_mo, nD); D2H(v_ho, o_vo, nD); }
        if (loss_sum) { D2H(loss_sum, o_ls, 8); }
        if (n_correct) { D2H(n_correct, o_nc, 8); }
#undef H2D
#undef D2H
        if (cudaStreamSynchronize(st) != cudaSuccess) break;
        rc = 0;
    } while (0);
    if (rc == 1) set_error("g2v_cbow_step_host: CUDA failure: %s", cudaGetErrorString(cudaGetLastError()));
    cudaFree(d);
    if (st) cudaStreamDestroy(st);
    return rc;
}
