// g2v_cbow_rank1.cu -- HOT PATH 2, collapsed form (SURVEY.md 8f-3).
//
// The reference's model has no nonlinearity:  O = (X.W_ih).W_ho = X.(W_ih.W_ho)  (G2Vec.py:239-240).
// With  s = W_ih.W_ho  [V]  and  c = X^T.dO  [V]  the same optimizer step is, exactly,
//     o[n]     = sum_{g in window n} s[g]
//     dO[n]    = (sigmoid(o[n]) - y[n]) / N
//     dW_ih[g] = c[g] * W_ho            (rank-1: the dense [V,D] gradient is never formed)
//     dW_ho    = W_ih^T . c
// so the per-window work touches 4-byte scalars instead of D-wide rows, and the only dense traffic
// is the optimizer pass itself.  Results differ from the row formulation by float32 reassociation only
// (tests/test_gpu_cbow.py holds both to the same oracle and tolerance).
//
//   r1_prepare_kernel   s[g] = <W_ih[g,:], W_ho>                        reads 4*V*D
//   r1_windows_kernel   per window: gather s, logit, loss/acc, dO, c[g] += dO   12*l + 5 bytes / window
//   r1_update_kernel    per row: g = c[g]*W_ho, g_ho += c[g]*W_ih[g,:], Adam/SGD on the row   24*V*D (Adam)
//   r1_update_ho_kernel Adam/SGD on W_ho from g_ho
// Multi-GPU exchanges only c (4*V bytes) per step instead of the dense gradient (4*V*D bytes).
#include "g2v_cbow_common.cuh"

namespace g2v {

// ---- s = W_ih . W_ho ----------------------------------------------------------------------------
// WITH_T (the certified accuracy pass of g2v_cbow.cu, DESIGN.md §4.16): also t[g] = sum_d |W_ih[g,d] * W_ho[d]|,
// +inf when an element of the row has magnitude > 2^64, stored as the float2 {s[g], t[g]}.
template <bool WITH_T>
__global__ void __launch_bounds__(kCbowWarps * 32)
r1_prepare_kernel(const float *__restrict__ W_ih, const float *__restrict__ W_ho, float *__restrict__ s,
                  int32_t V, int32_t D, const int32_t *__restrict__ skip) {
    G2V_SKIP_IF_STOPPED(skip);
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * kCbowWarps + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * kCbowWarps;
    const bool vec4 = (D & 3) == 0;
    for (int64_t g = warp; g < V; g += nwarps) {
        const float *row = W_ih + (size_t)g * D;
        float part = 0.f, tpart = 0.f;
        bool big = false;
        if (vec4) {
            const float4 *r4 = reinterpret_cast<const float4 *>(row);
            const float4 *h4 = reinterpret_cast<const float4 *>(W_ho);
            for (int i = lane; i < (D >> 2); i += 32) {
                const float4 a = __ldg(r4 + i), b = __ldg(h4 + i);
                part += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
                if (WITH_T) {
                    tpart += fabsf(__fmul_rn(a.x, b.x)) + fabsf(__fmul_rn(a.y, b.y)) + fabsf(__fmul_rn(a.z, b.z))
                             + fabsf(__fmul_rn(a.w, b.w));
                    big |= fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))) > 0x1p64f;
                }
            }
        } else {
            for (int d = lane; d < D; d += 32) {
                const float a = __ldg(row + d), b = __ldg(W_ho + d);
                part += a * b;
                if (WITH_T) {
                    tpart += fabsf(__fmul_rn(a, b));
                    big |= fabsf(a) > 0x1p64f;
                }
            }
        }
        part = warp_sum(part);
        if (WITH_T) {
            tpart = warp_sum(tpart);
            if (__any_sync(0xffffffffu, big)) tpart = __int_as_float(0x7f800000);
            if (lane == 0) reinterpret_cast<float2 *>(s)[g] = make_float2(part, tpart);
        } else if (lane == 0) {
            s[g] = part;
        }
    }
}

// ---- per-window forward (+ backward into c) -------------------------------------------------------
// MODE 0: accuracy only.  MODE 1: backward with c[gene] += dO (scalar red).  MODE 2: backward that only
// stores dO[i] for list position i; c is then formed without atomics by r1_csc_reduce_kernel.
// CW (backward): the class-weighted dO and loss (class_weighted, DESIGN.md §4.20) with weights cw.
template <int MODE, bool CW>
__global__ void __launch_bounds__(kCbowWarps * 32)
r1_windows_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                  const uint8_t *__restrict__ label, const int32_t *__restrict__ win, int64_t win_begin,
                  int64_t n_win, float inv_n, const float *__restrict__ s, float *__restrict__ c,
                  double *__restrict__ loss_sum, unsigned long long *__restrict__ n_correct,
                  int32_t reduce_mean, const int32_t *__restrict__ skip, float2 cw) {
    G2V_SKIP_IF_STOPPED(skip);
    constexpr bool BACKWARD = MODE != 0;
    __shared__ CtaAcc sh;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & 7, slot = lane >> 3;          // 8 lanes per window, 4 windows per warp
    if (threadIdx.x == 0) { sh.loss = 0.0; sh.correct = 0ull; }
    __syncthreads();
    float loss_acc = 0.f;
    unsigned correct_acc = 0;
    const int64_t stride = (int64_t)gridDim.x * kCbowWarps * 4;
    for (int64_t base = ((int64_t)blockIdx.x * kCbowWarps + warp) * 4; base < n_win; base += stride) {
        const int64_t i = base + slot;
        const bool active = i < n_win;
        int32_t b = 0, e = 0;
        float y = 0.f;
        if (active) {
            const int64_t n = win ? (int64_t)__ldg(win + win_begin + i) : win_begin + i;
            b = __ldg(rowptr + n); e = __ldg(rowptr + n + 1);
            y = (float)__ldg(label + n);
        }
        float part = 0.f;
        for (int32_t j = b + sub; j < e; j += 8) part += __ldg(s + __ldg(gene + j));
        part += __shfl_xor_sync(0xffffffffu, part, 4);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        const float scale = (reduce_mean && e > b) ? 1.f / (float)(e - b) : 1.f;
        const float o = part * scale;
        float dO = 0.f;
        if (active && sub == 0) {                        // one lane per window does the scalar math
            correct_acc += ((o > 0.f) == (y != 0.f)) ? 1u : 0u;
            if (BACKWARD) {
                loss_acc += class_weighted<CW>(fmaxf(o, 0.f) - o * y + log1pf(expf(-fabsf(o))), y, cw);
                dO = class_weighted<CW>((sigmoid_stable(o) - y) * inv_n, y, cw) * scale;
                if (MODE == 2) c[i] = dO;                // c is the dO array here
            }
        }
        if (MODE == 1) {
            dO = __shfl_sync(0xffffffffu, dO, lane & ~7);
            for (int32_t j = b + sub; j < e; j += 8) atomicAdd(c + __ldg(gene + j), dO);
        }
    }
    loss_acc = warp_sum(loss_acc);
    correct_acc = __reduce_add_sync(0xffffffffu, correct_acc);
    if (lane == 0) {
        if (BACKWARD) atomicAdd(&sh.loss, (double)loss_acc);
        atomicAdd(&sh.correct, (unsigned long long)correct_acc);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (BACKWARD && loss_sum) atomicAdd(loss_sum, sh.loss);
        if (n_correct) atomicAdd(n_correct, sh.correct);
    }
}

// c[g] += sum over the list positions whose window contains g of dO[pos]: one warp per gene, fixed lane
// assignment and shuffle tree => bit-reproducible from run to run (no floating-point atomics).
__global__ void __launch_bounds__(kCbowWarps * 32)
r1_csc_reduce_kernel(const int32_t *__restrict__ cscptr, const int32_t *__restrict__ csc_pos,
                     const float *__restrict__ dO, float *__restrict__ c, int32_t V,
                     const int32_t *__restrict__ skip) {
    G2V_SKIP_IF_STOPPED(skip);
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * kCbowWarps + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * kCbowWarps;
    for (int64_t g = warp; g < V; g += nwarps) {
        const int32_t b = __ldg(cscptr + g), e = __ldg(cscptr + g + 1);
        if (b == e) continue;
        const float tot = csc_segment_sum(csc_pos, dO, b, e, lane);
        if (lane == 0) c[g] += tot;
    }
}

// ---- dense optimizer pass over the rows -----------------------------------------------------------
// VEC > 0: D = 128*VEC, register accumulators for g_ho.  VEC == 0: any D, shared-memory accumulators.
// WD: every row is decayed (decay1) before its step, rows with c[g] = 0 included; g_ho takes the pre-decay row.
template <int VEC, int OPT, bool WD>
__global__ void __launch_bounds__(kCbowWarps * 32)
r1_update_kernel(float *__restrict__ W_ih, float *__restrict__ M, float *__restrict__ Vv,
                 const float *__restrict__ W_ho, float *__restrict__ c, float *__restrict__ g_part, int32_t V,
                 int32_t D, float alpha_host, float omb1, float omb2, float eps,
                 const float *__restrict__ alpha_dev, const int32_t *__restrict__ skip, float wd) {
    G2V_SKIP_IF_STOPPED(skip);
    const float alpha = alpha_dev ? __ldg(alpha_dev + 2) : alpha_host;
    // g_ho = W_ih^T . c is reduced WITHOUT atomics so that the step is bit-reproducible: every warp owns a
    // row of sh_gho, the block sums its rows in warp order into g_part[blockIdx.x][:], and
    // r1_update_ho_kernel sums the blocks in block order.
    extern __shared__ float sh_gho[];              // [kCbowWarps][D]
    const int lane = threadIdx.x & 31;
    float *my = sh_gho + (size_t)(threadIdx.x >> 5) * D;
    for (int i = threadIdx.x; i < kCbowWarps * D; i += blockDim.x) sh_gho[i] = 0.f;
    __syncthreads();
    const int64_t warp = (int64_t)blockIdx.x * kCbowWarps + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * kCbowWarps;
    if (VEC > 0) {
        constexpr int NV = VEC > 0 ? VEC : 1;  // (dead code when VEC == 0)
        float4 who[NV], acc[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
            who[v] = __ldg(reinterpret_cast<const float4 *>(W_ho) + v * 32 + lane);
            acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int64_t g = warp; g < V; g += nwarps) {
            const float cg = c[g];
            float4 *w4 = reinterpret_cast<float4 *>(W_ih + (size_t)g * D) + lane;
            float4 *m4 = reinterpret_cast<float4 *>(M + (size_t)g * D) + lane;
            float4 *v4 = reinterpret_cast<float4 *>(Vv + (size_t)g * D) + lane;
#pragma unroll
            for (int v = 0; v < NV; ++v) {
                float4 w = w4[v * 32];
                acc[v].x += cg * w.x; acc[v].y += cg * w.y; acc[v].z += cg * w.z; acc[v].w += cg * w.w;
                decay4<WD>(w, wd);
                if (OPT == G2V_OPT_ADAM_TF1) {
                    float4 m = m4[v * 32], vv = v4[v * 32];
                    adam1(w.x, m.x, vv.x, cg * who[v].x, alpha, omb1, omb2, eps);
                    adam1(w.y, m.y, vv.y, cg * who[v].y, alpha, omb1, omb2, eps);
                    adam1(w.z, m.z, vv.z, cg * who[v].z, alpha, omb1, omb2, eps);
                    adam1(w.w, m.w, vv.w, cg * who[v].w, alpha, omb1, omb2, eps);
                    m4[v * 32] = m; v4[v * 32] = vv;
                    w4[v * 32] = w;
                } else {
                    // SGD skips the arithmetic of a row with c[g] = 0; with WD the decayed row is still stored
                    if (cg != 0.f) {
                        w.x -= alpha * cg * who[v].x; w.y -= alpha * cg * who[v].y;
                        w.z -= alpha * cg * who[v].z; w.w -= alpha * cg * who[v].w;
                    }
                    if (WD || cg != 0.f) w4[v * 32] = w;
                }
            }
            __syncwarp();
            if (lane == 0) c[g] = 0.f;
        }
#pragma unroll
        for (int v = 0; v < NV; ++v) reinterpret_cast<float4 *>(my)[v * 32 + lane] = acc[v];
    } else {
        for (int64_t g = warp; g < V; g += nwarps) {
            const float cg = c[g];
            float *w = W_ih + (size_t)g * D;
            for (int d = lane; d < D; d += 32) {
                float x = w[d];
                if (cg != 0.f) my[d] += cg * x;            // lane-owned element of the warp's row
                decay1<WD>(x, wd);
                if (OPT == G2V_OPT_ADAM_TF1) {
                    float m = M[(size_t)g * D + d], vv = Vv[(size_t)g * D + d];
                    adam1(x, m, vv, cg * __ldg(W_ho + d), alpha, omb1, omb2, eps);
                    M[(size_t)g * D + d] = m; Vv[(size_t)g * D + d] = vv;
                } else {
                    x -= alpha * cg * __ldg(W_ho + d);
                }
                w[d] = x;
            }
            __syncwarp();
            if (lane == 0) c[g] = 0.f;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
        float x = 0.f;
#pragma unroll
        for (int w = 0; w < kCbowWarps; ++w) x += sh_gho[(size_t)w * D + i];
        g_part[(size_t)blockIdx.x * D + i] = x;
    }
}

// W_ho step: g_ho[i] = sum over the update kernel's blocks of g_part[p][i], in a fixed order (32 interleaved
// slices, then the slices in order) so the result is bit-reproducible, then TF1 Adam / SGD.
template <int OPT, bool WD>
__global__ void __launch_bounds__(1024)
r1_update_ho_kernel(float *__restrict__ W_ho, float *__restrict__ m, float *__restrict__ v,
                    const float *__restrict__ g_part, int32_t n_part, int32_t D, float alpha_host, float omb1,
                    float omb2, float eps, const float *__restrict__ alpha_dev, const int32_t *__restrict__ skip,
                    float wd) {
    G2V_SKIP_IF_STOPPED(skip);
    const float alpha = alpha_dev ? __ldg(alpha_dev + 2) : alpha_host;
    __shared__ float sh[32][33];
    const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + lane;
    float a = 0.f;
    if (i < D)
        for (int p = slice; p < n_part; p += 32) a += g_part[(size_t)p * D + i];
    sh[slice][lane] = a;
    __syncthreads();
    if (slice == 0 && i < D) {
        float g = 0.f;
#pragma unroll
        for (int q = 0; q < 32; ++q) g += sh[q][lane];
        float w = W_ho[i];
        decay1<WD>(w, wd);
        if (OPT == G2V_OPT_ADAM_TF1) {
            float mm = m[i], vv = v[i];
            adam1(w, mm, vv, g, alpha, omb1, omb2, eps);
            m[i] = mm; v[i] = vv;
        } else {
            w -= alpha * g;
        }
        W_ho[i] = w;
    }
}

}  // namespace g2v

using namespace g2v;

namespace g2v {
int launch_r1_prepare(const float *W_ih, const float *W_ho, float *s, int32_t V, int32_t D, bool with_t,
                      cudaStream_t stream) {
    const void *kern = with_t ? (const void *)r1_prepare_kernel<true> : (const void *)r1_prepare_kernel<false>;
    int grid = 0, rc;
    if ((rc = rows_grid(kern, 0, V, &grid))) return rc;
    if (with_t)
        r1_prepare_kernel<true><<<grid, kCbowWarps * 32, 0, stream>>>(W_ih, W_ho, s, V, D, loop_skip_flag());
    else
        r1_prepare_kernel<false><<<grid, kCbowWarps * 32, 0, stream>>>(W_ih, W_ho, s, V, D, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
}  // namespace g2v

extern "C" int g2v_cbow_r1_prepare(const float *W_ih, const float *W_ho, float *s, int32_t V, int32_t D,
                                   void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && W_ih && W_ho && s, "g2v_cbow_r1_prepare: bad arguments");
    return launch_r1_prepare(W_ih, W_ho, s, V, D, false, (cudaStream_t)stream);
}

// One body for the plain and the class-weighted (_cw, DESIGN.md §4.20) forms; `name` is the entry point's, for errors.
// c == NULL: the accuracy pass, which has no class weights.
template <bool CW>
static int r1_windows_impl(const char *name, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                           const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total, const float *s,
                           float *c, double *loss_sum, int64_t *n_correct, int32_t V, int32_t reduce, float2 cw,
                           void *stream) {
    G2V_REQUIRE(V > 0 && n_win >= 0 && win_begin >= 0, "%s: bad sizes", name);
    G2V_REQUIRE(rowptr && label && s, "%s: null pointer", name);
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "%s: unknown reduce %d", name, reduce);
    if (n_win == 0) return 0;
    unsigned long long *nc = reinterpret_cast<unsigned long long *>(n_correct);
    int grid = 0, rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (c) {
        if ((rc = rows_grid((const void *)r1_windows_kernel<1, CW>, 0, (n_win + 3) / 4, &grid))) return rc;
        r1_windows_kernel<1, CW><<<grid, kCbowWarps * 32, 0, st>>>(rowptr, gene, label, win, win_begin, n_win,
                                                                  inv_n_total, s, c, loss_sum, nc, reduce,
                                                                  loop_skip_flag(), cw);
    } else {
        if ((rc = rows_grid((const void *)r1_windows_kernel<0, false>, 0, (n_win + 3) / 4, &grid))) return rc;
        r1_windows_kernel<0, false><<<grid, kCbowWarps * 32, 0, st>>>(rowptr, gene, label, win, win_begin, n_win, 0.f,
                                                                     s, nullptr, nullptr, nc, reduce, loop_skip_flag(),
                                                                     cw);
    }
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_r1_windows(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                   const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total,
                                   const float *s, float *c, double *loss_sum, int64_t *n_correct, int32_t V,
                                   int32_t reduce, void *stream) {
    return r1_windows_impl<false>("g2v_cbow_r1_windows", rowptr, gene, label, win, win_begin, n_win, inv_n_total, s, c,
                                  loss_sum, n_correct, V, reduce, float2{1.f, 1.f}, stream);
}

extern "C" int g2v_cbow_r1_windows_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                      const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total,
                                      const float *s, float *c, double *loss_sum, int64_t *n_correct, int32_t V,
                                      int32_t reduce, float w0, float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_r1_windows_cw");
    return r1_windows_impl<true>("g2v_cbow_r1_windows_cw", rowptr, gene, label, win, win_begin, n_win, inv_n_total, s,
                                 c, loss_sum, n_correct, V, reduce, float2{w0, w1}, stream);
}

template <bool CW>
static int r1_windows_csc_impl(const char *name, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                               const int32_t *win, int64_t n_win, float inv_n_total, const float *s,
                               const int32_t *cscptr, const int32_t *csc_pos, float *dO, float *c, double *loss_sum,
                               int64_t *n_correct, int32_t V, int32_t reduce, float2 cw, void *stream) {
    G2V_REQUIRE(V > 0 && n_win >= 0, "%s: bad sizes", name);
    G2V_REQUIRE(rowptr && label && s && cscptr && dO && c, "%s: null pointer", name);
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "%s: unknown reduce %d", name, reduce);
    if (n_win == 0) return 0;
    unsigned long long *nc = reinterpret_cast<unsigned long long *>(n_correct);
    int grid = 0, rc;
    cudaStream_t st = (cudaStream_t)stream;
    if ((rc = rows_grid((const void *)r1_windows_kernel<2, CW>, 0, (n_win + 3) / 4, &grid))) return rc;
    r1_windows_kernel<2, CW><<<grid, kCbowWarps * 32, 0, st>>>(rowptr, gene, label, win, 0, n_win, inv_n_total, s, dO,
                                                              loss_sum, nc, reduce, loop_skip_flag(), cw);
    G2V_CUDA_OK(cudaGetLastError());
    if ((rc = rows_grid((const void *)r1_csc_reduce_kernel, 0, V, &grid))) return rc;
    r1_csc_reduce_kernel<<<grid, kCbowWarps * 32, 0, st>>>(cscptr, csc_pos, dO, c, V, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch(2);
    return 0;
}

extern "C" int g2v_cbow_r1_windows_csc(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                       const int32_t *win, int64_t n_win, float inv_n_total, const float *s,
                                       const int32_t *cscptr, const int32_t *csc_pos, float *dO, float *c,
                                       double *loss_sum, int64_t *n_correct, int32_t V, int32_t reduce,
                                       void *stream) {
    return r1_windows_csc_impl<false>("g2v_cbow_r1_windows_csc", rowptr, gene, label, win, n_win, inv_n_total, s,
                                      cscptr, csc_pos, dO, c, loss_sum, n_correct, V, reduce, float2{1.f, 1.f}, stream);
}

extern "C" int g2v_cbow_r1_windows_csc_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                          const int32_t *win, int64_t n_win, float inv_n_total, const float *s,
                                          const int32_t *cscptr, const int32_t *csc_pos, float *dO, float *c,
                                          double *loss_sum, int64_t *n_correct, int32_t V, int32_t reduce, float w0,
                                          float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_r1_windows_csc_cw");
    return r1_windows_csc_impl<true>("g2v_cbow_r1_windows_csc_cw", rowptr, gene, label, win, n_win, inv_n_total, s,
                                     cscptr, csc_pos, dO, c, loss_sum, n_correct, V, reduce, float2{w0, w1}, stream);
}

constexpr int kR1MaxParts = 1024;   // upper bound on the update kernel's grid (scratch = kR1MaxParts * D floats)

template <int VEC, int OPT, bool WD>
static int launch_r1_update(float *W_ih, float *M, float *Vv, const float *W_ho, float *c, float *g_ho, int32_t V,
                            int32_t D, float alpha, float omb1, float omb2, float eps, const float *alpha_dev,
                            float wd, cudaStream_t st, int *grid_out) {
    const size_t smem = (size_t)kCbowWarps * D * sizeof(float);
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    G2V_REQUIRE(smem <= (size_t)dp.max_smem_optin, "sizeHiddenlayer %d too large", D);
    if (smem > 48 * 1024)
        G2V_CUDA_OK(cudaFuncSetAttribute(r1_update_kernel<VEC, OPT, WD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
    int grid = 0, rc;
    if ((rc = rows_grid((const void *)r1_update_kernel<VEC, OPT, WD>, smem, V, &grid))) return rc;
    if (grid > kR1MaxParts) grid = kR1MaxParts;
    r1_update_kernel<VEC, OPT, WD><<<grid, kCbowWarps * 32, smem, st>>>(W_ih, M, Vv, W_ho, c, g_ho, V, D, alpha, omb1,
                                                                        omb2, eps, alpha_dev, loop_skip_flag(), wd);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    *grid_out = grid;
    return 0;
}

extern "C" size_t g2v_cbow_r1_scratch_bytes(int32_t D) { return (size_t)kR1MaxParts * (size_t)(D > 0 ? D : 1) * sizeof(float); }

extern "C" int g2v_cbow_r1_update_wd(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                                     float *c, float *g_ho, float *s, int32_t V, int32_t D, int32_t optimizer,
                                     float lr, float beta1, float beta2, float eps, float weight_decay, int32_t t,
                                     const float *alpha_dev, void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && (t >= 1 || alpha_dev), "g2v_cbow_r1_update: bad sizes (V=%d D=%d t=%d)", V, D, t);
    if (optimizer != G2V_OPT_ADAM_TF1) alpha_dev = nullptr;
    G2V_REQUIRE(W_ih && W_ho && c && g_ho && s, "g2v_cbow_r1_update: null pointer");
    G2V_REQUIRE(optimizer == G2V_OPT_ADAM_TF1 || optimizer == G2V_OPT_SGD, "g2v_cbow_r1_update: unknown optimizer %d", optimizer);
    G2V_REQUIRE(optimizer == G2V_OPT_SGD || (m_ih && v_ih && m_ho && v_ho), "g2v_cbow_r1_update: Adam needs m/v buffers");
    G2V_REQUIRE(weight_decay_ok(weight_decay),
                "g2v_cbow_r1_update_wd: weight_decay must be finite with 0 <= wd < 1 (got %g)", (double)weight_decay);
    cudaStream_t st = (cudaStream_t)stream;
    const bool adam = optimizer == G2V_OPT_ADAM_TF1;
    float alpha = lr, omb1 = 0.f, omb2 = 0.f;
    if (adam) {
        alpha = adam_tf1_alpha(lr, beta1, beta2, t);
        omb1 = 1.f - beta1; omb2 = 1.f - beta2;
    } else {
        m_ih = v_ih = m_ho = v_ho = nullptr;
    }
    int rc = 0, parts = 0;
#define G2V_R1(OPT, WD)                                                                                               \
    do {                                                                                                              \
        if (D == 128) rc = launch_r1_update<1, OPT, WD>(W_ih, m_ih, v_ih, W_ho, c, g_ho, V, D, alpha, omb1, omb2, eps, \
                                                        alpha_dev, weight_decay, st, &parts);                         \
        else if (D == 256) rc = launch_r1_update<2, OPT, WD>(W_ih, m_ih, v_ih, W_ho, c, g_ho, V, D, alpha, omb1, omb2, \
                                                             eps, alpha_dev, weight_decay, st, &parts);               \
        else if (D == 512) rc = launch_r1_update<4, OPT, WD>(W_ih, m_ih, v_ih, W_ho, c, g_ho, V, D, alpha, omb1, omb2, \
                                                             eps, alpha_dev, weight_decay, st, &parts);               \
        else rc = launch_r1_update<0, OPT, WD>(W_ih, m_ih, v_ih, W_ho, c, g_ho, V, D, alpha, omb1, omb2, eps,          \
                                               alpha_dev, weight_decay, st, &parts);                                  \
        if (rc) return rc;                                                                                            \
        r1_update_ho_kernel<OPT, WD><<<(D + 31) / 32, 1024, 0, st>>>(W_ho, m_ho, v_ho, g_ho, parts, D, alpha, omb1,    \
                                                                     omb2, eps, alpha_dev, loop_skip_flag(),          \
                                                                     weight_decay);                                   \
    } while (0)
    if (adam) { if (weight_decay > 0.f) G2V_R1(G2V_OPT_ADAM_TF1, true); else G2V_R1(G2V_OPT_ADAM_TF1, false); }
    else { if (weight_decay > 0.f) G2V_R1(G2V_OPT_SGD, true); else G2V_R1(G2V_OPT_SGD, false); }
#undef G2V_R1
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return g2v_cbow_r1_prepare(W_ih, W_ho, s, V, D, stream);
}

extern "C" int g2v_cbow_r1_update(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                                  float *c, float *g_ho, float *s, int32_t V, int32_t D, int32_t optimizer,
                                  float lr, float beta1, float beta2, float eps, int32_t t, const float *alpha_dev,
                                  void *stream) {
    return g2v_cbow_r1_update_wd(W_ih, W_ho, m_ih, v_ih, m_ho, v_ho, c, g_ho, s, V, D, optimizer, lr, beta1, beta2, eps,
                                 0.f, t, alpha_dev, stream);
}
