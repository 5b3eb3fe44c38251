// g2v_cbow.cu -- HOT PATH 2: modified CBOW (G2Vec.py:217-286) as fused sm_90a kernels.
//
// The reference builds  H = X.W_ih ; O = H.W_ho ; cost = mean(sigmoid_BCE(O, Y))  on a dense
// multi-hot X [N, V] (99.7 % zeros) and lets TF1 autodiff + ApplyAdam train W_ih, W_ho
// (G2Vec.py:239-246).  Here X is CSR (window -> gene ids) and one warp owns one window:
//
//   cbow_rows_kernel<VEC, MODE>          D = 128*VEC, each lane owns VEC float4 of the row; MODE: eval (the
//                                         accuracy pass: gather and logit only), scatter, or CSC (below)
//     gather   h   = sum_{g in window} W_ih[g, :]          (512*VEC B coalesced per row, 8 rows in flight)
//     logit    o   = <h, W_ho>                            (warp shuffle reduction)
//     loss/acc     max(o,0) - o*y + log1p(exp(-|o|)),  (o > 0) == y
//     grad     dO  = (sigmoid(o) - y) / N                 (N known up front: no global barrier)
//     scatter  g_ih[g, :] += dO * W_ho  for g in window   (red.global.add.v4.f32, 16 B per lane)
//              g_ho       += h * dO                       (registers -> smem -> one atomic per CTA)
//   cbow_rows_kernel<VEC, kRowsCsc>       the same up to dO; then, instead of the scatter,
//                                         dO_pos[i] = dO * scale  at the window's list position i (4 B per window)
//   cbow_csc_expand_kernel                one warp per gene: c = sum of dO_pos over the gene's segment of the list's
//                                         transposed incidence (CSC), then g_ih[g, :] += c * W_ho, one plain
//                                         read-modify-write per touched row.  Exact because the model is linear:
//                                         every window adds the same row W_ho to its genes, only the scale differs.
//                                         This is the backward of a prepared full list (g2v_cbow_fwdbwd_csc): it
//                                         replaces l*D*4 bytes of L2 atomics per window by 8 bytes per incidence.
//   cbow_update_kernel                   dense epilogue over [V*D] (+[D]): TF1 Adam or SGD,
//                                         float4, zeroes the gradient for the next step
//   cbow_lazy_adam_rows_kernel            lazy (touched-row) Adam of a batch: one warp per gene the batch gathered,
//                                         c = its segmented dO sum, then TF1 Adam on the W/m/v row with g = c * W_ho;
//                                         g_ih is never materialised (g2v_cbow_fwd_do + g2v_cbow_lazy_adam)
//                                         The optimizer kernels take a bool WD: decoupled weight decay of every
//                                         element they update, fused before the step (the *_wd entry points)
//   adam_tick_kernel                      TF1's beta1_power / beta2_power / alpha_t kept on the device so
//                                         that a whole step can be replayed as one CUDA graph; adam_tick_lr_kernel
//                                         reads the learning rate from device memory as well
//   lr_plateau_kernel                     the reduce-on-plateau rule on the step's validation count (one thread)
//   val_loss_kernel                       the validation loss as an exact fixed-point integer Q from the collapsed
//                                         logits (s gathered, no rows); loop_decide[_best]_score_kernel decide on it
//
// No tensor cores: the 128..512-wide reduction is a memory-bound gather/scatter, not a dense
// contraction.  Algorithmic bytes per window: l*(8D+4)+5 with the scatter, l*(4D+12)+9 with the CSC backward
// (+ 8*D per touched gene row) (DESIGN.md), per step + 32*V*D (Adam).
#include "g2v_cbow_common.cuh"

namespace g2v {

// MODE of cbow_rows_kernel.  kRowsCsc: the backward stops at dO -- it stores dO*scale at the window's list position i
// (dO_pos[i]) instead of scattering rows into g_ih; cbow_csc_expand_kernel then sums those scalars per gene and writes
// each gene row once.
constexpr int kRowsEval = 0, kRowsScatter = 1, kRowsCsc = 2;

// carried != NULL and set: the loop's tail pass already ran this forward at these weights (g2v_cbow_loop_tail).
// CW: the training term of a window of label y is weighted by cw.{x,y}[y] (class_weighted, DESIGN.md §4.20).
template <int VEC, int MODE, bool CW>
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_rows_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                 const uint8_t *__restrict__ label, const int32_t *__restrict__ win,
                 int64_t win_begin, int64_t n_win, float inv_n, const float *__restrict__ W_ih,
                 const float *__restrict__ W_ho, float *__restrict__ g_ih, float *__restrict__ g_ho,
                 double *__restrict__ loss_sum, unsigned long long *__restrict__ n_correct,
                 int32_t reduce_mean, const int32_t *__restrict__ skip, float *__restrict__ dO_pos,
                 const int32_t *__restrict__ carried, float2 cw) {
    G2V_SKIP_IF_STOPPED(skip);
    G2V_SKIP_IF_STOPPED(carried);
    constexpr bool BACKWARD = MODE != kRowsEval;
    constexpr int D = 128 * VEC;
    __shared__ float sh_gho[BACKWARD ? D : 1];
    __shared__ CtaAcc sh_acc;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (BACKWARD) for (int i = threadIdx.x; i < D; i += blockDim.x) sh_gho[i] = 0.f;
    if (threadIdx.x == 0) { sh_acc.loss = 0.0; sh_acc.correct = 0ull; }
    __syncthreads();

    const float4 *__restrict__ W4 = reinterpret_cast<const float4 *>(W_ih);
    float4 who[VEC], gho[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
        who[v] = ldg4(reinterpret_cast<const float4 *>(W_ho) + v * 32 + lane);
        gho[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    unsigned correct_acc = 0;
    float loss_acc = 0.f;

    const int64_t warps_total = (int64_t)gridDim.x * kCbowWarps;
    for (int64_t i = (int64_t)blockIdx.x * kCbowWarps + warp; i < n_win; i += warps_total) {
        const int64_t n = win ? (int64_t)__ldg(win + win_begin + i) : win_begin + i;
        const int32_t b = __ldg(rowptr + n), e = __ldg(rowptr + n + 1);
        const float y = (float)__ldg(label + n);
        float4 h[VEC];
        float scale;
        const float o = rows_logit<VEC>(gene, W4, b, e, lane, reduce_mean, who, h, scale);
        if (lane == 0) {
            correct_acc += ((o > 0.f) == (y != 0.f)) ? 1u : 0u;
            if (BACKWARD) loss_acc += class_weighted<CW>(fmaxf(o, 0.f) - o * y + log1pf(expf(-fabsf(o))), y, cw);
        }
        if (MODE == kRowsCsc) {
            const float dO = class_weighted<CW>((sigmoid_stable(o) - y) * inv_n, y, cw);
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
                gho[v].x += h[v].x * dO; gho[v].y += h[v].y * dO; gho[v].z += h[v].z * dO; gho[v].w += h[v].w * dO;
            }
            if (lane == 0) dO_pos[i] = dO * scale;
        } else if (MODE == kRowsScatter) {
            const float dO = class_weighted<CW>((sigmoid_stable(o) - y) * inv_n, y, cw);
            float4 gv[VEC];
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
                gho[v].x += h[v].x * dO; gho[v].y += h[v].y * dO; gho[v].z += h[v].z * dO; gho[v].w += h[v].w * dO;
                const float s = dO * scale;
                gv[v] = make_float4(who[v].x * s, who[v].y * s, who[v].z * s, who[v].w * s);
            }
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
    cta_epilogue<VEC, BACKWARD, true>(sh_gho, sh_acc, gho, loss_acc, correct_acc, lane, g_ho, loss_sum, n_correct);
}

// Any D (not a multiple of 128): h and the g_ho partial live in shared memory per warp.
// dO_pos != NULL: the CSC backward of cbow_rows_kernel (dO*scale stored per list position, no scatter).
template <bool BACKWARD, bool CW>
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_rows_generic_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                         const uint8_t *__restrict__ label, const int32_t *__restrict__ win,
                         int64_t win_begin, int64_t n_win, float inv_n, const float *__restrict__ W_ih,
                         const float *__restrict__ W_ho, float *__restrict__ g_ih,
                         float *__restrict__ g_ho, double *__restrict__ loss_sum,
                         unsigned long long *__restrict__ n_correct, int32_t D, int32_t reduce_mean,
                         const int32_t *__restrict__ skip, float *__restrict__ dO_pos,
                         const int32_t *__restrict__ carried, float2 cw) {
    G2V_SKIP_IF_STOPPED(skip);
    G2V_SKIP_IF_STOPPED(carried);
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
        float scale;
        const float o = rows_generic_logit(gene, W_ih, W_ho, b, e, lane, D, reduce_mean, h, scale);
        if (lane == 0) {
            correct_acc += ((o > 0.f) == (y != 0.f)) ? 1u : 0u;
            if (BACKWARD) loss_acc += class_weighted<CW>(fmaxf(o, 0.f) - o * y + log1pf(expf(-fabsf(o))), y, cw);
        }
        if (BACKWARD) {
            const float dO = class_weighted<CW>((sigmoid_stable(o) - y) * inv_n, y, cw);
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

// ---- certified accuracy pass (DESIGN.md §4.16) ----------------------------------------------------------------
// The count of (o > 0) == y over the windows, the same integer cbow_rows_kernel's eval mode gives, from the collapsed
// logit o' = scale * sum_{g in n} s[g] where it provably has o's sign.  st[g] = {s[g], t[g]} (r1_prepare_kernel<true>):
// s[g] = <W_ih[g,:], W_ho>, t[g] = sum_d |W_ih[g,d] W_ho[d]|.  Both o and o' are float32 evaluations of the same real
// number with at most k = l + D + 16 roundings on any term's path, so |o - o'| <= certified_tau(T, scale, l, D, A)
// with T = sum_{g in n} t[g] and A = sum_d |W_ho[d]|; a window with |o'| > tau is decided by o', every other one
// (empty, tau or o' not finite, |o'| within the band) gets o from rows_logit / rows_generic_logit, the code
// cbow_rows_kernel runs.  The absolute term covers underflowing products: each product of o and o' may lose 2^-150,
// and in o the product scale * h[d] (mean) is then multiplied by W_ho[d], so its loss counts |W_ho[d]| times.
__device__ __forceinline__ float certified_tau(float T, float scale, int32_t l, int32_t D, float A) {
    const int64_t k = (int64_t)l + D + 16;
    if (!(T <= 0x1p126f) || k > (1 << 22)) return __int_as_float(0x7f800000);
    const float rel = __fmul_rn(__fmul_rn((float)k, 0x1p-21f), scale);           // 8 k u s, u = 2^-24
    // 32 ((l + 3) D + A) 2^-150; A = +inf or NaN makes tau so, and the window is gathered
    const float abs_ = __fmul_rn(__fadd_rn((float)(((int64_t)l + 3) * D), A), 0x1p-145f);
    return __fadd_rn(__fmul_rn(rel, T), abs_);
}

// 8 lanes per window, 4 windows per warp (r1_windows_kernel's layout) for o' and T; then the whole warp gathers the
// rows of each undecided window of the four in turn.  VEC > 0: D = 128 * VEC; VEC == 0: any D, h in shared memory
// ([kCbowWarps][D], dynamic).  force_gather: every window takes the row gather (tests).  n_gathered (nullable): the
// number of windows that took it.
template <int VEC>
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_eval_certified_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                           const uint8_t *__restrict__ label, const int32_t *__restrict__ win, int64_t win_begin,
                           int64_t n_win, const float *__restrict__ W_ih, const float *__restrict__ W_ho,
                           const float2 *__restrict__ st, unsigned long long *__restrict__ n_correct,
                           unsigned long long *__restrict__ n_gathered, int32_t D, int32_t reduce_mean,
                           int32_t force_gather, const int32_t *__restrict__ skip) {
    G2V_SKIP_IF_STOPPED(skip);
    constexpr int NV = VEC > 0 ? VEC : 1;
    extern __shared__ float shf[];
    __shared__ unsigned long long sh_cnt[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & 7, slot = lane >> 3;
    if (threadIdx.x < 2) sh_cnt[threadIdx.x] = 0ull;
    __syncthreads();
    const float4 *__restrict__ W4 = reinterpret_cast<const float4 *>(W_ih);
    float4 who[NV];
    if (VEC > 0) {
#pragma unroll
        for (int v = 0; v < NV; ++v) who[v] = ldg4(reinterpret_cast<const float4 *>(W_ho) + v * 32 + lane);
    }
    float *h_generic = shf + (size_t)warp * D;
    // A = sum_d |W_ho[d]| (certified_tau's underflow term).  VEC > 0: from the lanes' who, summed where it is first
    // needed, so that the warp does not wait for W_ho before its first window's loads are issued
    float A = 0.f;
    if (VEC == 0) {
        for (int d = lane; d < D; d += 32) A += fabsf(__ldg(W_ho + d));
        A = warp_sum(A);
    }
    unsigned correct_acc = 0, gathered_acc = 0;
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
        float ps = 0.f, pt = 0.f;
        for (int32_t j = b + sub; j < e; j += 8) {
            const float2 q = __ldg(st + __ldg(gene + j));
            ps += q.x; pt += q.y;
        }
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
            ps += __shfl_xor_sync(0xffffffffu, ps, o);
            pt += __shfl_xor_sync(0xffffffffu, pt, o);
        }
        if (VEC > 0) {
            A = 0.f;
#pragma unroll
            for (int v = 0; v < NV; ++v)
                A += (fabsf(who[v].x) + fabsf(who[v].y)) + (fabsf(who[v].z) + fabsf(who[v].w));
            A = warp_sum(A);
        }
        const float scale = (reduce_mean && e > b) ? 1.f / (float)(e - b) : 1.f;
        const float o1 = ps * scale;
        const bool decided = !force_gather && fabsf(o1) <= 0x1.fffffep127f
                             && fabsf(o1) > certified_tau(pt, scale, e - b, D, A);
        if (active && sub == 0 && decided) correct_acc += ((o1 > 0.f) == (y != 0.f)) ? 1u : 0u;
        unsigned todo = __ballot_sync(0xffffffffu, active && sub == 0 && !decided);
        while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const int32_t wb = __shfl_sync(0xffffffffu, b, src), we = __shfl_sync(0xffffffffu, e, src);
            const float wy = __shfl_sync(0xffffffffu, y, src);
            float wscale, o;
            if (VEC > 0) {
                float4 h[NV];
                o = rows_logit<NV>(gene, W4, wb, we, lane, reduce_mean, who, h, wscale);
            } else {
                o = rows_generic_logit(gene, W_ih, W_ho, wb, we, lane, D, reduce_mean, h_generic, wscale);
            }
            if (lane == 0) {
                correct_acc += ((o > 0.f) == (wy != 0.f)) ? 1u : 0u;
                ++gathered_acc;
            }
        }
    }
    correct_acc = __reduce_add_sync(0xffffffffu, correct_acc);
    if (lane == 0) {
        atomicAdd(&sh_cnt[0], (unsigned long long)correct_acc);
        atomicAdd(&sh_cnt[1], (unsigned long long)gathered_acc);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(n_correct, sh_cnt[0]);
        if (n_gathered) atomicAdd(n_gathered, sh_cnt[1]);
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

// ---- deterministic mode (DESIGN.md §4.13): the CSC forward with every floating-point sum in a fixed order ----
// The list is cut into tiles of kDetTile positions.  A CTA takes whole tiles (t = blockIdx.x, + gridDim.x, ...); inside
// tile t warp w takes positions t*kDetTile + w, + kCbowWarps, ... in order and accumulates its g_ho partial and loss from
// zero.  The warp partials are added in warp order in shared memory and stored as the tile's partial in a workspace
// (loss: double [n_tiles], then g_ho: float [n_tiles][D]); cbow_det_sum_kernel then adds the tiles in a fixed order.
// No value depends on the grid, so the result is the same bits for any number of CTAs.  dO_pos and the correct count
// are the CSC mode's (integers need no order).
constexpr int kDetTile = 64;
constexpr int kDetSumWarps = 32;

__host__ __device__ __forceinline__ size_t det_ws_loss_bytes(int64_t n_tiles) {
    return ((size_t)n_tiles * sizeof(double) + 255) & ~(size_t)255;
}

template <int VEC, bool CW>
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_rows_det_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                     const uint8_t *__restrict__ label, const int32_t *__restrict__ win, int64_t n_win, float inv_n,
                     const float *__restrict__ W_ih, const float *__restrict__ W_ho, float *__restrict__ dO_pos,
                     double *__restrict__ tile_loss, float *__restrict__ tile_gho,
                     unsigned long long *__restrict__ n_correct, int32_t reduce_mean, const int32_t *__restrict__ skip,
                     const int32_t *__restrict__ carried, float2 cw) {
    G2V_SKIP_IF_STOPPED(skip);
    G2V_SKIP_IF_STOPPED(carried);
    constexpr int D = 128 * VEC;
    constexpr int D4 = D / 4;
    constexpr int UNR = 8 / VEC;
    __shared__ float4 sh_gho[kCbowWarps][D4];
    __shared__ float sh_loss[kCbowWarps];
    __shared__ unsigned long long sh_correct;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) sh_correct = 0ull;
    __syncthreads();
    const float4 *__restrict__ W4 = reinterpret_cast<const float4 *>(W_ih);
    float4 who[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) who[v] = ldg4(reinterpret_cast<const float4 *>(W_ho) + v * 32 + lane);
    unsigned correct_acc = 0;
    const int64_t n_tiles = (n_win + kDetTile - 1) / kDetTile;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        float4 gho[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) gho[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        float loss_acc = 0.f;
        const int64_t i_end = min(n_win, (t + 1) * kDetTile);
        for (int64_t i = t * kDetTile + warp; i < i_end; i += kCbowWarps) {
            const int64_t n = __ldg(win + i);
            const int32_t b = __ldg(rowptr + n), e = __ldg(rowptr + n + 1);
            const float y = (float)__ldg(label + n);
            float4 h[VEC];
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
                loss_acc += class_weighted<CW>(fmaxf(o, 0.f) - o * y + log1pf(expf(-fabsf(o))), y, cw);
            }
            const float dO = class_weighted<CW>((sigmoid_stable(o) - y) * inv_n, y, cw);
#pragma unroll
            for (int v = 0; v < VEC; ++v) {
                gho[v].x += h[v].x * dO; gho[v].y += h[v].y * dO; gho[v].z += h[v].z * dO; gho[v].w += h[v].w * dO;
            }
            if (lane == 0) dO_pos[i] = dO * scale;
        }
#pragma unroll
        for (int v = 0; v < VEC; ++v) sh_gho[warp][v * 32 + lane] = gho[v];
        if (lane == 0) sh_loss[warp] = loss_acc;
        __syncthreads();
        float4 *out = reinterpret_cast<float4 *>(tile_gho + (size_t)t * D);
        for (int k = threadIdx.x; k < D4; k += blockDim.x) {
            float4 s = sh_gho[0][k];
#pragma unroll
            for (int w = 1; w < kCbowWarps; ++w) {
                const float4 x = sh_gho[w][k];
                s.x += x.x; s.y += x.y; s.z += x.z; s.w += x.w;
            }
            out[k] = s;
        }
        if (threadIdx.x == 0) {
            double l = 0.0;
            for (int w = 0; w < kCbowWarps; ++w) l += (double)sh_loss[w];
            tile_loss[t] = l;
        }
        __syncthreads();                                   // the next tile overwrites sh_gho / sh_loss
    }
    if (lane == 0) atomicAdd(&sh_correct, (unsigned long long)correct_acc);
    __syncthreads();
    if (threadIdx.x == 0 && n_correct) atomicAdd(n_correct, sh_correct);
}

// Any D: cbow_rows_generic_kernel's CSC mode with the tiles of cbow_rows_det_kernel.
template <bool CW>
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_rows_generic_det_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                             const uint8_t *__restrict__ label, const int32_t *__restrict__ win, int64_t n_win,
                             float inv_n, const float *__restrict__ W_ih, const float *__restrict__ W_ho,
                             float *__restrict__ dO_pos, double *__restrict__ tile_loss, float *__restrict__ tile_gho,
                             unsigned long long *__restrict__ n_correct, int32_t D, int32_t reduce_mean,
                             const int32_t *__restrict__ skip, const int32_t *__restrict__ carried, float2 cw) {
    G2V_SKIP_IF_STOPPED(skip);
    G2V_SKIP_IF_STOPPED(carried);
    extern __shared__ float shf[];
    __shared__ float sh_loss[kCbowWarps];
    __shared__ unsigned long long sh_correct;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *h = shf + (size_t)warp * 2 * D;
    float *gho = h + D;
    if (threadIdx.x == 0) sh_correct = 0ull;
    __syncthreads();
    unsigned correct_acc = 0;
    const int64_t n_tiles = (n_win + kDetTile - 1) / kDetTile;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        for (int d = lane; d < D; d += 32) gho[d] = 0.f;
        float loss_acc = 0.f;
        const int64_t i_end = min(n_win, (t + 1) * kDetTile);
        for (int64_t i = t * kDetTile + warp; i < i_end; i += kCbowWarps) {
            const int64_t n = __ldg(win + i);
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
                loss_acc += class_weighted<CW>(fmaxf(o, 0.f) - o * y + log1pf(expf(-fabsf(o))), y, cw);
            }
            const float dO = class_weighted<CW>((sigmoid_stable(o) - y) * inv_n, y, cw);
            for (int d = lane; d < D; d += 32) gho[d] += h[d] * dO;
            if (lane == 0) dO_pos[i] = dO * scale;
        }
        if (lane == 0) sh_loss[warp] = loss_acc;
        __syncthreads();
        float *out = tile_gho + (size_t)t * D;
        for (int d = threadIdx.x; d < D; d += blockDim.x) {
            float s = shf[D + d];
            for (int w = 1; w < kCbowWarps; ++w) s += shf[(size_t)w * 2 * D + D + d];
            out[d] = s;
        }
        if (threadIdx.x == 0) {
            double l = 0.0;
            for (int w = 0; w < kCbowWarps; ++w) l += (double)sh_loss[w];
            tile_loss[t] = l;
        }
        __syncthreads();
    }
    if (lane == 0) atomicAdd(&sh_correct, (unsigned long long)correct_acc);
    __syncthreads();
    if (threadIdx.x == 0 && n_correct) atomicAdd(n_correct, sh_correct);
}

// Second step of the deterministic forward: g_ho[d] += the sum of the tile partials, *loss_sum += the sum of the tile
// losses.  One CTA per 32 columns; warp w sums tiles w, w + kDetSumWarps, ... in order, then the warp sums are added
// in warp order.  The losses: CTA 0, thread j sums tiles j, j + 32*kDetSumWarps, ... in order, then a fixed shuffle
// tree per warp and the warps in order.  The launch shape depends on D only.
__global__ void __launch_bounds__(kDetSumWarps * 32)
cbow_det_sum_kernel(const double *__restrict__ tile_loss, const float *__restrict__ tile_gho, int64_t n_tiles,
                    int32_t D, float *__restrict__ g_ho, double *__restrict__ loss_sum, const int32_t *__restrict__ skip,
                    const int32_t *__restrict__ carried) {
    G2V_SKIP_IF_STOPPED(skip);
    G2V_SKIP_IF_STOPPED(carried);
    __shared__ float sh[kDetSumWarps][32];
    __shared__ double shl[kDetSumWarps];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int d = blockIdx.x * 32 + lane;
    float s = 0.f;
    if (d < D)
#pragma unroll 8
        for (int64_t t = warp; t < n_tiles; t += kDetSumWarps) s += __ldg(tile_gho + (size_t)t * D + d);
    sh[warp][lane] = s;
    if (blockIdx.x == 0) {
        double l = 0.0;
        for (int64_t t = threadIdx.x; t < n_tiles; t += kDetSumWarps * 32) l += __ldg(tile_loss + t);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
        if (lane == 0) shl[warp] = l;
    }
    __syncthreads();
    if (warp == 0) {
        if (d < D) {
            float a = sh[0][lane];
            for (int w = 1; w < kDetSumWarps; ++w) a += sh[w][lane];
            g_ho[d] += a;
        }
        if (blockIdx.x == 0 && lane == 0 && loss_sum) {
            double a = shl[0];
            for (int w = 1; w < kDetSumWarps; ++w) a += shl[w];
            *loss_sum += a;
        }
    }
}

// The CSC expansion on one batch's plan (g2v_cbow_batch_plan): rows[r] = a gene the batch gathered, its batch-relative
// positions pos[segptr[r] .. segptr[r+1]).  One warp per row, as cbow_csc_expand_kernel: c = its segmented dO sum,
// g_ih[row,:] += c * W_ho; no atomics.
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_batch_expand_kernel(const int32_t *__restrict__ rows, const int32_t *__restrict__ segptr,
                         const int32_t *__restrict__ pos, const float *__restrict__ dO_pos, int64_t n_rows,
                         const float *__restrict__ W_ho, float *__restrict__ g_ih, int32_t D,
                         const int32_t *__restrict__ skip) {
    G2V_SKIP_IF_STOPPED(skip);
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * kCbowWarps + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * kCbowWarps;
    for (int64_t r = warp; r < n_rows; r += nwarps) {
        const float c = csc_segment_sum(pos, dO_pos, __ldg(segptr + r), __ldg(segptr + r + 1), lane);
        float *row = g_ih + (size_t)__ldg(rows + r) * D;
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
// WD: decoupled weight decay wd on every element before the step (decay1); WD = false is the plain update.
template <int OPT, bool WD>
__global__ void __launch_bounds__(256)
cbow_update_kernel(float *__restrict__ W, float *__restrict__ M, float *__restrict__ Vv,
                   float *__restrict__ G, int64_t n, float *__restrict__ W2, float *__restrict__ M2,
                   float *__restrict__ V2, float *__restrict__ G2, int64_t n2, float alpha_host, float omb1,
                   float omb2, float eps, const float *__restrict__ alpha_dev, const int32_t *__restrict__ skip,
                   float wd) {
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
        decay4<WD>(w, wd);
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
        decay1<WD>(*w, wd);
        if (OPT == G2V_OPT_ADAM_TF1) adam1(*w, *m, *v, *g, alpha, omb1, omb2, eps);
        else *w -= alpha * *g;
        *g = 0.f;
    }
}

// ---- lazy (touched-row) Adam over the rows of one batch -------------------------------------
// TF1 LazyAdam on the embedding-lookup form of the model: only the rows a batch gathered are updated.  The gradient
// of gene row g is c[g] * W_ho with c[g] = sum of dO*scale over the gene's positions in the batch, so the optimizer
// step is fused with that per-gene segmented sum and g_ih is never materialised.  One warp per touched gene:
// rows[r] = the gene, its positions pos[segptr[r] .. segptr[r+1]) index dO (batch-relative list positions).
// Rows outside the list keep W, m and v bit for bit.  W_ho must be the value before this step: its own update is a
// second launch (cbow_update_kernel with n = 0).  The gradient is rounded on its own (__fmul_rn, never contracted
// into Adam's first subtraction), as the stored g_ih of the CSC backward is, so the step is the dense one bit for bit.
// WD: each listed row is decayed once (rows are distinct) before its step, as TF1 decays the deduplicated indices.
template <bool WD>
__global__ void __launch_bounds__(kCbowWarps * 32)
cbow_lazy_adam_rows_kernel(const int32_t *__restrict__ rows, const int32_t *__restrict__ segptr,
                           const int32_t *__restrict__ pos, const float *__restrict__ dO, int64_t n_rows,
                           float *__restrict__ W, float *__restrict__ M, float *__restrict__ Vv,
                           const float *__restrict__ W_ho, int32_t D, float alpha_host, float omb1, float omb2,
                           float eps, const float *__restrict__ alpha_dev, const int32_t *__restrict__ skip,
                           float wd) {
    G2V_SKIP_IF_STOPPED(skip);
    const float alpha = alpha_dev ? __ldg(alpha_dev + 2) : alpha_host;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * kCbowWarps + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * kCbowWarps;
    for (int64_t r = warp; r < n_rows; r += nwarps) {
        const size_t off = (size_t)__ldg(rows + r) * D;
        const float c = csc_segment_sum(pos, dO, __ldg(segptr + r), __ldg(segptr + r + 1), lane);
        if ((D & 3) == 0) {
            float4 *w4 = reinterpret_cast<float4 *>(W + off), *m4 = reinterpret_cast<float4 *>(M + off);
            float4 *v4 = reinterpret_cast<float4 *>(Vv + off);
            for (int k = lane; k < (D >> 2); k += 32) {
                const float4 h = ldg4(reinterpret_cast<const float4 *>(W_ho) + k);
                float4 w = w4[k], m = m4[k], v = v4[k];
                decay4<WD>(w, wd);
                adam1(w.x, m.x, v.x, __fmul_rn(c, h.x), alpha, omb1, omb2, eps);
                adam1(w.y, m.y, v.y, __fmul_rn(c, h.y), alpha, omb1, omb2, eps);
                adam1(w.z, m.z, v.z, __fmul_rn(c, h.z), alpha, omb1, omb2, eps);
                adam1(w.w, m.w, v.w, __fmul_rn(c, h.w), alpha, omb1, omb2, eps);
                w4[k] = w; m4[k] = m; v4[k] = v;
            }
        } else {
            for (int d = lane; d < D; d += 32) {
                decay1<WD>(W[off + d], wd);
                adam1(W[off + d], M[off + d], Vv[off + d], __fmul_rn(c, __ldg(W_ho + d)), alpha, omb1, omb2, eps);
            }
        }
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

// WD: the owned slice is decayed (decay1) after the reduce and before Adam / SGD, then all-gathered as before.
template <int OPT, bool MC, bool WD>
__global__ void __launch_bounds__(256)
cbow_update_nvl_kernel(float *const *__restrict__ g_ptrs, float *const *__restrict__ w_ptrs, float *__restrict__ g_mc,
                       float *__restrict__ w_mc, float *__restrict__ M, float *__restrict__ Vv, int64_t n, int32_t rank,
                       int32_t world, float alpha_host, float omb1, float omb2, float eps,
                       const float *__restrict__ alpha_dev, const int32_t *__restrict__ skip, float wd) {
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
        decay4<WD>(w, wd);
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
            decay1<WD>(w, wd);
            if (OPT == G2V_OPT_ADAM_TF1) adam1(w, M[i], Vv[i], g, alpha, omb1, omb2, eps);
            else w -= alpha * g;
            for (int p = 0; p < world; ++p) { volatile float *wp = w_ptrs[p] + i; *wp = w; }
        }
}

int rows_grid(const void *kernel, size_t smem, int64_t n_items, int *grid_out) {
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    if (dp.cc_major != 9) { set_error("needs an sm_90 device (found sm_%d%d); no CPU fallback", dp.cc_major, dp.cc_minor); return 2; }
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kCbowWarps * 32, smem);
    if (e != cudaSuccess || per_sm <= 0) { set_error("occupancy query failed: %s", cudaGetErrorString(e)); return 1; }
    int64_t grid = (int64_t)dp.sm_count * per_sm;
    const int64_t need = (n_items + kCbowWarps - 1) / kCbowWarps;
    if (grid > need) grid = need;
    *grid_out = (int)(grid > 0 ? grid : 1);
    return 0;
}

// dO_pos != NULL (backward only): the CSC backward -- dO*scale per list position instead of the scatter into g_ih.
// carried: the word that makes the launched kernel return at once when set (besides `stopped`), or NULL.
// CW (backward only): the class-weighted kernels with weights cw (DESIGN.md §4.20).
template <bool BACKWARD, bool CW = false>
static int launch_rows(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                       int64_t win_begin, int64_t n_win, float inv_n, const float *W_ih, const float *W_ho,
                       float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t D,
                       int32_t reduce, cudaStream_t st, float *dO_pos = nullptr, const int32_t *carried = nullptr,
                       float2 cw = float2{1.f, 1.f}) {
    static_assert(BACKWARD || !CW, "the accuracy pass has no class weights");
    unsigned long long *nc = reinterpret_cast<unsigned long long *>(n_correct);
    int grid = 0, rc;
#define G2V_LAUNCH_VEC(VEC)                                                                                            \
    {                                                                                                                  \
        auto kern = !BACKWARD ? cbow_rows_kernel<VEC, kRowsEval, false>                                                \
                    : dO_pos  ? cbow_rows_kernel<VEC, kRowsCsc, CW> : cbow_rows_kernel<VEC, kRowsScatter, CW>;         \
        if ((rc = rows_grid((const void *)kern, 0, n_win, &grid))) return rc;                                          \
        kern<<<grid, kCbowWarps * 32, 0, st>>>(rowptr, gene, label, win, win_begin, n_win, inv_n, W_ih, W_ho, g_ih, \
                                               g_ho, loss_sum, nc, reduce, loop_skip_flag(), dO_pos, carried, cw); \
    }
    if (D == 128) G2V_LAUNCH_VEC(1)
    else if (D == 256) G2V_LAUNCH_VEC(2)
    else if (D == 512) G2V_LAUNCH_VEC(4)
    else {
        const size_t smem = (size_t)kCbowWarps * 2 * D * sizeof(float);
        DeviceProps dp;
        if (device_props(&dp)) return 1;
        // the opt-in limit covers the kernel's static shared memory (sh_acc) as well as the dynamic part
        cudaFuncAttributes fa;
        G2V_CUDA_OK(cudaFuncGetAttributes(&fa, cbow_rows_generic_kernel<BACKWARD, CW>));
        G2V_REQUIRE(smem + fa.sharedSizeBytes <= (size_t)dp.max_smem_optin,
                    "sizeHiddenlayer %d too large for the generic kernel", D);
        G2V_CUDA_OK(cudaFuncSetAttribute(cbow_rows_generic_kernel<BACKWARD, CW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if ((rc = rows_grid((const void *)cbow_rows_generic_kernel<BACKWARD, CW>, smem, n_win, &grid))) return rc;
        cbow_rows_generic_kernel<BACKWARD, CW><<<grid, kCbowWarps * 32, smem, st>>>(
            rowptr, gene, label, win, win_begin, n_win, inv_n, W_ih, W_ho, g_ih, g_ho, loss_sum, nc, D, reduce, loop_skip_flag(),
            dO_pos, carried, cw);
    }
#undef G2V_LAUNCH_VEC
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

// Grid of a deterministic launch over n_items: rows_grid's, at most max_ctas CTAs when max_ctas > 0.  The results do
// not depend on it; tests vary it to show that.
static int det_grid(const void *kernel, size_t smem, int64_t n_items, int32_t max_ctas, int *grid) {
    int rc = rows_grid(kernel, smem, n_items, grid);
    if (rc == 0 && max_ctas > 0 && *grid > max_ctas) *grid = max_ctas;
    return rc;
}

// The deterministic forward over win[0..n_win-1] (cbow_rows_det_kernel / cbow_rows_generic_det_kernel) and the fixed-
// order sum of its tiles into g_ho and loss_sum (cbow_det_sum_kernel).  Both launches also test `carried` (nullable).
// CW: the class-weighted forward kernels with weights cw (DESIGN.md §4.20).
template <bool CW = false>
static int launch_rows_det(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                           int64_t n_win, float inv_n, const float *W_ih, const float *W_ho, float *dO_pos,
                           float *g_ho, double *loss_sum, int64_t *n_correct, int32_t D, int32_t reduce,
                           void *workspace, int32_t max_ctas, cudaStream_t st, const int32_t *carried,
                           float2 cw = float2{1.f, 1.f}) {
    unsigned long long *nc = reinterpret_cast<unsigned long long *>(n_correct);
    const int64_t n_tiles = (n_win + kDetTile - 1) / kDetTile;
    double *tile_loss = reinterpret_cast<double *>(workspace);
    float *tile_gho = reinterpret_cast<float *>(reinterpret_cast<char *>(workspace) + det_ws_loss_bytes(n_tiles));
    int grid = 0, rc;
#define G2V_LAUNCH_DET(VEC)                                                                                            \
    {                                                                                                                  \
        if ((rc = det_grid((const void *)cbow_rows_det_kernel<VEC, CW>, 0, n_tiles * kCbowWarps, max_ctas, &grid)))  \
            return rc;                                                                                                 \
        cbow_rows_det_kernel<VEC, CW><<<grid, kCbowWarps * 32, 0, st>>>(rowptr, gene, label, win, n_win, inv_n, W_ih, \
                                                                        W_ho, dO_pos, tile_loss, tile_gho, nc, reduce, \
                                                                        loop_skip_flag(), carried, cw);                \
    }
    if (D == 128) G2V_LAUNCH_DET(1)
    else if (D == 256) G2V_LAUNCH_DET(2)
    else if (D == 512) G2V_LAUNCH_DET(4)
    else {
        const size_t smem = (size_t)kCbowWarps * 2 * D * sizeof(float);
        DeviceProps dp;
        if (device_props(&dp)) return 1;
        G2V_REQUIRE(smem + 1024 <= (size_t)dp.max_smem_optin, "sizeHiddenlayer %d too large for the generic kernel", D);
        G2V_CUDA_OK(cudaFuncSetAttribute(cbow_rows_generic_det_kernel<CW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if ((rc = det_grid((const void *)cbow_rows_generic_det_kernel<CW>, smem, n_tiles * kCbowWarps, max_ctas, &grid)))
            return rc;
        cbow_rows_generic_det_kernel<CW><<<grid, kCbowWarps * 32, smem, st>>>(rowptr, gene, label, win, n_win, inv_n,
                                                                              W_ih, W_ho, dO_pos, tile_loss, tile_gho,
                                                                              nc, D, reduce, loop_skip_flag(), carried, cw);
    }
#undef G2V_LAUNCH_DET
    G2V_CUDA_OK(cudaGetLastError());
    cbow_det_sum_kernel<<<(D + 31) / 32, kDetSumWarps * 32, 0, st>>>(tile_loss, tile_gho, n_tiles, D, g_ho, loss_sum,
                                                                       loop_skip_flag(), carried);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch(2);
    return 0;
}


// ---- device-side training loop control (SURVEY 8f-4; G2Vec.py:262-283) ------------------------------------
// ctl (int64 x 8 in device memory):
//   [0] stopped      1 once the loop is over: the validation accuracy dropped (strict <, :276) or max_steps ran
//   [1] step         optimizer steps decided so far
//   [2] stop_step    step whose validation accuracy dropped, -1 if none (the reference breaks there, :279)
//   [3] before_val   correct validation windows of the last passed step (before_acc_val, :280; -1 = the -1. of :261)
//   [4] max_steps    cap on optimizer steps (--epoch)       [5] early_stop   0 = never stop early
//   [6] carried      1 once a tail pass (g2v_cbow_loop_tail) has run the training forward of the current weights:
//                    dO per list position, the g_ho partial and the carry counters acc[4..5] are pending, and the
//                    forward of g2v_cbow_fwdbwd_csc returns at once while the loop is attached
//   [7] unused
// acc (int64): [0] loss sum (f64 bits)  [1] pre-update train correct  [2] validation correct  [3] train correct;
//   with tail passes also [4] carried loss sum (f64 bits)  [5] carried train correct (this rank's own count, kept
//   out of [1..3], the range a multi-GPU step sums over the ranks).
// loop_begin:  if not stopped, copy the weights into `snapshot` (they are the result if THIS step's validation
//   accuracy drops: the reference returns the W_ih read at :283 after the previous step) and zero the 4 counters;
//   with a carry pending, acc[0..1] take the carried loss and count instead and acc[4..5] are zeroed.
// loop_carry:  after a tail pass, ACC[tr] of this step (acc[3]) is the carried count; sets ctl[6].
// loop_decide: if not stopped, record the step's counters in hist[step][0..3], apply the early-stop rule on the
//   validation count (same ordering as the float32 ratios the reference compares while n_val < 2^24), advance.
__global__ void __launch_bounds__(256)
loop_begin_kernel(const long long *__restrict__ ctl, long long *__restrict__ acc, const float4 *__restrict__ W4,
                  float4 *__restrict__ S4, int64_t n4, const float *__restrict__ W, float *__restrict__ S, int64_t n) {
    if (ctl[0] != 0) return;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
    if (tid == 0) {
        if (ctl[6] != 0) {
            acc[0] = acc[4]; acc[1] = acc[5];
            acc[4] = 0; acc[5] = 0;
        } else {
            acc[0] = 0; acc[1] = 0;
        }
        acc[2] = 0; acc[3] = 0;
    }
    if (S == nullptr) return;
    for (int64_t i = tid; i < n4; i += nth) S4[i] = W4[i];
    for (int64_t i = (n4 << 2) + tid; i < n; i += nth) S[i] = W[i];
}

__global__ void loop_carry_kernel(long long *__restrict__ ctl, long long *__restrict__ acc) {
    if (ctl[0] != 0) return;
    acc[3] += acc[5];
    ctl[6] = 1;
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

// ---- early stopping with patience (DESIGN.md §4.15) ------------------------------------------------------------
// best (int64 x 4 in device memory, kept apart from ctl): {patience, best_step, bad_steps, improved}.  ctl[3] holds
// the best validation count so far, which is the previous step's count whenever patience is 1.
// loop_decide_best: loop_decide with the patience rule -- a count >= the best is the new best (ties: the later step),
//   a lower one is a bad step, and the patience-th bad step in a row stops the loop.  `improved` says whether THIS
//   step's weights must be kept; it is cleared on the no-op steps enqueued after the stop.
// loop_keep_best: copy W_ih into `result` if `improved`.  It does not test `stopped`: the step that ends the loop at
//   max_steps can be the best one.
__global__ void loop_decide_best_kernel(long long *__restrict__ ctl, long long *__restrict__ best,
                                        const long long *__restrict__ acc, long long *__restrict__ hist) {
    if (ctl[0] != 0) {
        best[3] = 0;
        return;
    }
    const long long step = ctl[1];
    if (acc)
        for (int k = 0; k < 4; ++k) hist[step * 4 + k] = acc[k];
    const long long val = hist[step * 4 + 2];
    if (val >= ctl[3]) {
        ctl[3] = val; best[1] = step; best[2] = 0; best[3] = 1;
    } else {
        best[2] += 1; best[3] = 0;
        if (ctl[5] != 0 && best[2] >= best[0]) {
            ctl[0] = 1; ctl[2] = step;               // the patience-th bad step: the kept weights are the result
        }
    }
    if (step + 1 >= ctl[4]) ctl[0] = 1;              // ran --epoch steps
    ctl[1] = step + 1;
}

__global__ void __launch_bounds__(256)
loop_keep_best_kernel(const long long *__restrict__ best, const float4 *__restrict__ W4, float4 *__restrict__ R4,
                      int64_t n4, const float *__restrict__ W, float *__restrict__ R, int64_t n) {
    if (best[3] == 0) return;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = tid; i < n4; i += nth) R4[i] = W4[i];
    for (int64_t i = (n4 << 2) + tid; i < n; i += nth) R[i] = W[i];
}

// ---- reduce-on-plateau learning rate (DESIGN.md §4.17) ---------------------------------------------------------
// st (int64 x 8, then float32 x (4 + cap)): {K, best, wait, n_reductions, steps, cap, -, -}, then
//   f = {lr, factor, min_lr, -, rate[0 .. cap-1]}.  Applies the rule to every step from st.steps up to (excluding)
//   *n_decided -- or to exactly one step if n_decided is NULL -- reading step s's validation count at
//   counts[s * stride].  rate[s] records the rate step s trained with (the one before its own decision).  It does not
//   test the loop's `stopped` word: the step that stops the loop is decided like any other, and the no-op steps
//   enqueued after it find st.steps == *n_decided.
__global__ void lr_plateau_kernel(long long *__restrict__ st, const long long *__restrict__ counts, int64_t stride,
                                  const long long *__restrict__ n_decided) {
    float *f = reinterpret_cast<float *>(st + 8);
    const long long end = n_decided ? *n_decided : st[4] + 1;
    for (long long s = st[4]; s < end; ++s) {
        const long long v = counts[s * stride];
        const float lr = f[0];
        if (s < st[5]) f[4 + s] = lr;
        if (v > st[1]) {                             // strict: a tie is not an improvement
            st[1] = v; st[2] = 0;
        } else if (++st[2] >= st[0]) {
            if (lr > f[2]) {
                f[0] = fmaxf(__fmul_rn(lr, f[1]), f[2]);
                st[3] += 1;
            }
            st[2] = 0;
        }
    }
    if (end > st[4]) st[4] = end;
}

// ---- validation loss (DESIGN.md §4.19) -------------------------------------------------------------------------
// Q = sum over the listed windows of q_n = rint(min(l_n, 64) 2^24), l_n = max(z,0) - z y + log1p(exp(-|z|)) in float64
// (64 for a z that is not finite), z = scale * sum_{g in n} s[g] in float32.  The sum over g is r1_windows_kernel's
// order: lane `sub` of the window's 8 lanes adds s of its genes j = b + sub, b + sub + 8, ... in turn, then the 8
// partials are combined by the xor-shuffle tree 4, 2, 1.  z therefore depends only on s and the window, and Q, an
// integer sum, on nothing but the list: not on the grid, the order of the windows or a split of the list.
// q_n <= 2^30, so a list of fewer than 2^32 windows sums to Q < 2^62 without overflow.
constexpr double kValLossCap = 64.0, kValLossUnit = 0x1p24;
constexpr long long kScoreTop = 1ll << 62;

__device__ __forceinline__ unsigned long long val_loss_term(float z, float y) {
    double l = kValLossCap;
    if (isfinite(z)) {
        const double zd = (double)z;
        l = fmin(fmax(zd, 0.0) - zd * (double)y + log1p(exp(-fabs(zd))), kValLossCap);
    }
    return (unsigned long long)rint(l * kValLossUnit);
}

// s[g] at s[g * s_stride]: 2 for the certified pass's st = {s, t}, 1 for the rank-1 model's s
__global__ void __launch_bounds__(kCbowWarps * 32)
val_loss_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene,
                const uint8_t *__restrict__ label, const int32_t *__restrict__ win, int64_t win_begin, int64_t n_win,
                const float *__restrict__ s, int32_t s_stride, unsigned long long *__restrict__ q_sum,
                int32_t reduce_mean, const int32_t *__restrict__ skip) {
    G2V_SKIP_IF_STOPPED(skip);
    __shared__ unsigned long long sh_q;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & 7, slot = lane >> 3;          // 8 lanes per window, 4 windows per warp
    if (threadIdx.x == 0) sh_q = 0ull;
    __syncthreads();
    unsigned long long q_acc = 0ull;
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
        for (int32_t j = b + sub; j < e; j += 8) part += __ldg(s + (int64_t)__ldg(gene + j) * s_stride);
        part += __shfl_xor_sync(0xffffffffu, part, 4);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        const float scale = (reduce_mean && e > b) ? 1.f / (float)(e - b) : 1.f;
        if (active && sub == 0) q_acc += val_loss_term(part * scale, y);
    }
    q_acc = warp_sum_u64(q_acc);
    if (lane == 0) atomicAdd(&sh_q, q_acc);
    __syncthreads();
    if (threadIdx.x == 0 && sh_q) atomicAdd(q_sum, sh_q);
}

// The monitored score of a step is 2^62 - Q (Q summed over the ranks): non-negative and higher-is-better, like a
// validation count, so ctl.before_val = -1 and the plateau state's best = -1 stay "worse than any step".  q != NULL:
// Q is *q, which is cleared for the next step; q == NULL: score[step] holds the Q the ranks added (loop_score_nvl).
// score[step] is left holding the score.
__device__ __forceinline__ long long take_score(long long *__restrict__ score, long long step,
                                                unsigned long long *__restrict__ q) {
    const unsigned long long Q = q ? *q : (unsigned long long)score[step];
    if (q) *q = 0ull;
    const long long v = kScoreTop - (long long)Q;
    score[step] = v;
    return v;
}

// loop_decide_kernel / loop_decide_best_kernel deciding on score[step] instead of the validation count hist[step][2]
__global__ void loop_decide_score_kernel(long long *__restrict__ ctl, const long long *__restrict__ acc,
                                         long long *__restrict__ hist, unsigned long long *__restrict__ q,
                                         long long *__restrict__ score) {
    if (ctl[0] != 0) return;
    const long long step = ctl[1];
    if (acc)
        for (int k = 0; k < 4; ++k) hist[step * 4 + k] = acc[k];
    const long long val = take_score(score, step, q);
    if (ctl[5] != 0 && val < ctl[3]) {
        ctl[0] = 1; ctl[2] = step;
    } else {
        ctl[3] = val;
        if (step + 1 >= ctl[4]) ctl[0] = 1;
    }
    ctl[1] = step + 1;
}

__global__ void loop_decide_best_score_kernel(long long *__restrict__ ctl, long long *__restrict__ best,
                                              const long long *__restrict__ acc, long long *__restrict__ hist,
                                              unsigned long long *__restrict__ q, long long *__restrict__ score) {
    if (ctl[0] != 0) {
        best[3] = 0;
        return;
    }
    const long long step = ctl[1];
    if (acc)
        for (int k = 0; k < 4; ++k) hist[step * 4 + k] = acc[k];
    const long long val = take_score(score, step, q);
    if (val >= ctl[3]) {
        ctl[3] = val; best[1] = step; best[2] = 0; best[3] = 1;
    } else {
        best[2] += 1; best[3] = 0;
        if (ctl[5] != 0 && best[2] >= best[0]) {
            ctl[0] = 1; ctl[2] = step;
        }
    }
    if (step + 1 >= ctl[4]) ctl[0] = 1;
    ctl[1] = step + 1;
}

// Multi-GPU: add this rank's Q into score[step] of every rank's symmetric-memory buffer (at element `offset` of it),
// as loop_counters_nvl_kernel adds the counters, and clear Q.  The caller puts a cross-GPU barrier before the decision.
__global__ void loop_score_nvl_kernel(const long long *__restrict__ ctl, unsigned long long *__restrict__ q,
                                      long long *const *__restrict__ ptrs, long long *__restrict__ mc, int64_t offset,
                                      int32_t world) {
    if (ctl[0] != 0) return;
    const long long step = ctl[1];
    const unsigned long long v = *q;
    *q = 0ull;
    if (mc) {
        asm volatile("multimem.red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(mc + offset + step), "l"(v) : "memory");
    } else {
        for (int p = 0; p < world; ++p)
            atomicAdd_system(reinterpret_cast<unsigned long long *>(ptrs[p] + offset + step), v);
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
    // the low 32 bits of ctl[0] (little endian) are the `stopped` word every step kernel tests; those of ctl[6]
    // the `carried` word the forward of g2v_cbow_fwdbwd_csc also tests
    set_loop_skip_flag(reinterpret_cast<const int32_t *>(ctl));
    set_loop_carry_flag(ctl ? reinterpret_cast<const int32_t *>(ctl + 6) : nullptr);
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

extern "C" int g2v_cbow_loop_decide_best(int64_t *ctl, int64_t *best, const int64_t *acc, int64_t *hist, void *stream) {
    G2V_REQUIRE(ctl && best && hist, "g2v_cbow_loop_decide_best: null pointer");
    loop_decide_best_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<long long *>(ctl), reinterpret_cast<long long *>(best),
        reinterpret_cast<const long long *>(acc), reinterpret_cast<long long *>(hist));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_loop_keep_best(const int64_t *best, const float *W_ih, float *result, int64_t n, void *stream) {
    G2V_REQUIRE(best && W_ih && result && n >= 0, "g2v_cbow_loop_keep_best: bad arguments");
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    int64_t blocks = (n / 4 + 255) / 256;
    if (blocks > (int64_t)dp.sm_count * 8) blocks = (int64_t)dp.sm_count * 8;
    if (blocks < 1) blocks = 1;
    loop_keep_best_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const long long *>(best), reinterpret_cast<const float4 *>(W_ih),
        reinterpret_cast<float4 *>(result), n >> 2, W_ih, result, n);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_lr_plateau(int64_t *state, const int64_t *counts, int64_t stride, const int64_t *n_decided,
                                   void *stream) {
    G2V_REQUIRE(state && counts && stride >= 0, "g2v_cbow_lr_plateau: bad arguments");
    lr_plateau_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<long long *>(state), reinterpret_cast<const long long *>(counts), stride,
        reinterpret_cast<const long long *>(n_decided));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_val_loss(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                                 int64_t win_begin, int64_t n_win, const float *s, int32_t s_stride, uint64_t *q_sum,
                                 int32_t V, int32_t reduce, void *stream) {
    G2V_REQUIRE(V > 0 && n_win >= 0 && win_begin >= 0 && n_win < (1ll << 32) && (s_stride == 1 || s_stride == 2),
                "g2v_cbow_val_loss: bad sizes (V=%d n_win=%lld s_stride=%d)", V, (long long)n_win, s_stride);
    G2V_REQUIRE(rowptr && label && s && q_sum, "g2v_cbow_val_loss: null pointer");
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "g2v_cbow_val_loss: unknown reduce %d", reduce);
    if (n_win == 0) return 0;
    int grid = 0, rc;
    if ((rc = rows_grid((const void *)val_loss_kernel, 0, (n_win + 3) / 4, &grid))) return rc;
    val_loss_kernel<<<grid, kCbowWarps * 32, 0, (cudaStream_t)stream>>>(
        rowptr, gene, label, win, win_begin, n_win, s, s_stride, reinterpret_cast<unsigned long long *>(q_sum),
        reduce == G2V_REDUCE_MEAN, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_st_prepare(const float *W_ih, const float *W_ho, float *st, int32_t V, int32_t D,
                                   void *stream) {
    G2V_REQUIRE(V > 0 && D > 0, "g2v_cbow_st_prepare: bad sizes (V=%d D=%d)", V, D);
    G2V_REQUIRE(W_ih && W_ho && st, "g2v_cbow_st_prepare: null pointer");
    return launch_r1_prepare(W_ih, W_ho, st, V, D, true, (cudaStream_t)stream);
}

extern "C" int g2v_cbow_loop_decide_score(int64_t *ctl, const int64_t *acc, int64_t *hist, uint64_t *q,
                                          int64_t *score, void *stream) {
    G2V_REQUIRE(ctl && hist && score, "g2v_cbow_loop_decide_score: null pointer");
    loop_decide_score_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<long long *>(ctl), reinterpret_cast<const long long *>(acc),
        reinterpret_cast<long long *>(hist), reinterpret_cast<unsigned long long *>(q),
        reinterpret_cast<long long *>(score));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_loop_decide_best_score(int64_t *ctl, int64_t *best, const int64_t *acc, int64_t *hist,
                                               uint64_t *q, int64_t *score, void *stream) {
    G2V_REQUIRE(ctl && best && hist && score, "g2v_cbow_loop_decide_best_score: null pointer");
    loop_decide_best_score_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<long long *>(ctl), reinterpret_cast<long long *>(best),
        reinterpret_cast<const long long *>(acc), reinterpret_cast<long long *>(hist),
        reinterpret_cast<unsigned long long *>(q), reinterpret_cast<long long *>(score));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_loop_score_nvl(const int64_t *ctl, uint64_t *q, int64_t *const *ptrs_dev, int64_t *multicast,
                                       int64_t offset, int32_t world, void *stream) {
    G2V_REQUIRE(ctl && q && ptrs_dev && offset >= 0 && world >= 1, "g2v_cbow_loop_score_nvl: bad arguments");
    loop_score_nvl_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const long long *>(ctl), reinterpret_cast<unsigned long long *>(q),
        reinterpret_cast<long long *const *>(ptrs_dev), reinterpret_cast<long long *>(multicast), offset, world);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

// ---- the entry points that form dO and their class-weighted *_cw forms (DESIGN.md §4.20) ------------------------
// One body per entry point, a template on CW: the plain form launches the unweighted kernels, the _cw form checks its
// weights (G2V_CW_CHECK) and launches the weighted instantiations with cw = {w0, w1}.  `name` is the entry point's,
// for errors.

template <bool CW>
static int fwdbwd_impl(const char *name, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                       const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total, const float *W_ih,
                       const float *W_ho, float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V,
                       int32_t D, int32_t reduce, float2 cw, void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_win >= 0 && win_begin >= 0, "%s: bad sizes (V=%d D=%d n_win=%lld)", name, V, D, (long long)n_win);
    G2V_REQUIRE(rowptr && label && W_ih && W_ho && g_ih && g_ho, "%s: null pointer", name);
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "%s: unknown reduce %d", name, reduce);
    if (n_win == 0) return 0;
    return launch_rows<true, CW>(rowptr, gene, label, win, win_begin, n_win, inv_n_total, W_ih, W_ho, g_ih, g_ho,
                                 loss_sum, n_correct, D, reduce, (cudaStream_t)stream, nullptr, nullptr, cw);
}

extern "C" int g2v_cbow_fwdbwd(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                               const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total,
                               const float *W_ih, const float *W_ho, float *g_ih, float *g_ho,
                               double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                               void *stream) {
    return fwdbwd_impl<false>("g2v_cbow_fwdbwd", rowptr, gene, label, win, win_begin, n_win, inv_n_total, W_ih, W_ho,
                              g_ih, g_ho, loss_sum, n_correct, V, D, reduce, float2{1.f, 1.f}, stream);
}

extern "C" int g2v_cbow_fwdbwd_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                  const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total,
                                  const float *W_ih, const float *W_ho, float *g_ih, float *g_ho,
                                  double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                                  float w0, float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_fwdbwd_cw");
    return fwdbwd_impl<true>("g2v_cbow_fwdbwd_cw", rowptr, gene, label, win, win_begin, n_win, inv_n_total, W_ih, W_ho,
                             g_ih, g_ho, loss_sum, n_correct, V, D, reduce, float2{w0, w1}, stream);
}

template <bool CW>
static int fwdbwd_csc_impl(const char *name, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                           const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                           const int32_t *cscptr, const int32_t *csc_pos, float *dO, float *g_ih, float *g_ho,
                           double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce, float2 cw,
                           void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_win >= 0, "%s: bad sizes (V=%d D=%d n_win=%lld)", name, V, D, (long long)n_win);
    G2V_REQUIRE(rowptr && label && W_ih && W_ho && cscptr && dO && g_ih && g_ho, "%s: null pointer", name);
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "%s: unknown reduce %d", name, reduce);
    if (n_win == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    // with a tail pass pending (attached loop, ctl[6] set) the forward returns at once and the expansion reads its dO
    int rc = launch_rows<true, CW>(rowptr, gene, label, win, 0, n_win, inv_n_total, W_ih, W_ho, g_ih, g_ho, loss_sum,
                                   n_correct, D, reduce, st, dO, loop_carry_flag(), cw);
    if (rc) return rc;
    int grid = 0;
    if ((rc = rows_grid((const void *)cbow_csc_expand_kernel, 0, V, &grid))) return rc;
    cbow_csc_expand_kernel<<<grid, kCbowWarps * 32, 0, st>>>(cscptr, csc_pos, dO, W_ho, g_ih, V, D, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_fwdbwd_csc(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                   const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                   const float *W_ho, const int32_t *cscptr, const int32_t *csc_pos, float *dO,
                                   float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V,
                                   int32_t D, int32_t reduce, void *stream) {
    return fwdbwd_csc_impl<false>("g2v_cbow_fwdbwd_csc", rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho,
                                  cscptr, csc_pos, dO, g_ih, g_ho, loss_sum, n_correct, V, D, reduce, float2{1.f, 1.f},
                                  stream);
}

extern "C" int g2v_cbow_fwdbwd_csc_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                      const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                      const float *W_ho, const int32_t *cscptr, const int32_t *csc_pos, float *dO,
                                      float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V,
                                      int32_t D, int32_t reduce, float w0, float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_fwdbwd_csc_cw");
    return fwdbwd_csc_impl<true>("g2v_cbow_fwdbwd_csc_cw", rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho,
                                 cscptr, csc_pos, dO, g_ih, g_ho, loss_sum, n_correct, V, D, reduce, float2{w0, w1},
                                 stream);
}

template <bool CW>
static int fwd_do_impl(const char *name, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                       const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                       float *dO, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D,
                       int32_t reduce, float2 cw, void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_win >= 0, "%s: bad sizes (V=%d D=%d n_win=%lld)", name, V, D, (long long)n_win);
    G2V_REQUIRE(rowptr && label && W_ih && W_ho && dO && g_ho, "%s: null pointer", name);
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "%s: unknown reduce %d", name, reduce);
    if (n_win == 0) return 0;
    return launch_rows<true, CW>(rowptr, gene, label, win, 0, n_win, inv_n_total, W_ih, W_ho, nullptr, g_ho, loss_sum,
                                 n_correct, D, reduce, (cudaStream_t)stream, dO, nullptr, cw);
}

extern "C" int g2v_cbow_fwd_do(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                               int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho, float *dO,
                               float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                               void *stream) {
    return fwd_do_impl<false>("g2v_cbow_fwd_do", rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho, dO, g_ho,
                              loss_sum, n_correct, V, D, reduce, float2{1.f, 1.f}, stream);
}

extern "C" int g2v_cbow_fwd_do_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                                  int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho, float *dO,
                                  float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D,
                                  int32_t reduce, float w0, float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_fwd_do_cw");
    return fwd_do_impl<true>("g2v_cbow_fwd_do_cw", rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho, dO, g_ho,
                             loss_sum, n_correct, V, D, reduce, float2{w0, w1}, stream);
}

template <bool CW>
static int loop_tail_impl(const char *name, int64_t *ctl, const int32_t *rowptr, const int32_t *gene,
                          const uint8_t *label, const int32_t *win, int64_t n_win, float inv_n_total,
                          const float *W_ih, const float *W_ho, float *dO, float *g_ho, int64_t *acc, int32_t V,
                          int32_t D, int32_t reduce, float2 cw, void *stream) {
    G2V_REQUIRE(ctl && acc, "%s: null loop state", name);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = fwd_do_impl<CW>(CW ? "g2v_cbow_fwd_do_cw" : "g2v_cbow_fwd_do", rowptr, gene, label, win, n_win,
                             inv_n_total, W_ih, W_ho, dO, g_ho, reinterpret_cast<double *>(acc + 4), acc + 5, V, D,
                             reduce, cw, st);
    if (rc) return rc;
    loop_carry_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long *>(ctl), reinterpret_cast<long long *>(acc));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_loop_tail(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                  const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                  const float *W_ho, float *dO, float *g_ho, int64_t *acc, int32_t V, int32_t D,
                                  int32_t reduce, void *stream) {
    return loop_tail_impl<false>("g2v_cbow_loop_tail", ctl, rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho,
                                 dO, g_ho, acc, V, D, reduce, float2{1.f, 1.f}, stream);
}

extern "C" int g2v_cbow_loop_tail_cw(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                     const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                     const float *W_ho, float *dO, float *g_ho, int64_t *acc, int32_t V, int32_t D,
                                     int32_t reduce, float w0, float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_loop_tail_cw");
    return loop_tail_impl<true>("g2v_cbow_loop_tail_cw", ctl, rowptr, gene, label, win, n_win, inv_n_total, W_ih,
                                W_ho, dO, g_ho, acc, V, D, reduce, float2{w0, w1}, stream);
}

extern "C" size_t g2v_cbow_det_workspace_bytes(int64_t n_win, int32_t D) {
    if (n_win < 0 || D <= 0) return 0;
    const int64_t n_tiles = (n_win + kDetTile - 1) / kDetTile;
    return det_ws_loss_bytes(n_tiles) + (size_t)n_tiles * (size_t)D * sizeof(float);
}

// name: the entry point's, a runtime string (errors)
#define G2V_DET_CHECK(name)                                                                                            \
    G2V_REQUIRE(V > 0 && D > 0 && n_win >= 0 && max_ctas >= 0, "%s: bad sizes (V=%d D=%d n_win=%lld max_ctas=%d)",  \
                name, V, D, (long long)n_win, max_ctas);                                                               \
    G2V_REQUIRE(n_win == 0 || (rowptr && gene && label && win && W_ih && W_ho && dO && g_ho && workspace),            \
                "%s: null pointer", name);                                                                             \
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "%s: unknown reduce %d", name, reduce)

template <bool CW>
static int fwdbwd_csc_det_impl(const char *name, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                               const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                               const float *W_ho, const int32_t *cscptr, const int32_t *csc_pos, float *dO,
                               float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D,
                               int32_t reduce, void *workspace, int32_t max_ctas, float2 cw, void *stream) {
    G2V_DET_CHECK(name);
    // csc_pos may be NULL: a list of empty windows has no incidences (every CSC segment is empty)
    G2V_REQUIRE(n_win == 0 || (cscptr && g_ih), "%s: null pointer", name);
    if (n_win == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = launch_rows_det<CW>(rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho, dO, g_ho, loss_sum,
                                 n_correct, D, reduce, workspace, max_ctas, st, loop_carry_flag(), cw);
    if (rc) return rc;
    int grid = 0;
    if ((rc = det_grid((const void *)cbow_csc_expand_kernel, 0, V, max_ctas, &grid))) return rc;
    cbow_csc_expand_kernel<<<grid, kCbowWarps * 32, 0, st>>>(cscptr, csc_pos, dO, W_ho, g_ih, V, D, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_fwdbwd_csc_det(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                       const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                       const float *W_ho, const int32_t *cscptr, const int32_t *csc_pos, float *dO,
                                       float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V,
                                       int32_t D, int32_t reduce, void *workspace, int32_t max_ctas, void *stream) {
    return fwdbwd_csc_det_impl<false>("g2v_cbow_fwdbwd_csc_det", rowptr, gene, label, win, n_win, inv_n_total, W_ih,
                                      W_ho, cscptr, csc_pos, dO, g_ih, g_ho, loss_sum, n_correct, V, D, reduce,
                                      workspace, max_ctas, float2{1.f, 1.f}, stream);
}

extern "C" int g2v_cbow_fwdbwd_csc_det_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                          const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                          const float *W_ho, const int32_t *cscptr, const int32_t *csc_pos, float *dO,
                                          float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V,
                                          int32_t D, int32_t reduce, void *workspace, int32_t max_ctas, float w0,
                                          float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_fwdbwd_csc_det_cw");
    return fwdbwd_csc_det_impl<true>("g2v_cbow_fwdbwd_csc_det_cw", rowptr, gene, label, win, n_win, inv_n_total, W_ih,
                                     W_ho, cscptr, csc_pos, dO, g_ih, g_ho, loss_sum, n_correct, V, D, reduce,
                                     workspace, max_ctas, float2{w0, w1}, stream);
}

template <bool CW>
static int fwd_do_det_impl(const char *name, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                           const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                           float *dO, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D,
                           int32_t reduce, void *workspace, int32_t max_ctas, float2 cw, void *stream) {
    G2V_DET_CHECK(name);
    if (n_win == 0) return 0;
    return launch_rows_det<CW>(rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho, dO, g_ho, loss_sum, n_correct,
                               D, reduce, workspace, max_ctas, (cudaStream_t)stream, nullptr, cw);
}
#undef G2V_DET_CHECK

extern "C" int g2v_cbow_fwd_do_det(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                   const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                   const float *W_ho, float *dO, float *g_ho, double *loss_sum, int64_t *n_correct,
                                   int32_t V, int32_t D, int32_t reduce, void *workspace, int32_t max_ctas,
                                   void *stream) {
    return fwd_do_det_impl<false>("g2v_cbow_fwd_do_det", rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho, dO,
                                  g_ho, loss_sum, n_correct, V, D, reduce, workspace, max_ctas, float2{1.f, 1.f},
                                  stream);
}

extern "C" int g2v_cbow_fwd_do_det_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                      const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                      const float *W_ho, float *dO, float *g_ho, double *loss_sum, int64_t *n_correct,
                                      int32_t V, int32_t D, int32_t reduce, void *workspace, int32_t max_ctas,
                                      float w0, float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_fwd_do_det_cw");
    return fwd_do_det_impl<true>("g2v_cbow_fwd_do_det_cw", rowptr, gene, label, win, n_win, inv_n_total, W_ih, W_ho,
                                 dO, g_ho, loss_sum, n_correct, V, D, reduce, workspace, max_ctas, float2{w0, w1},
                                 stream);
}

template <bool CW>
static int loop_tail_det_impl(const char *name, int64_t *ctl, const int32_t *rowptr, const int32_t *gene,
                              const uint8_t *label, const int32_t *win, int64_t n_win, float inv_n_total,
                              const float *W_ih, const float *W_ho, float *dO, float *g_ho, int64_t *acc, int32_t V,
                              int32_t D, int32_t reduce, void *workspace, int32_t max_ctas, float2 cw, void *stream) {
    G2V_REQUIRE(ctl && acc, "%s: null loop state", name);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = fwd_do_det_impl<CW>(CW ? "g2v_cbow_fwd_do_det_cw" : "g2v_cbow_fwd_do_det", rowptr, gene, label, win,
                                 n_win, inv_n_total, W_ih, W_ho, dO, g_ho, reinterpret_cast<double *>(acc + 4),
                                 acc + 5, V, D, reduce, workspace, max_ctas, cw, st);
    if (rc) return rc;
    loop_carry_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long *>(ctl), reinterpret_cast<long long *>(acc));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_loop_tail_det(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                      const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                                      const float *W_ho, float *dO, float *g_ho, int64_t *acc, int32_t V, int32_t D,
                                      int32_t reduce, void *workspace, int32_t max_ctas, void *stream) {
    return loop_tail_det_impl<false>("g2v_cbow_loop_tail_det", ctl, rowptr, gene, label, win, n_win, inv_n_total,
                                     W_ih, W_ho, dO, g_ho, acc, V, D, reduce, workspace, max_ctas, float2{1.f, 1.f},
                                     stream);
}

extern "C" int g2v_cbow_loop_tail_det_cw(int64_t *ctl, const int32_t *rowptr, const int32_t *gene,
                                         const uint8_t *label, const int32_t *win, int64_t n_win, float inv_n_total,
                                         const float *W_ih, const float *W_ho, float *dO, float *g_ho, int64_t *acc,
                                         int32_t V, int32_t D, int32_t reduce, void *workspace, int32_t max_ctas,
                                         float w0, float w1, void *stream) {
    G2V_CW_CHECK("g2v_cbow_loop_tail_det_cw");
    return loop_tail_det_impl<true>("g2v_cbow_loop_tail_det_cw", ctl, rowptr, gene, label, win, n_win, inv_n_total,
                                    W_ih, W_ho, dO, g_ho, acc, V, D, reduce, workspace, max_ctas, float2{w0, w1},
                                    stream);
}

extern "C" int g2v_cbow_batch_expand(const int32_t *rows, const int32_t *segptr, const int32_t *pos, const float *dO,
                                     int64_t n_rows, const float *W_ho, float *g_ih, int32_t V, int32_t D,
                                     int32_t max_ctas, void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_rows >= 0 && n_rows <= V && max_ctas >= 0,
                "g2v_cbow_batch_expand: bad sizes (V=%d D=%d n_rows=%lld max_ctas=%d)", V, D, (long long)n_rows, max_ctas);
    G2V_REQUIRE(n_rows == 0 || (rows && segptr && pos && dO && W_ho && g_ih), "g2v_cbow_batch_expand: null pointer");
    if (n_rows == 0) return 0;
    int grid = 0, rc;
    if ((rc = det_grid((const void *)cbow_batch_expand_kernel, 0, n_rows, max_ctas, &grid))) return rc;
    cbow_batch_expand_kernel<<<grid, kCbowWarps * 32, 0, (cudaStream_t)stream>>>(rows, segptr, pos, dO, n_rows, W_ho,
                                                                                  g_ih, D, loop_skip_flag());
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

extern "C" int g2v_cbow_eval_certified(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                                       const int32_t *win, int64_t win_begin, int64_t n_win, const float *W_ih,
                                       const float *W_ho, float *st, int64_t *n_correct, int64_t *n_gathered,
                                       int32_t V, int32_t D, int32_t reduce, int32_t force_gather, void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_win >= 0 && win_begin >= 0, "g2v_cbow_eval_certified: bad sizes");
    G2V_REQUIRE(rowptr && label && W_ih && W_ho && st && n_correct, "g2v_cbow_eval_certified: null pointer");
    G2V_REQUIRE(reduce == G2V_REDUCE_SUM || reduce == G2V_REDUCE_MEAN, "g2v_cbow_eval_certified: unknown reduce %d",
                reduce);
    if (n_win == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const bool generic = D != 128 && D != 256 && D != 512;
    const size_t smem = generic ? (size_t)kCbowWarps * D * sizeof(float) : 0;
    if (generic) {
        // the D range of g2v_cbow_eval: its generic kernel holds h and the g_ho partial, 2 D floats per warp
        DeviceProps dp;
        if (device_props(&dp)) return 1;
        cudaFuncAttributes fa;
        G2V_CUDA_OK(cudaFuncGetAttributes(&fa, cbow_rows_generic_kernel<false, false>));
        G2V_REQUIRE((size_t)kCbowWarps * 2 * D * sizeof(float) + fa.sharedSizeBytes <= (size_t)dp.max_smem_optin,
                    "sizeHiddenlayer %d too large for the generic kernel", D);
        G2V_CUDA_OK(cudaFuncSetAttribute(cbow_eval_certified_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
    }
    int rc = launch_r1_prepare(W_ih, W_ho, st, V, D, true, s);
    if (rc) return rc;
    auto kern = D == 128 ? cbow_eval_certified_kernel<1> : D == 256 ? cbow_eval_certified_kernel<2>
              : D == 512 ? cbow_eval_certified_kernel<4> : cbow_eval_certified_kernel<0>;
    int grid = 0;
    if ((rc = rows_grid((const void *)kern, smem, (n_win + 3) / 4, &grid))) return rc;
    kern<<<grid, kCbowWarps * 32, smem, s>>>(rowptr, gene, label, win, win_begin, n_win, W_ih, W_ho,
                                            reinterpret_cast<const float2 *>(st),
                                            reinterpret_cast<unsigned long long *>(n_correct),
                                            reinterpret_cast<unsigned long long *>(n_gathered), D,
                                            reduce == G2V_REDUCE_MEAN, force_gather, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
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

// adam_tick_kernel with the learning rate read from device memory (the rate g2v_cbow_lr_plateau keeps)
__global__ void adam_tick_lr_kernel(float *state, const float *lr_dev, float beta1, float beta2, const int32_t *skip) {
    G2V_SKIP_IF_STOPPED(skip);
    const float lr = *lr_dev;
    const float b1p = state[0] * beta1, b2p = state[1] * beta2;
    state[0] = b1p; state[1] = b2p;
    state[2] = lr * sqrtf(1.f - b2p) / (1.f - b1p);
}

extern "C" int g2v_cbow_adam_tick_lr(float *state, const float *lr_dev, float beta1, float beta2, void *stream) {
    G2V_REQUIRE(state != nullptr && lr_dev != nullptr, "g2v_cbow_adam_tick_lr: null pointer");
    adam_tick_lr_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state, lr_dev, beta1, beta2, loop_skip_flag());
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

// The template arguments <OPT, WD> of an optimizer kernel as runtime values: WD = weight_decay > 0, so that 0 launches
// the plain instantiation.
#define G2V_OPT_WD_DISPATCH(optimizer, weight_decay, MACRO)                                                            \
    do {                                                                                                               \
        if ((optimizer) == G2V_OPT_ADAM_TF1) { if ((weight_decay) > 0.f) MACRO(G2V_OPT_ADAM_TF1, true);              \
                                               else MACRO(G2V_OPT_ADAM_TF1, false); }                                 \
        else { if ((weight_decay) > 0.f) MACRO(G2V_OPT_SGD, true); else MACRO(G2V_OPT_SGD, false); }                  \
    } while (0)

extern "C" int g2v_cbow_update_wd(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                                  float *g_ih, float *g_ho, int32_t V, int32_t D, int32_t optimizer, float lr,
                                  float beta1, float beta2, float eps, float weight_decay, int32_t t,
                                  const float *alpha_dev, void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && (t >= 1 || alpha_dev), "g2v_cbow_update: bad sizes (V=%d D=%d t=%d)", V, D, t);
    G2V_REQUIRE(W_ih && W_ho && g_ih && g_ho, "g2v_cbow_update: null pointer");
    G2V_REQUIRE(optimizer == G2V_OPT_ADAM_TF1 || optimizer == G2V_OPT_SGD, "g2v_cbow_update: unknown optimizer %d", optimizer);
    G2V_REQUIRE(optimizer == G2V_OPT_SGD || (m_ih && v_ih && m_ho && v_ho), "g2v_cbow_update: Adam needs m/v buffers");
    G2V_REQUIRE(weight_decay_ok(weight_decay), "g2v_cbow_update_wd: weight_decay must be finite with 0 <= wd < 1 (got %g)",
                (double)weight_decay);
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    const int64_t n = (int64_t)V * D;
    int64_t blocks = (n / 4 + 255) / 256;
    const int64_t cap = (int64_t)dp.sm_count * 8;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    cudaStream_t st = (cudaStream_t)stream;
    const bool adam = optimizer == G2V_OPT_ADAM_TF1;
    const float alpha = !adam ? lr : alpha_dev ? 0.f : adam_tf1_alpha(lr, beta1, beta2, t);
    const float omb1 = adam ? 1.f - beta1 : 0.f, omb2 = adam ? 1.f - beta2 : 0.f, eps_ = adam ? eps : 0.f;
    if (!adam) { m_ih = v_ih = m_ho = v_ho = nullptr; alpha_dev = nullptr; }
#define G2V_UPDATE(OPT, WD)                                                                                           \
    cbow_update_kernel<OPT, WD><<<(unsigned)blocks, 256, 0, st>>>(W_ih, m_ih, v_ih, g_ih, n, W_ho, m_ho, v_ho, g_ho,   \
                                                                  (int64_t)D, alpha, omb1, omb2, eps_, alpha_dev,     \
                                                                  loop_skip_flag(), weight_decay)
    G2V_OPT_WD_DISPATCH(optimizer, weight_decay, G2V_UPDATE);
#undef G2V_UPDATE
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_update(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                               float *g_ih, float *g_ho, int32_t V, int32_t D, int32_t optimizer, float lr,
                               float beta1, float beta2, float eps, int32_t t, const float *alpha_dev,
                               void *stream) {
    return g2v_cbow_update_wd(W_ih, W_ho, m_ih, v_ih, m_ho, v_ho, g_ih, g_ho, V, D, optimizer, lr, beta1, beta2, eps, 0.f,
                              t, alpha_dev, stream);
}

extern "C" int g2v_cbow_lazy_adam_wd(const int32_t *rows, const int32_t *segptr, const int32_t *pos, const float *dO,
                                     int64_t n_rows, float *W_ih, float *m_ih, float *v_ih, float *W_ho, float *m_ho,
                                     float *v_ho, float *g_ho, int32_t V, int32_t D, float lr, float beta1, float beta2,
                                     float eps, float weight_decay, int32_t t, const float *alpha_dev, void *stream) {
    G2V_REQUIRE(V > 0 && D > 0 && n_rows >= 0 && n_rows <= V && (t >= 1 || alpha_dev),
                "g2v_cbow_lazy_adam: bad sizes (V=%d D=%d n_rows=%lld t=%d)", V, D, (long long)n_rows, t);
    G2V_REQUIRE(W_ih && m_ih && v_ih && W_ho && m_ho && v_ho && g_ho, "g2v_cbow_lazy_adam: null pointer");
    G2V_REQUIRE(n_rows == 0 || (rows && segptr && pos && dO), "g2v_cbow_lazy_adam: null row list");
    G2V_REQUIRE(weight_decay_ok(weight_decay),
                "g2v_cbow_lazy_adam_wd: weight_decay must be finite with 0 <= wd < 1 (got %g)", (double)weight_decay);
    cudaStream_t st = (cudaStream_t)stream;
    const float alpha = alpha_dev ? 0.f : adam_tf1_alpha(lr, beta1, beta2, t);
    const bool wd = weight_decay > 0.f;
    int rc, launches = 1;
    if (n_rows > 0) {
        int grid = 0;
        auto kern = wd ? cbow_lazy_adam_rows_kernel<true> : cbow_lazy_adam_rows_kernel<false>;
        if ((rc = rows_grid((const void *)kern, 0, n_rows, &grid))) return rc;
        kern<<<grid, kCbowWarps * 32, 0, st>>>(rows, segptr, pos, dO, n_rows, W_ih, m_ih, v_ih, W_ho, D, alpha,
                                               1.f - beta1, 1.f - beta2, eps, alpha_dev, loop_skip_flag(), weight_decay);
        G2V_CUDA_OK(cudaGetLastError());
        ++launches;
    }
    // W_ho (dense TF1 Adam from g_ho, which it zeroes) after every row has read the pre-step W_ho
    auto ho = wd ? cbow_update_kernel<G2V_OPT_ADAM_TF1, true> : cbow_update_kernel<G2V_OPT_ADAM_TF1, false>;
    ho<<<(unsigned)((D + 255) / 256), 256, 0, st>>>(nullptr, nullptr, nullptr, nullptr, 0, W_ho, m_ho, v_ho, g_ho,
                                                    (int64_t)D, alpha, 1.f - beta1, 1.f - beta2, eps, alpha_dev,
                                                    loop_skip_flag(), weight_decay);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch(launches);
    return 0;
}

extern "C" int g2v_cbow_lazy_adam(const int32_t *rows, const int32_t *segptr, const int32_t *pos, const float *dO,
                                  int64_t n_rows, float *W_ih, float *m_ih, float *v_ih, float *W_ho, float *m_ho,
                                  float *v_ho, float *g_ho, int32_t V, int32_t D, float lr, float beta1, float beta2,
                                  float eps, int32_t t, const float *alpha_dev, void *stream) {
    return g2v_cbow_lazy_adam_wd(rows, segptr, pos, dO, n_rows, W_ih, m_ih, v_ih, W_ho, m_ho, v_ho, g_ho, V, D, lr, beta1,
                                 beta2, eps, 0.f, t, alpha_dev, stream);
}

extern "C" int g2v_cbow_update_nvl_wd(float *const *g_ptrs_dev, float *const *w_ptrs_dev, float *g_multicast,
                                      float *w_multicast, float *m_flat, float *v_flat, int64_t n, int32_t rank,
                                      int32_t world, int32_t optimizer, float lr, float beta1, float beta2, float eps,
                                      float weight_decay, int32_t t, const float *alpha_dev, void *stream) {
    G2V_REQUIRE(n > 0 && world >= 1 && rank >= 0 && rank < world && (t >= 1 || alpha_dev), "g2v_cbow_update_nvl: bad sizes");
    G2V_REQUIRE(g_ptrs_dev && w_ptrs_dev, "g2v_cbow_update_nvl: null pointer tables");
    G2V_REQUIRE((g_multicast == nullptr) == (w_multicast == nullptr), "g2v_cbow_update_nvl: both or neither multicast pointer");
    G2V_REQUIRE(optimizer == G2V_OPT_ADAM_TF1 || optimizer == G2V_OPT_SGD, "g2v_cbow_update_nvl: unknown optimizer %d", optimizer);
    G2V_REQUIRE(optimizer == G2V_OPT_SGD || (m_flat && v_flat), "g2v_cbow_update_nvl: Adam needs m/v buffers");
    G2V_REQUIRE(weight_decay_ok(weight_decay),
                "g2v_cbow_update_nvl_wd: weight_decay must be finite with 0 <= wd < 1 (got %g)", (double)weight_decay);
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
        alpha = alpha_dev ? 0.f : adam_tf1_alpha(lr, beta1, beta2, t);
        omb1 = 1.f - beta1; omb2 = 1.f - beta2;
    } else {
        alpha_dev = nullptr;
    }
#define G2V_NVL(OPT, WD)                                                                                              \
    do {                                                                                                              \
        auto kern = mc ? cbow_update_nvl_kernel<OPT, true, WD> : cbow_update_nvl_kernel<OPT, false, WD>;              \
        kern<<<(unsigned)blocks, 256, 0, st>>>(g_ptrs_dev, w_ptrs_dev, g_multicast, w_multicast, m_flat, v_flat, n,   \
                                               rank, world, alpha, omb1, omb2, eps, alpha_dev, loop_skip_flag(),      \
                                               weight_decay);                                                         \
    } while (0)
    G2V_OPT_WD_DISPATCH(optimizer, weight_decay, G2V_NVL);
#undef G2V_NVL
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cbow_update_nvl(float *const *g_ptrs_dev, float *const *w_ptrs_dev, float *g_multicast,
                                   float *w_multicast, float *m_flat, float *v_flat, int64_t n, int32_t rank,
                                   int32_t world, int32_t optimizer, float lr, float beta1, float beta2, float eps,
                                   int32_t t, const float *alpha_dev, void *stream) {
    return g2v_cbow_update_nvl_wd(g_ptrs_dev, w_ptrs_dev, g_multicast, w_multicast, m_flat, v_flat, n, rank, world,
                                  optimizer, lr, beta1, beta2, eps, 0.f, t, alpha_dev, stream);
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
