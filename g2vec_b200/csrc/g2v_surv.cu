// g2v_surv.cu -- permutation Cox score test of every gene against survival (DESIGN.md §4.31).
//   surv_rows_kernel    one warp per permutation: Fisher-Yates on the identity in shared memory with exactly the
//                       draws of perm_labels_kernel's row b (lanes draw 32 swap targets at a time, lane 0 swaps in
//                       order), then the scatter idx[slot[pi_b(s)]] = s: the sample whose expression sits at each
//                       time position.
//   surv_scores_kernel  one thread per (gene, permutation); a warp holds 32 consecutive genes of one permutation, a CTA
//                       kScoreWarps permutations of the same 32-gene tile, and the grid runs the permutations fastest
//                       so that the CTAs in flight share the tile's column of q in L1/L2.  The warp walks the time
//                       positions in descending time: every step loads one 128-byte line of q (warp-uniform row) and
//                       adds it into the exact int64 risk-set sums S1 = sum q and S2 = sum q^2 (and E1, d over the
//                       events); at the end of a time group with events it forms num_u = S0 E1 - d S1 and
//                       num_v = S0 S2 - S1^2 (exact int64) and adds u = num_u * a and v = double(num_v) * c into U and V.
// Every floating-point operation is one correctly rounded float64 operation in a fixed order (no fma contraction, no
// division in the loop), so U, V and T = U^2 / V are the bits a NumPy restatement computes.
#include "g2v_common.cuh"

namespace g2v {

// ---- permutation rows ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
surv_rows_kernel(const int32_t *__restrict__ slot, int32_t n, uint64_t seed, int64_t b_begin,
                 uint16_t *__restrict__ idx) {
    extern __shared__ uint16_t arr[];                  // [n]: pi_b(s) at s
    __shared__ uint32_t js[32];                        // the swap targets of one round of 32 draws
    const int lane = threadIdx.x;
    const int64_t r = blockIdx.x;
    const uint64_t subseq = (1ull << 63) + (uint64_t)(b_begin + r + 1);
    for (int s = lane; s < n; s += 32) arr[s] = (uint16_t)s;
    __syncwarp();
    for (int base = 0; base < n - 1; base += 32) {
        const int s = base + lane;                     // draw s swaps position i = n-1-s
        js[lane] = s < n - 1 ? (uint32_t)__umul64hi(draw64(seed, subseq, (uint32_t)s), (uint64_t)(n - s)) : 0u;
        __syncwarp();
        if (lane == 0) {
            const int cnt = min(32, n - 1 - base);
            for (int t = 0; t < cnt; ++t) {
                const int i = n - 1 - (base + t);
                const uint32_t jt = js[t];
                const uint16_t x = arr[i];
                arr[i] = arr[jt];
                arr[jt] = x;
            }
        }
        __syncwarp();                                  // the swaps are done before js is rewritten or arr read
    }
    uint16_t *row = idx + r * n;
    for (int s = lane; s < n; s += 32) row[__ldg(slot + arr[s])] = (uint16_t)s;
}

// ---- scores -------------------------------------------------------------------------------------------------
constexpr int kScoreWarps = 8, kScoreThreads = 32 * kScoreWarps, kScoreUnroll = 8;

__global__ void __launch_bounds__(kScoreThreads)
surv_scores_kernel(const int32_t *__restrict__ q, int32_t n, int32_t G, const uint16_t *__restrict__ idx,
                   int64_t n_b, const uint8_t *__restrict__ flags, const double *__restrict__ a,
                   const double *__restrict__ c, double *__restrict__ T, double *__restrict__ UV) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * kScoreWarps + (threadIdx.x >> 5);
    if (r >= n_b) return;                              // whole warps only
    const int64_t g = (int64_t)blockIdx.y * 32 + lane;
    const bool ok = g < G;
    const int32_t *qg = q + (ok ? g : 0);
    const uint16_t *row = idx + r * n;
    int64_t S1 = 0, S2 = 0, E1 = 0;
    int32_t d = 0;
    double U = 0.0, V = 0.0;
    for (int i0 = 0; i0 < n; i0 += 32) {
        // lane l holds position i0 + l: the sample (low 16 bits) and the position's flags (bits 16, 17)
        const uint32_t word = i0 + lane < n ? (uint32_t)__ldg(row + i0 + lane) | ((uint32_t)__ldg(flags + i0 + lane) << 16)
                                            : 0u;
        const int cnt = min(32, n - i0);
        for (int j0 = 0; j0 < cnt; j0 += kScoreUnroll) {
            int32_t x[kScoreUnroll];
            uint32_t f[kScoreUnroll];
#pragma unroll
            for (int u = 0; u < kScoreUnroll; ++u) {   // the loads first, so that they are in flight together
                const uint32_t w = __shfl_sync(0xffffffffu, word, (j0 + u) & 31);
                f[u] = j0 + u < cnt ? w >> 16 : 0u;
                x[u] = j0 + u < cnt ? __ldg(qg + (int64_t)(w & 0xffffu) * G) : 0;
            }
#pragma unroll
            for (int u = 0; u < kScoreUnroll; ++u) {
                if (j0 + u >= cnt) break;              // warp-uniform
                S1 += x[u];
                S2 += (int64_t)x[u] * x[u];
                if (f[u] & 1u) {
                    E1 += x[u];
                    ++d;
                }
                if (f[u] & 2u) {                       // the last position of its time group
                    if (d > 0) {
                        const int64_t S0 = i0 + j0 + u + 1;
                        const int64_t num_u = S0 * E1 - (int64_t)d * S1;      // |num_u| <= 2^47: exact as a double
                        const int64_t num_v = S0 * S2 - S1 * S1;              // 0 <= num_v <= 2^62
                        const int p = i0 + j0 + u;
                        U = __dadd_rn(U, __dmul_rn(__ll2double_rn(num_u), __ldg(a + p)));
                        V = __dadd_rn(V, __dmul_rn(__ll2double_rn(num_v), __ldg(c + p)));
                    }
                    E1 = 0;
                    d = 0;
                }
            }
        }
    }
    if (!ok) return;
    T[r * G + g] = V > 0.0 ? __ddiv_rn(__dmul_rn(U, U), V) : 0.0;
    if (UV) {
        UV[r * G + g] = U;
        UV[(n_b + r) * G + g] = V;
    }
}

}  // namespace g2v

using namespace g2v;

#define G2V_SURV_CHECK_SAMPLES(fn, n)                                                                        \
    G2V_REQUIRE((n) >= 3 && (n) <= G2V_SURV_MAX_SAMPLES, fn ": n = %d samples, must be in [3, %d]", (int)(n),       \
                G2V_SURV_MAX_SAMPLES)

extern "C" int g2v_surv_rows(const int32_t *slot, int32_t n, uint64_t seed, int64_t b_begin, int64_t n_b,
                             uint16_t *idx, void *stream) {
    G2V_REQUIRE(slot && idx, "g2v_surv_rows: null pointer");
    G2V_SURV_CHECK_SAMPLES("g2v_surv_rows", n);
    G2V_REQUIRE(b_begin >= 0 && n_b >= 1 && b_begin + n_b <= G2V_SURV_MAX_PERMUTATIONS,
                "g2v_surv_rows: permutations %lld + [1, %lld] out of [1, %d]", (long long)b_begin, (long long)n_b,
                G2V_SURV_MAX_PERMUTATIONS);
    const size_t smem = (size_t)n * sizeof(uint16_t);
    G2V_CUDA_OK(cudaFuncSetAttribute(surv_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    surv_rows_kernel<<<(unsigned)n_b, 32, smem, (cudaStream_t)stream>>>(slot, n, seed, b_begin, idx);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_surv_scores(const int32_t *q, int32_t n, int32_t G, const uint16_t *idx, int64_t n_b,
                               const uint8_t *flags, const double *a, const double *c, double *T, double *UV,
                               void *stream) {
    G2V_REQUIRE(q && idx && flags && a && c && T, "g2v_surv_scores: null pointer");
    G2V_SURV_CHECK_SAMPLES("g2v_surv_scores", n);
    G2V_REQUIRE(G >= 1 && G <= G2V_SURV_MAX_GENES, "g2v_surv_scores: G = %d genes, must be in [1, %d]", (int)G,
                G2V_SURV_MAX_GENES);
    G2V_REQUIRE(n_b >= 1 && n_b <= G2V_SURV_MAX_PERMUTATIONS, "g2v_surv_scores: n_b = %lld rows, must be in [1, %d]",
                (long long)n_b, G2V_SURV_MAX_PERMUTATIONS);
    const dim3 grid((unsigned)((n_b + kScoreWarps - 1) / kScoreWarps), (unsigned)((G + 31) / 32));
    surv_scores_kernel<<<grid, kScoreThreads, 0, (cudaStream_t)stream>>>(q, n, G, idx, n_b, flags, a, c, T, UV);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
