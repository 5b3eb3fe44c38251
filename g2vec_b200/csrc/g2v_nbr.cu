// g2v_nbr.cu -- exact cosine K nearest genes of every gene (DESIGN.md §4.25).
//   nbr_norms_kernel    one warp per 32 genes: a 32 x 32 float chunk staged in shared memory, each lane running its
//                       gene's float64 chain n_i = sum_d W_id^2 in ascending d; inv_i = 1 / sqrt(n_i), 0 when n_i = 0.
//   nbr_partial_kernel  a CTA owns 64 rows and sweeps the 64-column tiles of its column range in ascending order:
//                       register-tiled FP64 FMA "GEMM" of W against itself (256 threads x 4 x 4 outputs, W converted to
//                       float64 in shared memory in chunks of 32 d consumed in ascending d, so every accumulator is
//                       the contract's sequential chain), then s = (dot * inv_i) * inv_j into shared memory and a
//                       top-K update of each row's list (one warp per 8 rows).  The similarity matrix is never stored.
//   nbr_merge_kernel    one warp per row, one lane per column split: a K-step merge of the splits' sorted lists.
// No tensor cores: the order of summation inside an FP64 MMA is unspecified, and the result here must be the
// sequential float64 chain bit for bit.  The lists are ordered by the total order (s descending, j ascending), so
// the result does not depend on the grid, the column split or the launch order.
#include "g2v_common.cuh"

#include <math.h>

namespace g2v {

constexpr int kNbrTile = 64;                           // rows and columns of a CTA tile
constexpr int kNbrDK = 32;                             // d per staged chunk
constexpr int kNbrThreads = 256, kNbrWarps = kNbrThreads / 32;
constexpr int kNbrLd = kNbrDK + 1;                     // padded staged row (doubles): conflict-free column reads
constexpr int kNbrSLd = kNbrTile + 1;                  // padded row of the similarity tile
constexpr int kNbrCtasPerSm = 2;                       // what the split plans for (83 KB of shared memory per CTA)
constexpr int kNbrMaxSplits = 32;                      // one merge lane per split
constexpr int kNbrRowsPerWarp = kNbrTile / kNbrWarps;

struct NbrSmem {
    union {
        double stage[2][kNbrTile][kNbrLd];             // [0] the CTA's rows, [1] the tile's columns, one d chunk
        double s[kNbrTile][kNbrSLd];                   // the tile's similarities
    } u;
    double ls[kNbrTile][G2V_NBR_MAX_K];                // each row's list, sorted by (s desc, j asc)
    int32_t lj[kNbrTile][G2V_NBR_MAX_K];
    int32_t cnt[kNbrTile];
};

// a precedes b in a list
__device__ __forceinline__ bool nbr_before(double sa, int32_t ja, double sb, int32_t jb) {
    return sa > sb || (sa == sb && ja < jb);
}

// ---- norms ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kNbrThreads)
nbr_norms_kernel(const float *__restrict__ W, int32_t m, int32_t D, double *__restrict__ inv) {
    __shared__ float tile[kNbrWarps][32][33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t g0 = ((int64_t)blockIdx.x * kNbrWarps + warp) * 32;
    if (g0 >= m) return;                               // warp-uniform; only __syncwarp below
    double acc = 0.0;
    for (int d0 = 0; d0 < D; d0 += 32) {
        const int d = d0 + lane;
        for (int g = 0; g < 32; ++g) {
            const int64_t row = g0 + g;
            tile[warp][g][lane] = (row < m && d < D) ? __ldg(W + row * D + d) : 0.f;
        }
        __syncwarp();
        const int kn = min(32, D - d0);
        for (int k = 0; k < kn; ++k) {
            const double x = (double)tile[warp][lane][k];
            acc = __fma_rn(x, x, acc);
        }
        __syncwarp();
    }
    const int64_t i = g0 + lane;
    if (i < m) inv[i] = acc > 0.0 ? __ddiv_rn(1.0, __dsqrt_rn(acc)) : 0.0;
}

// ---- partial lists -------------------------------------------------------------------------------------------
// Insert (s, j) into a row's sorted list of n entries (n < K, or n == K and s above the K-th): the entries that
// precede it are a prefix, the rest move one place down and the K-th of a full list falls off.
__device__ __forceinline__ void nbr_insert(double *ls, int32_t *lj, int n, int K, double s, int32_t j, int lane) {
    const int q0 = lane, q1 = lane + 32;
    const bool b0 = q0 < n && nbr_before(ls[q0], lj[q0], s, j);
    const bool b1 = q1 < n && nbr_before(ls[q1], lj[q1], s, j);
    const int p = __popc(__ballot_sync(0xffffffffu, b0)) + __popc(__ballot_sync(0xffffffffu, b1));
    const int last = min(n, K - 1);
    const bool m0 = q0 > p && q0 <= last, m1 = q1 > p && q1 <= last;
    double v0 = 0.0, v1 = 0.0;
    int32_t w0 = 0, w1 = 0;
    if (m0) { v0 = ls[q0 - 1]; w0 = lj[q0 - 1]; }
    if (m1) { v1 = ls[q1 - 1]; w1 = lj[q1 - 1]; }
    __syncwarp();
    if (m0) { ls[q0] = v0; lj[q0] = w0; }
    if (m1) { ls[q1] = v1; lj[q1] = w1; }
    if (q0 == p) { ls[q0] = s; lj[q0] = j; }
    if (q1 == p) { ls[q1] = s; lj[q1] = j; }
    __syncwarp();
}

// Chunk loads: warp w fetches rows w + 8 q (q < 8) of a 64-row block, lane = d offset; out of range -> 0.
__device__ __forceinline__ void nbr_load(const float *__restrict__ W, int32_t m, int32_t D, int32_t base, int d0,
                                         int warp, int lane, float r[8]) {
    const int d = d0 + lane;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const int32_t row = base + warp + 8 * q;
        r[q] = (row < m && d < D) ? __ldg(W + (int64_t)row * D + d) : 0.f;
    }
}

// Zero padding past D (rows past m) adds fma(0, 0, acc) = acc exactly: acc is never -0, since it starts at +0 and a
// round-to-nearest sum is -0 only when both terms are.  So every chunk runs all 32 steps.
__global__ void __launch_bounds__(kNbrThreads, kNbrCtasPerSm)
nbr_partial_kernel(const float *__restrict__ W, const double *__restrict__ inv, int32_t m, int32_t D, int32_t K,
                   int32_t splits, int32_t *__restrict__ part_idx, double *__restrict__ part_sim) {
    extern __shared__ __align__(16) unsigned char nbr_smem_raw[];
    NbrSmem &sm = *reinterpret_cast<NbrSmem *>(nbr_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tx = tid & 15, ty = tid >> 4;            // outputs: rows ty + 16 r, columns tx + 16 c
    const int32_t row0 = (int32_t)blockIdx.x * kNbrTile;
    const int32_t n_ct = (m + kNbrTile - 1) / kNbrTile;
    const int32_t t_begin = (int32_t)((int64_t)blockIdx.y * n_ct / splits);
    const int32_t t_end = (int32_t)((int64_t)(blockIdx.y + 1) * n_ct / splits);
    if (tid < kNbrTile) sm.cnt[tid] = 0;
    double inv_r[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int32_t i = row0 + ty + 16 * r;
        inv_r[r] = i < m ? inv[i] : 0.0;
    }
    for (int32_t t = t_begin; t < t_end; ++t) {
        const int32_t col0 = t * kNbrTile;
        double acc[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
        float ra[8], rb[8];
        nbr_load(W, m, D, row0, 0, warp, lane, ra);
        nbr_load(W, m, D, col0, 0, warp, lane, rb);
        for (int d0 = 0; d0 < D; d0 += kNbrDK) {
            __syncthreads();                           // the last chunk (or the last tile's epilogue) is done with u
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                sm.u.stage[0][warp + 8 * q][lane] = (double)ra[q];
                sm.u.stage[1][warp + 8 * q][lane] = (double)rb[q];
            }
            __syncthreads();
            if (d0 + kNbrDK < D) {                     // the next chunk is in flight while this one is consumed
                nbr_load(W, m, D, row0, d0 + kNbrDK, warp, lane, ra);
                nbr_load(W, m, D, col0, d0 + kNbrDK, warp, lane, rb);
            }
#pragma unroll
            for (int k = 0; k < kNbrDK; ++k) {
                double a[4], b[4];
#pragma unroll
                for (int r = 0; r < 4; ++r) a[r] = sm.u.stage[0][ty + 16 * r][k];
#pragma unroll
                for (int c = 0; c < 4; ++c) b[c] = sm.u.stage[1][tx + 16 * c][k];
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[r][c] = __fma_rn(a[r], b[c], acc[r][c]);
            }
        }
        __syncthreads();                               // every warp is done with the stage: it becomes s
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int32_t j = col0 + tx + 16 * c;
            const double inv_c = j < m ? inv[j] : 0.0;
#pragma unroll
            for (int r = 0; r < 4; ++r)
                sm.u.s[ty + 16 * r][tx + 16 * c] =
                    (inv_r[r] == 0.0 || inv_c == 0.0) ? 0.0 : __dmul_rn(__dmul_rn(acc[r][c], inv_r[r]), inv_c);
        }
        __syncthreads();
        for (int rr = 0; rr < kNbrRowsPerWarp; ++rr) {
            const int r = warp * kNbrRowsPerWarp + rr;
            const int32_t i = row0 + r;
            if (i >= m) break;                         // warp-uniform
            double *ls = sm.ls[r];
            int32_t *lj = sm.lj[r];
            int n = sm.cnt[r];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int32_t j = col0 + h * 32 + lane;
                const double s = sm.u.s[r][h * 32 + lane];
                const bool pass = j < m && j != i && (n < K || s > ls[K - 1]);
                unsigned mask = __ballot_sync(0xffffffffu, pass);
                while (mask) {                         // ascending j; a candidate enters a full list only if it
                    const int b = __ffs(mask) - 1;     // is strictly above the current K-th value
                    mask &= mask - 1;
                    const double cs = __shfl_sync(0xffffffffu, s, b);
                    if (n == K && !(cs > ls[K - 1])) continue;
                    nbr_insert(ls, lj, n, K, cs, col0 + h * 32 + b, lane);
                    n = min(n + 1, K);
                }
            }
            __syncwarp();
            if (lane == 0) sm.cnt[r] = n;
        }
    }
    __syncthreads();
    // the list of row i from split y at [(y * m + i) * K]; a split with fewer than K columns pads with j = -1
    for (int rr = 0; rr < kNbrRowsPerWarp; ++rr) {
        const int r = warp * kNbrRowsPerWarp + rr;
        const int32_t i = row0 + r;
        if (i >= m) break;
        const int n = sm.cnt[r];
        const size_t base = ((size_t)blockIdx.y * m + i) * K;
        for (int q = lane; q < K; q += 32) {
            part_sim[base + q] = q < n ? sm.ls[r][q] : -INFINITY;
            part_idx[base + q] = q < n ? sm.lj[r][q] : -1;
        }
    }
}

// ---- merge ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kNbrThreads)
nbr_merge_kernel(const int32_t *__restrict__ part_idx, const double *__restrict__ part_sim, int32_t splits, int32_t m,
                 int32_t K, int32_t *__restrict__ idx, double *__restrict__ sim) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kNbrWarps + (threadIdx.x >> 5);
    if (i >= m) return;
    const size_t off = ((size_t)lane * m + i) * K;
    const int32_t *pj = part_idx + off;
    const double *ps = part_sim + off;
    int h = 0;
    // the head of this lane's list; exhausted or padded heads lose to every real entry (s is finite)
    double s = -INFINITY;
    int32_t j = 0x7fffffff;
    if (lane < splits && pj[0] >= 0) { s = ps[0]; j = pj[0]; }
    for (int q = 0; q < K; ++q) {
        double bs = s;
        int32_t bj = j;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double os = __shfl_xor_sync(0xffffffffu, bs, o);
            const int32_t oj = __shfl_xor_sync(0xffffffffu, bj, o);
            if (nbr_before(os, oj, bs, bj)) { bs = os; bj = oj; }
        }
        if (lane == 0) {
            idx[i * K + q] = bj;
            sim[i * K + q] = bs;
        }
        if (j == bj) {                                 // column ranges are disjoint: one lane holds bj
            ++h;
            s = -INFINITY;
            j = 0x7fffffff;
            if (h < K && pj[h] >= 0) { s = ps[h]; j = pj[h]; }
        }
    }
}

// The column split: a function of m and the SM count only.  With rb = ceil(m / 64) row blocks (= column tiles) and
// kNbrCtasPerSm CTAs per SM, it minimises the column tiles on the critical path, waves * ceil(rb / splits); the
// smallest such split wins.
int nbr_splits_for(int32_t m, int sm_count) {
    const int64_t rb = (m + kNbrTile - 1) / kNbrTile;
    const int64_t slots = (int64_t)sm_count * kNbrCtasPerSm;
    int best = 1;
    int64_t best_cost = INT64_MAX;
    for (int s = 1; s <= kNbrMaxSplits && s <= rb; ++s) {
        const int64_t cost = ((rb * s + slots - 1) / slots) * ((rb + s - 1) / s);
        if (cost < best_cost) { best_cost = cost; best = s; }
    }
    return best;
}

}  // namespace g2v

using namespace g2v;

#define G2V_NBR_CHECK_SIZES(fn, m, D)                                                                             \
    do {                                                                                                        \
        G2V_REQUIRE((m) >= 2 && (m) <= G2V_NBR_MAX_GENES, fn ": m = %lld genes, must be in [2, %d]", (long long)(m), \
                    G2V_NBR_MAX_GENES);                                                                         \
        G2V_REQUIRE((D) >= 1, fn ": D = %d, must be >= 1", (int)(D));                                             \
    } while (0)

#define G2V_NBR_CHECK_K(fn, m, K)                                                                                 \
    G2V_REQUIRE((K) >= 1 && (K) <= G2V_NBR_MAX_K && (int64_t)(K) < (m), fn ": K = %d, must be in [1, min(%d, m - 1)]", \
                (int)(K), G2V_NBR_MAX_K)

extern "C" int32_t g2v_nbr_splits(int64_t m) {
    if (m < 2 || m > G2V_NBR_MAX_GENES) {
        set_error("g2v_nbr_splits: m = %lld genes, must be in [2, %d]", (long long)m, G2V_NBR_MAX_GENES);
        return 0;
    }
    DeviceProps dp;
    if (device_props(&dp)) return 0;
    return nbr_splits_for((int32_t)m, dp.sm_count);
}

extern "C" int g2v_nbr_norms(const float *W, int64_t m, int32_t D, double *inv, void *stream) {
    G2V_REQUIRE(W && inv, "g2v_nbr_norms: null pointer");
    G2V_NBR_CHECK_SIZES("g2v_nbr_norms", m, D);
    const int64_t genes_per_cta = 32 * kNbrWarps;
    nbr_norms_kernel<<<(unsigned)((m + genes_per_cta - 1) / genes_per_cta), kNbrThreads, 0, (cudaStream_t)stream>>>(
        W, (int32_t)m, D, inv);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_nbr_partial(const float *W, const double *inv, int64_t m, int32_t D, int32_t K, int32_t *part_idx,
                               double *part_sim, void *stream) {
    G2V_REQUIRE(W && inv && part_idx && part_sim, "g2v_nbr_partial: null pointer");
    G2V_NBR_CHECK_SIZES("g2v_nbr_partial", m, D);
    G2V_NBR_CHECK_K("g2v_nbr_partial", m, K);
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    const int splits = nbr_splits_for((int32_t)m, dp.sm_count);
    const size_t smem = sizeof(NbrSmem);
    G2V_REQUIRE(smem <= (size_t)dp.max_smem_optin, "g2v_nbr_partial: needs %zu B of shared memory per block", smem);
    G2V_CUDA_OK(cudaFuncSetAttribute(nbr_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((unsigned)((m + kNbrTile - 1) / kNbrTile), (unsigned)splits);
    nbr_partial_kernel<<<grid, kNbrThreads, smem, (cudaStream_t)stream>>>(W, inv, (int32_t)m, D, K, splits, part_idx,
                                                                         part_sim);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_nbr_merge(const int32_t *part_idx, const double *part_sim, int32_t splits, int64_t m, int32_t K,
                             int32_t *idx, double *sim, void *stream) {
    G2V_REQUIRE(part_idx && part_sim && idx && sim, "g2v_nbr_merge: null pointer");
    G2V_REQUIRE(m >= 2 && m <= G2V_NBR_MAX_GENES, "g2v_nbr_merge: m = %lld genes, must be in [2, %d]", (long long)m,
                G2V_NBR_MAX_GENES);
    G2V_NBR_CHECK_K("g2v_nbr_merge", m, K);
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    const int want = nbr_splits_for((int32_t)m, dp.sm_count);
    G2V_REQUIRE(splits == want && splits > 1, "g2v_nbr_merge: splits = %d, g2v_nbr_splits(%lld) = %d (must be > 1)",
                (int)splits, (long long)m, want);
    nbr_merge_kernel<<<(unsigned)((m + kNbrWarps - 1) / kNbrWarps), kNbrThreads, 0, (cudaStream_t)stream>>>(
        part_idx, part_sim, splits, (int32_t)m, K, idx, sim);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
