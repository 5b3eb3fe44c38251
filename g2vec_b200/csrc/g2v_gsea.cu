// g2v_gsea.cu -- phenotype-permutation gene-set enrichment of the good / poor contrast (DESIGN.md §4.28).
//   gsea_keys_kernel    one pass over [n_b, G]: the exact N = n A - k Q of every (labelling, gene), the point-biserial
//                       r = (s N) / sqrt(W) in float64, rq = rint(r 2^32), the weight u = |rq| and the unique sort key
//                       ((2^32 - rq) << 20) | g, so that ascending keys are rq descending, ties by gene ascending.
//   g2v_gsea_rank       CUB's segmented radix sort of each row's keys over bits [0, 54), then gsea_scatter_kernel
//                       writes pos[row][g] = the rank of gene g.
//   gsea_es_kernel      the hot path: one warp per (row, set).  The warp gathers its members' pos and u from the row
//                       (which the CTAs of one row share through the L2), packs (pos << 34 | u), bitonic-sorts the
//                       packed words in shared memory, takes the prefix sums S_j with an integer warp scan, forms the
//                       two running-sum terms with three correctly rounded float64 operations each and reduces their
//                       max and min.  No floating-point atomics.
//   gsea_norm_kernel    one thread per set, sequential over the permutations (coalesced over the sets): mean+ and
//                       mean-, the observed NES, the null NES column and the nominal counts.
// Everything ES depends on is integer up to its last three float64 operations, so ES, NES and the counts equal the
// NumPy restatement bit for bit whatever the grid, the chunking or the sort.
#include <cub/device/device_segmented_radix_sort.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "g2v_common.cuh"

namespace g2v {

constexpr int kGseaGeneBits = 20;                      // G <= 2^20: the gene index in the low bits of the key
constexpr int kGseaKeyBits = 54;                       // 2^32 - rq <= 2^33 above the gene bits
constexpr int kGseaUBits = 34;                         // u <= 2^32 below pos in the packed member word
constexpr uint64_t kGseaUMask = (1ull << kGseaUBits) - 1;

// ---- keys ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gsea_keys_kernel(const int64_t *__restrict__ A, int64_t n_b, int32_t G, int32_t n, int32_t k, int32_t s,
                 const int64_t *__restrict__ Q, const double *__restrict__ W, uint64_t *__restrict__ key,
                 uint64_t *__restrict__ u) {
    const int64_t total = n_b * (int64_t)G;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t g = (int32_t)(i % G);
        const int64_t N = (int64_t)n * A[i] - (int64_t)k * __ldg(Q + g);
        const double w = __ldg(W + g);
        const double r = w > 0.0 ? __ddiv_rn(__ll2double_rn(s > 0 ? N : -N), __dsqrt_rn(w)) : 0.0;
        const int64_t rq = __double2ll_rn(__dmul_rn(r, 4294967296.0));
        key[i] = ((uint64_t)((1ll << 32) - rq) << kGseaGeneBits) | (uint64_t)g;
        u[i] = (uint64_t)(rq < 0 ? -rq : rq);
    }
}

// ---- rank ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gsea_scatter_kernel(const uint64_t *__restrict__ sorted, int64_t n_b, int32_t G, int32_t *__restrict__ pos) {
    const int64_t total = n_b * (int64_t)G;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / G;
        const int32_t rank = (int32_t)(i - row * G);
        pos[row * G + (int64_t)(sorted[i] & ((1ull << kGseaGeneBits) - 1))] = rank;
    }
}

struct RowOffset {
    int32_t G;
    __host__ __device__ int operator()(int r) const { return r * G; }
};

// ---- enrichment scores --------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t warp_inclusive_scan_u64(uint64_t v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// grid (ceil(n_sets / warps), n_b); warp w of CTA x owns set x * warps + w of row blockIdx.y, with `cap` packed words
// of dynamic shared memory (cap = the power of two >= the largest set, at least 32).
__global__ void __launch_bounds__(256)
gsea_es_kernel(const int32_t *__restrict__ pos, const uint64_t *__restrict__ u, int32_t G,
               const int32_t *__restrict__ set_ptr, const int32_t *__restrict__ set_gene, int32_t n_sets, int32_t cap,
               double *__restrict__ es) {
    extern __shared__ uint64_t sh_es[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int32_t set = blockIdx.x * (blockDim.x >> 5) + warp;
    if (set >= n_sets) return;
    const int64_t row = blockIdx.y;
    uint64_t *w = sh_es + (size_t)warp * cap;
    const int32_t b = __ldg(set_ptr + set), k = __ldg(set_ptr + set + 1) - b;
    int32_t kp = 32;
    while (kp < k) kp <<= 1;
    const int32_t *prow = pos + row * G;
    const uint64_t *urow = u + row * G;
    uint64_t tot = 0;
    for (int32_t j = lane; j < kp; j += 32) {
        uint64_t v = ~0ull;                             // padding sorts last
        if (j < k) {
            const int32_t g = __ldg(set_gene + b + j);
            const uint64_t uj = __ldg(urow + g);
            tot += uj;
            v = ((uint64_t)__ldg(prow + g) << kGseaUBits) | uj;
        }
        w[j] = v;
    }
    const uint64_t NR = warp_sum_u64(tot);
    __syncwarp();
    for (int32_t size = 2; size <= kp; size <<= 1)
        for (int32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (int32_t i = lane; i < (kp >> 1); i += 32) {
                const int32_t lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const uint64_t x = w[lo], y = w[hi];
                if ((x > y) == ((lo & size) == 0)) {
                    w[lo] = y;
                    w[hi] = x;
                }
            }
            __syncwarp();
        }
    double dp = 0.0, dm = 0.0;
    if (NR != 0) {
        const double nr = __ull2double_rn(NR), miss = (double)(G - k);
        uint64_t carry = 0;
        for (int32_t base = 0; base < k; base += 32) {
            const int32_t j = base + lane;
            const uint64_t v = j < k ? w[j] : 0ull;
            const uint64_t uj = v & kGseaUMask;
            const uint64_t S = carry + warp_inclusive_scan_u64(uj, lane);
            carry = __shfl_sync(0xffffffffu, S, 31);
            if (j < k) {
                const double m = __int2double_rn((int32_t)(v >> kGseaUBits) - j);
                const double mq = __ddiv_rn(m, miss);
                const double tp = __dsub_rn(__ddiv_rn(__ull2double_rn(S), nr), mq);
                const double tm = __dsub_rn(__ddiv_rn(__ull2double_rn(S - uj), nr), mq);
                if (tp > dp) dp = tp;
                if (tm < dm) dm = tm;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            dp = fmax(dp, __shfl_xor_sync(0xffffffffu, dp, o));
            dm = fmin(dm, __shfl_xor_sync(0xffffffffu, dm, o));
        }
    }
    if (lane == 0) es[row * n_sets + set] = dp >= -dm ? dp : dm;
}

// ---- normalisation ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
gsea_norm_kernel(const double *__restrict__ es, int64_t B, int32_t n_sets, const double *__restrict__ es_obs,
                 double *__restrict__ nes, double *__restrict__ mean_pos, double *__restrict__ mean_neg,
                 double *__restrict__ nes_obs, int64_t *__restrict__ counts) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_sets) return;
    const double e0 = es_obs[s];
    double sp = 0.0, sn = 0.0;
    int64_t np_ = 0, nn = 0, ext = 0;
    for (int64_t b = 0; b < B; ++b) {
        const double e = es[b * n_sets + s];
        if (e >= 0.0) {
            sp = __dadd_rn(sp, e);
            ++np_;
        } else {
            sn = __dadd_rn(sn, -e);
            ++nn;
        }
        ext += e0 >= 0.0 ? (e >= e0) : (e <= e0);
    }
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    const double mp = np_ ? __ddiv_rn(sp, __ll2double_rn(np_)) : qnan;
    const double mn = nn ? __ddiv_rn(sn, __ll2double_rn(nn)) : qnan;
    const double n0 = e0 >= 0.0 ? (np_ ? __ddiv_rn(e0, mp) : qnan) : (nn ? __ddiv_rn(e0, mn) : qnan);
    const bool valid = !isnan(n0);
    for (int64_t b = 0; b < B; ++b) {
        const double e = es[b * n_sets + s];
        nes[b * n_sets + s] = valid ? __ddiv_rn(e, e >= 0.0 ? mp : mn) : qnan;
    }
    mean_pos[s] = mp;
    mean_neg[s] = mn;
    nes_obs[s] = n0;
    counts[s] = np_;
    counts[n_sets + s] = nn;
    counts[2 * (int64_t)n_sets + s] = ext;
}

static int es_cap(int32_t max_k) {
    int cap = 32;
    while (cap < max_k) cap <<= 1;
    return cap;
}

}  // namespace g2v

using namespace g2v;

#define G2V_GSEA_CHECK_ROWS(fn, n_b, G)                                                                             \
    G2V_REQUIRE((G) >= 2 && (G) <= G2V_GSEA_MAX_GENES, fn ": G = %d genes, must be in [2, %d]", (int)(G),             \
                G2V_GSEA_MAX_GENES);                                                                                \
    G2V_REQUIRE((n_b) >= 1 && (n_b) <= G2V_GSEA_MAX_ROWS && (n_b) * (int64_t)(G) <= INT32_MAX,                      \
                fn ": n_b = %lld rows of %d genes, must be in [1, %d] with n_b * G < 2^31", (long long)(n_b), (int)(G), \
                G2V_GSEA_MAX_ROWS)

static unsigned grid_1d(int64_t total) {
    const int64_t g = (total + 255) / 256;
    return (unsigned)(g < 8192 ? g : 8192);
}

extern "C" int g2v_gsea_keys(const int64_t *A, int64_t n_b, int32_t G, int32_t n, int32_t k, int32_t s,
                             const int64_t *Q, const double *W, uint64_t *key, uint64_t *u, void *stream) {
    G2V_REQUIRE(A && Q && W && key && u, "g2v_gsea_keys: null pointer");
    G2V_GSEA_CHECK_ROWS("g2v_gsea_keys", n_b, G);
    G2V_REQUIRE(n >= 3 && n <= G2V_PERM_MAX_SAMPLES, "g2v_gsea_keys: n = %d samples, must be in [3, %d]", (int)n,
                G2V_PERM_MAX_SAMPLES);
    G2V_REQUIRE(k >= 1 && k < n, "g2v_gsea_keys: k = %d, must be in [1, n - 1 = %d]", (int)k, (int)n - 1);
    G2V_REQUIRE(s == 1 || s == -1, "g2v_gsea_keys: s = %d, must be +1 or -1", (int)s);
    gsea_keys_kernel<<<grid_1d(n_b * G), 256, 0, (cudaStream_t)stream>>>(A, n_b, G, n, k, s, Q, W, key, u);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" size_t g2v_gsea_rank_workspace_bytes(int64_t n_b, int32_t G) {
    if (G < 2 || G > G2V_GSEA_MAX_GENES || n_b < 1 || n_b > G2V_GSEA_MAX_ROWS || n_b * (int64_t)G > INT32_MAX)
        return 0;
    auto offs = thrust::make_transform_iterator(thrust::make_counting_iterator<int>(0), RowOffset{G});
    size_t tmp = 0;
    if (cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tmp, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                                (int)(n_b * G), (int)n_b, offs, offs + 1, 0, kGseaKeyBits) !=
        cudaSuccess)
        return 0;
    const size_t keys = ((size_t)n_b * G * sizeof(uint64_t) + 255) & ~(size_t)255;
    return keys + tmp;
}

extern "C" int g2v_gsea_rank(const uint64_t *key, int64_t n_b, int32_t G, int32_t *pos, void *workspace,
                             size_t workspace_bytes, void *stream) {
    G2V_REQUIRE(key && pos && workspace, "g2v_gsea_rank: null pointer");
    G2V_GSEA_CHECK_ROWS("g2v_gsea_rank", n_b, G);
    const size_t need = g2v_gsea_rank_workspace_bytes(n_b, G);
    G2V_REQUIRE(need > 0 && workspace_bytes >= need, "g2v_gsea_rank: workspace of %zu bytes, needs %zu",
                workspace_bytes, need);
    const size_t keys = ((size_t)n_b * G * sizeof(uint64_t) + 255) & ~(size_t)255;
    uint64_t *sorted = static_cast<uint64_t *>(workspace);
    size_t tmp = need - keys;
    auto offs = thrust::make_transform_iterator(thrust::make_counting_iterator<int>(0), RowOffset{G});
    G2V_CUDA_OK(cub::DeviceSegmentedRadixSort::SortKeys(static_cast<char *>(workspace) + keys, tmp, key, sorted,
                                                        (int)(n_b * G), (int)n_b, offs, offs + 1, 0, kGseaKeyBits,
                                                        (cudaStream_t)stream));
    gsea_scatter_kernel<<<grid_1d(n_b * G), 256, 0, (cudaStream_t)stream>>>(sorted, n_b, G, pos);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch(2);
    return 0;
}

extern "C" int g2v_gsea_es(const int32_t *pos, const uint64_t *u, int64_t n_b, int32_t G, const int32_t *set_ptr,
                           const int32_t *set_gene, int32_t n_sets, int32_t max_k, double *es, void *stream) {
    G2V_REQUIRE(pos && u && set_ptr && set_gene && es, "g2v_gsea_es: null pointer");
    G2V_GSEA_CHECK_ROWS("g2v_gsea_es", n_b, G);
    G2V_REQUIRE(n_sets >= 1 && n_sets <= G2V_GSEA_MAX_SETS, "g2v_gsea_es: %d sets, must be in [1, %d]", (int)n_sets,
                G2V_GSEA_MAX_SETS);
    G2V_REQUIRE(max_k >= 1 && max_k <= G2V_GSEA_MAX_SET_SIZE && max_k < G,
                "g2v_gsea_es: max_k = %d, must be in [1, min(%d, G - 1 = %d)]", (int)max_k, G2V_GSEA_MAX_SET_SIZE,
                (int)G - 1);
    const int cap = es_cap(max_k);
    int warps = (48 * 1024) / (cap * (int)sizeof(uint64_t));
    warps = warps < 1 ? 1 : (warps > 8 ? 8 : warps);
    const size_t smem = (size_t)warps * cap * sizeof(uint64_t);
    const dim3 grid((unsigned)((n_sets + warps - 1) / warps), (unsigned)n_b);
    gsea_es_kernel<<<grid, 32 * warps, smem, (cudaStream_t)stream>>>(pos, u, G, set_ptr, set_gene, n_sets, cap, es);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_gsea_norm(const double *es, int64_t B, int32_t n_sets, const double *es_obs, double *nes,
                             double *mean_pos, double *mean_neg, double *nes_obs, int64_t *counts, void *stream) {
    G2V_REQUIRE(es && es_obs && nes && mean_pos && mean_neg && nes_obs && counts, "g2v_gsea_norm: null pointer");
    G2V_REQUIRE(B >= 1 && B <= G2V_GSEA_MAX_PERMUTATIONS, "g2v_gsea_norm: B = %lld, must be in [1, %d]",
                (long long)B, G2V_GSEA_MAX_PERMUTATIONS);
    G2V_REQUIRE(n_sets >= 1 && n_sets <= G2V_GSEA_MAX_SETS && B * (int64_t)n_sets <= G2V_GSEA_MAX_ES,
                "g2v_gsea_norm: %d sets x %lld permutations, must be 1 <= S <= %d with B * S <= %d", (int)n_sets,
                (long long)B, G2V_GSEA_MAX_SETS, G2V_GSEA_MAX_ES);
    gsea_norm_kernel<<<(unsigned)((n_sets + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        es, B, n_sets, es_obs, nes, mean_pos, mean_neg, nes_obs, counts);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
