// g2v_corr.cu -- rank-based and robust edge weights (DESIGN.md §4.22): Spearman's rho and the biweight
// midcorrelation ("bicor", WGCNA; Langfelder & Horvath 2012) as a per-gene transform z of one group's expression,
// with mean_s z[a][s] * z[b][s] equal to the coefficient, so that pcc_edge_kernel (g2v_pcc.cu) computes the edge
// weights unchanged.
//   corr_transpose_kernel  32x32 tiles: expr [S][V] sample-major -> z [V][S] gene-major (the values themselves)
//   corr_rank_kernel       one CTA per gene: bitonic sort of the row's order-preserving uint32 keys in dynamic
//                          shared memory (padded to a power of two), then
//                          spearman: 2r - (S+1) = #{< x} + #{<= x} - S per value (two binary searches), z-score of r;
//                          bicor:    median, MAD (a selection over the two sorted halves |x - med|), Tukey's
//                                    biweight, z = t * sqrt(S) / ||t||; MAD = 0 falls back to the Pearson z-score
//                                    with pcc_zscore_kernel's own arithmetic (g2v_pcc.cuh);
//                          and overwrites the row with z.
// Arithmetic in double, z stored as float32.  Every sum has a fixed order (integer for Spearman), there are no
// atomics, and a gene's result depends only on S (which fixes the block size), not on the grid.
#include "g2v_common.cuh"
#include "g2v_pcc.cuh"

namespace g2v {

constexpr int kCorrMaxThreads = 1024;

__global__ void __launch_bounds__(256)
corr_transpose_kernel(const float *__restrict__ expr, int32_t S, int32_t V, float *__restrict__ z) {
    __shared__ float t[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t g0 = (int64_t)blockIdx.x * 32, s0 = (int64_t)blockIdx.y * 32;
    for (int k = ty; k < 32; k += 8)
        if (s0 + k < S && g0 + tx < V) t[k][tx] = expr[(s0 + k) * V + g0 + tx];
    __syncthreads();
    for (int k = ty; k < 32; k += 8)
        if (g0 + k < V && s0 + tx < S) z[(g0 + k) * S + s0 + tx] = t[tx][k];
}

// float -> uint32 with the same order; -0.0 is keyed as +0.0 so that the two tie
__device__ __forceinline__ uint32_t order_key(float x) {
    uint32_t u = __float_as_uint(x);
    if (u == 0x80000000u) u = 0u;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ double key_value(uint32_t k) {
    return (double)__uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
constexpr uint32_t kKeyPad = 0xffffffffu;            // above every finite key (and +inf's)

// ascending bitonic sort of k[0..N), N a power of two, by the whole block; ends on a barrier
__device__ __forceinline__ void bitonic_sort(uint32_t *k, int N) {
    for (int size = 2; size <= N; size <<= 1)
        for (int j = size >> 1; j > 0; j >>= 1) {
            for (int p = threadIdx.x; p < (N >> 1); p += blockDim.x) {
                const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1)), l = i + j;
                const uint32_t a = k[i], b = k[l];
                if ((i & size) == 0 ? a > b : a < b) { k[i] = b; k[l] = a; }
            }
            __syncthreads();
        }
}

// #{k[0..n) < key} (upper = false) or #{k[0..n) <= key} (upper = true) on a sorted k
__device__ __forceinline__ int count_below(const uint32_t *k, int n, uint32_t key, bool upper) {
    int lo = 0;
    while (n > 0) {
        const int half = n >> 1;
        const uint32_t v = k[lo + half];
        if (v < key || (upper && v == key)) { lo += half + 1; n -= half + 1; } else n = half;
    }
    return lo;
}

// Sum over the block in a fixed order: lane tree 16, 8, 4, 2, 1 (lane 0's value), then the warps in index order.
// Every thread gets the same bits; `sh` holds 32 values and is free again on return.
template <class T>
__device__ __forceinline__ T block_sum(T v, T *sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    T r = sh[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r += sh[w];
    __syncthreads();
    return r;
}

// k-th smallest (0-based) of the union of the two ascending sequences A[j] = med - y[m-1-j] (j < m) and
// B[j] = y[m+j] - med (j < S-m), y = the sorted row: the values |x - med| without a second sort
__device__ double abs_dev_select(const uint32_t *y, int S, int m, double med, int k) {
    const auto A = [&](int j) { return med - key_value(y[m - 1 - j]); };
    const auto B = [&](int j) { return key_value(y[m + j]) - med; };
    const int need = k + 1, nA = m, nB = S - m;
    int lo = max(0, need - nB), hi = min(need, nA);
    while (lo < hi) {                                  // smallest i with A[i] >= B[need-i-1] (or i = hi)
        const int i = (lo + hi) >> 1;
        if (A(i) >= B(need - i - 1)) hi = i; else lo = i + 1;
    }
    const int i = lo, j = need - lo;
    const double a = i > 0 ? A(i - 1) : 0.0, b = j > 0 ? B(j - 1) : 0.0;
    return a > b ? a : b;
}

// Tukey's biweight of one value: t = (x - med) * (1 - u^2)^2 for |u| < 1, else 0, u = (x - med) / (9 mad)
__device__ __forceinline__ double biweight(float x, double med, double c9) {
    const double d = (double)x - med, u = d / c9;
    const double a = 1.0 - u * u;
    return fabs(u) < 1.0 ? d * (a * a) : 0.0;
}

template <int METHOD>
__global__ void __launch_bounds__(kCorrMaxThreads)
corr_rank_kernel(float *__restrict__ z, int32_t S, int32_t V, int32_t N) {
    extern __shared__ uint32_t keys[];                 // [N]
    __shared__ double red[32];
    __shared__ unsigned long long redu[32];
    __shared__ double stat[2 + 2 * kZscoreLanes];
    for (int64_t g = blockIdx.x; g < V; g += gridDim.x) {
        float *row = z + g * S;
        for (int i = threadIdx.x; i < N; i += blockDim.x) keys[i] = i < S ? order_key(row[i]) : kKeyPad;
        __syncthreads();
        bitonic_sort(keys, N);
        if (METHOD == G2V_CORR_SPEARMAN) {
            // d = 2r - (S+1), r = the average rank (#{<} + #{<=} + 1) / 2; sum d^2 exactly in integers.  Each thread
            // parks its d in the row slot it read (exact in float) and is the only one to touch it again.
            unsigned long long ss = 0;
            for (int i = threadIdx.x; i < S; i += blockDim.x) {
                const uint32_t k = order_key(row[i]);
                const int d = count_below(keys, S, k, false) + count_below(keys, S, k, true) - S;
                row[i] = (float)d;
                ss += (unsigned long long)((int64_t)d * d);
            }
            ss = block_sum(ss, redu);
            // Pearson z-score of r: mean (S+1)/2 and sum (r - mean)^2 = ss/4 are exact
            const double sd = sqrt((double)ss * 0.25 / (double)S);
            for (int i = threadIdx.x; i < S; i += blockDim.x)
                row[i] = sd > 0.0 ? (float)((double)row[i] * 0.5 / sd) : 0.f;
        } else {
            if (threadIdx.x == 0) {
                const int h = S >> 1;
                const double med = (S & 1) ? key_value(keys[h]) : 0.5 * (key_value(keys[h - 1]) + key_value(keys[h]));
                int lo = 0, n = S;                     // m = #{y < med}
                while (n > 0) {
                    const int half = n >> 1;
                    if (key_value(keys[lo + half]) < med) { lo += half + 1; n -= half + 1; } else n = half;
                }
                stat[0] = med;
                stat[1] = (S & 1) ? abs_dev_select(keys, S, lo, med, h)
                                  : 0.5 * (abs_dev_select(keys, S, lo, med, h - 1) + abs_dev_select(keys, S, lo, med, h));
            }
            __syncthreads();
            const double med = stat[0], mad = stat[1];
            if (mad > 0.0) {
                const double c9 = 9.0 * mad;
                double tt = 0.0;
                for (int i = threadIdx.x; i < S; i += blockDim.x) { const double t = biweight(row[i], med, c9); tt += t * t; }
                tt = block_sum(tt, red);               // > 0: the upper middle |x - med| lies in (0, 2 mad]
                const double scale = sqrt((double)S) / sqrt(tt);
                for (int i = threadIdx.x; i < S; i += blockDim.x) row[i] = (float)(biweight(row[i], med, c9) * scale);
            } else {
                // MAD = 0: the gene's Pearson z-score, the bits g2v_pcc_zscore gives it (WGCNA's individual fallback)
                const auto x = [&](int s) { return row[s]; };
                double *lane = stat + 2;
                if (threadIdx.x < kZscoreLanes) lane[threadIdx.x] = zscore_lane_sum(x, threadIdx.x, S);
                __syncthreads();
                double mu = 0.0;
                for (int k = 0; k < kZscoreLanes; ++k) mu += lane[k];
                mu /= (double)S;
                if (threadIdx.x < kZscoreLanes) lane[kZscoreLanes + threadIdx.x] = zscore_lane_ss(x, threadIdx.x, S, mu);
                __syncthreads();
                double var = 0.0;
                for (int k = 0; k < kZscoreLanes; ++k) var += lane[kZscoreLanes + k];
                const double sd = sqrt(var / (double)S);
                for (int i = threadIdx.x; i < S; i += blockDim.x) row[i] = zscore_value(row[i], mu, sd);
            }
        }
        __syncthreads();                               // keys and stat are rewritten by the next gene
    }
}

// block size of corr_rank_kernel for a padded row of N keys: one thread per compare-exchange pair, 32..1024
inline int corr_threads(int N) { return N / 2 < 32 ? 32 : (N / 2 > kCorrMaxThreads ? kCorrMaxThreads : N / 2); }

template <int METHOD>
int launch_corr(const float *expr, float *z, int32_t S, int32_t V, int32_t N, size_t smem, cudaStream_t st) {
    if (smem > 48 * 1024)
        G2V_CUDA_OK(cudaFuncSetAttribute(corr_rank_kernel<METHOD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
    corr_transpose_kernel<<<dim3((unsigned)((V + 31) / 32), (unsigned)((S + 31) / 32)), 256, 0, st>>>(expr, S, V, z);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    corr_rank_kernel<METHOD><<<(unsigned)V, corr_threads(N), smem, st>>>(z, S, V, N);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

}  // namespace g2v

using namespace g2v;

extern "C" int g2v_corr_transform(const float *expr, int32_t S, int32_t V, int32_t method, float *z, void *stream) {
    G2V_REQUIRE(expr && z, "g2v_corr_transform: null pointer");
    G2V_REQUIRE(method == G2V_CORR_SPEARMAN || method == G2V_CORR_BICOR,
                "g2v_corr_transform: method must be %d (spearman) or %d (bicor), got %d", G2V_CORR_SPEARMAN,
                G2V_CORR_BICOR, (int)method);
    G2V_REQUIRE(S >= 1 && S <= G2V_CORR_MAX_SAMPLES, "g2v_corr_transform: S = %d samples, must be in [1, %d]",
                (int)S, G2V_CORR_MAX_SAMPLES);
    G2V_REQUIRE(V >= 1, "g2v_corr_transform: V = %d genes, must be >= 1", (int)V);
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    int32_t N = 1;
    while (N < S) N <<= 1;
    const size_t smem = (size_t)N * sizeof(uint32_t);
    G2V_REQUIRE((long long)smem <= dp.max_smem_optin, "g2v_corr_transform: %zu bytes of shared memory per row, the "
                "device allows %d", smem, dp.max_smem_optin);
    cudaStream_t st = (cudaStream_t)stream;
    return method == G2V_CORR_SPEARMAN ? launch_corr<G2V_CORR_SPEARMAN>(expr, z, S, V, N, smem, st)
                                       : launch_corr<G2V_CORR_BICOR>(expr, z, S, V, N, smem, st);
}
