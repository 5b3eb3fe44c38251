// g2v_pcc.cu -- edge weighting upstream of the walk sampler (SURVEY.md 8f-1).
//
// Replaces construct_adjMat / compute_PCC (/root/reference/G2Vec.py:354-391): for one patient
// group, weight(src,dest) = |PCC(expr[:,src], expr[:,dest])| over that group's samples, population
// std (ddof = 0), weight 0 when either gene has zero variance (:359,366-367).  The reference loops over
// 216 540 edges in Python (8-9 s per group) and writes a dense [V,V] matrix; here
//   pcc_zscore_kernel  one thread-column per gene: mean, std, z = (x - mean)/std, stored gene-major
//                      z[V][S] so that an edge's two vectors are two contiguous rows
//   pcc_edge_kernel    8 lanes per edge: w = |mean_s z[src][s] * z[dest][s]|
// Accumulation is in double (the reference's float32 NumPy pairwise sums are not reproducible bit for
// bit; agreement is ~1e-7, tests compare at 2e-6 and the kept-edge set away from the 0.5 threshold).
// Thresholding and CSR assembly stay with the host (torch sort as plumbing, g2vec_b200/graph.py).
#include "g2v_common.cuh"
#include "g2v_pcc.cuh"

namespace g2v {

__global__ void __launch_bounds__(256)
pcc_zscore_kernel(const float *__restrict__ expr, int32_t S, int32_t V, float *__restrict__ z) {
    // block = 32 genes x 8 sample-lanes; expr is sample-major [S][V] (the reference's data['expr'] rows)
    // (the arithmetic is g2v_pcc.cuh's, which the bicor transform's Pearson fallback shares)
    __shared__ double sh[kZscoreLanes][33];
    const int gx = threadIdx.x & 31, sy = threadIdx.x >> 5;
    const int g = blockIdx.x * 32 + gx;
    const auto x = [&](int s) { return expr[(size_t)s * V + g]; };
    double sum = 0.0;
    if (g < V) sum = zscore_lane_sum(x, sy, S);
    sh[sy][gx] = sum;
    __syncthreads();
    double mu = 0.0;
    for (int k = 0; k < kZscoreLanes; ++k) mu += sh[k][gx];
    mu /= (double)S;
    __syncthreads();
    double ss = 0.0;
    if (g < V) ss = zscore_lane_ss(x, sy, S, mu);
    sh[sy][gx] = ss;
    __syncthreads();
    double var = 0.0;
    for (int k = 0; k < kZscoreLanes; ++k) var += sh[k][gx];
    const double sd = sqrt(var / (double)S);
    if (g < V)
        for (int s = sy; s < S; s += kZscoreLanes) z[(size_t)g * S + s] = zscore_value(x(s), mu, sd);
}

__global__ void __launch_bounds__(256)
pcc_edge_kernel(const float *__restrict__ z, int32_t S, const int32_t *__restrict__ src,
                const int32_t *__restrict__ dst, int64_t E, float *__restrict__ w) {
    const int sub = threadIdx.x & 7;
    const int64_t e = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    double acc = 0.0;
    if (e < E) {
        const float *a = z + (size_t)__ldg(src + e) * S, *b = z + (size_t)__ldg(dst + e) * S;
        for (int s = sub; s < S; s += 8) acc += (double)__ldg(a + s) * (double)__ldg(b + s);
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    if (e < E && sub == 0) w[e] = (float)fabs(acc / (double)S);
}

}  // namespace g2v

using namespace g2v;

extern "C" int g2v_pcc_zscore(const float *expr, int32_t S, int32_t V, float *z, void *stream) {
    G2V_REQUIRE(expr && z && S > 0 && V > 0, "g2v_pcc_zscore: bad arguments");
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    pcc_zscore_kernel<<<(V + 31) / 32, 256, 0, (cudaStream_t)stream>>>(expr, S, V, z);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_pcc_edge_weights(const float *z, int32_t S, int32_t V, const int32_t *src, const int32_t *dst,
                                    int64_t E, float *w, void *stream) {
    G2V_REQUIRE(z && S > 0 && V > 0 && E >= 0, "g2v_pcc_edge_weights: bad arguments");
    if (E == 0) return 0;
    G2V_REQUIRE(src && dst && w, "g2v_pcc_edge_weights: null pointer");
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    const int64_t blocks = (E * 8 + 255) / 256;
    pcc_edge_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(z, S, src, dst, E, w);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
