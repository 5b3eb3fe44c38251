// g2v_pcc.cuh -- the z-score arithmetic of pcc_zscore_kernel (g2v_pcc.cu), shared with the bicor transform's
// Pearson fallback (g2v_corr.cu) so that both give a gene the same bits.
//
// Order of the sums: lane sy of 8 adds the samples s = sy, sy + 8, sy + 16, ... in ascending order, in double; the
// caller then adds the 8 lane sums in lane order 0..7 (mean = that / S, then the same for the squared deviations).
#pragma once
#include "g2v_common.cuh"

namespace g2v {

constexpr int kZscoreLanes = 8;

template <class Load>
__device__ __forceinline__ double zscore_lane_sum(Load x, int sy, int32_t S) {
    double sum = 0.0;
    for (int s = sy; s < S; s += kZscoreLanes) sum += (double)x(s);
    return sum;
}

template <class Load>
__device__ __forceinline__ double zscore_lane_ss(Load x, int sy, int32_t S, double mu) {
    double ss = 0.0;
    for (int s = sy; s < S; s += kZscoreLanes) { const double d = (double)x(s) - mu; ss += d * d; }
    return ss;
}

// z of one value given the mean and the population std; 0 for a zero-variance gene (G2Vec.py:359,366-367)
__device__ __forceinline__ float zscore_value(float x, double mu, double sd) {
    return sd > 0.0 ? (float)(((double)x - mu) / sd) : 0.f;
}

}  // namespace g2v
