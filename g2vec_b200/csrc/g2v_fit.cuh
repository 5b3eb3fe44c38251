// g2v_fit.cuh -- the one-CTA-per-fit damped-Newton machinery shared by the signature fits (g2v_sig.cu, ridge logistic
// regression, DESIGN.md §4.29) and the survival fits (g2v_cox.cu, ridge Cox regression, §4.33): the training-fold
// standardisation, the FP64 mma.sync wrapper the Gram tiles use, the shared-memory Cholesky solve and the Newton loop
// with its Armijo search.  Each model supplies its own sample passes.
#pragma once
#include "g2v_common.cuh"

namespace g2v {

constexpr int kFitThreads = 512, kFitWarps = kFitThreads / 32;
constexpr int kTileS = 32;                             // samples per tile
constexpr int kPerSample = kFitThreads / kTileS;      // threads per sample in the linear-predictor sums
constexpr int kTS = kTileS + 4;                        // row stride of the tiles in doubles (conflict-free DMMA loads)
constexpr int kMaxPad = ((G2V_SIG_MAX_SIZE + 1 + 7) / 8) * 8;            // 136
constexpr int kMaxTiles = (kMaxPad / 8) * (kMaxPad / 8 + 1) / 2;           // 153 lower-triangle 8 x 8 tiles
constexpr int kTilesPerWarp = (kMaxTiles + kFitWarps - 1) / kFitWarps;     // 10
constexpr int kMaxIter = 100, kMaxHalvings = 40;
constexpr double kStepTol = 1e-10, kArmijo = 1e-4;
// The Armijo test allows the rounding of the loss sum: near the minimum the decrease it asks for falls below the
// loss's last bits, and without the slack the search would halve 40 times and the tiny step t d would meet the stop
// rule with the minimiser still a full Newton step away.
constexpr double kLossSlack = 0x1p-40;

__device__ __forceinline__ void dmma_8x8x4(double c[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

// Coefficient slot 0 is the intercept of the logistic fits; the Cox fits have none and keep z = 0, beta = 0 there.
__host__ __device__ __forceinline__ int fit_pad(int p) { return ((p + 1 + 7) / 8) * 8; }
__host__ __device__ __forceinline__ int tri(int i) { return i * (i + 1) / 2; }

struct Fit {
    const double *X;
    int64_t n_pad;
    int n, p, P1, P, f, n_tiles;
    const uint8_t *y;                                  // labels (logistic) or time flags (Cox)
    const int8_t *fold;                                // this repeat's row
    const int32_t *genes;                              // this signature's row
    double *Zs, *WZs, *Hp;                             // Hp aliases the tiles once a pass is over
    double *mu, *sd, *g;
};

// Per-CTA scratch of a fit at fixed size: the scalars the threads share, and the 8 x 8 tiles of H's lower triangle as
// (I << 8) | J, I >= J.
static __shared__ double fit_scal[4];
static __shared__ uint16_t fit_tiles[kMaxTiles];

__device__ __forceinline__ void fit_init_tiles(int n_tiles) {
    for (int t = threadIdx.x; t < n_tiles; t += kFitThreads) {
        int I = 0;
        while (tri(I + 1) <= t) ++I;
        fit_tiles[t] = (uint16_t)((I << 8) | (t - tri(I)));
    }
}

// Training-fold mean and population SD of every feature, in fixed order; a feature constant over the training fold
// (min == max) gets mu = that value and sd = 1, so its z is exactly 0.
__device__ inline void fit_standardise(const Fit &c) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = 1 + warp; j <= c.p; j += kFitWarps) {
        const double *xr = c.X + (int64_t)__ldg(c.genes + j - 1) * c.n_pad;
        double s = 0.0, mn = INFINITY, mx = -INFINITY;
        int cnt = 0;
        for (int i = lane; i < c.n; i += 32)
            if (c.fold[i] != c.f) {
                const double v = __ldg(xr + i);
                s += v; mn = fmin(mn, v); mx = fmax(mx, v); ++cnt;
            }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s += __shfl_xor_sync(0xffffffffu, s, o);
            mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        }
        double mu = mn, sd = 1.0;
        if (mn != mx) {
            mu = s / cnt;
            double ss = 0.0;
            for (int i = lane; i < c.n; i += 32)
                if (c.fold[i] != c.f) {
                    const double d = __ldg(xr + i) - mu;
                    ss = fma(d, d, ss);
                }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
            sd = sqrt(ss / cnt);
        }
        if (lane == 0) { c.mu[j] = mu; c.sd[j] = sd; }
    }
    if (threadIdx.x == 0) { c.mu[0] = 0.0; c.sd[0] = 1.0; }
    __syncthreads();
}

// Solves H d = g in place of the packed lower triangle Hp (Cholesky, right-looking, one barrier per column), then
// L y = g and L^T d = y in one warp.  y and d go through tmp.
__device__ inline void fit_solve(const Fit &c, double *d, double *tmp) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double *H = c.Hp;
    for (int j = 0; j < c.P1; ++j) {
        const double inv = 1.0 / sqrt(H[tri(j) + j]);
        for (int i = j + 1 + warp; i < c.P1; i += kFitWarps) {
            const double lij = H[tri(i) + j] * inv;
            for (int k = j + 1 + lane; k <= i; k += 32) H[tri(i) + k] = fma(-lij, H[tri(k) + j] * inv, H[tri(i) + k]);
        }
        __syncthreads();                               // every thread has read column j and the diagonal
        for (int i = j + tid; i < c.P1; i += kFitThreads) H[tri(i) + j] = i == j ? sqrt(H[tri(j) + j]) : H[tri(i) + j] * inv;
        // column j is not read again before the next barrier: step j+1 reads columns j+1.. only
    }
    __syncthreads();
    if (warp == 0) {
        for (int j = lane; j < c.P1; j += 32) tmp[j] = c.g[j];
        __syncwarp();
        for (int j = 0; j < c.P1; ++j) {
            const double yj = tmp[j] / H[tri(j) + j];
            for (int i = j + 1 + lane; i < c.P1; i += 32) tmp[i] = fma(-H[tri(i) + j], yj, tmp[i]);
            __syncwarp();
            if (lane == 0) tmp[j] = yj;
            __syncwarp();
        }
        for (int j = c.P1 - 1; j >= 0; --j) {
            const double dj = tmp[j] / H[tri(j) + j];
            for (int i = lane; i < j; i += 32) tmp[i] = fma(-H[tri(j) + i], dj, tmp[i]);
            __syncwarp();
            if (lane == 0) d[j] = dj;
            __syncwarp();
        }
    }
    __syncthreads();
}

// Damped Newton from the coefficients in bt [P1] (zero on entry): Armijo backtracking with the loss slack, at most
// kMaxHalvings halvings, stop when t max|d| <= kStepTol or after kMaxIter iterations.  model.gram(b) returns the loss
// at b and leaves the gradient in c.g and the packed H in c.Hp; model.loss(b) returns the loss only.  Every thread
// returns the iteration count and whether the step rule was met; bt holds the last accepted coefficients.
template <class Model>
__device__ void fit_newton(const Fit &c, Model &model, double *bt, double *bc, double *d, double *tmp, int &n_iter,
                           bool &converged) {
    double L = model.gram(bt);
    int it = 0;
    bool conv = false;
    while (it < kMaxIter) {
        fit_solve(c, d, tmp);
        if (threadIdx.x == 0) {
            double gd = 0.0, dmax = 0.0;
            for (int j = 0; j < c.P1; ++j) { gd = fma(c.g[j], d[j], gd); dmax = fmax(dmax, fabs(d[j])); }
            fit_scal[1] = gd; fit_scal[2] = dmax;
        }
        __syncthreads();
        const double gd = fit_scal[1], dmax = fit_scal[2];
        double t = 1.0;
        for (int h = 0;; ++h) {
            for (int j = threadIdx.x; j < c.P1; j += kFitThreads) bc[j] = bt[j] - t * d[j];
            __syncthreads();
            const double Lc = model.loss(bc);
            if (Lc <= L - kArmijo * t * gd + kLossSlack * fabs(L) || h == kMaxHalvings) break;
            t *= 0.5;
        }
        for (int j = threadIdx.x; j < c.P1; j += kFitThreads) bt[j] = bc[j];
        __syncthreads();
        ++it;
        if (t * dmax <= kStepTol) { conv = true; break; }
        if (it == kMaxIter) break;
        L = model.gram(bt);
    }
    n_iter = it;
    converged = conv;
}

}  // namespace g2v
