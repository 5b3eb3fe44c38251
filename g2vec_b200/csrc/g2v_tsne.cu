// g2v_tsne.cu -- exact 2-D t-SNE of the learned gene vectors (DESIGN.md §4.27).
//   tsne_dist_kernel      all-pairs squared distances: a register-tiled FP64 "GEMM" (64 x 64 tiles, 256 threads with
//                         4 x 4 outputs each), W converted to float64 in shared memory in chunks of 32 d consumed in
//                         ascending d, so every output is the contract's chain; writes the m x m buffer that later
//                         holds P.
//   tsne_affinity_kernel  one CTA per row: scikit-learn's perplexity bisection over the row of d (at most 100 steps),
//                         then the row is overwritten with the conditional affinities c_i.
//   tsne_sym_kernel       in place P_ij = (c_ij + c_ji) / 2m, one CTA per 32 x 32 tile pair (I, J), I <= J.
//   tsne_grad_kernel      one thread per (row i, block of G2V_TSNE_BLOCK columns): the chains of w, p w t_c and
//                         w^2 t_c over the block's j in ascending order, y_j staged in shared memory, p_ij read as
//                         P[j][i] (P is symmetric bit for bit) so that a warp's loads are coalesced.
//   tsne_rows_kernel      per row the chains of the block partials, and per block of 256 rows the chain of Z_i.
//   tsne_step_kernel      Z from the row-block chains, then scikit-learn's gains, momentum and step per coordinate.
//   tsne_kl_kernel, tsne_sum_kernel  the final KL divergence (reported only; fixed order, not part of the bit contract).
// Every operation of the distance chain and of the iteration is a correctly rounded __dsub_rn / __dmul_rn / __dadd_rn /
// __drcp_rn / __ddiv_rn (the library is built with -fmad=true, so the chains must not be left to the compiler), every
// sum has a fixed order and nothing uses atomics, so d and the iterates equal the NumPy restatement bit for bit.
#include <math_constants.h>

#include "g2v_common.cuh"

namespace g2v {

constexpr int kTsThreads = 256;
constexpr int kTsTile = 64;                            // rows and columns of a distance tile
constexpr int kTsDK = 32;                              // d per staged chunk
constexpr int kTsLd = kTsDK + 1;                       // padded staged row (doubles)
constexpr int kTsSym = 32;                             // edge of a symmetrisation tile
constexpr int kTsMaxSteps = 100;
constexpr int kTsExploration = 250;                    // iterations with early exaggeration
constexpr int kTsSumThreads = 1024;
static_assert(G2V_TSNE_BLOCK == kTsThreads, "a grad / rows CTA is one block of rows");

// ---- distances -------------------------------------------------------------------------------------------------
// Zero padding past D adds (0 - 0)^2 = +0 to acc >= +0, which leaves it unchanged, so every chunk runs all 32 steps.
// x_j - x_i is -(x_i - x_j) exactly, so d_ji has the bits of d_ij, and d_ii = +0.
__global__ void __launch_bounds__(kTsThreads)
tsne_dist_kernel(const float *__restrict__ W, int64_t m, int32_t D, double *__restrict__ P) {
    __shared__ double sa[kTsTile][kTsLd];
    __shared__ double sb[kTsTile][kTsLd];
    const int tid = threadIdx.x;
    const int tx = tid % 16, ty = tid / 16;
    const int64_t i0 = (int64_t)blockIdx.y * kTsTile, j0 = (int64_t)blockIdx.x * kTsTile;
    double acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
    for (int d0 = 0; d0 < D; d0 += kTsDK) {
        __syncthreads();                               // the last chunk is consumed
        for (int e = tid; e < kTsTile * kTsDK; e += kTsThreads) {
            const int rr = e / kTsDK, dd = e % kTsDK;
            const int d = d0 + dd;
            const int64_t i = i0 + rr, j = j0 + rr;
            sa[rr][dd] = (i < m && d < D) ? (double)__ldg(W + i * D + d) : 0.0;
            sb[rr][dd] = (j < m && d < D) ? (double)__ldg(W + j * D + d) : 0.0;
        }
        __syncthreads();
#pragma unroll 8
        for (int dd = 0; dd < kTsDK; ++dd) {
            double a[4], b[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) a[r] = sa[ty + 16 * r][dd];
#pragma unroll
            for (int c = 0; c < 4; ++c) b[c] = sb[tx + 16 * c][dd];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const double t = __dsub_rn(a[r], b[c]);
                    acc[r][c] = __dadd_rn(acc[r][c], __dmul_rn(t, t));
                }
        }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int64_t i = i0 + ty + 16 * r;
        if (i >= m) break;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int64_t j = j0 + tx + 16 * c;
            if (j < m) P[i * m + j] = acc[r][c];
        }
    }
}

// ---- conditional affinities ------------------------------------------------------------------------------------
// Fixed-order CTA sum: each thread's chain over its strided j, a shuffle tree per warp, then the warps in order.
__device__ __forceinline__ double tsne_block_sum(double v, double *sred) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();                                   // sred of the previous call is read
    if (lane == 0) sred[warp] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += sred[w];
    return s;
}

// scikit-learn's _binary_search_perplexity for row i in float64: beta = 1, at most 100 evaluations of
// H = log S + beta * sum_j d_ij e_ij / S with e_ij = exp(-d_ij beta) (j != i) and S = sum_j e_ij (0 -> float32(1e-8));
// accept when |H - log Perp| <= float32(1e-5); otherwise double / halve beta until bracketed, then bisect.  beta_i is
// the beta the row's c was computed from, steps_i the 0-based evaluation that met the tolerance (100: none did).
__global__ void __launch_bounds__(kTsThreads)
tsne_affinity_kernel(double *__restrict__ P, int64_t m, double log_perp, double *__restrict__ beta_out,
                     int32_t *__restrict__ steps_out) {
    __shared__ double sred[kTsThreads / 32];
    const int64_t i = blockIdx.x;
    double *row = P + i * m;
    const double tol = (double)1e-5f, floor_sum = (double)1e-8f;
    double beta = 1.0, lo = -CUDART_INF, hi = CUDART_INF, S = 0.0;
    int steps = kTsMaxSteps;
    for (int l = 0; l < kTsMaxSteps; ++l) {
        double s = 0.0, t = 0.0;
        for (int64_t j = threadIdx.x; j < m; j += kTsThreads) {
            if (j == i) continue;
            const double d = row[j];
            const double e = exp(-(d * beta));
            s += e;
            t += d * e;
        }
        S = tsne_block_sum(s, sred);
        const double T = tsne_block_sum(t, sred);
        if (S == 0.0) S = floor_sum;
        const double diff = (log(S) + beta * (T / S)) - log_perp;
        if (fabs(diff) <= tol) { steps = l; break; }
        if (l == kTsMaxSteps - 1) break;               // beta is the one S belongs to
        if (diff > 0.0) {
            lo = beta;
            beta = hi == CUDART_INF ? beta * 2.0 : (beta + hi) / 2.0;
        } else {
            hi = beta;
            beta = lo == -CUDART_INF ? beta / 2.0 : (beta + lo) / 2.0;
        }
    }
    for (int64_t j = threadIdx.x; j < m; j += kTsThreads)
        row[j] = j == i ? 0.0 : exp(-(row[j] * beta)) / S;
    if (threadIdx.x == 0) {
        beta_out[i] = beta;
        steps_out[i] = steps;
    }
}

// ---- joint affinities ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTsThreads)
tsne_sym_kernel(double *__restrict__ P, int64_t m) {
    const int64_t I = blockIdx.y, J = blockIdx.x;
    if (I > J) return;
    __shared__ double sa[kTsSym][kTsSym + 1];          // tile (I, J)
    __shared__ double sb[kTsSym][kTsSym + 1];          // tile (J, I)
    const int tx = threadIdx.x % kTsSym, ty = threadIdx.x / kTsSym;
    const double two_m = (double)(2 * m);
    for (int r = ty; r < kTsSym; r += kTsThreads / kTsSym) {
        const int64_t ia = I * kTsSym + r, ja = J * kTsSym + tx;
        const int64_t ib = J * kTsSym + r, jb = I * kTsSym + tx;
        sa[r][tx] = (ia < m && ja < m) ? P[ia * m + ja] : 0.0;
        sb[r][tx] = (ib < m && jb < m) ? P[ib * m + jb] : 0.0;
    }
    __syncthreads();
    for (int r = ty; r < kTsSym; r += kTsThreads / kTsSym) {
        const int64_t ia = I * kTsSym + r, ja = J * kTsSym + tx;
        if (ia < m && ja < m) P[ia * m + ja] = __ddiv_rn(__dadd_rn(sa[r][tx], sb[tx][r]), two_m);
        const int64_t ib = J * kTsSym + r, jb = I * kTsSym + tx;
        if (I != J && ib < m && jb < m) P[ib * m + jb] = __ddiv_rn(__dadd_rn(sb[r][tx], sa[tx][r]), two_m);
    }
}

// ---- gradient partials -----------------------------------------------------------------------------------------
// part [nb][5][m]: per column block b and row i the chains of w, a t_0, a t_1, r t_0, r t_1 over the block's j != i.
__global__ void __launch_bounds__(kTsThreads)
tsne_grad_kernel(const double *__restrict__ P, const double *__restrict__ Y, int64_t m, double *__restrict__ part) {
    __shared__ double sy[G2V_TSNE_BLOCK][2];
    const int tid = threadIdx.x;
    const int64_t b = blockIdx.y, j0 = b * G2V_TSNE_BLOCK;
    const int64_t i = (int64_t)blockIdx.x * kTsThreads + tid;
    if (j0 + tid < m) {
        sy[tid][0] = Y[(j0 + tid) * 2];
        sy[tid][1] = Y[(j0 + tid) * 2 + 1];
    }
    __syncthreads();
    if (i >= m) return;
    const int len = (int)min((int64_t)G2V_TSNE_BLOCK, m - j0);
    const double yi0 = Y[i * 2], yi1 = Y[i * 2 + 1];
    double z = 0.0, a0 = 0.0, a1 = 0.0, r0 = 0.0, r1 = 0.0;
    const double *p = P + j0 * m + i;
#pragma unroll 4
    for (int jj = 0; jj < len; ++jj) {
        if (j0 + jj == i) continue;
        const double pij = p[(int64_t)jj * m];
        const double t0 = __dsub_rn(yi0, sy[jj][0]), t1 = __dsub_rn(yi1, sy[jj][1]);
        const double d = __dadd_rn(__dmul_rn(t0, t0), __dmul_rn(t1, t1));
        const double w = __drcp_rn(__dadd_rn(1.0, d));
        const double a = __dmul_rn(pij, w), r = __dmul_rn(w, w);
        z = __dadd_rn(z, w);
        a0 = __dadd_rn(a0, __dmul_rn(a, t0));
        a1 = __dadd_rn(a1, __dmul_rn(a, t1));
        r0 = __dadd_rn(r0, __dmul_rn(r, t0));
        r1 = __dadd_rn(r1, __dmul_rn(r, t1));
    }
    double *o = part + b * 5 * m + i;
    o[0] = z; o[m] = a0; o[2 * m] = a1; o[3 * m] = r0; o[4 * m] = r1;
}

// rows [5][m]: the chains of the nb block partials per row; zblk [nb]: the chain of Z_i over each block of 256 rows.
// Rows past m add +0 to a chain >= +0, which leaves it unchanged.
__global__ void __launch_bounds__(kTsThreads)
tsne_rows_kernel(const double *__restrict__ part, int64_t m, int64_t nb, double *__restrict__ rows,
                 double *__restrict__ zblk) {
    __shared__ double sz[kTsThreads];
    const int tid = threadIdx.x;
    const int64_t i = (int64_t)blockIdx.x * kTsThreads + tid;
    double v[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    if (i < m) {
        for (int64_t b = 0; b < nb; ++b)
#pragma unroll
            for (int k = 0; k < 5; ++k) v[k] = __dadd_rn(v[k], part[(b * 5 + k) * m + i]);
#pragma unroll
        for (int k = 0; k < 5; ++k) rows[k * m + i] = v[k];
    }
    sz[tid] = v[0];
    __syncthreads();
    if (tid == 0) {
        double zb = 0.0;
        for (int t = 0; t < kTsThreads; ++t) zb = __dadd_rn(zb, sz[t]);
        zblk[blockIdx.x] = zb;
    }
}

__device__ __forceinline__ double tsne_total_z(const double *__restrict__ zblk, int64_t nb, double *sZ) {
    if (threadIdx.x == 0) {
        double Z = 0.0;
        for (int64_t b = 0; b < nb; ++b) Z = __dadd_rn(Z, zblk[b]);
        *sZ = Z;
    }
    __syncthreads();
    return *sZ;
}

// ---- the step --------------------------------------------------------------------------------------------------
// g = 4 ((alpha A) - (R / Z)); scikit-learn's _gradient_descent update per coordinate.  u and the gains start over at
// iterations 0 and 250, as in scikit-learn's two _gradient_descent calls.
__global__ void __launch_bounds__(kTsThreads)
tsne_step_kernel(const double *__restrict__ rows, const double *__restrict__ zblk, int64_t m, int64_t nb, int32_t it,
                 double eta, double *__restrict__ Y, double *__restrict__ U, double *__restrict__ gains) {
    __shared__ double sZ;
    const double Z = tsne_total_z(zblk, nb, &sZ);
    const int64_t i = (int64_t)blockIdx.x * kTsThreads + threadIdx.x;
    if (i >= m) return;
    const bool early = it < kTsExploration, reset = it == 0 || it == kTsExploration;
    const double alpha = early ? 12.0 : 1.0, mu = early ? 0.5 : 0.8;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        const double A = rows[(1 + c) * m + i], R = rows[(3 + c) * m + i];
        double g = __dmul_rn(4.0, __dsub_rn(__dmul_rn(alpha, A), __ddiv_rn(R, Z)));
        double u = reset ? 0.0 : U[i * 2 + c];
        double gain = reset ? 1.0 : gains[i * 2 + c];
        gain = __dmul_rn(u, g) < 0.0 ? __dadd_rn(gain, 0.2) : __dmul_rn(gain, 0.8);
        if (gain < 0.01) gain = 0.01;
        g = __dmul_rn(g, gain);
        u = __dsub_rn(__dmul_rn(mu, u), __dmul_rn(eta, g));
        Y[i * 2 + c] = __dadd_rn(Y[i * 2 + c], u);
        U[i * 2 + c] = u;
        gains[i * 2 + c] = gain;
    }
}

// ---- KL --------------------------------------------------------------------------------------------------------
// part[b][0][i] = sum over the block's j != i of p log(max(p, eps) / max(w / Z, eps)).
__global__ void __launch_bounds__(kTsThreads)
tsne_kl_kernel(const double *__restrict__ P, const double *__restrict__ Y, const double *__restrict__ zblk, int64_t m,
               int64_t nb, double *__restrict__ part) {
    __shared__ double sy[G2V_TSNE_BLOCK][2];
    __shared__ double sZ;
    const int tid = threadIdx.x;
    const int64_t b = blockIdx.y, j0 = b * G2V_TSNE_BLOCK;
    const int64_t i = (int64_t)blockIdx.x * kTsThreads + tid;
    if (j0 + tid < m) {
        sy[tid][0] = Y[(j0 + tid) * 2];
        sy[tid][1] = Y[(j0 + tid) * 2 + 1];
    }
    const double Z = tsne_total_z(zblk, nb, &sZ);      // synchronises the CTA
    if (i >= m) return;
    const double eps = 2.220446049250313e-16;          // float64 machine epsilon
    const int len = (int)min((int64_t)G2V_TSNE_BLOCK, m - j0);
    const double yi0 = Y[i * 2], yi1 = Y[i * 2 + 1];
    double kl = 0.0;
    const double *p = P + j0 * m + i;
    for (int jj = 0; jj < len; ++jj) {
        if (j0 + jj == i) continue;
        const double pij = p[(int64_t)jj * m];
        const double t0 = yi0 - sy[jj][0], t1 = yi1 - sy[jj][1];
        const double q = (1.0 / (1.0 + (t0 * t0 + t1 * t1))) / Z;
        kl += pij * log(fmax(pij, eps) / fmax(q, eps));
    }
    part[b * 5 * m + i] = kl;
}

__global__ void __launch_bounds__(kTsSumThreads)
tsne_sum_kernel(const double *__restrict__ part, int64_t m, int64_t nb, double *__restrict__ out) {
    __shared__ double sred[kTsSumThreads / 32];
    double s = 0.0;
    for (int64_t e = threadIdx.x; e < nb * m; e += kTsSumThreads) s += part[(e / m) * 5 * m + e % m];
    s = tsne_block_sum(s, sred);
    if (threadIdx.x == 0) *out = s;
}

}  // namespace g2v

using namespace g2v;

#define G2V_TSNE_CHECK_M(fn, m)                                                                                    \
    G2V_REQUIRE((m) >= 2 && (m) <= G2V_TSNE_MAX_GENES, fn ": m = %lld genes, must be in [2, %d]", (long long)(m), \
                G2V_TSNE_MAX_GENES)

static int64_t tsne_blocks(int64_t m) { return (m + G2V_TSNE_BLOCK - 1) / G2V_TSNE_BLOCK; }

extern "C" size_t g2v_tsne_workspace_bytes(int64_t m) {
    if (m < 2 || m > G2V_TSNE_MAX_GENES) return 0;
    const int64_t nb = tsne_blocks(m);
    return sizeof(double) * (size_t)(5 * m * nb + 5 * m + nb);
}

extern "C" int g2v_tsne_dist(const float *W, int64_t m, int32_t D, double *P, void *stream) {
    G2V_REQUIRE(W && P, "g2v_tsne_dist: null pointer");
    G2V_TSNE_CHECK_M("g2v_tsne_dist", m);
    G2V_REQUIRE(D >= 1, "g2v_tsne_dist: D = %d, must be >= 1", (int)D);
    const unsigned t = (unsigned)((m + kTsTile - 1) / kTsTile);
    tsne_dist_kernel<<<dim3(t, t), kTsThreads, 0, (cudaStream_t)stream>>>(W, m, D, P);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_tsne_affinity(double *P, int64_t m, double perplexity, double *beta, int32_t *steps,
                                 void *stream) {
    G2V_REQUIRE(P && beta && steps, "g2v_tsne_affinity: null pointer");
    G2V_TSNE_CHECK_M("g2v_tsne_affinity", m);
    G2V_REQUIRE(perplexity >= 1.0 && perplexity < (double)m,
                "g2v_tsne_affinity: perplexity %g, must be finite with 1 <= perplexity < m = %lld", perplexity,
                (long long)m);
    tsne_affinity_kernel<<<(unsigned)m, kTsThreads, 0, (cudaStream_t)stream>>>(P, m, log(perplexity), beta, steps);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_tsne_symmetrize(double *P, int64_t m, void *stream) {
    G2V_REQUIRE(P, "g2v_tsne_symmetrize: null pointer");
    G2V_TSNE_CHECK_M("g2v_tsne_symmetrize", m);
    const unsigned t = (unsigned)((m + kTsSym - 1) / kTsSym);
    tsne_sym_kernel<<<dim3(t, t), kTsThreads, 0, (cudaStream_t)stream>>>(P, m);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_tsne_grad(const double *P, const double *Y, int64_t m, double *ws, void *stream) {
    G2V_REQUIRE(P && Y && ws, "g2v_tsne_grad: null pointer");
    G2V_TSNE_CHECK_M("g2v_tsne_grad", m);
    const int64_t nb = tsne_blocks(m);
    tsne_grad_kernel<<<dim3((unsigned)nb, (unsigned)nb), kTsThreads, 0, (cudaStream_t)stream>>>(P, Y, m, ws);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_tsne_update(double *ws, int64_t m, int32_t it, double eta, double *Y, double *u, double *gains,
                               void *stream) {
    G2V_REQUIRE(ws && Y && u && gains, "g2v_tsne_update: null pointer");
    G2V_TSNE_CHECK_M("g2v_tsne_update", m);
    G2V_REQUIRE(it >= 0, "g2v_tsne_update: iteration %d, must be >= 0", (int)it);
    G2V_REQUIRE(eta > 0.0 && eta <= 1.7976931348623157e308, "g2v_tsne_update: learning rate %g, must be finite and > 0", eta);
    const int64_t nb = tsne_blocks(m);
    double *rows = ws + 5 * m * nb, *zblk = rows + 5 * m;
    tsne_rows_kernel<<<(unsigned)nb, kTsThreads, 0, (cudaStream_t)stream>>>(ws, m, nb, rows, zblk);
    G2V_CUDA_OK(cudaGetLastError());
    tsne_step_kernel<<<(unsigned)nb, kTsThreads, 0, (cudaStream_t)stream>>>(rows, zblk, m, nb, it, eta, Y, u, gains);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch(2);
    return 0;
}

extern "C" int g2v_tsne_kl(const double *P, const double *Y, int64_t m, double *ws, double *kl, void *stream) {
    G2V_REQUIRE(P && Y && ws && kl, "g2v_tsne_kl: null pointer");
    G2V_TSNE_CHECK_M("g2v_tsne_kl", m);
    const int64_t nb = tsne_blocks(m);
    double *rows = ws + 5 * m * nb, *zblk = rows + 5 * m;
    cudaStream_t st = (cudaStream_t)stream;
    tsne_grad_kernel<<<dim3((unsigned)nb, (unsigned)nb), kTsThreads, 0, st>>>(P, Y, m, ws);
    G2V_CUDA_OK(cudaGetLastError());
    tsne_rows_kernel<<<(unsigned)nb, kTsThreads, 0, st>>>(ws, m, nb, rows, zblk);
    G2V_CUDA_OK(cudaGetLastError());
    tsne_kl_kernel<<<dim3((unsigned)nb, (unsigned)nb), kTsThreads, 0, st>>>(P, Y, zblk, m, nb, ws);
    G2V_CUDA_OK(cudaGetLastError());
    tsne_sum_kernel<<<1, kTsSumThreads, 0, st>>>(ws, m, nb, kl);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch(4);
    return 0;
}
