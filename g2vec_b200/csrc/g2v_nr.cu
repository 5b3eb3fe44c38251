// g2v_nr.cu -- network-propagated gene scores with a label-permutation test, NetRank (DESIGN.md §4.35).
//   nr_seed_kernel   per labelling (row of A) and gene: N = n A - k Q, rho = N^2 / W, s = sqrt(rho); a 32 x 32 tile
//                    through shared memory turns the labelling-major A into the gene-major S [G][ld], so that each
//                    gene's labellings are contiguous.
//   nr_step_kernel   one power iteration over a column range of the labellings: a warp owns one gene j and 32
//                    columns, each lane one column b, and sums x[i][b] w_i over j's CSR neighbours in ascending i
//                    (each x row is one coalesced 256-byte read).  Warps take the genes in a host-given order
//                    (descending degree), so the hubs start first.
//   nr_tally_kernel  a warp per gene: count[j] += #{b : x[j][b] >= score_obs[j]}.
// Every float64 operation is a correctly rounded __dmul_rn / __dadd_rn / __ddiv_rn / __dsqrt_rn in a fixed order, and
// each (j, b) sum belongs to one thread, so the bits do not depend on the launch shape, the column tile or the chunk.
#include "g2v_common.cuh"

namespace g2v {

// ---- seed ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
nr_seed_kernel(const int64_t *__restrict__ A, int64_t n_b, int32_t G, int32_t n, int32_t k,
               const int64_t *__restrict__ Q, const double *__restrict__ W, double *__restrict__ S, int64_t ld) {
    __shared__ double tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 8 rows of 32 threads
    const int64_t g0 = (int64_t)blockIdx.x * 32, b0 = (int64_t)blockIdx.y * 32;
    const int64_t g = g0 + tx;
    const int64_t q = g < G ? Q[g] : 0;
    const double w = g < G ? W[g] : 0.0;
    for (int r = ty; r < 32; r += 8) {
        const int64_t b = b0 + r;
        double s = 0.0;
        if (g < G && b < n_b) {
            const int64_t N = (int64_t)n * A[b * G + g] - (int64_t)k * q;
            const double d = (double)N;
            s = w > 0.0 ? __dsqrt_rn(__ddiv_rn(__dmul_rn(d, d), w)) : 0.0;
        }
        tile[r][tx] = s;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {                            // thread tx now writes labelling b0 + tx of gene g0 + r
        const int64_t gg = g0 + r, b = b0 + tx;
        if (gg < G && b < n_b) S[gg * ld + b] = tile[tx][r];
    }
}

// ---- step ---------------------------------------------------------------------------------------------------
constexpr int kStepThreads = 256, kStepWarps = kStepThreads / 32, kStepUnroll = 8;

__global__ void __launch_bounds__(kStepThreads)
nr_step_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ col, const double *__restrict__ w,
               const int32_t *__restrict__ rows, const double *__restrict__ S, const double *__restrict__ x_in,
               double *__restrict__ x_out, int32_t G, int64_t ld, int64_t c0, int64_t n_cols, int32_t n_groups,
               double one_minus_d, double d) {
    const int lane = threadIdx.x & 31;
    const int64_t gw = (int64_t)blockIdx.x * kStepWarps + (threadIdx.x >> 5);
    if (gw >= (int64_t)G * n_groups) return;
    const int32_t j = __ldg(rows + gw / n_groups);
    const int64_t c = (gw % n_groups) * 32 + lane;                // column within the range
    const bool ok = c < n_cols;
    const int64_t b = c0 + (ok ? c : 0);
    const int32_t p0 = __ldg(rowptr + j), p1 = __ldg(rowptr + j + 1);
    double acc = 0.0;
    int32_t p = p0;
    for (; p + kStepUnroll <= p1; p += kStepUnroll) {            // the loads of a group are in flight together
        double v[kStepUnroll], wi[kStepUnroll];
#pragma unroll
        for (int u = 0; u < kStepUnroll; ++u) {
            const int32_t i = __ldg(col + p + u);
            wi[u] = __ldg(w + i);
            v[u] = ok ? __ldg(x_in + (int64_t)i * ld + b) : 0.0;
        }
#pragma unroll
        for (int u = 0; u < kStepUnroll; ++u) acc = __dadd_rn(acc, __dmul_rn(v[u], wi[u]));
    }
    for (; p < p1; ++p) {
        const int32_t i = __ldg(col + p);
        const double v = ok ? __ldg(x_in + (int64_t)i * ld + b) : 0.0;
        acc = __dadd_rn(acc, __dmul_rn(v, __ldg(w + i)));
    }
    if (ok) x_out[(int64_t)j * ld + b] = __dadd_rn(__dmul_rn(one_minus_d, __ldg(S + (int64_t)j * ld + b)),
                                                   __dmul_rn(d, acc));
}

// ---- tally --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
nr_tally_kernel(const double *__restrict__ x, int32_t G, int64_t n_b, int64_t ld, const double *__restrict__ score_obs,
                unsigned long long *__restrict__ count) {
    const int lane = threadIdx.x & 31;
    const int64_t j = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (j >= G) return;
    const double o = score_obs[j];
    const double *row = x + j * ld;
    uint32_t c = 0;
    for (int64_t b = lane; b < n_b; b += 32) c += __ldg(row + b) >= o ? 1u : 0u;
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
    if (lane == 0 && c) count[j] += c;                           // one warp owns gene j in a launch
}

}  // namespace g2v

using namespace g2v;

#define G2V_NR_CHECK_GENES(fn, G)                                                                             \
    G2V_REQUIRE((G) >= 1 && (G) <= G2V_NR_MAX_GENES, fn ": G = %d genes, must be in [1, %d]", (int)(G),         \
                G2V_NR_MAX_GENES)
#define G2V_NR_CHECK_COLS(fn, n_b, ld)                                                                        \
    G2V_REQUIRE((n_b) >= 1 && (ld) >= (n_b) && (ld) <= G2V_NR_MAX_ROWS,                                       \
                fn ": n_b = %lld labellings with ld = %lld, must be 1 <= n_b <= ld <= %d", (long long)(n_b),   \
                (long long)(ld), G2V_NR_MAX_ROWS)

extern "C" int64_t g2v_nr_tile_cols(int32_t G) {
    if (G < 1 || G > G2V_NR_MAX_GENES) return 0;
    DeviceProps dp;
    if (device_props(&dp)) return 0;
    // S and the two x buffers of a tile (24 G bytes per column) in half of the L2
    int64_t cols = dp.l2_bytes / 2 / (24 * (int64_t)G) / 32 * 32;
    if (cols < 32) cols = 32;
    if (cols > G2V_NR_MAX_ROWS) cols = G2V_NR_MAX_ROWS;
    return cols;
}

extern "C" int g2v_nr_seed(const int64_t *A, int64_t n_b, int32_t G, int32_t n, int32_t k, const int64_t *Q,
                           const double *W, double *S, int64_t ld, void *stream) {
    G2V_REQUIRE(A && Q && W && S, "g2v_nr_seed: null pointer");
    G2V_REQUIRE(n >= 3 && n <= G2V_PERM_MAX_SAMPLES, "g2v_nr_seed: n = %d samples, must be in [3, %d]", (int)n,
                G2V_PERM_MAX_SAMPLES);
    G2V_REQUIRE(k >= 1 && k < n, "g2v_nr_seed: k = %d, must be in [1, n - 1 = %d]", (int)k, (int)n - 1);
    G2V_NR_CHECK_GENES("g2v_nr_seed", G);
    G2V_NR_CHECK_COLS("g2v_nr_seed", n_b, ld);
    const dim3 grid((unsigned)((G + 31) / 32), (unsigned)((n_b + 31) / 32));
    nr_seed_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A, n_b, G, n, k, Q, W, S, ld);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_nr_step(const int32_t *rowptr, const int32_t *col, const double *w, const int32_t *rows,
                           const double *S, const double *x_in, double *x_out, int32_t G, int64_t ld, int64_t c0,
                           int64_t n_cols, double damping, void *stream) {
    G2V_REQUIRE(rowptr && col && w && rows && S && x_in && x_out, "g2v_nr_step: null pointer");
    G2V_REQUIRE(x_in != x_out && x_out != S, "g2v_nr_step: x_out must differ from x_in and S");
    G2V_NR_CHECK_GENES("g2v_nr_step", G);
    G2V_REQUIRE(ld >= 1 && ld <= G2V_NR_MAX_ROWS && c0 >= 0 && n_cols >= 1 && c0 + n_cols <= ld,
                "g2v_nr_step: columns %lld + [1, %lld] out of ld = %lld (at most %d)", (long long)c0, (long long)n_cols,
                (long long)ld, G2V_NR_MAX_ROWS);
    G2V_REQUIRE(damping >= 0.0 && damping <= G2V_NR_MAX_DAMPING, "g2v_nr_step: damping = %g, must be in [0, %g]",
                damping, G2V_NR_MAX_DAMPING);
    const int32_t n_groups = (int32_t)((n_cols + 31) / 32);
    const int64_t warps = (int64_t)G * n_groups;
    G2V_REQUIRE((warps + kStepWarps - 1) / kStepWarps <= 0x7fffffff, "g2v_nr_step: G x column groups too large");
    nr_step_kernel<<<(unsigned)((warps + kStepWarps - 1) / kStepWarps), kStepThreads, 0, (cudaStream_t)stream>>>(
        rowptr, col, w, rows, S, x_in, x_out, G, ld, c0, n_cols, n_groups, 1.0 - damping, damping);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_nr_tally(const double *x, int32_t G, int64_t n_b, int64_t ld, const double *score_obs,
                            int64_t *count, void *stream) {
    G2V_REQUIRE(x && score_obs && count, "g2v_nr_tally: null pointer");
    G2V_NR_CHECK_GENES("g2v_nr_tally", G);
    G2V_NR_CHECK_COLS("g2v_nr_tally", n_b, ld);
    nr_tally_kernel<<<(unsigned)((G + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
        x, G, n_b, ld, score_obs, reinterpret_cast<unsigned long long *>(count));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
