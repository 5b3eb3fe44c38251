// g2v_dcx.cu -- label-permutation test of differential co-expression for every network pair (DESIGN.md §4.30).
//   dcx_sums_kernel<D>  P = M . (q_i q_j) on the FP64 tensor cores (mma.sync m8n8k4, DMMA): a CTA owns 128 rows
//                       (labellings) x 64 pairs and walks the samples in slabs of 32.  Per slab the indicator bytes
//                       go to shared memory as doubles and the pair products q_i q_j are formed there from the
//                       gene-major q (never materialised in global memory); each warp then multiplies 32 rows x 32
//                       pairs from shared memory.  Every product is an integer <= 2^32 and every partial sum <= 2^47,
//                       so the sums are exact in any order.  Without D the epilogue writes the int64 sums; with D it
//                       forms both groups' r from the int64 sums and writes the statistic D = |r1 - r0| / (1 - r0 r1).
//   dcx_tally_kernel    perm_tally_kernel's design over D in rank order: a CTA owns a run of rows and walks the pair
//                       axis from the right in tiles of 128, carrying each row's running max in shared memory;
//                       integer atomics only.
// r and D are correctly rounded float64 operations in a fixed order (no fma contraction), so they are the bits a
// NumPy restatement computes.
#include "g2v_common.cuh"

namespace g2v {

// ---- r and D ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double dcx_corr(int64_t C, int64_t Vi, int64_t Vj) {
    if (Vi == 0 || Vj == 0) return 0.0;
    const double den = __dsqrt_rn(__dmul_rn(__ll2double_rn(Vi), __ll2double_rn(Vj)));
    const double r = __ddiv_rn(__ll2double_rn(C), den);
    return r > 1.0 ? 1.0 : (r < -1.0 ? -1.0 : r);
}

__device__ __forceinline__ double dcx_stat(double r0, double r1) {
    if (r0 == r1) return 0.0;
    return __ddiv_rn(fabs(__dsub_rn(r1, r0)), __dsub_rn(1.0, __dmul_rn(r0, r1)));
}

// ---- sums ---------------------------------------------------------------------------------------------------
constexpr int kRows = 128, kPairs = 64, kSlab = 32, kStride = kSlab + 4;   // stride 36: conflict-free fragment loads
constexpr int kSumThreads = 256;
constexpr size_t kSumSmem = (size_t)(kRows + kPairs) * kStride * sizeof(double);

__device__ __forceinline__ void dmma_8x8x4(double c[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

struct DcxEpilogue {                                   // the D form's inputs (see g2v_dcx_sums in the header)
    int32_t n, k;
    const int64_t *A, *Bq, *A_tot, *B_tot, *P_tot;
};

template <bool kD>
__global__ void __launch_bounds__(kSumThreads)
dcx_sums_kernel(const uint8_t *__restrict__ M, int64_t n_b, int32_t S_pad, const int32_t *__restrict__ q, int32_t G,
                const int32_t *__restrict__ pi, const int32_t *__restrict__ pj, int64_t E, DcxEpilogue ep,
                int64_t *__restrict__ P, double *__restrict__ D) {
    extern __shared__ double smem[];
    double *As = smem;                                 // [kRows][kStride]: indicator of row, sample
    double *Bs = smem + kRows * kStride;               // [kPairs][kStride]: q_i q_j of pair, sample
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    const int wr = warp & 3, wc = warp >> 2;           // warp tile: rows wr*32 .., pairs wc*32 ..
    const int64_t rb = (int64_t)blockIdx.y * kRows, eb = (int64_t)blockIdx.x * kPairs;
    double acc[4][4][2];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = 0.0;
    for (int s0 = 0; s0 < S_pad; s0 += kSlab) {
        for (int x = tid; x < kRows * kSlab; x += kSumThreads) {
            const int row = x >> 5, s = x & 31;
            const int64_t r = rb + row;
            As[row * kStride + s] = r < n_b ? (double)__ldg(M + r * S_pad + s0 + s) : 0.0;
        }
        for (int x = tid; x < kPairs * kSlab; x += kSumThreads) {
            const int pr = x >> 5, s = x & 31;
            const int64_t e = eb + pr;
            double v = 0.0;
            if (e < E) {
                const int32_t a = __ldg(q + (int64_t)__ldg(pi + e) * S_pad + s0 + s);
                const int32_t b = __ldg(q + (int64_t)__ldg(pj + e) * S_pad + s0 + s);
                v = __dmul_rn((double)a, (double)b);  // exact: |q_i q_j| <= 2^32
            }
            Bs[pr * kStride + s] = v;
        }
        __syncthreads();
        const double *ap = As + (wr * 32 + gid) * kStride + tig;
        const double *bp = Bs + (wc * 32 + gid) * kStride + tig;
#pragma unroll
        for (int kk = 0; kk < kSlab; kk += 4) {
            double a[4], b[4];
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                a[t] = ap[t * 8 * kStride + kk];
                b[t] = bp[t * 8 * kStride + kk];
            }
#pragma unroll
            for (int mt = 0; mt < 4; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) dmma_8x8x4(acc[mt][nt], a[mt], b[nt]);
        }
        __syncthreads();                               // the slab is consumed before the next one is written
    }
    // accumulator e of tile (mt, nt): row wr*32 + mt*8 + gid, pair wc*32 + nt*8 + 2 tig + e
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int64_t p = eb + wc * 32 + nt * 8 + 2 * tig + e;
            if (p >= E) continue;
            int32_t gi = 0, gj = 0;
            int64_t pt = 0, ati = 0, atj = 0, bti = 0, btj = 0;
            if (kD) {
                gi = __ldg(pi + p); gj = __ldg(pj + p);
                pt = __ldg(ep.P_tot + p);
                ati = __ldg(ep.A_tot + gi); atj = __ldg(ep.A_tot + gj);
                bti = __ldg(ep.B_tot + gi); btj = __ldg(ep.B_tot + gj);
            }
#pragma unroll
            for (int mt = 0; mt < 4; ++mt) {
                const int64_t r = rb + wr * 32 + mt * 8 + gid;
                if (r >= n_b) continue;
                const int64_t s = __double2ll_rn(acc[mt][nt][e]);
                if (!kD) {
                    P[r * E + p] = s;
                    continue;
                }
                // group 1 = the row's selected samples (k), group 2 = the rest (n - k); every product fits in int64
                const int64_t k1 = ep.k, k2 = (int64_t)ep.n - ep.k;
                const int64_t a1i = __ldg(ep.A + r * G + gi), a1j = __ldg(ep.A + r * G + gj);
                const int64_t b1i = __ldg(ep.Bq + r * G + gi), b1j = __ldg(ep.Bq + r * G + gj);
                const int64_t a2i = ati - a1i, a2j = atj - a1j, b2i = bti - b1i, b2j = btj - b1j, s2 = pt - s;
                const double r1 = dcx_corr(k1 * s - a1i * a1j, k1 * b1i - a1i * a1i, k1 * b1j - a1j * a1j);
                const double r2 = dcx_corr(k2 * s2 - a2i * a2j, k2 * b2i - a2i * a2i, k2 * b2j - a2j * a2j);
                D[r * E + p] = dcx_stat(r1, r2);
            }
        }
}

// ---- tally --------------------------------------------------------------------------------------------------
constexpr int kTallyThreads = 256, kTallyWarps = kTallyThreads / 32, kTallyV = 4, kTallyTile = 32 * kTallyV;
constexpr int kTallyMaxRows = 1024;                    // rows per CTA (the carries live in shared memory)

__global__ void __launch_bounds__(kTallyThreads)
dcx_tally_kernel(const double *__restrict__ D, int64_t n_b, int64_t E, const double *__restrict__ D_obs,
                 int32_t rows_per_cta, unsigned long long *__restrict__ count,
                 unsigned long long *__restrict__ count_maxt) {
    __shared__ double carry[kTallyMaxRows];
    __shared__ uint32_t cnt[2][kTallyTile];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t rb = (int64_t)blockIdx.x * rows_per_cta;
    const int R = (int)min((int64_t)rows_per_cta, n_b - rb);
    for (int i = threadIdx.x; i < R; i += kTallyThreads) carry[i] = 0.0;
    const int64_t n_tiles = (E + kTallyTile - 1) / kTallyTile;
    for (int64_t t = n_tiles - 1; t >= 0; --t) {
        double dob[kTallyV];
        bool ok[kTallyV];
#pragma unroll
        for (int v = 0; v < kTallyV; ++v) {
            const int64_t j = t * kTallyTile + v * 32 + lane;
            ok[v] = j < E;
            dob[v] = ok[v] ? D_obs[j] : 0.0;
        }
        cnt[threadIdx.x / kTallyTile][threadIdx.x % kTallyTile] = 0u;
        __syncthreads();
        uint32_t c1[kTallyV] = {}, c2[kTallyV] = {};
        for (int r = warp; r < R; r += kTallyWarps) {
            const double *row = D + (rb + r) * E + t * kTallyTile + lane;
            double d[kTallyV];
#pragma unroll
            for (int v = 0; v < kTallyV; ++v) d[v] = ok[v] ? __ldg(row + v * 32) : 0.0;
            double cr = carry[r];                      // max of D over the pairs right of this sub-tile
#pragma unroll
            for (int v = kTallyV - 1; v >= 0; --v) {
                c1[v] += (ok[v] && d[v] >= dob[v]) ? 1u : 0u;
                double u = d[v];
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {     // inclusive suffix max over the lanes
                    const double x = __shfl_down_sync(0xffffffffu, u, o);
                    if (lane + o < 32 && x > u) u = x;
                }
                if (cr > u) u = cr;
                c2[v] += (ok[v] && u >= dob[v]) ? 1u : 0u;
                cr = __shfl_sync(0xffffffffu, u, 0);
            }
            if (lane == 0) carry[r] = cr;
        }
#pragma unroll
        for (int v = 0; v < kTallyV; ++v) {
            if (c1[v]) atomicAdd(&cnt[0][v * 32 + lane], c1[v]);
            if (c2[v]) atomicAdd(&cnt[1][v * 32 + lane], c2[v]);
        }
        __syncthreads();
        {
            const int which = threadIdx.x / kTallyTile, jj = threadIdx.x % kTallyTile;
            const int64_t j = t * kTallyTile + jj;
            const uint32_t c = cnt[which][jj];
            if (j < E && c) atomicAdd((which ? count_maxt : count) + j, (unsigned long long)c);
        }
        __syncthreads();                               // cnt is cleared for the next tile
    }
}
static_assert(2 * kTallyTile == kTallyThreads, "one thread per tile counter");

}  // namespace g2v

using namespace g2v;

extern "C" int g2v_dcx_sums(const uint8_t *M, int64_t n_b, int32_t S_pad, const int32_t *q, int32_t G,
                            const int32_t *pair_i, const int32_t *pair_j, int64_t E, int32_t n, int32_t k,
                            const int64_t *A, const int64_t *Bq, const int64_t *A_tot, const int64_t *B_tot,
                            const int64_t *P_tot, int64_t *P, double *D, void *stream) {
    G2V_REQUIRE(M && q && pair_i && pair_j, "g2v_dcx_sums: null pointer");
    G2V_REQUIRE((P == nullptr) != (D == nullptr), "g2v_dcx_sums: exactly one of P and D must be given");
    G2V_REQUIRE(S_pad >= 32 && S_pad % 32 == 0 && S_pad <= G2V_DCX_MAX_SAMPLES,
                "g2v_dcx_sums: S_pad = %d, must be a multiple of 32 in [32, %d]", (int)S_pad, G2V_DCX_MAX_SAMPLES);
    G2V_REQUIRE(n_b >= 1 && n_b <= G2V_DCX_MAX_ROWS, "g2v_dcx_sums: n_b = %lld rows, must be in [1, %d]",
                (long long)n_b, G2V_DCX_MAX_ROWS);
    G2V_REQUIRE(G >= 1, "g2v_dcx_sums: G = %d genes, must be >= 1", (int)G);
    G2V_REQUIRE(E >= 1 && E <= G2V_DCX_MAX_PAIRS, "g2v_dcx_sums: E = %lld pairs, must be in [1, %d]", (long long)E,
                G2V_DCX_MAX_PAIRS);
    DcxEpilogue ep{n, k, A, Bq, A_tot, B_tot, P_tot};
    if (D) {
        G2V_REQUIRE(A && Bq && A_tot && B_tot && P_tot, "g2v_dcx_sums: null pointer");
        G2V_REQUIRE(n >= 8 && n <= S_pad, "g2v_dcx_sums: n = %d samples, must be in [8, S_pad = %d]", (int)n,
                    (int)S_pad);
        G2V_REQUIRE(k >= 4 && n - k >= 4, "g2v_dcx_sums: k = %d, must be in [4, n - 4 = %d]", (int)k, (int)n - 4);
    }
    if (D) G2V_CUDA_OK(cudaFuncSetAttribute(dcx_sums_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                            (int)kSumSmem));
    else G2V_CUDA_OK(cudaFuncSetAttribute(dcx_sums_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)kSumSmem));
    const dim3 grid((unsigned)((E + kPairs - 1) / kPairs), (unsigned)((n_b + kRows - 1) / kRows));
    if (D)
        dcx_sums_kernel<true><<<grid, kSumThreads, kSumSmem, (cudaStream_t)stream>>>(M, n_b, S_pad, q, G, pair_i,
                                                                                    pair_j, E, ep, P, D);
    else
        dcx_sums_kernel<false><<<grid, kSumThreads, kSumSmem, (cudaStream_t)stream>>>(M, n_b, S_pad, q, G, pair_i,
                                                                                     pair_j, E, ep, P, D);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_dcx_tally(const double *D, int64_t n_b, int64_t E, const double *D_obs, int64_t *count,
                             int64_t *count_maxt, void *stream) {
    G2V_REQUIRE(D && D_obs && count && count_maxt, "g2v_dcx_tally: null pointer");
    G2V_REQUIRE(n_b >= 1 && n_b <= G2V_DCX_MAX_ROWS, "g2v_dcx_tally: n_b = %lld rows, must be in [1, %d]",
                (long long)n_b, G2V_DCX_MAX_ROWS);
    G2V_REQUIRE(E >= 1 && E <= G2V_DCX_MAX_PAIRS, "g2v_dcx_tally: E = %lld pairs, must be in [1, %d]", (long long)E,
                G2V_DCX_MAX_PAIRS);
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    // about two CTAs per SM; each CTA adds its counts to global memory once per pair tile
    int64_t rows = (n_b + 2 * dp.sm_count - 1) / (2 * dp.sm_count);
    if (rows > kTallyMaxRows) rows = kTallyMaxRows;
    const int64_t grid = (n_b + rows - 1) / rows;
    dcx_tally_kernel<<<(unsigned)grid, kTallyThreads, 0, (cudaStream_t)stream>>>(
        D, n_b, E, D_obs, (int32_t)rows, reinterpret_cast<unsigned long long *>(count),
        reinterpret_cast<unsigned long long *>(count_maxt));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
