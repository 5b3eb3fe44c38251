// g2v_perm.cu -- label-permutation test of the gene t statistics (DESIGN.md §4.24).
//   perm_labels_kernel  one warp per permutation: Fisher-Yates on the observed indicator in shared memory, the
//                       lanes drawing 32 swap targets at a time from the walk sampler's Philox stream into shared
//                       memory, lane 0 swapping in order; the row goes out with the zero padding.
//   perm_sums_kernel    A = M . q on the INT8 tensor cores: mma.sync m16n8k32 u8 x s8 (high plane) and u8 x u8
//                       (middle and low planes), fragments loaded straight from global memory (L1/L2 serve the
//                       reuse); a warp owns 32 permutations x 32 genes and all three planes of them, so the int64
//                       A = 2^16 h + 2^8 m + l is formed in registers in the epilogue.
//   perm_tally_kernel   a CTA owns a run of rows and walks the gene axis (rank order) from the right in tiles of
//                       128 genes, carrying each row's running max of rho in shared memory; counts are kept per
//                       lane, summed per CTA with shared-memory atomics and added to global memory once per tile.
// Everything the counts depend on is integer or one correctly rounded float64 operation (__dmul_rn, IEEE
// division), so they equal the NumPy restatement bit for bit whatever the grid or the chunking.
#include "g2v_common.cuh"

namespace g2v {

// ---- labels -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
perm_labels_kernel(const uint8_t *__restrict__ obs, int32_t n, int32_t S_pad, uint64_t seed, int64_t b_begin,
                   uint8_t *__restrict__ M) {
    extern __shared__ uint4 row4[];                    // [S_pad / 16]
    __shared__ uint32_t js[32];                        // the swap targets of one round of 32 draws
    uint8_t *row = reinterpret_cast<uint8_t *>(row4);
    const int lane = threadIdx.x;
    const int64_t r = blockIdx.x;
    const uint64_t subseq = (1ull << 63) + (uint64_t)(b_begin + r + 1);
    for (int s = lane; s < S_pad; s += 32) row[s] = s < n ? obs[s] : (uint8_t)0;
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
                const uint8_t x = row[i];
                row[i] = row[jt];
                row[jt] = x;
            }
        }
        __syncwarp();                                  // the swaps are done before js is rewritten or row read
    }
    uint4 *out = reinterpret_cast<uint4 *>(M + r * S_pad);
    for (int w = lane; w < (S_pad >> 4); w += 32) out[w] = row4[w];
}

// ---- sums ---------------------------------------------------------------------------------------------------
constexpr int kSumTile = 64;                           // CTA: 64 permutations x 64 genes, 2 x 2 warps of 32 x 32

__device__ __forceinline__ void mma_u8s8(int c[4], const uint32_t a[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_u8u8(int c[4], const uint32_t a[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// The k order inside a 32-sample step is free (the sums are exact), so each lane loads 8 contiguous bytes of its row
// (tig*8 .. tig*8+7) and hands the first 4 to the fragment's k block tig and the last 4 to block tig + 4: the A and
// B fragments use the same map, so every product pairs the same sample.
__global__ void __launch_bounds__(128)
perm_sums_kernel(const uint8_t *__restrict__ M, const uint8_t *__restrict__ planes, int64_t n_b, int32_t S_pad,
                 int32_t G, int64_t *__restrict__ A) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gid = lane >> 2, tig = lane & 3;
    const int64_t r0 = (int64_t)blockIdx.x * kSumTile + (warp & 1) * 32;
    const int64_t g0 = (int64_t)blockIdx.y * kSumTile + (warp >> 1) * 32;
    const size_t plane = (size_t)G * S_pad;
    const uint8_t *ap[2][2];                           // rows r0 + 16 mt + gid + 8 h
    bool aok[2][2];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t r = r0 + mt * 16 + gid + h * 8;
            aok[mt][h] = r < n_b;
            ap[mt][h] = M + (aok[mt][h] ? r : 0) * S_pad + tig * 8;
        }
    const uint8_t *bp[4];                              // genes g0 + 8 nt + gid
    bool bok[4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        const int64_t g = g0 + nt * 8 + gid;
        bok[nt] = g < G;
        bp[nt] = planes + (bok[nt] ? g : 0) * S_pad + tig * 8;
    }
    int acc[3][2][4][4];
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[p][mt][nt][e] = 0;
    const uint2 zero = make_uint2(0u, 0u);
    for (int k0 = 0; k0 < S_pad; k0 += 32) {
        uint2 a[2][2], b[3][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int h = 0; h < 2; ++h)
                a[mt][h] = aok[mt][h] ? __ldg(reinterpret_cast<const uint2 *>(ap[mt][h] + k0)) : zero;
#pragma unroll
        for (int p = 0; p < 3; ++p)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
                b[p][nt] = bok[nt] ? __ldg(reinterpret_cast<const uint2 *>(bp[nt] + p * plane + k0)) : zero;
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const uint32_t af[4] = {a[mt][0].x, a[mt][1].x, a[mt][0].y, a[mt][1].y};
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                mma_u8s8(acc[0][mt][nt], af, b[0][nt].x, b[0][nt].y);
                mma_u8u8(acc[1][mt][nt], af, b[1][nt].x, b[1][nt].y);
                mma_u8u8(acc[2][mt][nt], af, b[2][nt].x, b[2][nt].y);
            }
        }
    }
    // accumulator e: row gid (e < 2) or gid + 8, gene 2 tig + (e & 1)
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int64_t r = r0 + mt * 16 + gid + (e >> 1) * 8, g = g0 + nt * 8 + tig * 2 + (e & 1);
                if (r < n_b && g < G)
                    A[r * G + g] = (int64_t)acc[0][mt][nt][e] * 65536 + (int64_t)acc[1][mt][nt][e] * 256 +
                                   (int64_t)acc[2][mt][nt][e];
            }
}

// ---- tally --------------------------------------------------------------------------------------------------
constexpr int kTallyThreads = 256, kTallyWarps = kTallyThreads / 32, kTallyV = 4, kTallyTile = 32 * kTallyV;
constexpr int kTallyMaxRows = 1024;                    // rows per CTA (the carries live in shared memory)

__global__ void __launch_bounds__(kTallyThreads)
perm_tally_kernel(const int64_t *__restrict__ A, int64_t n_b, int32_t G, int32_t n, int32_t k,
                  const int64_t *__restrict__ Q, const double *__restrict__ W, const int64_t *__restrict__ absN_obs,
                  const double *__restrict__ rho_obs, int32_t rows_per_cta, unsigned long long *__restrict__ count,
                  unsigned long long *__restrict__ count_maxt) {
    __shared__ double carry[kTallyMaxRows];
    __shared__ uint32_t cnt[2][kTallyTile];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t rb = (int64_t)blockIdx.x * rows_per_cta;
    const int R = (int)min((int64_t)rows_per_cta, n_b - rb);
    for (int i = threadIdx.x; i < R; i += kTallyThreads) carry[i] = 0.0;
    const int n_tiles = (G + kTallyTile - 1) / kTallyTile;
    for (int t = n_tiles - 1; t >= 0; --t) {
        int64_t q[kTallyV], an[kTallyV];
        double w[kTallyV], ro[kTallyV];
        bool ok[kTallyV];
#pragma unroll
        for (int v = 0; v < kTallyV; ++v) {
            const int j = t * kTallyTile + v * 32 + lane;
            ok[v] = j < G;
            q[v] = ok[v] ? Q[j] : 0;
            an[v] = ok[v] ? absN_obs[j] : 0;
            w[v] = ok[v] ? W[j] : 0.0;
            ro[v] = ok[v] ? rho_obs[j] : 0.0;
        }
        cnt[threadIdx.x / kTallyTile][threadIdx.x % kTallyTile] = 0u;
        __syncthreads();
        uint32_t c1[kTallyV] = {}, c2[kTallyV] = {};
        for (int r = warp; r < R; r += kTallyWarps) {
            const int64_t *row = A + (rb + r) * G + t * kTallyTile + lane;
            int64_t a[kTallyV];
#pragma unroll
            for (int v = 0; v < kTallyV; ++v) a[v] = ok[v] ? __ldg(row + v * 32) : 0;
            double cr = carry[r];                      // max of rho over the genes right of this sub-tile
#pragma unroll
            for (int v = kTallyV - 1; v >= 0; --v) {
                const int64_t N = (int64_t)n * a[v] - (int64_t)k * q[v];
                const int64_t absN = N < 0 ? -N : N;
                c1[v] += (ok[v] && absN >= an[v]) ? 1u : 0u;
                const double d = (double)N;
                double rho = w[v] > 0.0 ? __ddiv_rn(__dmul_rn(d, d), w[v]) : 0.0;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {     // inclusive suffix max over the lanes
                    const double x = __shfl_down_sync(0xffffffffu, rho, o);
                    if (lane + o < 32 && x > rho) rho = x;
                }
                if (cr > rho) rho = cr;
                c2[v] += (ok[v] && rho >= ro[v]) ? 1u : 0u;
                cr = __shfl_sync(0xffffffffu, rho, 0);
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
            const int j = t * kTallyTile + jj;
            const uint32_t c = cnt[which][jj];
            if (j < G && c) atomicAdd((which ? count_maxt : count) + j, (unsigned long long)c);
        }
        __syncthreads();                               // cnt is cleared for the next tile
    }
}
static_assert(2 * kTallyTile == kTallyThreads, "one thread per tile counter");

}  // namespace g2v

using namespace g2v;

#define G2V_PERM_CHECK_SAMPLES(fn, n)                                                                        \
    G2V_REQUIRE((n) >= 3 && (n) <= G2V_PERM_MAX_SAMPLES, fn ": n = %d samples, must be in [3, %d]", (int)(n),       \
                G2V_PERM_MAX_SAMPLES)

extern "C" int g2v_perm_labels(const uint8_t *obs, int32_t n, int32_t S_pad, uint64_t seed, int64_t b_begin,
                               int64_t n_b, uint8_t *M, void *stream) {
    G2V_REQUIRE(obs && M, "g2v_perm_labels: null pointer");
    G2V_PERM_CHECK_SAMPLES("g2v_perm_labels", n);
    G2V_REQUIRE(S_pad >= n && S_pad % 32 == 0 && S_pad <= G2V_PERM_MAX_SAMPLES,
                "g2v_perm_labels: S_pad = %d, must be a multiple of 32 in [n = %d, %d]", (int)S_pad, (int)n,
                G2V_PERM_MAX_SAMPLES);
    G2V_REQUIRE(b_begin >= 0 && n_b >= 1 && b_begin + n_b <= G2V_PERM_MAX_PERMUTATIONS,
                "g2v_perm_labels: permutations %lld + [1, %lld] out of [1, %d]", (long long)b_begin, (long long)n_b,
                G2V_PERM_MAX_PERMUTATIONS);
    perm_labels_kernel<<<(unsigned)n_b, 32, (size_t)S_pad, (cudaStream_t)stream>>>(obs, n, S_pad, seed, b_begin, M);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_perm_sums(const uint8_t *M, const uint8_t *planes, int64_t n_b, int32_t S_pad, int32_t G,
                             int64_t *A, void *stream) {
    G2V_REQUIRE(M && planes && A, "g2v_perm_sums: null pointer");
    G2V_REQUIRE(S_pad >= 32 && S_pad % 32 == 0 && S_pad <= G2V_PERM_MAX_SAMPLES,
                "g2v_perm_sums: S_pad = %d, must be a multiple of 32 in [32, %d]", (int)S_pad, G2V_PERM_MAX_SAMPLES);
    G2V_REQUIRE(n_b >= 1 && n_b <= G2V_PERM_MAX_PERMUTATIONS, "g2v_perm_sums: n_b = %lld rows, must be in [1, %d]",
                (long long)n_b, G2V_PERM_MAX_PERMUTATIONS);
    G2V_REQUIRE(G >= 1 && (G + kSumTile - 1) / kSumTile <= 65535, "g2v_perm_sums: G = %d genes, must be in [1, %d]",
                (int)G, 65535 * kSumTile);
    const dim3 grid((unsigned)((n_b + kSumTile - 1) / kSumTile), (unsigned)((G + kSumTile - 1) / kSumTile));
    perm_sums_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(M, planes, n_b, S_pad, G, A);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_perm_tally(const int64_t *A, int64_t n_b, int32_t G, int32_t n, int32_t k, const int64_t *Q,
                              const double *W, const int64_t *absN_obs, const double *rho_obs, int64_t *count,
                              int64_t *count_maxt, void *stream) {
    G2V_REQUIRE(A && Q && W && absN_obs && rho_obs && count && count_maxt, "g2v_perm_tally: null pointer");
    G2V_PERM_CHECK_SAMPLES("g2v_perm_tally", n);
    G2V_REQUIRE(k >= 1 && k < n, "g2v_perm_tally: k = %d, must be in [1, n - 1 = %d]", (int)k, (int)n - 1);
    G2V_REQUIRE(n_b >= 1 && n_b <= G2V_PERM_MAX_PERMUTATIONS, "g2v_perm_tally: n_b = %lld rows, must be in [1, %d]",
                (long long)n_b, G2V_PERM_MAX_PERMUTATIONS);
    G2V_REQUIRE(G >= 1, "g2v_perm_tally: G = %d genes, must be >= 1", (int)G);
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    // about two CTAs per SM; each CTA adds its counts to global memory once per gene tile
    int64_t rows = (n_b + 2 * dp.sm_count - 1) / (2 * dp.sm_count);
    if (rows > kTallyMaxRows) rows = kTallyMaxRows;
    const int64_t grid = (n_b + rows - 1) / rows;
    perm_tally_kernel<<<(unsigned)grid, kTallyThreads, 0, (cudaStream_t)stream>>>(
        A, n_b, G, n, k, Q, W, absN_obs, rho_obs, (int32_t)rows, reinterpret_cast<unsigned long long *>(count),
        reinterpret_cast<unsigned long long *>(count_maxt));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
