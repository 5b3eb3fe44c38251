// g2v_km.cu -- best-of-R k-means (k = 3) restarts of the L-groups (DESIGN.md §4.26).
//   km_assign_kernel<RT>  a CTA owns a tile of rows and RT restarts: a register-tiled FP64 "GEMM" of the rows against
//                         the restarts' 3 centres (256 threads, 4 rows x 1 restart x 3 centres each), W converted to
//                         float64 in shared memory in chunks of 32 d consumed in ascending d, so every accumulator is
//                         the contract's chain; the argmin, mind and the changed / occupancy flags (shared-memory then
//                         global integer atomics) are fused into the epilogue.
//   km_seed_kernel        one CTA per restart: the k-means++ pick by an integer inverse CDF (max, q_i, Q, block scan).
//   km_blocks_kernel      one CTA per block of G2V_KM_BLOCK rows and up to 8 restarts: per cluster and d the
//                         sequential chain of x over the block's rows, the counts and the chain of mind.
//   km_update_kernel      one CTA per restart: the stop decision, the block chains / count, the relocation of empty
//                         clusters and the inertia.
//   km_contingency_kernel, km_agree_kernel  integer counts of the agreement between restarts.
// Every floating-point operation is a correctly rounded __dsub_rn / __dmul_rn / __dadd_rn / __ddiv_rn (the library is
// built with -fmad=true, so the chain must not be left to the compiler), every sum has a fixed order and every atomic
// is on integers, so the result equals the NumPy restatement bit for bit whatever the grid or the chunking.
#include "g2v_common.cuh"

namespace g2v {

constexpr int kKmThreads = 256;
constexpr int kKmDK = 32;                              // d per staged chunk
constexpr int kKmLd = kKmDK + 1;                       // padded staged row (doubles)
constexpr int kKmRowsPerThread = 4;
constexpr int kKmGroup = 8;                            // restarts per CTA of km_blocks_kernel
constexpr int kKmBlockThreads = 128;
constexpr int kKmSeedThreads = 1024;
constexpr int kKmSeedItems = 4;                        // consecutive rows per thread in a scan tile
constexpr int32_t kKmChanged = 8;

template <int RT> struct KmTile {
    static constexpr int TY = kKmThreads / RT;         // thread rows
    static constexpr int ROWS = TY * kKmRowsPerThread;
    static constexpr size_t smem = sizeof(double) * ((size_t)ROWS * kKmLd + (size_t)RT * 3 * kKmLd);
};

// ---- assign ----------------------------------------------------------------------------------------------------
// Zero padding past D adds (0 - 0)^2 = +0 to acc, which leaves it unchanged: acc >= +0 from the start, and a sum of
// +0 and +0 is +0.  So every chunk runs all 32 steps.
template <int RT>
__global__ void __launch_bounds__(kKmThreads)
km_assign_kernel(const float *__restrict__ W, int64_t n, int32_t D, const double *__restrict__ centres, int32_t kc,
                 const int32_t *__restrict__ active, int32_t n_active, int8_t *__restrict__ labels,
                 double *__restrict__ mind, int32_t *__restrict__ flags) {
    using T = KmTile<RT>;
    extern __shared__ __align__(16) unsigned char km_smem_raw[];
    double (*sx)[kKmLd] = reinterpret_cast<double (*)[kKmLd]>(km_smem_raw);
    double (*sc)[kKmLd] = sx + T::ROWS;                // [RT * 3][kKmLd]
    __shared__ int32_t sflag[RT];
    const int tid = threadIdx.x;
    const int tx = tid % RT, ty = tid / RT;
    const int64_t row0 = (int64_t)blockIdx.x * T::ROWS;
    const int k = blockIdx.y * RT + tx;                // position in the active list
    const int32_t slot = k < n_active ? active[k] : -1;
    if (tid < RT) sflag[tid] = 0;
    double acc[kKmRowsPerThread][3];
#pragma unroll
    for (int r = 0; r < kKmRowsPerThread; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[r][c] = 0.0;
    for (int d0 = 0; d0 < D; d0 += kKmDK) {
        __syncthreads();                               // the last chunk is consumed
        for (int e = tid; e < T::ROWS * kKmDK; e += kKmThreads) {
            const int rr = e / kKmDK, dd = e % kKmDK;
            const int64_t i = row0 + rr;
            const int d = d0 + dd;
            sx[rr][dd] = (i < n && d < D) ? (double)__ldg(W + i * D + d) : 0.0;
        }
        for (int e = tid; e < RT * 3 * kKmDK; e += kKmThreads) {
            const int q = e / kKmDK, dd = e % kKmDK;    // q = restart * 3 + centre
            const int kk = blockIdx.y * RT + q / 3;
            const int d = d0 + dd;
            sc[q][dd] = (kk < n_active && d < D) ? centres[((size_t)active[kk] * 3 + q % 3) * D + d] : 0.0;
        }
        __syncthreads();
#pragma unroll 8
        for (int dd = 0; dd < kKmDK; ++dd) {
            double x[kKmRowsPerThread], c[3];
#pragma unroll
            for (int r = 0; r < kKmRowsPerThread; ++r) x[r] = sx[ty + T::TY * r][dd];
#pragma unroll
            for (int q = 0; q < 3; ++q) c[q] = sc[tx * 3 + q][dd];
#pragma unroll
            for (int r = 0; r < kKmRowsPerThread; ++r)
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    const double t = __dsub_rn(x[r], c[q]);
                    acc[r][q] = __dadd_rn(acc[r][q], __dmul_rn(t, t));
                }
        }
    }
    int32_t bits = 0;
    if (slot >= 0) {
#pragma unroll
        for (int r = 0; r < kKmRowsPerThread; ++r) {
            const int64_t i = row0 + ty + T::TY * r;
            if (i >= n) break;
            int a = 0;
            double best = acc[r][0];
#pragma unroll
            for (int q = 1; q < 3; ++q)
                if (q < kc && acc[r][q] < best) { best = acc[r][q]; a = q; }
            const size_t at = (size_t)slot * n + i;
            mind[at] = best;
            if (kc == 3) {
                if (labels[at] != a) bits |= kKmChanged;
                labels[at] = (int8_t)a;
                bits |= 1 << a;
            }
        }
    }
    if (bits) atomicOr(&sflag[tx], bits);
    __syncthreads();
    if (tid < RT && blockIdx.y * RT + tid < n_active && sflag[tid]) atomicOr(flags + active[blockIdx.y * RT + tid], sflag[tid]);
}

// ---- block reductions ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t warp_scan_u64(uint64_t v, int lane) {          // inclusive
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// q_i = floor(2^32 * fl(D_i / maxD)), an integer in [0, 2^32]; the product by 2^32 is exact.
__device__ __forceinline__ uint64_t km_q(double Di, double maxD) {
    return (uint64_t)__double2ull_rz(__dmul_rn(__ddiv_rn(Di, maxD), 4294967296.0));
}

// ---- seeding ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kKmSeedThreads)
km_seed_kernel(const float *__restrict__ W, int64_t n, int32_t D, const double *__restrict__ mind, uint64_t seed,
               int64_t r_begin, int32_t t, double *__restrict__ centres, int32_t *__restrict__ seeds) {
    __shared__ double smax[kKmSeedThreads / 32];
    __shared__ uint64_t ssum[kKmSeedThreads / 32];
    __shared__ int64_t srow;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int32_t slot = blockIdx.x;
    const uint64_t u = draw64(seed, (1ull << 62) + (uint64_t)(r_begin + slot), (uint32_t)t);
    int64_t row = (int64_t)__umul64hi(u, (uint64_t)n);
    if (t > 0) {
        const double *m = mind + (size_t)slot * n;
        double mx = 0.0;                               // every D_i >= +0
        for (int64_t i = tid; i < n; i += kKmSeedThreads) mx = fmax(mx, m[i]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) smax[warp] = mx;
        __syncthreads();
        mx = smax[0];
        for (int w = 1; w < kKmSeedThreads / 32; ++w) mx = fmax(mx, smax[w]);
        if (mx > 0.0) {
            uint64_t s = 0;
            for (int64_t i = tid; i < n; i += kKmSeedThreads) s += km_q(m[i], mx);
            s = warp_sum_u64(s);
            if (lane == 0) ssum[warp] = s;
            __syncthreads();
            uint64_t Q = 0;
            for (int w = 0; w < kKmSeedThreads / 32; ++w) Q += ssum[w];
            const uint64_t target = __umul64hi(u, Q);  // < Q: the smallest i whose inclusive prefix exceeds it
            if (tid == 0) srow = -1;
            uint64_t base = 0;                         // the prefix before the tile
            for (int64_t i0 = 0; i0 < n; i0 += (int64_t)kKmSeedThreads * kKmSeedItems) {
                __syncthreads();                       // ssum and srow of the last tile are read
                uint64_t q[kKmSeedItems], own = 0;
                const int64_t ib = i0 + (int64_t)tid * kKmSeedItems;
#pragma unroll
                for (int j = 0; j < kKmSeedItems; ++j) {
                    q[j] = ib + j < n ? km_q(m[ib + j], mx) : 0;
                    own += q[j];
                }
                const uint64_t incl = warp_scan_u64(own, lane);
                if (lane == 31) ssum[warp] = incl;
                __syncthreads();
                uint64_t before = base, tile = 0;
                for (int w = 0; w < kKmSeedThreads / 32; ++w) {
                    if (w < warp) before += ssum[w];
                    tile += ssum[w];
                }
                uint64_t p = before + incl - own;      // exclusive prefix of this thread's first row
                if (p <= target && target < p + own) { // exactly one thread holds the crossing
#pragma unroll
                    for (int j = 0; j < kKmSeedItems; ++j) {
                        p += q[j];
                        if (p > target) { srow = ib + j; break; }
                    }
                }
                base += tile;
                __syncthreads();
                if (srow >= 0) break;
            }
            row = srow;
        }
    }
    if (tid == 0) seeds[slot * 3 + t] = (int32_t)row;
    for (int d = tid; d < D; d += kKmSeedThreads)
        centres[((size_t)slot * 3 + t) * D + d] = (double)__ldg(W + row * D + d);
}

// ---- block sums ------------------------------------------------------------------------------------------------
// acc + (+0) = acc for every acc the chain can hold (it starts at +0 and is never -0), so adding +0 for the rows of
// the other clusters gives the chain over the cluster's own rows.
__global__ void __launch_bounds__(kKmBlockThreads)
km_blocks_kernel(const float *__restrict__ W, const int8_t *__restrict__ labels, const double *__restrict__ mind,
                 int64_t n, int32_t D, const int32_t *__restrict__ active, int32_t n_active, double *__restrict__ psum,
                 int32_t *__restrict__ pcnt, double *__restrict__ pin) {
    __shared__ int8_t sl[kKmGroup][G2V_KM_BLOCK];
    const int tid = threadIdx.x;
    const int64_t b = blockIdx.x, nb = (n + G2V_KM_BLOCK - 1) / G2V_KM_BLOCK;
    const int64_t i0 = b * G2V_KM_BLOCK;
    const int len = (int)min((int64_t)G2V_KM_BLOCK, n - i0);
    const int g0 = blockIdx.y * kKmGroup;
    const int ng = min(kKmGroup, n_active - g0);
    for (int e = tid; e < kKmGroup * G2V_KM_BLOCK; e += kKmBlockThreads) {
        const int g = e / G2V_KM_BLOCK, j = e % G2V_KM_BLOCK;
        sl[g][j] = (g < ng && j < len) ? labels[(size_t)active[g0 + g] * n + i0 + j] : (int8_t)-1;
    }
    __syncthreads();
    if (tid < ng) {                                    // counts and the chain of mind
        const int32_t slot = active[g0 + tid];
        int32_t cnt[3] = {0, 0, 0};
        double in = 0.0;
        const double *m = mind + (size_t)slot * n + i0;
        for (int j = 0; j < len; ++j) {
            const int a = sl[tid][j];
            cnt[0] += a == 0; cnt[1] += a == 1; cnt[2] += a == 2;
            in = __dadd_rn(in, m[j]);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) pcnt[((size_t)slot * nb + b) * 3 + c] = cnt[c];
        pin[(size_t)slot * nb + b] = in;
    }
    for (int d = tid; d < D; d += kKmBlockThreads) {
        double acc[kKmGroup][3];
#pragma unroll
        for (int g = 0; g < kKmGroup; ++g)
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[g][c] = 0.0;
        const float *w = W + i0 * D + d;
        for (int j = 0; j < len; ++j) {
            const double x = (double)__ldg(w + (int64_t)j * D);
#pragma unroll
            for (int g = 0; g < kKmGroup; ++g) {
                const int a = sl[g][j];
#pragma unroll
                for (int c = 0; c < 3; ++c) acc[g][c] = __dadd_rn(acc[g][c], a == c ? x : 0.0);
            }
        }
#pragma unroll
        for (int g = 0; g < kKmGroup; ++g) {
            if (g >= ng) break;
            const int32_t slot = active[g0 + g];
#pragma unroll
            for (int c = 0; c < 3; ++c) psum[(((size_t)slot * nb + b) * 3 + c) * D + d] = acc[g][c];
        }
    }
}

// ---- update ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kKmThreads)
km_update_kernel(const float *__restrict__ W, const double *__restrict__ mind, const double *__restrict__ psum,
                 const int32_t *__restrict__ pcnt, const double *__restrict__ pin, int64_t n, int32_t D,
                 const int32_t *__restrict__ active, int32_t it, int32_t max_iter, int32_t *__restrict__ flags,
                 double *__restrict__ centres, int32_t *__restrict__ state, double *__restrict__ inertia,
                 int32_t *__restrict__ n_iter) {
    __shared__ int64_t scnt[3];
    __shared__ double sbm[kKmThreads / 32];
    __shared__ int64_t sbi[kKmThreads / 32];
    __shared__ int64_t srow[3];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int32_t slot = active[blockIdx.x];
    const int64_t nb = (n + G2V_KM_BLOCK - 1) / G2V_KM_BLOCK;
    const int32_t f = flags[slot];
    if (tid < 3) {
        int64_t c = 0;
        for (int64_t b = 0; b < nb; ++b) c += pcnt[((size_t)slot * nb + b) * 3 + tid];
        scnt[tid] = c;
    }
    const bool stop = it >= max_iter || (it > 1 && !(f & kKmChanged) && (f & 7) == 7);
    if (stop) {
        if (tid == 0) {
            double in = 0.0;
            for (int64_t b = 0; b < nb; ++b) in = __dadd_rn(in, pin[(size_t)slot * nb + b]);
            inertia[slot] = in;
            n_iter[slot] = it;
            state[slot] = 1;
            flags[slot] = 0;
        }
        return;
    }
    __syncthreads();
    double *C = centres + (size_t)slot * 3 * D;
    for (int e = tid; e < 3 * D; e += kKmThreads) {
        const int c = e / D;
        if (scnt[c] == 0) continue;
        double s = 0.0;
        for (int64_t b = 0; b < nb; ++b) s = __dadd_rn(s, psum[((size_t)slot * nb + b) * 3 * D + e]);
        C[e] = __ddiv_rn(s, (double)scnt[c]);
    }
    const double *m = mind + (size_t)slot * n;
    int n_moved = 0;
    for (int c = 0; c < 3; ++c) {                      // uniform: scnt is shared
        if (scnt[c] != 0) continue;
        double bm = -1.0;                              // every mind >= +0
        int64_t bi = -1;
        for (int64_t i = tid; i < n; i += kKmThreads) {
            bool taken = false;
            for (int p = 0; p < n_moved; ++p) taken |= srow[p] == i;
            if (!taken && m[i] > bm) { bm = m[i]; bi = i; }       // ascending i: the first of equal values stays
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double om = __shfl_xor_sync(0xffffffffu, bm, o);
            const int64_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (om > bm || (om == bm && oi >= 0 && (bi < 0 || oi < bi))) { bm = om; bi = oi; }
        }
        if (lane == 0) { sbm[warp] = bm; sbi[warp] = bi; }
        __syncthreads();
        if (tid == 0) {
            double m0 = sbm[0];
            int64_t i0 = sbi[0];
            for (int w = 1; w < kKmThreads / 32; ++w)
                if (sbm[w] > m0 || (sbm[w] == m0 && sbi[w] >= 0 && (i0 < 0 || sbi[w] < i0))) { m0 = sbm[w]; i0 = sbi[w]; }
            srow[n_moved] = i0;
        }
        __syncthreads();
        const int64_t row = srow[n_moved];
        for (int d = tid; d < D; d += kKmThreads) C[(size_t)c * D + d] = (double)__ldg(W + row * D + d);
        ++n_moved;
    }
    if (tid == 0) flags[slot] = 0;
}

// ---- agreement -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kKmThreads)
km_contingency_kernel(const int8_t *__restrict__ labels, const int8_t *__restrict__ best, int64_t n,
                      int64_t *__restrict__ table) {
    __shared__ int32_t st[9];
    const int tid = threadIdx.x;
    const int32_t slot = blockIdx.y;
    if (tid < 9) st[tid] = 0;
    __syncthreads();
    int32_t c[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    const int8_t *l = labels + (size_t)slot * n;
    for (int64_t i = (int64_t)blockIdx.x * kKmThreads + tid; i < n; i += (int64_t)gridDim.x * kKmThreads) {
        const int cell = l[i] * 3 + best[i];
#pragma unroll
        for (int q = 0; q < 9; ++q) c[q] += cell == q;
    }
#pragma unroll
    for (int q = 0; q < 9; ++q) {
        int32_t v = c[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((tid & 31) == 0 && v) atomicAdd(&st[q], v);
    }
    __syncthreads();
    if (tid < 9 && st[tid])
        atomicAdd(reinterpret_cast<unsigned long long *>(table + (size_t)slot * 9 + tid), (unsigned long long)st[tid]);
}

__global__ void __launch_bounds__(kKmThreads)
km_agree_kernel(const int8_t *__restrict__ labels, const int8_t *__restrict__ best, const int8_t *__restrict__ perm,
                int64_t n, int32_t n_slots, int32_t *__restrict__ count) {
    const int64_t i = (int64_t)blockIdx.x * kKmThreads + threadIdx.x;
    if (i >= n) return;
    const int b = best[i];
    int32_t c = 0;
    for (int32_t s = 0; s < n_slots; ++s) c += perm[s * 3 + labels[(size_t)s * n + i]] == b;
    count[i] += c;
}

}  // namespace g2v

using namespace g2v;

#define G2V_KM_CHECK_N(fn, n)                                                                                    \
    G2V_REQUIRE((n) >= 3 && (n) <= G2V_KM_MAX_GENES, fn ": n = %lld genes, must be in [3, %d]", (long long)(n), \
                G2V_KM_MAX_GENES)
#define G2V_KM_CHECK_D(fn, D) G2V_REQUIRE((D) >= 1, fn ": D = %d, must be >= 1", (int)(D))
#define G2V_KM_CHECK_SLOTS(fn, r)                                                                                \
    G2V_REQUIRE((r) >= 1 && (r) <= G2V_KM_MAX_RESTARTS, fn ": %d restarts, must be in [1, %d]", (int)(r),       \
                G2V_KM_MAX_RESTARTS)

template <int RT>
static int km_assign_launch(const float *W, int64_t n, int32_t D, const double *centres, int32_t kc,
                            const int32_t *active, int32_t n_active, int8_t *labels, double *mind, int32_t *flags,
                            cudaStream_t st) {
    using T = KmTile<RT>;
    G2V_CUDA_OK(cudaFuncSetAttribute(km_assign_kernel<RT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T::smem));
    const dim3 grid((unsigned)((n + T::ROWS - 1) / T::ROWS), (unsigned)((n_active + RT - 1) / RT));
    km_assign_kernel<RT><<<grid, kKmThreads, T::smem, st>>>(W, n, D, centres, kc, active, n_active, labels, mind, flags);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_km_assign(const float *W, int64_t n, int32_t D, const double *centres, int32_t kc,
                             const int32_t *active, int32_t n_active, int8_t *labels, double *mind, int32_t *flags,
                             void *stream) {
    G2V_REQUIRE(W && centres && active && mind, "g2v_km_assign: null pointer");
    G2V_KM_CHECK_N("g2v_km_assign", n);
    G2V_KM_CHECK_D("g2v_km_assign", D);
    G2V_KM_CHECK_SLOTS("g2v_km_assign", n_active);
    G2V_REQUIRE(kc >= 1 && kc <= 3, "g2v_km_assign: kc = %d centres, must be in [1, 3]", (int)kc);
    G2V_REQUIRE(kc < 3 || (labels && flags), "g2v_km_assign: null pointer");
    // 16 restarts per CTA when there are enough of them to fill the tile, else 4 (less padding for small R)
    if (n_active >= 16)
        return km_assign_launch<16>(W, n, D, centres, kc, active, n_active, labels, mind, flags, (cudaStream_t)stream);
    return km_assign_launch<4>(W, n, D, centres, kc, active, n_active, labels, mind, flags, (cudaStream_t)stream);
}

extern "C" int g2v_km_seed(const float *W, int64_t n, int32_t D, const double *mind, uint64_t seed, int64_t r_begin,
                           int32_t t, int32_t n_slots, double *centres, int32_t *seeds, void *stream) {
    G2V_REQUIRE(W && centres && seeds && (t == 0 || mind), "g2v_km_seed: null pointer");
    G2V_KM_CHECK_N("g2v_km_seed", n);
    G2V_KM_CHECK_D("g2v_km_seed", D);
    G2V_KM_CHECK_SLOTS("g2v_km_seed", n_slots);
    G2V_REQUIRE(t >= 0 && t <= 2, "g2v_km_seed: t = %d, must be in [0, 2]", (int)t);
    G2V_REQUIRE(r_begin >= 0 && r_begin + n_slots <= G2V_KM_MAX_RESTARTS,
                "g2v_km_seed: restarts %lld .. %lld, must lie in [0, %d)", (long long)r_begin,
                (long long)(r_begin + n_slots - 1), G2V_KM_MAX_RESTARTS);
    km_seed_kernel<<<(unsigned)n_slots, kKmSeedThreads, 0, (cudaStream_t)stream>>>(W, n, D, mind, seed, r_begin, t,
                                                                                  centres, seeds);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_km_blocks(const float *W, const int8_t *labels, const double *mind, int64_t n, int32_t D,
                             const int32_t *active, int32_t n_active, double *psum, int32_t *pcnt, double *pin,
                             void *stream) {
    G2V_REQUIRE(W && labels && mind && active && psum && pcnt && pin, "g2v_km_blocks: null pointer");
    G2V_KM_CHECK_N("g2v_km_blocks", n);
    G2V_KM_CHECK_D("g2v_km_blocks", D);
    G2V_KM_CHECK_SLOTS("g2v_km_blocks", n_active);
    const dim3 grid((unsigned)((n + G2V_KM_BLOCK - 1) / G2V_KM_BLOCK), (unsigned)((n_active + kKmGroup - 1) / kKmGroup));
    km_blocks_kernel<<<grid, kKmBlockThreads, 0, (cudaStream_t)stream>>>(W, labels, mind, n, D, active, n_active, psum,
                                                                        pcnt, pin);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_km_update(const float *W, const double *mind, const double *psum, const int32_t *pcnt,
                             const double *pin, int64_t n, int32_t D, const int32_t *active, int32_t n_active,
                             int32_t it, int32_t max_iter, int32_t *flags, double *centres, int32_t *state,
                             double *inertia, int32_t *n_iter, void *stream) {
    G2V_REQUIRE(W && mind && psum && pcnt && pin && active && flags && centres && state && inertia && n_iter,
                "g2v_km_update: null pointer");
    G2V_KM_CHECK_N("g2v_km_update", n);
    G2V_KM_CHECK_D("g2v_km_update", D);
    G2V_KM_CHECK_SLOTS("g2v_km_update", n_active);
    G2V_REQUIRE(max_iter >= 1 && it >= 1 && it <= max_iter, "g2v_km_update: iteration %d of %d", (int)it,
                (int)max_iter);
    km_update_kernel<<<(unsigned)n_active, kKmThreads, 0, (cudaStream_t)stream>>>(
        W, mind, psum, pcnt, pin, n, D, active, it, max_iter, flags, centres, state, inertia, n_iter);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_km_contingency(const int8_t *labels, const int8_t *best, int64_t n, int32_t n_slots,
                                  int64_t *table, void *stream) {
    G2V_REQUIRE(labels && best && table, "g2v_km_contingency: null pointer");
    G2V_KM_CHECK_N("g2v_km_contingency", n);
    G2V_KM_CHECK_SLOTS("g2v_km_contingency", n_slots);
    const int64_t tiles = (n + kKmThreads - 1) / kKmThreads;
    const dim3 grid((unsigned)min(tiles, (int64_t)256), (unsigned)n_slots);
    km_contingency_kernel<<<grid, kKmThreads, 0, (cudaStream_t)stream>>>(labels, best, n, table);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_km_agree(const int8_t *labels, const int8_t *best, const int8_t *perm, int64_t n, int32_t n_slots,
                            int32_t *count, void *stream) {
    G2V_REQUIRE(labels && best && perm && count, "g2v_km_agree: null pointer");
    G2V_KM_CHECK_N("g2v_km_agree", n);
    G2V_KM_CHECK_SLOTS("g2v_km_agree", n_slots);
    km_agree_kernel<<<(unsigned)((n + kKmThreads - 1) / kKmThreads), kKmThreads, 0, (cudaStream_t)stream>>>(
        labels, best, perm, n, n_slots, count);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
