// g2v_cbow_plan.cu -- mini-batch epochs on the device (DESIGN.md §4.12): the reshuffled epoch order of the training
// list (a keyed Feistel permutation, no sort) and the per-batch transposed incidence that lazy_adam steps read
// (a counting transpose per batch: count, scan, scatter, then the positions of each gene put back in ascending order).
#include <algorithm>
#include <climits>

#include "g2v_common.cuh"

namespace g2v {
namespace {

// ---- epoch order ---------------------------------------------------------------------------------------------------
// P(seed, epoch, n): a 4-round Feistel network on b bits (the smallest even b >= 2 with 2^b >= n), cycle-walked back
// into [0, n).  Round r of the network maps (L, R) -> (R, L ^ F_r(R)) with
//   F_r(R) = word 0 of Philox4x32-10(counter {R, kOrderDomain | r, epoch, n}, key {seed lo, seed hi}) & (2^(b/2) - 1).
// The walk sampler's counters have word 1 == 0 (g2v_common.cuh draw64), these never do: the two streams are disjoint.
constexpr uint32_t kOrderDomain = 0x53480000u;

__host__ __device__ __forceinline__ int order_half_bits(int64_t n) {
    int b = 2;
    while (b < 32 && (1ull << b) < (uint64_t)n) b += 2;
    return b / 2;
}

__device__ __forceinline__ uint32_t feistel(uint32_t x, int h, uint32_t mask, uint32_t k0, uint32_t k1, uint32_t epoch,
                                            uint32_t n32) {
    uint32_t L = x >> h, R = x & mask;
#pragma unroll
    for (uint32_t r = 0; r < 4; ++r) {
        uint32_t w[4];
        philox4x32_10(R, kOrderDomain | r, epoch, n32, k0, k1, w);
        const uint32_t t = L ^ (w[0] & mask);
        L = R;
        R = t;
    }
    return (L << h) | R;
}

__global__ void __launch_bounds__(256)
epoch_order_kernel(const int32_t *__restrict__ tr, int64_t n, uint64_t seed, uint32_t epoch, int64_t rank, int64_t world,
                   int64_t n_loc, int32_t *__restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_loc) return;
    const int h = order_half_bits(n);
    const uint32_t mask = (1u << h) - 1u;
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32), n32 = (uint32_t)n;
    uint32_t y = feistel((uint32_t)(rank + i * world), h, mask, k0, k1, epoch, n32);
    while ((int64_t)y >= n) y = feistel(y, h, mask, k0, k1, epoch, n32);
    out[i] = __ldg(tr + y);
}

// ---- batch plan ----------------------------------------------------------------------------------------------------
// Batches are processed in waves of K consecutive batches with one int32 counter per (batch of the wave, gene):
// K * V <= kCounterBudget, so the counters stay L2-sized at any V.  Per wave, 7 launches:
//   count      one warp per window: cnt[batch][gene] += 1 per incidence
//   tile_sums  per tile of kTile counters: packed sum (count << 32 | nonzero)
//   tile_scan  one CTA: exclusive scan of the tile sums; advances the running totals (rows, incidences) in hdr
//   emit       per counter with count > 0: rows[r] = gene, segptr[r] = first incidence q; cnt becomes the cursor q;
//              batch_rowptr[batch] = the batch's first row
//   scatter    one warp per window: tmp[cursor++] = position of the window relative to its batch
//   sort_short one lane per segment of 1 or 2 positions; one warp per segment of 3..32: rank sort in registers;
//              tmp -> pos
//   sort_long  one CTA per longer segment (listed by sort_short): bitonic sort in shared memory up to kLongCap
//              positions, else a counting pass over position ranges of kLongCap
// hdr (int64): [0] rows so far, [1] incidences so far, [2] first row of the wave, [3] first incidence of the wave,
// [4] long segments of the wave, [5] overflow (the list has more incidences than the caller's nnz).
constexpr int kPlanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kTile = kPlanThreads * kScanItems;
constexpr int kLongCap = 4096;
constexpr int64_t kCounterBudget = int64_t(1) << 22;
constexpr int kHdr = 8;

struct PlanGeometry {
    int64_t n_b, K, n_tiles;
    size_t off_long, off_toff, off_cnt, off_tmp, bytes;
};

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

PlanGeometry plan_geometry(int64_t n_win, int64_t nnz, int64_t B, int32_t V) {
    PlanGeometry g;
    g.n_b = n_win > 0 ? (n_win + B - 1) / B : 0;
    g.K = kCounterBudget / (V > 0 ? V : 1);
    if (g.K < 1) g.K = 1;
    if (g.K > g.n_b) g.K = g.n_b > 0 ? g.n_b : 1;
    g.n_tiles = (g.K * (int64_t)V + kTile - 1) / kTile;
    const int64_t n_long = std::min<int64_t>(g.K * (int64_t)V, nnz) + 1;
    g.off_long = align256(kHdr * sizeof(int64_t));
    g.off_toff = g.off_long + align256((size_t)n_long * sizeof(int32_t));
    g.off_cnt = g.off_toff + align256((size_t)g.n_tiles * sizeof(uint64_t));
    g.off_tmp = g.off_cnt + align256((size_t)g.n_tiles * kTile * sizeof(int32_t));
    g.bytes = g.off_tmp + align256((size_t)(nnz > 0 ? nnz : 1) * sizeof(int32_t));
    return g;
}

// Exclusive scan over the CTA of one value per thread; *total = the CTA's sum.  `sh` = 32 words of shared memory.
__device__ __forceinline__ uint64_t block_exclusive_scan(uint64_t v, uint64_t *sh, uint64_t *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    uint64_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint64_t s = lane < nwarps ? sh[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        if (lane < nwarps) sh[lane] = s;
    }
    __syncthreads();
    const uint64_t base = warp ? sh[warp - 1] : 0;
    *total = sh[nwarps - 1];
    __syncthreads();
    return base + inc - v;
}

__device__ __forceinline__ bool overflowed(const int64_t *hdr) { return *reinterpret_cast<const volatile int64_t *>(hdr + 5) != 0; }

template <bool SCATTER>
__global__ void __launch_bounds__(kPlanThreads)
plan_windows_kernel(const int32_t *__restrict__ rowptr, const int32_t *__restrict__ gene, const int32_t *__restrict__ win,
                    int64_t w_begin, int64_t w_end, int64_t B, int64_t b0, int32_t V, int32_t *__restrict__ cnt,
                    int32_t *__restrict__ tmp, const int64_t *hdr) {
    if (SCATTER && overflowed(hdr)) return;
    const int lane = threadIdx.x & 31;
    const int64_t i = w_begin + (int64_t)blockIdx.x * (kPlanThreads / 32) + (threadIdx.x >> 5);
    if (i >= w_end) return;
    const int64_t b = i / B;
    const int32_t rel = (int32_t)(i - b * B);
    int32_t *c = cnt + (b - b0) * (int64_t)V;
    const int32_t w = __ldg(win + i);
    const int32_t s = __ldg(rowptr + w), e = __ldg(rowptr + w + 1);
    for (int32_t k = s + lane; k < e; k += 32) {
        const int32_t g = __ldg(gene + k);
        if (SCATTER) tmp[atomicAdd(c + g, 1)] = rel;
        else atomicAdd(c + g, 1);
    }
}

__device__ __forceinline__ uint64_t packed(int32_t c) { return ((uint64_t)(uint32_t)c << 32) | (uint64_t)(c > 0); }

__global__ void __launch_bounds__(kPlanThreads) plan_tile_sums_kernel(const int32_t *__restrict__ cnt, uint64_t *toff) {
    __shared__ uint64_t sh[32];
    const int32_t *c = cnt + (int64_t)blockIdx.x * kTile;
    uint64_t s = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) s += packed(c[j * kPlanThreads + threadIdx.x]);
    uint64_t total;
    block_exclusive_scan(s, sh, &total);
    if (threadIdx.x == 0) toff[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kPlanThreads)
plan_tile_scan_kernel(uint64_t *toff, int64_t n_tiles, int64_t nnz_cap, int64_t b_end, int64_t n_b,
                      int32_t *__restrict__ segptr, int32_t *__restrict__ batch_rowptr, int64_t *hdr) {
    __shared__ uint64_t sh[32];
    if (overflowed(hdr)) return;
    uint64_t carry = 0;
    for (int64_t base = 0; base < n_tiles; base += kPlanThreads) {
        const int64_t t = base + threadIdx.x;
        const uint64_t v = t < n_tiles ? toff[t] : 0;
        uint64_t total;
        const uint64_t ex = block_exclusive_scan(v, sh, &total);
        if (t < n_tiles) toff[t] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) {
        const int64_t rows = hdr[0] + (int64_t)(carry & 0xffffffffu), inc = hdr[1] + (int64_t)(carry >> 32);
        if (inc > nnz_cap) {                           // more incidences than the caller allocated for: write nothing
            hdr[5] = 1;
            batch_rowptr[n_b] = -1;
            return;
        }
        hdr[2] = hdr[0]; hdr[3] = hdr[1];
        hdr[0] = rows; hdr[1] = inc; hdr[4] = 0;
        segptr[rows] = (int32_t)inc;
        batch_rowptr[b_end] = (int32_t)rows;
    }
}

__global__ void __launch_bounds__(kPlanThreads)
plan_emit_kernel(int32_t *__restrict__ cnt, const uint64_t *__restrict__ toff, int64_t n_used, int32_t V, int64_t b0,
                 int32_t *__restrict__ rows, int32_t *__restrict__ segptr, int32_t *__restrict__ batch_rowptr,
                 const int64_t *hdr) {
    __shared__ uint64_t sh[32];
    if (overflowed(hdr)) return;
    const int64_t e0 = (int64_t)blockIdx.x * kTile + threadIdx.x * kScanItems;
    int32_t c[kScanItems];
    const int4 *p4 = reinterpret_cast<const int4 *>(cnt + e0);
    const int4 a = p4[0], b = p4[1];
    c[0] = a.x; c[1] = a.y; c[2] = a.z; c[3] = a.w; c[4] = b.x; c[5] = b.y; c[6] = b.z; c[7] = b.w;
    uint64_t s = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) s += packed(c[j]);
    uint64_t total;
    uint64_t p = toff[blockIdx.x] + block_exclusive_scan(s, sh, &total);
    const int64_t r0 = hdr[2], q0 = hdr[3];
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        const int64_t e = e0 + j;
        const int32_t r = (int32_t)(r0 + (int64_t)(p & 0xffffffffu)), q = (int32_t)(q0 + (int64_t)(p >> 32));
        if (e < n_used) {
            const int64_t bl = e / V, g = e - bl * V;
            if (c[j] > 0) {
                rows[r] = (int32_t)g;
                segptr[r] = q;
                cnt[e] = q;
            }
            if (g == 0) batch_rowptr[b0 + bl] = r;
        }
        p += packed(c[j]);
    }
}

__global__ void __launch_bounds__(kPlanThreads)
plan_sort_short_kernel(const int32_t *__restrict__ segptr, const int32_t *__restrict__ tmp, int32_t *__restrict__ pos,
                       int32_t *__restrict__ long_list, int64_t *hdr) {
    if (overflowed(hdr)) return;
    const int lane = threadIdx.x & 31;
    const int64_t r_begin = hdr[2], r_end = hdr[0];
    const int64_t stride = (int64_t)gridDim.x * kPlanThreads;
    // each warp takes 32 consecutive segments, one per lane: a lane finishes its own segment when it holds at most 2
    // positions (most segments of a batch that touches a large share of the genes), the warp rank-sorts the segments
    // of 3..32 positions one after the other, and longer ones go to the long list
    for (int64_t base = r_begin + (int64_t)blockIdx.x * kPlanThreads + (threadIdx.x & ~31); base < r_end;
         base += stride) {
        const int64_t r = base + lane;
        int32_t s = 0, L = 0;
        if (r < r_end) {
            s = segptr[r];
            L = segptr[r + 1] - s;
            if (L == 1) {
                pos[s] = tmp[s];
            } else if (L == 2) {
                const int32_t a = tmp[s], b = tmp[s + 1];
                pos[s] = min(a, b);
                pos[s + 1] = max(a, b);
            } else if (L > 32) {
                long_list[atomicAdd(reinterpret_cast<unsigned long long *>(hdr + 4), 1ull)] = (int32_t)r;
            }
        }
        for (unsigned mid = __ballot_sync(0xffffffffu, L > 2 && L <= 32); mid; mid &= mid - 1) {
            const int src = __ffs(mid) - 1;
            const int32_t ss = __shfl_sync(0xffffffffu, s, src), LL = __shfl_sync(0xffffffffu, L, src);
            const int32_t v = lane < LL ? tmp[ss + lane] : INT_MAX;
            int rank = 0;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const int32_t u = __shfl_sync(0xffffffffu, v, j);
                rank += (u < v) || (u == v && j < lane);
            }
            if (lane < LL) pos[ss + rank] = v;
        }
    }
}

__global__ void __launch_bounds__(kPlanThreads)
plan_sort_long_kernel(const int32_t *__restrict__ segptr, const int32_t *__restrict__ tmp, int32_t *__restrict__ pos,
                      const int32_t *__restrict__ long_list, int64_t B, const int64_t *hdr) {
    __shared__ int32_t sm[kLongCap];
    __shared__ uint64_t sh[32];
    if (overflowed(hdr)) return;
    const int64_t n_long = hdr[4];
    for (int64_t li = blockIdx.x; li < n_long; li += gridDim.x) {
        const int64_t r = long_list[li];
        const int32_t s = segptr[r], L = segptr[r + 1] - s;
        if (L <= kLongCap) {                           // bitonic sort of the segment padded to a power of two
            int P = 64;
            while (P < L) P <<= 1;
            for (int k = threadIdx.x; k < P; k += kPlanThreads) sm[k] = k < L ? tmp[s + k] : INT_MAX;
            for (int size = 2; size <= P; size <<= 1) {
                for (int stride = size >> 1; stride > 0; stride >>= 1) {
                    __syncthreads();
                    for (int k = threadIdx.x; k < (P >> 1); k += kPlanThreads) {
                        const int i = 2 * stride * (k / stride) + (k % stride), j = i + stride;
                        const int32_t x = sm[i], y = sm[j];
                        if ((x > y) == ((i & size) == 0)) { sm[i] = y; sm[j] = x; }
                    }
                }
            }
            __syncthreads();
            for (int k = threadIdx.x; k < L; k += kPlanThreads) pos[s + k] = sm[k];
            __syncthreads();
            continue;
        }
        // counting over position ranges [v0, v0 + kLongCap): positions lie in [0, B)
        int64_t out = s;
        for (int64_t v0 = 0; v0 < B; v0 += kLongCap) {
            for (int k = threadIdx.x; k < kLongCap; k += kPlanThreads) sm[k] = 0;
            __syncthreads();
            for (int32_t k = threadIdx.x; k < L; k += kPlanThreads) {
                const int64_t d = (int64_t)tmp[s + k] - v0;
                if (d >= 0 && d < kLongCap) atomicAdd(sm + d, 1);
            }
            __syncthreads();
            constexpr int per = kLongCap / kPlanThreads;
            const int k0 = threadIdx.x * per;
            uint64_t mine = 0;
            for (int k = 0; k < per; ++k) mine += (uint64_t)sm[k0 + k];
            uint64_t total;
            int64_t o = out + (int64_t)block_exclusive_scan(mine, sh, &total);
            for (int k = 0; k < per; ++k)
                for (int32_t m = 0; m < sm[k0 + k]; ++m) pos[o++] = (int32_t)(v0 + k0 + k);
            out += (int64_t)total;
            __syncthreads();
        }
    }
}

}  // namespace
}  // namespace g2v

using namespace g2v;

extern "C" int g2v_cbow_epoch_order(const int32_t *tr, int64_t n, uint64_t seed, int32_t epoch, int64_t rank,
                                    int64_t world, int32_t *out, void *stream) {
    G2V_REQUIRE(n >= 0 && n <= INT32_MAX && epoch >= 0 && world >= 1 && rank >= 0 && rank < world,
                "g2v_cbow_epoch_order: bad sizes (n=%lld epoch=%d rank=%lld world=%lld)", (long long)n, epoch,
                (long long)rank, (long long)world);
    const int64_t n_loc = rank < n ? (n - rank + world - 1) / world : 0;
    if (n_loc == 0) return 0;
    G2V_REQUIRE(tr && out, "g2v_cbow_epoch_order: null pointer");
    epoch_order_kernel<<<(unsigned)((n_loc + 255) / 256), 256, 0, (cudaStream_t)stream>>>(tr, n, seed, (uint32_t)epoch,
                                                                                           rank, world, n_loc, out);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" size_t g2v_cbow_batch_plan_workspace_bytes(int64_t n_win, int64_t nnz, int64_t B, int32_t V) {
    if (n_win < 0 || nnz < 0 || B < 1 || V < 1) return 0;
    return plan_geometry(n_win, nnz, B, V).bytes;
}

extern "C" int g2v_cbow_batch_plan(const int32_t *rowptr, const int32_t *gene, const int32_t *win, int64_t n_win,
                                   int64_t nnz, int64_t B, int32_t V, int32_t *rows, int32_t *segptr, int32_t *pos,
                                   int32_t *batch_rowptr, void *workspace, void *stream) {
    G2V_REQUIRE(n_win >= 0 && n_win <= INT32_MAX && nnz >= 0 && nnz < INT32_MAX && B >= 1 && V >= 1,
                "g2v_cbow_batch_plan: bad sizes (n_win=%lld nnz=%lld B=%lld V=%d)", (long long)n_win, (long long)nnz,
                (long long)B, V);
    if (n_win == 0) return 0;
    G2V_REQUIRE(rowptr && gene && win && rows && segptr && pos && batch_rowptr && workspace,
                "g2v_cbow_batch_plan: null pointer");
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    const PlanGeometry g = plan_geometry(n_win, nnz, B, V);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = static_cast<char *>(workspace);
    int64_t *hdr = reinterpret_cast<int64_t *>(ws);
    int32_t *long_list = reinterpret_cast<int32_t *>(ws + g.off_long);
    uint64_t *toff = reinterpret_cast<uint64_t *>(ws + g.off_toff);
    int32_t *cnt = reinterpret_cast<int32_t *>(ws + g.off_cnt);
    int32_t *tmp = reinterpret_cast<int32_t *>(ws + g.off_tmp);
    G2V_CUDA_OK(cudaMemsetAsync(hdr, 0, kHdr * sizeof(int64_t), st));
    const unsigned sort_grid = (unsigned)dp.sm_count * 8;
    int launches = 0;
    for (int64_t b0 = 0; b0 < g.n_b; b0 += g.K) {
        const int64_t b1 = std::min(b0 + g.K, g.n_b);
        const int64_t w0 = b0 * B, w1 = std::min(b1 * B, n_win);
        const int64_t n_used = (b1 - b0) * (int64_t)V, tiles = (n_used + kTile - 1) / kTile;
        const unsigned wgrid = (unsigned)((w1 - w0 + kPlanThreads / 32 - 1) / (kPlanThreads / 32));
        G2V_CUDA_OK(cudaMemsetAsync(cnt, 0, (size_t)tiles * kTile * sizeof(int32_t), st));
        plan_windows_kernel<false><<<wgrid, kPlanThreads, 0, st>>>(rowptr, gene, win, w0, w1, B, b0, V, cnt, tmp, hdr);
        plan_tile_sums_kernel<<<(unsigned)tiles, kPlanThreads, 0, st>>>(cnt, toff);
        plan_tile_scan_kernel<<<1, kPlanThreads, 0, st>>>(toff, tiles, nnz, b1, g.n_b, segptr, batch_rowptr, hdr);
        plan_emit_kernel<<<(unsigned)tiles, kPlanThreads, 0, st>>>(cnt, toff, n_used, V, b0, rows, segptr, batch_rowptr,
                                                                   hdr);
        plan_windows_kernel<true><<<wgrid, kPlanThreads, 0, st>>>(rowptr, gene, win, w0, w1, B, b0, V, cnt, tmp, hdr);
        plan_sort_short_kernel<<<sort_grid, kPlanThreads, 0, st>>>(segptr, tmp, pos, long_list, hdr);
        plan_sort_long_kernel<<<sort_grid, kPlanThreads, 0, st>>>(segptr, tmp, pos, long_list, B, hdr);
        G2V_CUDA_OK(cudaGetLastError());
        launches += 7;
    }
    count_launch(launches);
    return 0;
}
