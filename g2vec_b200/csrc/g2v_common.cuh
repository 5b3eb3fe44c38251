// g2v_common.cuh -- shared device/host helpers of libg2vec_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "g2vec_b200.h"

namespace g2v {

// ---- error plumbing (C ABI: no exceptions, thread-local message) -----------------------
void set_error(const char *fmt, ...);
void count_launch(int n = 1);

#define G2V_CUDA_OK(expr)                                                                   \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            g2v::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                           __LINE__);                                                       \
            return 1;                                                                       \
        }                                                                                   \
    } while (0)

#define G2V_REQUIRE(cond, ...)          \
    do {                                \
        if (!(cond)) {                  \
            g2v::set_error(__VA_ARGS__); \
            return 2;                   \
        }                               \
    } while (0)

// Device-side loop control (g2v_cbow_loop_*): when a training loop is driven from a CUDA graph, every kernel of a
// step takes the address of the loop's `stopped` word and returns at once if it is set, so that the steps that
// follow the early stop (G2Vec.py:276-279) inside an already enqueued graph are no-ops.
void set_loop_skip_flag(const int32_t *p);
const int32_t *loop_skip_flag();   // thread-local, set by g2v_cbow_loop_attach (NULL = no loop control)
#define G2V_SKIP_IF_STOPPED(skip) \
    do { if ((skip) != nullptr && *reinterpret_cast<const volatile int32_t *>(skip) != 0) return; } while (0)

struct DeviceProps {
    int sm_count;
    int cc_major, cc_minor;
    long long l2_bytes;
    int max_smem_optin;
};
int device_props(DeviceProps *out);  // cached per current device; 0 on success

// ---- Philox4x32-10, curand-compatible (curand_philox4x32_x.h) ---------------------------
__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2,
                                                       uint32_t c3, uint32_t k0, uint32_t k1,
                                                       uint32_t out[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
#ifdef __CUDA_ARCH__
        uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
#else
        uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
#endif
        uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;   // the bump after round 10 is unused
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// 64-bit draw s of (seed, subsequence): words 2s (low) and 2s+1 (high) of the stream whose
// word k lives in counter (k/4, 0, subseq lo, subseq hi)  [curand_init(seed, subseq, 0)].
__host__ __device__ __forceinline__ uint64_t draw64(uint64_t seed, uint64_t subseq, uint32_t s) {
    uint32_t w[4];
    philox4x32_10(s >> 1, 0u, (uint32_t)subseq, (uint32_t)(subseq >> 32), (uint32_t)seed,
                  (uint32_t)(seed >> 32), w);
    return (s & 1u) ? (((uint64_t)w[3] << 32) | w[2]) : (((uint64_t)w[1] << 32) | w[0]);
}

// ---- canonical path rows (G2Vec.py:345 tuple(sorted(path))): padding value and the 64-bit row key ------
// key = finish(sum over sorted positions i of term(node_i, i)); equal rows have equal keys, the converse is
// never assumed (g2v_paths.cu compares rows in full).
constexpr int32_t kPathPad = 0x7fffffff;
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {      // splitmix64 finaliser
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27; x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}
__host__ __device__ __forceinline__ uint64_t path_key_term(int32_t v, int i) {
    return mix64(((uint64_t)(uint32_t)v << 20) ^ (uint64_t)(i + 1) * 0x9e3779b97f4a7c15ull);
}
__host__ __device__ __forceinline__ uint64_t path_key_finish(uint64_t h) {
    return mix64(h) >> 1;                                              // 63 bits: non-negative as int64
}

// ---- warp helpers ------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ uint32_t warp_inclusive_scan_u32(uint32_t v, int lane) {
    (void)lane;
    // shfl.up's own predicate output says whether the source lane exists: SHFL.UP P, ... ; @P IADD -- two
    // instructions per stage instead of shuffle + compare + select + add
#pragma unroll
    for (int o = 1; o < 32; o <<= 1)
        asm volatile("{ .reg .pred p; .reg .u32 t; shfl.sync.up.b32 t|p, %0, %1, 0, 0xffffffff; @p add.u32 %0, %0, t; }"
                     : "+r"(v) : "r"(o));
    return v;
}

// Segmented sum over the transposed incidence of a window list (CSC over list positions): the sum of
// vals[pos[j]] for j in [b, e), returned in every lane.  Fixed lane assignment and shuffle tree, so the result
// is the same bits from run to run (no floating-point atomics).  Used by the CBOW backward passes that reduce a
// per-window scalar dO into a per-gene coefficient (g2v_cbow.cu, g2v_cbow_rank1.cu).
__device__ __forceinline__ float csc_segment_sum(const int32_t *__restrict__ pos, const float *__restrict__ vals,
                                                 int32_t b, int32_t e, int lane) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int32_t j = b + lane;
    for (; j + 96 < e; j += 128) {
        a0 += __ldg(vals + __ldg(pos + j));      a1 += __ldg(vals + __ldg(pos + j + 32));
        a2 += __ldg(vals + __ldg(pos + j + 64)); a3 += __ldg(vals + __ldg(pos + j + 96));
    }
    for (; j < e; j += 32) a0 += __ldg(vals + __ldg(pos + j));
    return warp_sum((a0 + a1) + (a2 + a3));
}

}  // namespace g2v
