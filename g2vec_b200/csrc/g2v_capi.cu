// g2v_capi.cu -- error plumbing, device facts and the curand cross-check hook of the C ABI.
#include <curand_kernel.h>
#include <stdarg.h>

#include <atomic>

#include "g2v_common.cuh"

namespace g2v {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static thread_local const int32_t *g_skip = nullptr;
const int32_t *loop_skip_flag() { return g_skip; }
void set_loop_skip_flag(const int32_t *p) { g_skip = p; }
static thread_local const int32_t *g_carry = nullptr;
const int32_t *loop_carry_flag() { return g_carry; }
void set_loop_carry_flag(const int32_t *p) { g_carry = p; }

int device_props(DeviceProps *out) {
    static thread_local int cached_dev = -1;
    static thread_local DeviceProps cached;
    int dev = -1;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        set_error("no usable CUDA device: %s (there is no CPU fallback)", cudaGetErrorString(e));
        return 1;
    }
    if (dev != cached_dev) {
        int l2 = 0;
        if ((e = cudaDeviceGetAttribute(&cached.sm_count, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess ||
            (e = cudaDeviceGetAttribute(&cached.cc_major, cudaDevAttrComputeCapabilityMajor, dev)) != cudaSuccess ||
            (e = cudaDeviceGetAttribute(&cached.cc_minor, cudaDevAttrComputeCapabilityMinor, dev)) != cudaSuccess ||
            (e = cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev)) != cudaSuccess ||
            (e = cudaDeviceGetAttribute(&cached.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)) != cudaSuccess) {
            set_error("cudaDeviceGetAttribute failed: %s", cudaGetErrorString(e));
            return 1;
        }
        cached.l2_bytes = l2;
        cached_dev = dev;
    }
    *out = cached;
    return 0;
}

__global__ void curand_draws_kernel(uint64_t seed, uint64_t subseq, int32_t n, uint64_t *out) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        curandStatePhilox4_32_10_t st;
        curand_init(seed, subseq, 0, &st);
        for (int i = 0; i < n; ++i) {
            uint32_t lo = curand(&st);
            uint32_t hi = curand(&st);
            out[i] = ((uint64_t)hi << 32) | lo;
        }
    }
}

// Measurement hook (bench.py): the rate at which one warp per 32 row ids can (mode 0) read rows of a [V, D]
// float table with one LDG.128 per lane per 512 bytes, or (mode 1) add a constant row into them with
// red.global.add.v4.f32 -- the two memory operations of the CBOW kernels with the arithmetic removed.  On a table
// that fits the L2 this is the L2 / L1TEX ceiling the fused kernel is compared with.
template <int MODE, int VEC>
__global__ void __launch_bounds__(256)
l2_rows_kernel(const float *__restrict__ table, float *__restrict__ grad, const int32_t *__restrict__ idx, int64_t n_idx,
               float *__restrict__ sink) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
    constexpr int D4 = VEC * 32, UNR = 8 / VEC;          // 8 float4 in flight per lane, as in cbow_rows_kernel
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 one = make_float4(1e-9f, 1e-9f, 1e-9f, 1e-9f);
    for (int64_t base = warp * 32; base < n_idx; base += nwarps * 32) {
        const int cnt = (int)min((int64_t)32, n_idx - base);
        const int32_t g = lane < cnt ? __ldg(idx + base + lane) : 0;
        for (int k = 0; k < cnt; k += UNR) {
            float4 r[UNR][VEC];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const int32_t gk = __shfl_sync(0xffffffffu, g, (k + u) & 31);
#pragma unroll
                for (int v = 0; v < VEC; ++v) {
                    if (MODE == 0) {
                        r[u][v] = (k + u < cnt) ? __ldg(reinterpret_cast<const float4 *>(table) + (size_t)gk * D4 + v * 32 + lane)
                                                : make_float4(0.f, 0.f, 0.f, 0.f);
                    } else if (k + u < cnt) {
                        float *dst = grad + ((size_t)gk * D4 + v * 32 + lane) * 4;
                        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(one.x), "f"(one.y),
                                     "f"(one.z), "f"(one.w) : "memory");
                    }
                }
            }
            if (MODE == 0) {
#pragma unroll
                for (int u = 0; u < UNR; ++u)
#pragma unroll
                    for (int v = 0; v < VEC; ++v) { acc.x += r[u][v].x; acc.y += r[u][v].y; acc.z += r[u][v].z; acc.w += r[u][v].w; }
            }
        }
    }
    if (MODE == 0 && sink) sink[(warp * 32 + lane) & 1023] = acc.x + acc.y + acc.z + acc.w;
}

}  // namespace g2v

using namespace g2v;

extern "C" int g2v_test_l2_rows(const float *table, float *grad, const int32_t *idx, int64_t n_idx, int32_t D,
                                int32_t mode, float *sink, void *stream) {
    G2V_REQUIRE(idx && n_idx >= 0 && D > 0 && D % 128 == 0 && (mode == 0 ? (table && sink) : (grad != nullptr)),
                "g2v_test_l2_rows: bad arguments");
    if (n_idx == 0) return 0;
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    G2V_REQUIRE(D == 128 || D == 256 || D == 512, "g2v_test_l2_rows: D must be 128, 256 or 512 (got %d)", D);
    const int grid = dp.sm_count * 8;
    cudaStream_t st = (cudaStream_t)stream;
#define G2V_L2(VEC)                                                                                  \
    {                                                                                                \
        if (mode == 0) l2_rows_kernel<0, VEC><<<grid, 256, 0, st>>>(table, grad, idx, n_idx, sink);  \
        else l2_rows_kernel<1, VEC><<<grid, 256, 0, st>>>(table, grad, idx, n_idx, sink);            \
    }
    if (D == 128) G2V_L2(1) else if (D == 256) G2V_L2(2) else G2V_L2(4)
#undef G2V_L2
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_abi_version(void) { return G2V_ABI_VERSION; }
extern "C" const char *g2v_last_error(void) { return g_err; }
extern "C" int64_t g2v_launch_count(void) { return g_launches.load(); }

extern "C" int g2v_device_info(int32_t *sm_count, int32_t *cc_major, int32_t *cc_minor, int64_t *l2_bytes) {
    DeviceProps dp;
    if (device_props(&dp)) return 1;
    if (sm_count) *sm_count = dp.sm_count;
    if (cc_major) *cc_major = dp.cc_major;
    if (cc_minor) *cc_minor = dp.cc_minor;
    if (l2_bytes) *l2_bytes = dp.l2_bytes;
    return 0;
}

extern "C" int g2v_test_curand_draws(uint64_t seed, uint64_t subsequence, int32_t n, uint64_t *out_dev,
                                     void *stream) {
    G2V_REQUIRE(n >= 0 && out_dev, "g2v_test_curand_draws: bad arguments");
    if (n == 0) return 0;
    curand_draws_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(seed, subsequence, n, out_dev);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
