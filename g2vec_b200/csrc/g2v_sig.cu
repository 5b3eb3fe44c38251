// g2v_sig.cu -- cross-validated prediction of the good / poor label from a gene signature (DESIGN.md §4.29).
//   sig_folds_kernel  one warp per (repeat, class): the class's samples in ascending order, Fisher-Yates shuffled as
//                     perm_labels_kernel does (Philox subsequence 2^61 + 2k + c), position t -> fold t mod F.
//   sig_draw_kernel   one thread per random signature: Floyd's sampling of p of the G genes (subsequence
//                     2^61 + 2^40 + r), kept sorted by insertion in the output row.
//   sig_fit_kernel    one CTA per fit (signature, repeat, fold), the K F fits of a signature in adjacent CTAs: the
//                     training fold's standardisation, then damped Newton on the ridge logistic loss entirely on the
//                     device.  Each iteration streams the samples in tiles of 32 through shared memory (Z, and W Z),
//                     accumulates the lower triangle of H = Z^T W Z in 8 x 8 tiles with FP64 mma.sync m8n8k4 (DMMA),
//                     the gradient alongside; Cholesky and the two triangular solves run in shared memory.  The
//                     Armijo trials re-stream the samples for the loss only.  The test fold's logits go out last.
//   sig_auc_kernel    one CTA per fit: the test fold's scores split by label into shared memory, then exact integer
//                     counts of the (positive, negative) pairs ordered and tied, and of the correct predictions.
// Every floating-point sum is in a fixed order (per-thread chains, xor shuffle trees, fixed accumulator ownership);
// the only atomics are integer ones, so the results are the same bits whatever the grid or the chunking.
#include "g2v_fit.cuh"

namespace g2v {

// ---- folds --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32)
sig_folds_kernel(const uint8_t *__restrict__ y, int32_t n, int32_t F, uint64_t seed, int8_t *__restrict__ fold) {
    extern __shared__ uint16_t idx[];                  // [n]: the class's samples, then their shuffle
    __shared__ uint32_t js[32];
    const int lane = threadIdx.x;
    const int k = blockIdx.x >> 1, c = blockIdx.x & 1;
    int m = 0;
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool in = i < n && y[i] == c;
        const uint32_t bal = __ballot_sync(0xffffffffu, in);
        if (in) idx[m + __popc(bal & ((1u << lane) - 1u))] = (uint16_t)i;
        m += __popc(bal);
    }
    __syncwarp();
    const uint64_t subseq = (1ull << 61) + 2ull * (uint64_t)k + (uint64_t)c;
    for (int base = 0; base < m - 1; base += 32) {
        const int s = base + lane;                     // draw s swaps position m-1-s
        js[lane] = s < m - 1 ? (uint32_t)__umul64hi(draw64(seed, subseq, (uint32_t)s), (uint64_t)(m - s)) : 0u;
        __syncwarp();
        if (lane == 0) {
            const int cnt = min(32, m - 1 - base);
            for (int t = 0; t < cnt; ++t) {
                const int i = m - 1 - (base + t);
                const uint16_t x = idx[i];
                idx[i] = idx[js[t]];
                idx[js[t]] = x;
            }
        }
        __syncwarp();
    }
    for (int t = lane; t < m; t += 32) fold[(int64_t)k * n + idx[t]] = (int8_t)(t % F);
}

// ---- random signatures --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
sig_draw_kernel(int32_t G, int32_t p, uint64_t seed, int64_t r_begin, int64_t count, int32_t *__restrict__ genes) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= count) return;
    const uint64_t subseq = (1ull << 61) + (1ull << 40) + (uint64_t)(r_begin + q);
    int32_t *row = genes + q * p;                      // written and read by this thread only
    for (int t = 0; t < p; ++t) {
        const uint32_t j = (uint32_t)(G - p + t);
        const uint32_t v = (uint32_t)__umul64hi(draw64(seed, subseq, (uint32_t)t), (uint64_t)j + 1);
        int lo = 0, hi = t;                            // first position with row[pos] >= v
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((uint32_t)row[mid] < v) lo = mid + 1; else hi = mid;
        }
        if (lo < t && (uint32_t)row[lo] == v) {
            row[t] = (int32_t)j;                       // j exceeds every earlier pick: it goes last
        } else {
            for (int s = t; s > lo; --s) row[s] = row[s - 1];
            row[lo] = (int32_t)v;
        }
    }
}

// ---- fits (the shared Newton machinery is in g2v_fit.cuh) ---------------------------------------------------
__host__ __device__ __forceinline__ size_t fit_smem_doubles(int p) {
    const int P = fit_pad(p), P1 = p + 1;
    const int big = 2 * P * kTS > tri(P1) ? 2 * P * kTS : tri(P1);
    return (size_t)big + 7 * (size_t)P;
}

// Per-CTA scratch of a fit: one tile's weights, residuals and loss terms.
__shared__ double fit_w[kTileS], fit_r[kTileS], fit_lt[kTileS];

enum { kPassGram = 0, kPassLoss = 1, kPassScore = 2 };

// One pass over the samples at coefficients b [P1].  kPassGram: returns the loss and leaves g [P1] and the packed
// lower triangle of H in Hp (ridge included); kPassLoss: returns the loss; kPassScore: writes the test fold's logits.
template <int MODE>
__device__ double fit_pass(const Fit &c, const double *b, double *score_row) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    double acc[kTilesPerWarp][2];
    if (MODE == kPassGram) {
#pragma unroll
        for (int q = 0; q < kTilesPerWarp; ++q) acc[q][0] = acc[q][1] = 0.0;
    }
    double gacc = 0.0, lacc = 0.0;
    for (int i0 = 0; i0 < c.n; i0 += kTileS) {
        {
            const int i = i0 + lane;
            const bool in = i < c.n && (MODE == kPassScore ? c.fold[i] == c.f : c.fold[i] != c.f);
            for (int j = warp; j < c.P; j += kFitWarps) {
                double z = 0.0;
                if (in && j <= c.p)
                    z = j == 0 ? 1.0 : (__ldg(c.X + (int64_t)__ldg(c.genes + j - 1) * c.n_pad + i) - c.mu[j]) / c.sd[j];
                c.Zs[j * kTS + lane] = z;
            }
        }
        __syncthreads();
        {
            const int s = tid / kPerSample, part = tid % kPerSample;
            double e = 0.0;
            for (int j = part; j < c.P1; j += kPerSample) e = fma(c.Zs[j * kTS + s], b[j], e);
#pragma unroll
            for (int o = kPerSample / 2; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
            if (part == 0) {
                const int i = i0 + s;
                const bool in = i < c.n && (MODE == kPassScore ? c.fold[i] == c.f : c.fold[i] != c.f);
                if (MODE == kPassScore) {
                    if (in) score_row[i] = e;
                } else {
                    double wv = 0.0, rv = 0.0, lv = 0.0;
                    if (in) {
                        const double yv = (double)c.y[i];
                        const double ex = exp(-fabs(e));               // softplus(e) = max(e, 0) + log1p(e^-|e|)
                        const double den = 1.0 + ex;
                        lv = fmax(e, 0.0) + log1p(ex) - yv * e;
                        const double sg = e >= 0.0 ? 1.0 / den : ex / den;
                        wv = ex / (den * den);                         // sigma (1 - sigma)
                        rv = sg - yv;
                    }
                    fit_w[s] = wv; fit_r[s] = rv; fit_lt[s] = lv;
                }
            }
        }
        __syncthreads();
        if (MODE == kPassScore) continue;
        if (MODE == kPassGram) {
            for (int j = warp; j < c.P; j += kFitWarps) c.WZs[j * kTS + lane] = fit_w[lane] * c.Zs[j * kTS + lane];
            if (tid < c.P1)
#pragma unroll 4
                for (int t = 0; t < kTileS; ++t) gacc = fma(c.Zs[tid * kTS + t], fit_r[t], gacc);
        }
        if (tid == 0)
#pragma unroll 4
            for (int t = 0; t < kTileS; ++t) lacc += fit_lt[t];
        if (MODE == kPassGram) {
            __syncthreads();
#pragma unroll
            for (int q = 0; q < kTilesPerWarp; ++q) {
                const int tile = warp + q * kFitWarps;
                if (tile < c.n_tiles) {
                    const int IJ = fit_tiles[tile];
                    const double *ap = c.WZs + ((IJ >> 8) * 8 + gid) * kTS + tig;
                    const double *bp = c.Zs + ((IJ & 255) * 8 + gid) * kTS + tig;
#pragma unroll 2
                    for (int kk = 0; kk < kTileS; kk += 4) dmma_8x8x4(acc[q], ap[kk], bp[kk]);
                }
            }
        }
        __syncthreads();                               // the tile is consumed before the next one is written
    }
    if (MODE == kPassScore) return 0.0;
    if (MODE == kPassGram) {
#pragma unroll
        for (int q = 0; q < kTilesPerWarp; ++q) {      // accumulator e: row gid, column 2 tig + e of tile (I, J)
            const int tile = warp + q * kFitWarps;
            if (tile < c.n_tiles) {
                const int IJ = fit_tiles[tile];
                const int row = (IJ >> 8) * 8 + gid;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = (IJ & 255) * 8 + 2 * tig + e;
                    if (row < c.P1 && col <= row) c.Hp[tri(row) + col] = acc[q][e] + (row == col && row > 0 ? 1.0 : 0.0);
                }
            }
        }
        if (tid < c.P1) c.g[tid] = gacc + (tid > 0 ? b[tid] : 0.0);
    }
    if (tid == 0) {
        double pen = 0.0;
        for (int j = 1; j < c.P1; ++j) pen = fma(b[j], b[j], pen);
        fit_scal[0] = lacc + 0.5 * pen;
    }
    __syncthreads();
    return fit_scal[0];
}

struct LogisticModel {
    const Fit &c;
    __device__ double gram(const double *b) { return fit_pass<kPassGram>(c, b, nullptr); }
    __device__ double loss(const double *b) { return fit_pass<kPassLoss>(c, b, nullptr); }
};

__global__ void __launch_bounds__(kFitThreads, 1)
sig_fit_kernel(const double *__restrict__ X, int64_t n_pad, int32_t n, const uint8_t *__restrict__ y,
               const int8_t *__restrict__ fold, int32_t K, int32_t F, const int32_t *__restrict__ genes, int32_t p,
               double *__restrict__ scores, int32_t *__restrict__ n_iter, uint8_t *__restrict__ converged,
               double *__restrict__ beta, int32_t beta_rows) {
    extern __shared__ double sm[];
    const int64_t fit = blockIdx.x;
    const int64_t s = fit / ((int64_t)K * F);
    const int k = (int)((fit / F) % K), f = (int)(fit % F);
    Fit c;
    c.X = X; c.n_pad = n_pad; c.n = n; c.p = p; c.P1 = p + 1; c.P = fit_pad(p); c.f = f;
    c.y = y; c.fold = fold + (int64_t)k * n; c.genes = genes + s * p;
    const int nt = c.P / 8;
    c.n_tiles = nt * (nt + 1) / 2;
    const int big = 2 * c.P * kTS > tri(c.P1) ? 2 * c.P * kTS : tri(c.P1);
    c.Zs = sm; c.WZs = sm + c.P * kTS; c.Hp = sm;
    double *bt = sm + big, *bc = bt + c.P, *d = bc + c.P, *tmp = d + c.P;
    c.mu = tmp + c.P; c.sd = c.mu + c.P; c.g = c.sd + c.P;
    fit_init_tiles(c.n_tiles);
    for (int j = threadIdx.x; j < c.P; j += kFitThreads) bt[j] = 0.0;
    fit_standardise(c);                                // ends with a barrier
    LogisticModel model{c};
    int it;
    bool conv;
    fit_newton(c, model, bt, bc, d, tmp, it, conv);
    fit_pass<kPassScore>(c, bt, scores + (s * K + k) * (int64_t)n);
    if (threadIdx.x == 0) { n_iter[fit] = it; converged[fit] = conv ? 1 : 0; }
    if (s < beta_rows)
        for (int j = threadIdx.x; j < c.P1; j += kFitThreads) beta[fit * c.P1 + j] = bt[j];
}

// ---- AUC and accuracy ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
sig_auc_kernel(const double *__restrict__ scores, const uint8_t *__restrict__ y, const int8_t *__restrict__ fold,
               int32_t n, int32_t K, int32_t F, int32_t cap, double *__restrict__ auc, double *__restrict__ acc) {
    extern __shared__ double buf[];                    // [cap]: positives from the front, negatives from the back
    __shared__ unsigned int n_pos, n_neg, n_ok;
    __shared__ unsigned long long n_gt, n_eq;
    const int64_t fit = blockIdx.x;
    const int64_t s = fit / ((int64_t)K * F);
    const int k = (int)((fit / F) % K), f = (int)(fit % F);
    const double *sr = scores + (s * K + k) * (int64_t)n;
    const int8_t *fr = fold + (int64_t)k * n;
    if (threadIdx.x == 0) { n_pos = n_neg = n_ok = 0u; n_gt = n_eq = 0ull; }
    __syncthreads();
    unsigned int ok = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        if (fr[i] == f) {
            const double v = sr[i];
            const bool pos = y[i] != 0;
            ok += (v > 0.0) == pos;
            const unsigned int slot = atomicAdd(pos ? &n_pos : &n_neg, 1u);
            if (slot < (unsigned)cap) buf[pos ? slot : cap - 1 - slot] = v;
        }
    if (ok) atomicAdd(&n_ok, ok);
    __syncthreads();
    const unsigned int np = n_pos, nn = n_neg;
    if (np + nn > (unsigned)cap) {                     // not a fold the caller sized: no result
        if (threadIdx.x == 0) { auc[fit] = __longlong_as_double(0x7ff8000000000000ll); acc[fit] = auc[fit]; }
        return;
    }
    unsigned long long gt = 0, eq = 0;
    for (unsigned int a = threadIdx.x; a < np; a += blockDim.x) {
        const double v = buf[a];
        unsigned int g1 = 0, e1 = 0;
        for (unsigned int b = 0; b < nn; ++b) {
            const double u = buf[cap - 1 - b];
            g1 += v > u; e1 += v == u;
        }
        gt += g1; eq += e1;
    }
    if (gt) atomicAdd(&n_gt, gt);
    if (eq) atomicAdd(&n_eq, eq);
    __syncthreads();
    if (threadIdx.x == 0) {
        auc[fit] = (double)(2ull * n_gt + n_eq) / (2.0 * (double)np * (double)nn);
        acc[fit] = (double)n_ok / (double)(np + nn);
    }
}

}  // namespace g2v

using namespace g2v;

extern "C" int g2v_sig_folds(const uint8_t *y, int32_t n, int32_t K, int32_t F, uint64_t seed, int8_t *fold,
                             void *stream) {
    G2V_REQUIRE(y && fold, "g2v_sig_folds: null pointer");
    G2V_REQUIRE(n >= 3 && n <= G2V_SIG_MAX_SAMPLES, "g2v_sig_folds: n = %d samples, must be in [3, %d]", (int)n,
                G2V_SIG_MAX_SAMPLES);
    G2V_REQUIRE(K >= 1 && K <= G2V_SIG_MAX_REPEATS, "g2v_sig_folds: K = %d repeats, must be in [1, %d]", (int)K,
                G2V_SIG_MAX_REPEATS);
    G2V_REQUIRE(F >= 2 && F <= G2V_SIG_MAX_FOLDS && F <= n / 2, "g2v_sig_folds: F = %d folds, must be in [2, min(%d, "
                "n / 2)]", (int)F, G2V_SIG_MAX_FOLDS);
    const size_t smem = (size_t)n * sizeof(uint16_t);
    if (smem > 48 * 1024)
        G2V_CUDA_OK(cudaFuncSetAttribute(sig_folds_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    sig_folds_kernel<<<(unsigned)(2 * K), 32, smem, (cudaStream_t)stream>>>(y, n, F, seed, fold);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_sig_draw(int32_t G, int32_t p, uint64_t seed, int64_t r_begin, int64_t count, int32_t *genes,
                            void *stream) {
    G2V_REQUIRE(genes, "g2v_sig_draw: null pointer");
    G2V_REQUIRE(p >= 1 && p <= G2V_SIG_MAX_SIZE && p <= G, "g2v_sig_draw: p = %d genes of G = %d, must be in [1, "
                "min(%d, G)]", (int)p, (int)G, G2V_SIG_MAX_SIZE);
    G2V_REQUIRE(r_begin >= 1 && count >= 1 && r_begin + count - 1 <= G2V_SIG_MAX_RANDOM,
                "g2v_sig_draw: signatures %lld .. %lld out of [1, %d]", (long long)r_begin,
                (long long)(r_begin + count - 1), G2V_SIG_MAX_RANDOM);
    sig_draw_kernel<<<(unsigned)((count + 127) / 128), 128, 0, (cudaStream_t)stream>>>(G, p, seed, r_begin, count,
                                                                                          genes);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

#define G2V_SIG_CHECK_FITS(fn, n, K, F, n_sig)                                                                      \
    do {                                                                                                           \
        G2V_REQUIRE((n) >= 3 && (n) <= G2V_SIG_MAX_SAMPLES, fn ": n = %d samples, must be in [3, %d]", (int)(n),    \
                    G2V_SIG_MAX_SAMPLES);                                                                          \
        G2V_REQUIRE((K) >= 1 && (K) <= G2V_SIG_MAX_REPEATS && (F) >= 2 && (F) <= G2V_SIG_MAX_FOLDS,                 \
                    fn ": K = %d repeats and F = %d folds, must be in [1, %d] and [2, %d]", (int)(K), (int)(F),    \
                    G2V_SIG_MAX_REPEATS, G2V_SIG_MAX_FOLDS);                                                       \
        G2V_REQUIRE((n_sig) >= 1 && (int64_t)(n_sig) * (K) * (F) <= G2V_SIG_MAX_FITS,                               \
                    fn ": %d signatures x %d repeats x %d folds, must be 1 .. %d fits", (int)(n_sig), (int)(K),    \
                    (int)(F), G2V_SIG_MAX_FITS);                                                                   \
    } while (0)

extern "C" size_t g2v_sig_fit_smem_bytes(int32_t p) {
    if (p < 1 || p > G2V_SIG_MAX_SIZE) return 0;
    return fit_smem_doubles(p) * sizeof(double);
}

extern "C" int g2v_sig_fit(const double *X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *y, const int8_t *fold,
                           int32_t K, int32_t F, const int32_t *genes, int32_t n_sig, int32_t p, double *scores,
                           int32_t *n_iter, uint8_t *converged, double *beta, int32_t beta_rows, void *stream) {
    G2V_REQUIRE(X && y && fold && genes && scores && n_iter && converged, "g2v_sig_fit: null pointer");
    G2V_SIG_CHECK_FITS("g2v_sig_fit", n, K, F, n_sig);
    G2V_REQUIRE(p >= 1 && p <= G2V_SIG_MAX_SIZE && p <= G, "g2v_sig_fit: p = %d genes of G = %d, must be in [1, "
                "min(%d, G)]", (int)p, (int)G, G2V_SIG_MAX_SIZE);
    G2V_REQUIRE(n_pad >= n, "g2v_sig_fit: n_pad = %lld, must be >= n = %d", (long long)n_pad, (int)n);
    G2V_REQUIRE(beta_rows >= 0 && beta_rows <= n_sig && (beta_rows == 0 || beta),
                "g2v_sig_fit: beta_rows = %d, must be in [0, %d] with beta given when > 0", (int)beta_rows, (int)n_sig);
    const size_t smem = fit_smem_doubles(p) * sizeof(double);
    G2V_CUDA_OK(cudaFuncSetAttribute(sig_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t fits = (int64_t)n_sig * K * F;
    sig_fit_kernel<<<(unsigned)fits, kFitThreads, smem, (cudaStream_t)stream>>>(
        X, n_pad, n, y, fold, K, F, genes, p, scores, n_iter, converged, beta, beta_rows);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_sig_auc(const double *scores, const uint8_t *y, const int8_t *fold, int32_t n, int32_t K, int32_t F,
                           int32_t n_sig, int32_t cap, double *auc, double *acc, void *stream) {
    G2V_REQUIRE(scores && y && fold && auc && acc, "g2v_sig_auc: null pointer");
    G2V_SIG_CHECK_FITS("g2v_sig_auc", n, K, F, n_sig);
    G2V_REQUIRE(cap >= 2 && cap <= n, "g2v_sig_auc: cap = %d, must be in [2, n = %d]", (int)cap, (int)n);
    const size_t smem = (size_t)cap * sizeof(double);
    if (smem > 48 * 1024)
        G2V_CUDA_OK(cudaFuncSetAttribute(sig_auc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t fits = (int64_t)n_sig * K * F;
    sig_auc_kernel<<<(unsigned)fits, 256, smem, (cudaStream_t)stream>>>(scores, y, fold, n, K, F, cap, auc, acc);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
