// g2v_cox.cu -- cross-validated survival prediction from a gene signature: ridge Cox regression (DESIGN.md §4.33).
// Samples are in time positions: descending time, ties by sample index, so a time group is a run of positions and
// the risk set of a group is every position up to its end.  flags[pos]: bit 0 event, bit 1 last position of its group.
//   cox_fit_kernel   one CTA per fit (signature, repeat, fold), the K F fits of a signature in adjacent CTAs: the
//                    training fold's standardisation, then damped Newton (g2v_fit.cuh) on the Breslow negative log
//                    partial likelihood plus 1/2 |beta|^2.  A Gram pass streams the training samples twice in tiles of
//                    32 positions.  Pass 1, descending time: the risk-set sums S0 and S1 under a running shift (online
//                    softmax), l_k = log S0_k at every group end, m_k = S1_k / S0_k, the loss and the gradient, and
//                    the tiles of -sum d_k m_k m_k^T.  Pass 2, ascending time: the weights omega_i of sum omega_i z_i
//                    z_i^T from a scaled recurrence over the l_k.  Both Grams go into one set of FP64 mma.sync m8n8k4
//                    accumulators.  The Armijo trials run pass 1 for the loss only.  The test fold's eta goes out last.
//   cox_conc_kernel  one CTA per fit: the test fold staged in shared memory (or read from global memory when it does
//                    not fit), then exact integer counts of Harrell's comparable, concordant and tied pairs.
// Every floating-point sum is in a fixed order; the only atomics are integer ones, so the results are the same bits
// whatever the grid or the chunking.
#include "g2v_fit.cuh"

namespace g2v {

// The fit's shared memory: the tiles (Z, M and -d M in pass 1, Z and omega Z in pass 2; H after a pass), then
// bt, bc, d, tmp, mu, sd, g of P doubles each.
__host__ __device__ __forceinline__ size_t cox_smem_doubles(int p) {
    const int P = fit_pad(p), P1 = p + 1;
    const int big = 3 * P * kTS > tri(P1) ? 3 * P * kTS : tri(P1);
    return (size_t)big + 7 * (size_t)P;
}

// Per-CTA scratch of one tile: eta, the weights (e^{eta - M} in pass 1, omega in pass 2), the rescale factors of the
// running shift, d_k at the group ends, S0 at every position, and the training, event, end and m masks.
__shared__ double cox_eta[kTileS], cox_w[kTileS], cox_r[kTileS], cox_d[kTileS], cox_s0[kTileS];
__shared__ uint32_t cox_mask[4];

enum { kCoxGram = 0, kCoxLoss = 1, kCoxScore = 2 };

__device__ __forceinline__ uint32_t lanes_upto(int t) { return (2u << t) - 1u; }     // bits 0 .. t

// Stages the tile's z (training samples, or the test fold for kCoxScore; slot 0 and the pad rows are 0) into Zs and
// its linear predictors into cox_eta.  Ends with a barrier.
template <int MODE>
__device__ __forceinline__ void cox_stage(const Fit &c, const double *b, int i0) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    {
        const int i = i0 + lane;
        const bool in = i < c.n && (MODE == kCoxScore ? c.fold[i] == c.f : c.fold[i] != c.f);
        for (int j = warp; j < c.P; j += kFitWarps) {
            double z = 0.0;
            if (in && j >= 1 && j <= c.p)
                z = (__ldg(c.X + (int64_t)__ldg(c.genes + j - 1) * c.n_pad + i) - c.mu[j]) / c.sd[j];
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
        if (part == 0) cox_eta[s] = e;
    }
    __syncthreads();
}

// One run over the samples at coefficients b [P1].  kCoxGram: returns the loss and leaves g [P1], the packed lower
// triangle of H in Hp (ridge included) and the per-position scratch ell; kCoxLoss: returns the loss; kCoxScore:
// writes the test fold's eta into score_row.
//
// ell, written by pass 1 and read by pass 2: at a group end, l_k (NaN when the group holds no training sample); at
// the position before a group end inside the same group (never a group end itself), d_k.
template <int MODE>
__device__ double cox_pass(const Fit &c, const double *b, double *ell, double *score_row) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
    if (MODE == kCoxScore) {
        for (int i0 = 0; i0 < c.n; i0 += kTileS) {
            cox_stage<MODE>(c, b, i0);
            if (tid < kTileS && i0 + tid < c.n && c.fold[i0 + tid] == c.f) score_row[i0 + tid] = cox_eta[tid];
        }
        return 0.0;
    }
    double *Ms = c.Zs + c.P * kTS, *NMs = c.WZs;
    double acc[kTilesPerWarp][2];
    if (MODE == kCoxGram) {
#pragma unroll
        for (int q = 0; q < kTilesPerWarp; ++q) acc[q][0] = acc[q][1] = 0.0;
    }
    // warp 0's carries across tiles: the shift M, and the events and training presence of the open group; thread 0
    // carries S0 and the loss, thread j < P carries S1_j and g_j
    double M = -INFINITY, s0 = 0.0, s1 = 0.0, lacc = 0.0, gacc = 0.0;
    int d_open = 0;
    bool has_open = false;
    // ---- pass 1: descending time -------------------------------------------------------------------------------
    for (int i0 = 0; i0 < c.n; i0 += kTileS) {
        cox_stage<MODE>(c, b, i0);
        double d_lane = 0.0, l_lane = 0.0, eta = 0.0, Mt = 0.0;
        bool end = false, has = false, ev = false;
        if (warp == 0) {
            const int i = i0 + lane;
            const bool in = i < c.n && c.fold[i] != c.f;
            const uint8_t fl = i < c.n ? c.y[i] : 0;
            end = (fl & 2) != 0;
            ev = in && (fl & 1);
            eta = cox_eta[lane];
            double mx = in ? eta : -INFINITY;          // inclusive prefix max of the training eta, from the carry
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const double u = __shfl_up_sync(0xffffffffu, mx, o);
                if (lane >= o) mx = fmax(mx, u);
            }
            Mt = fmax(M, mx);
            const double up = __shfl_up_sync(0xffffffffu, Mt, 1);
            const double Mprev = lane == 0 ? M : up;
            const double r = Mt > Mprev ? exp(Mprev - Mt) : 1.0;
            const double w = in ? exp(eta - Mt) : 0.0;
            const uint32_t trm = __ballot_sync(0xffffffffu, in), evm = __ballot_sync(0xffffffffu, ev),
                           endm = __ballot_sync(0xffffffffu, end);
            const uint32_t before = endm & (lanes_upto(lane) >> 1);
            const int pe = before ? 31 - __clz(before) : -1;
            const uint32_t seg = lanes_upto(lane) & ~(pe >= 0 ? lanes_upto(pe) : 0u);   // this lane's group in tile
            const int d = __popc(evm & seg) + (pe < 0 ? d_open : 0);
            has = (trm & seg) != 0 || (pe < 0 && has_open);
            d_lane = end ? (double)d : 0.0;
            const uint32_t mm = __ballot_sync(0xffffffffu, end && d > 0);
            if (endm) {
                const uint32_t after = ~lanes_upto(31 - __clz(endm));
                d_open = __popc(evm & after);
                has_open = (trm & after) != 0;
            } else {
                d_open += __popc(evm);
                has_open = has_open || trm != 0;
            }
            M = __shfl_sync(0xffffffffu, Mt, 31);
            cox_w[lane] = w; cox_r[lane] = r; cox_d[lane] = d_lane;
            if (lane == 0) { cox_mask[0] = trm; cox_mask[1] = evm; cox_mask[2] = endm; cox_mask[3] = mm; }
            __syncwarp();
            if (lane == 0)
                for (int t = 0; t < kTileS; ++t) { s0 = fma(s0, cox_r[t], cox_w[t]); cox_s0[t] = s0; }
            __syncwarp();
            // l_k at the ends of groups with a training sample (S0 >= 1 there: the sample of the running maximum
            // entered with weight 1 and has only been rescaled since by factors that raised the shift past it)
            if (end && has) l_lane = log(cox_s0[lane]) + Mt;
            double term = (d > 0 && end ? d * l_lane : 0.0) - (ev ? eta : 0.0);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) term += __shfl_xor_sync(0xffffffffu, term, o);
            if (lane == 0) lacc += term;
        }
        if (MODE == kCoxGram) {
            __syncthreads();
            if (warp == 0 && end && i0 + lane < c.n) {
                const int i = i0 + lane;
                ell[i] = has ? l_lane : __longlong_as_double(0x7ff8000000000000ll);
                if (has && i >= 1 && !(c.y[i - 1] & 2)) ell[i - 1] = d_lane;
            }
            if (tid < c.P) {
                const uint32_t evm = cox_mask[1], mm = cox_mask[3];
                const double *zr = c.Zs + tid * kTS;
#pragma unroll 4
                for (int t = 0; t < kTileS; ++t) {
                    const double z = zr[t];
                    s1 = fma(cox_w[t], z, s1 * cox_r[t]);
                    double m = 0.0, dm = 0.0;
                    if ((mm >> t) & 1u) {
                        m = s1 / cox_s0[t];
                        dm = cox_d[t] * m;
                        gacc += dm;
                    }
                    if ((evm >> t) & 1u) gacc -= z;
                    Ms[tid * kTS + t] = m;
                    NMs[tid * kTS + t] = -dm;
                }
            }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < kTilesPerWarp; ++q) {
                const int tile = warp + q * kFitWarps;
                if (tile < c.n_tiles) {
                    const int IJ = fit_tiles[tile];
                    const double *ap = NMs + ((IJ >> 8) * 8 + gid) * kTS + tig;
                    const double *bp = Ms + ((IJ & 255) * 8 + gid) * kTS + tig;
#pragma unroll 2
                    for (int kk = 0; kk < kTileS; kk += 4) dmma_8x8x4(acc[q], ap[kk], bp[kk]);
                }
            }
        }
        __syncthreads();                               // the tile is consumed before the next one is written
    }
    if (MODE == kCoxGram) {
        // ---- pass 2: ascending time.  C = sum over the groups k' up to k of d_k' e^{l_k - l_k'}, carried as
        // C <- C e^{l_k - l_prev} + d_k over the groups with a training sample (factor <= 1), and omega_i =
        // e^{eta_i - l_k(i)} C_k(i) (first factor <= 1): 0 <= omega_i <= the training events.  Lane L takes
        // position i0 + 31 - L, so the lanes run in ascending time and the recurrence is an affine scan.
        double C = 0.0, l_open = -INFINITY;
        bool started = false;
        for (int i0 = ((c.n - 1) / kTileS) * kTileS; i0 >= 0; i0 -= kTileS) {
            cox_stage<MODE>(c, b, i0);
            if (warp == 0) {
                const int t = kTileS - 1 - lane, i = i0 + t;
                const bool in = i < c.n && c.fold[i] != c.f;
                const uint8_t fl = i < c.n ? c.y[i] : 0;
                double li = 0.0, dd = 0.0;
                bool valid = false;
                if (fl & 2) {
                    li = ell[i];
                    valid = !isnan(li);
                    if (valid) dd = i >= 1 && !(c.y[i - 1] & 2) ? ell[i - 1] : (in && (fl & 1) ? 1.0 : 0.0);
                }
                const uint32_t vm = __ballot_sync(0xffffffffu, valid);
                const uint32_t before = vm & (lanes_upto(lane) >> 1), upto = vm & lanes_upto(lane);
                const double lp = __shfl_sync(0xffffffffu, li, before ? 31 - __clz(before) : 0);
                const double lc = __shfl_sync(0xffffffffu, li, upto ? 31 - __clz(upto) : 0);
                const double l_prev = before ? lp : l_open, l_cur = upto ? lc : l_open;
                double A = valid ? (before || started ? exp(li - l_prev) : 0.0) : 1.0, B = valid ? dd : 0.0;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const double a2 = __shfl_up_sync(0xffffffffu, A, o), b2 = __shfl_up_sync(0xffffffffu, B, o);
                    if (lane >= o) { B = fma(A, b2, B); A *= a2; }
                }
                const double Ck = fma(A, C, B);
                cox_w[t] = in ? exp(cox_eta[t] - l_cur) * Ck : 0.0;
                C = __shfl_sync(0xffffffffu, Ck, 31);
                l_open = __shfl_sync(0xffffffffu, l_cur, 31);
                started = started || vm != 0;
            }
            __syncthreads();
            for (int j = warp; j < c.P; j += kFitWarps) c.WZs[j * kTS + lane] = cox_w[lane] * c.Zs[j * kTS + lane];
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
            __syncthreads();
        }
#pragma unroll
        for (int q = 0; q < kTilesPerWarp; ++q) {      // accumulator e: row gid, column 2 tig + e of tile (I, J)
            const int tile = warp + q * kFitWarps;
            if (tile < c.n_tiles) {
                const int IJ = fit_tiles[tile];
                const int row = (IJ >> 8) * 8 + gid;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = (IJ & 255) * 8 + 2 * tig + e;
                    if (row < c.P1 && col <= row) c.Hp[tri(row) + col] = acc[q][e] + (row == col ? 1.0 : 0.0);
                }
            }
        }
        if (tid < c.P1) c.g[tid] = gacc + b[tid];
    }
    if (tid == 0) {
        double pen = 0.0;
        for (int j = 1; j < c.P1; ++j) pen = fma(b[j], b[j], pen);
        fit_scal[0] = lacc + 0.5 * pen;
    }
    __syncthreads();
    return fit_scal[0];
}

struct CoxModel {
    const Fit &c;
    double *ell;
    __device__ double gram(const double *b) { return cox_pass<kCoxGram>(c, b, ell, nullptr); }
    __device__ double loss(const double *b) { return cox_pass<kCoxLoss>(c, b, ell, nullptr); }
};

__global__ void __launch_bounds__(kFitThreads, 1)
cox_fit_kernel(const double *__restrict__ X, int64_t n_pad, int32_t n, const uint8_t *__restrict__ flags,
               const int8_t *__restrict__ fold, int32_t K, int32_t F, const int32_t *__restrict__ genes, int32_t p,
               double *__restrict__ ell, double *__restrict__ scores, int32_t *__restrict__ n_iter,
               uint8_t *__restrict__ converged, double *__restrict__ beta, int32_t beta_rows) {
    extern __shared__ double sm[];
    const int64_t fit = blockIdx.x;
    const int64_t s = fit / ((int64_t)K * F);
    const int k = (int)((fit / F) % K), f = (int)(fit % F);
    Fit c;
    c.X = X; c.n_pad = n_pad; c.n = n; c.p = p; c.P1 = p + 1; c.P = fit_pad(p); c.f = f;
    c.y = flags; c.fold = fold + (int64_t)k * n; c.genes = genes + s * p;
    const int nt = c.P / 8;
    c.n_tiles = nt * (nt + 1) / 2;
    const int big = 3 * c.P * kTS > tri(c.P1) ? 3 * c.P * kTS : tri(c.P1);
    c.Zs = sm; c.WZs = sm + 2 * c.P * kTS; c.Hp = sm;
    double *bt = sm + big, *bc = bt + c.P, *d = bc + c.P, *tmp = d + c.P;
    c.mu = tmp + c.P; c.sd = c.mu + c.P; c.g = c.sd + c.P;
    fit_init_tiles(c.n_tiles);
    for (int j = threadIdx.x; j < c.P; j += kFitThreads) bt[j] = 0.0;
    fit_standardise(c);                                // ends with a barrier
    CoxModel model{c, ell + fit * (int64_t)n};
    int it;
    bool conv;
    fit_newton(c, model, bt, bc, d, tmp, it, conv);
    cox_pass<kCoxScore>(c, bt, nullptr, scores + (s * K + k) * (int64_t)n);
    if (threadIdx.x == 0) { n_iter[fit] = it; converged[fit] = conv ? 1 : 0; }
    if (s < beta_rows)
        for (int j = threadIdx.x; j < p; j += kFitThreads) beta[fit * p + j] = bt[j + 1];
}

// ---- Harrell's C ---------------------------------------------------------------------------------------------
// A pair (i, j) of the test fold is comparable when t_i < t_j (grp[i] > grp[j]) and i is an event; concordant when
// eta_i > eta_j, tied when equal.  counts [fit][3] = comparable, concordant, tied.
template <bool STAGED>
__device__ void conc_count(const double *sr, const int8_t *fr, const uint8_t *flags, const int32_t *grp, int n, int f,
                           const double *eta_s, const int32_t *key_s, int m, unsigned long long cnt[3]) {
    const int total = STAGED ? m : n;
    for (int a = threadIdx.x; a < total; a += blockDim.x) {
        int ga;
        double ea;
        if (STAGED) {
            if (!(key_s[a] & 1)) continue;
            ga = key_s[a] >> 1; ea = eta_s[a];
        } else {
            if (fr[a] != f || !(flags[a] & 1)) continue;
            ga = grp[a]; ea = sr[a];
        }
        unsigned int cmp = 0, con = 0, tie = 0;
        if (STAGED) {
            for (int b = 0; b < m; ++b) {
                const bool ok = (key_s[b] >> 1) < ga;
                const double eb = eta_s[b];
                cmp += ok; con += ok && ea > eb; tie += ok && ea == eb;
            }
        } else {
            for (int b = 0; b < a; ++b) {              // positions after a are never earlier in time
                const bool ok = fr[b] == f && grp[b] < ga;
                const double eb = sr[b];
                cmp += ok; con += ok && ea > eb; tie += ok && ea == eb;
            }
        }
        cnt[0] += cmp; cnt[1] += con; cnt[2] += tie;
    }
}

__global__ void __launch_bounds__(256)
cox_conc_kernel(const double *__restrict__ scores, const uint8_t *__restrict__ flags, const int32_t *__restrict__ grp,
                const int8_t *__restrict__ fold, int32_t n, int32_t K, int32_t F, int32_t cap,
                int64_t *__restrict__ counts) {
    extern __shared__ double eta_s[];                  // [cap] eta, then [cap] int32 keys (grp << 1) | event
    int32_t *key_s = reinterpret_cast<int32_t *>(eta_s + cap);
    __shared__ unsigned int n_test;
    __shared__ unsigned long long tot[3];
    const int64_t fit = blockIdx.x;
    const int64_t s = fit / ((int64_t)K * F);
    const int k = (int)((fit / F) % K), f = (int)(fit % F);
    const double *sr = scores + (s * K + k) * (int64_t)n;
    const int8_t *fr = fold + (int64_t)k * n;
    if (threadIdx.x == 0) { n_test = 0u; tot[0] = tot[1] = tot[2] = 0ull; }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        if (fr[i] == f) {
            const unsigned int slot = atomicAdd(&n_test, 1u);
            if (slot < (unsigned)cap) { eta_s[slot] = sr[i]; key_s[slot] = (grp[i] << 1) | (flags[i] & 1); }
        }
    __syncthreads();
    const int m = (int)n_test;
    unsigned long long cnt[3] = {0ull, 0ull, 0ull};
    if (m <= cap) conc_count<true>(sr, fr, flags, grp, n, f, eta_s, key_s, m, cnt);
    else conc_count<false>(sr, fr, flags, grp, n, f, eta_s, key_s, m, cnt);
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const unsigned long long v = warp_sum_u64(cnt[e]);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(&tot[e], v);
    }
    __syncthreads();
    if (threadIdx.x < 3) counts[fit * 3 + threadIdx.x] = (int64_t)tot[threadIdx.x];
}

}  // namespace g2v

using namespace g2v;

#define G2V_COX_CHECK_FITS(fn, n, K, F, n_sig)                                                                      \
    do {                                                                                                           \
        G2V_REQUIRE((n) >= 3 && (n) <= G2V_SIG_MAX_SAMPLES, fn ": n = %d samples, must be in [3, %d]", (int)(n),    \
                    G2V_SIG_MAX_SAMPLES);                                                                          \
        G2V_REQUIRE((K) >= 1 && (K) <= G2V_SIG_MAX_REPEATS && (F) >= 2 && (F) <= G2V_SIG_MAX_FOLDS &&               \
                        (F) <= (n) / 2,                                                                            \
                    fn ": K = %d repeats and F = %d folds, must be in [1, %d] and [2, min(%d, n / 2)]", (int)(K),  \
                    (int)(F), G2V_SIG_MAX_REPEATS, G2V_SIG_MAX_FOLDS);                                             \
        G2V_REQUIRE((n_sig) >= 1 && (int64_t)(n_sig) * (K) * (F) <= G2V_SIG_MAX_FITS,                               \
                    fn ": %d signatures x %d repeats x %d folds, must be 1 .. %d fits", (int)(n_sig), (int)(K),    \
                    (int)(F), G2V_SIG_MAX_FITS);                                                                   \
    } while (0)

extern "C" size_t g2v_cox_fit_smem_bytes(int32_t p) {
    if (p < 1 || p > G2V_SIG_MAX_SIZE) return 0;
    return cox_smem_doubles(p) * sizeof(double);
}

extern "C" int g2v_cox_fit(const double *X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *flags,
                           const int8_t *fold, int32_t K, int32_t F, const int32_t *genes, int32_t n_sig, int32_t p,
                           double *ell, double *scores, int32_t *n_iter, uint8_t *converged, double *beta,
                           int32_t beta_rows, void *stream) {
    G2V_REQUIRE(X && flags && fold && genes && ell && scores && n_iter && converged, "g2v_cox_fit: null pointer");
    G2V_COX_CHECK_FITS("g2v_cox_fit", n, K, F, n_sig);
    G2V_REQUIRE(p >= 1 && p <= G2V_SIG_MAX_SIZE && p <= G, "g2v_cox_fit: p = %d genes of G = %d, must be in [1, "
                "min(%d, G)]", (int)p, (int)G, G2V_SIG_MAX_SIZE);
    G2V_REQUIRE(n_pad >= n, "g2v_cox_fit: n_pad = %lld, must be >= n = %d", (long long)n_pad, (int)n);
    G2V_REQUIRE(beta_rows >= 0 && beta_rows <= n_sig && (beta_rows == 0 || beta),
                "g2v_cox_fit: beta_rows = %d, must be in [0, %d] with beta given when > 0", (int)beta_rows, (int)n_sig);
    const size_t smem = cox_smem_doubles(p) * sizeof(double);
    G2V_CUDA_OK(cudaFuncSetAttribute(cox_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t fits = (int64_t)n_sig * K * F;
    cox_fit_kernel<<<(unsigned)fits, kFitThreads, smem, (cudaStream_t)stream>>>(
        X, n_pad, n, flags, fold, K, F, genes, p, ell, scores, n_iter, converged, beta, beta_rows);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_cox_concordance(const double *scores, const uint8_t *flags, const int32_t *grp, const int8_t *fold,
                                   int32_t n, int32_t K, int32_t F, int32_t n_sig, int32_t cap, int64_t *counts,
                                   void *stream) {
    G2V_REQUIRE(scores && flags && grp && fold && counts, "g2v_cox_concordance: null pointer");
    G2V_COX_CHECK_FITS("g2v_cox_concordance", n, K, F, n_sig);
    G2V_REQUIRE(cap >= 0 && cap <= n && cap <= G2V_COX_MAX_STAGED, "g2v_cox_concordance: cap = %d, must be in [0, "
                "min(n = %d, %d)]", (int)cap, (int)n, G2V_COX_MAX_STAGED);
    const size_t smem = (size_t)cap * (sizeof(double) + sizeof(int32_t));
    if (smem > 48 * 1024)
        G2V_CUDA_OK(cudaFuncSetAttribute(cox_conc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t fits = (int64_t)n_sig * K * F;
    cox_conc_kernel<<<(unsigned)fits, 256, smem, (cudaStream_t)stream>>>(scores, flags, grp, fold, n, K, F, cap, counts);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
