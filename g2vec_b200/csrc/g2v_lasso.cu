// g2v_lasso.cu -- cross-validated lasso / elastic-net logistic regression over every gene, the glmnet path
// (DESIGN.md §4.37).  A fit is the full cohort (global fit 0) or the training samples of fold f of repeat k (global
// fit 1 + k F + f); a launch covers the fits fit0 .. fit0 + fits - 1 of a chunk, with their state in one workspace.
//   lasso_std_kernel    one CTA per fit: each gene's training mean and population SD (fit_standardise's rule; a gene
//                       constant over the training samples gets 1 / sd = 0 and never enters), the null model
//                       (intercept logit(ybar)), its deviance and residual, and a cleared path state.
//   lasso_grad_kernel   the full-gene gradient of every fit in one DGEMM: C = X [G x n_pad] times the masked residuals
//                       R^T [n_pad x fits] on the FP64 tensor cores (mma.sync m8n8k4), a warp owning 8 genes x 64
//                       fits; the epilogue applies each fit's standardisation, -(C - mu sum R) / (sd n_fit), and adds
//                       the ridge part lambda (1 - alpha) beta.
//   lasso_cd_kernel     one CTA per fit: the KKT certificate from the gradient, the working set (the sequential strong
//                       rule at a new lambda, KKT violators after), and when the fit is not certified, proximal Newton
//                       (IRLS weights p (1 - p), floored as glmnet floors them) with cyclic coordinate descent over the
//                       working set, then over its nonzero genes until they settle.  Samples are owned by fixed
//                       threads, so residual and linear predictor updates need no barrier; one barrier per coordinate
//                       for its two sums.  A certified fit records its lambda (df, deviance ratio, entries, stop rules)
//                       and does nothing until the next lambda.
//   lasso_score_kernel  each held-out sample's linear predictor and binomial deviance at lambda k.
// Every floating-point sum is in a fixed order (per-thread chains, xor shuffle trees, warp partials summed in warp
// order, DMMA over ascending samples); the only atomic is the integer count of pending fits.  So the results are the
// same bits whatever the chunking.
#include "g2v_fit.cuh"

namespace g2v {

constexpr int kLT = 256, kLW = kLT / 32;               // threads and warps of the per-fit kernels
constexpr double kPMin = 1e-5;                         // glmnet's probability clamp (weights, held-out deviance)
constexpr double kWMin = kPMin * (1.0 - kPMin);
constexpr double kTolCD = 1e-20;                       // max v d^2 of a sweep (gradient change ~ sqrt(v tol))
constexpr int kMaxNewton = 100;                        // Newton steps per (fit, lambda) before it is reported uncertified
constexpr int kMaxSweeps = 100000;                     // coordinate sweeps per Newton step
enum { D_B0, D_B0P, D_NFIT, D_DEVNULL, D_SR, D_DEVR, D_KKT, D_N };
enum { I_NWS, I_STOP, I_EVER, I_ITERS, I_DONE, I_DF, I_N = 8 };

struct LassoWs {
    double *mu, *isd, *beta, *bprev, *g, *eta, *etap, *R, *w, *r, *dsc;
    int32_t *wl, *al, *isc;
    uint8_t *inws, *tr;
};

__host__ __device__ inline LassoWs lasso_ws(void *base, int32_t G, int64_t n_pad, int32_t fits) {
    LassoWs s;
    const int64_t fg = (int64_t)fits * G, fn = (int64_t)fits * n_pad;
    double *d = static_cast<double *>(base);
    s.mu = d; d += fg; s.isd = d; d += fg; s.beta = d; d += fg; s.bprev = d; d += fg; s.g = d; d += fg;
    s.eta = d; d += fn; s.etap = d; d += fn; s.R = d; d += fn; s.w = d; d += fn; s.r = d; d += fn;
    s.dsc = d; d += (int64_t)fits * D_N;
    int32_t *i = reinterpret_cast<int32_t *>(d);
    s.wl = i; i += fg; s.al = i; i += fg; s.isc = i; i += (int64_t)fits * I_N;
    uint8_t *u = reinterpret_cast<uint8_t *>(i);
    s.inws = u; u += fg; s.tr = u;
    return s;
}

__host__ __device__ inline size_t lasso_ws_bytes(int32_t G, int64_t n_pad, int32_t fits) {
    const int64_t fg = (int64_t)fits * G, fn = (int64_t)fits * n_pad;
    return (size_t)(8 * (5 * fg + 5 * fn + (int64_t)fits * D_N) + 4 * (2 * fg + (int64_t)fits * I_N) + fg + fn);
}

// Sum of (a, b) over the CTA, the same bits in every thread.  buf [2][kLW]: alternate halves between calls (par), so
// one barrier per call suffices: a half is rewritten only after the barrier of the call in between.
__device__ __forceinline__ double2 lsum2(double a, double b, double2 *buf, int &par) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    double2 *h = buf + par * kLW;
    if ((threadIdx.x & 31) == 0) h[threadIdx.x >> 5] = make_double2(a, b);
    __syncthreads();
    double2 s = h[0];
#pragma unroll
    for (int w = 1; w < kLW; ++w) { s.x += h[w].x; s.y += h[w].y; }
    par ^= 1;
    return s;
}

__device__ __forceinline__ double lmax(double a, double2 *buf, int &par) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a = fmax(a, __shfl_xor_sync(0xffffffffu, a, o));
    double2 *h = buf + par * kLW;
    if ((threadIdx.x & 31) == 0) h[threadIdx.x >> 5].x = a;
    __syncthreads();
    double m = h[0].x;
#pragma unroll
    for (int w = 1; w < kLW; ++w) m = fmax(m, h[w].x);
    par ^= 1;
    return m;
}

// Appends, in ascending position, the entries whose flag is set: returns this thread's slot (or -1) and the total.
__device__ __forceinline__ int lcompact(bool flag, int *cnt, int &par, int &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t bal = __ballot_sync(0xffffffffu, flag);
    int *h = cnt + par * kLW;
    if (lane == 0) h[warp] = __popc(bal);
    __syncthreads();
    int off = 0;
    total = 0;
    for (int w = 0; w < kLW; ++w) { if (w < warp) off += h[w]; total += h[w]; }
    par ^= 1;
    return flag ? off + __popc(bal & ((1u << lane) - 1u)) : -1;
}

__device__ __forceinline__ double sigmoid(double e) { return 1.0 / (1.0 + exp(-e)); }
// log(1 + e^eta) - y eta, without overflow
__device__ __forceinline__ double nll(double e, double y) { return fmax(e, 0.0) + log1p(exp(-fabs(e))) - y * e; }

// ---- standardise --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLT)
lasso_std_kernel(const double *__restrict__ X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *__restrict__ y,
                 const int8_t *__restrict__ fold, int32_t F, int32_t fit0, int32_t fits, void *wsp,
                 int16_t *__restrict__ entry, double *__restrict__ entry_abs) {
    __shared__ double2 buf[2 * kLW];
    int par = 0;
    const int f = blockIdx.x, gf = fit0 + f, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    LassoWs s = lasso_ws(wsp, G, n_pad, fits);
    const int8_t *frow = gf ? fold + (int64_t)((gf - 1) / F) * n : nullptr;
    const int fout = gf ? (gf - 1) % F : -1;
    uint8_t *tr = s.tr + (int64_t)f * n_pad;
    for (int64_t i = threadIdx.x; i < n_pad; i += kLT) tr[i] = i < n && (!frow || frow[i] != fout);
    __syncthreads();
    const int64_t o = (int64_t)f * G;
    for (int j = warp; j < G; j += kLW) {
        const double *xr = X + (int64_t)j * n_pad;
        double sm = 0.0, mn = INFINITY, mx = -INFINITY;
        int cnt = 0;
        for (int i = lane; i < n; i += 32)
            if (tr[i]) { const double v = __ldg(xr + i); sm += v; mn = fmin(mn, v); mx = fmax(mx, v); ++cnt; }
#pragma unroll
        for (int q = 16; q > 0; q >>= 1) {
            sm += __shfl_xor_sync(0xffffffffu, sm, q);
            mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, q));
            mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, q));
            cnt += __shfl_xor_sync(0xffffffffu, cnt, q);
        }
        double mu = mn, isd = 0.0;
        if (mn != mx) {
            mu = sm / cnt;
            double ss = 0.0;
            for (int i = lane; i < n; i += 32)
                if (tr[i]) { const double d = __ldg(xr + i) - mu; ss = fma(d, d, ss); }
#pragma unroll
            for (int q = 16; q > 0; q >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, q);
            isd = 1.0 / sqrt(ss / cnt);
        }
        if (lane == 0) { s.mu[o + j] = mu; s.isd[o + j] = isd; }
    }
    for (int j = threadIdx.x; j < G; j += kLT) {
        s.beta[o + j] = 0.0; s.bprev[o + j] = 0.0; s.inws[o + j] = 0;
        entry[o + j] = -1; entry_abs[o + j] = 0.0;
    }
    double ys = 0.0, nt = 0.0;
    for (int i = threadIdx.x; i < n; i += kLT)
        if (tr[i]) { ys += y[i]; nt += 1.0; }
    const double2 t = lsum2(ys, nt, buf, par);
    const double ybar = t.x / t.y, b0 = log(ybar / (1.0 - ybar)), p0 = sigmoid(b0);
    double dv = 0.0, sr = 0.0;
    const int64_t on = (int64_t)f * n_pad;
    for (int64_t i = threadIdx.x; i < n_pad; i += kLT) {
        const bool in = tr[i];
        const double yi = in ? (double)y[i] : 0.0;
        s.eta[on + i] = i < n ? b0 : 0.0;
        s.etap[on + i] = s.eta[on + i];
        s.R[on + i] = in ? yi - p0 : 0.0;
        if (in) { dv += nll(b0, yi); sr += yi - p0; }
    }
    const double2 u = lsum2(dv, sr, buf, par);
    if (threadIdx.x == 0) {
        double *d = s.dsc + (int64_t)f * D_N;
        int32_t *c = s.isc + (int64_t)f * I_N;
        d[D_B0] = b0; d[D_B0P] = b0; d[D_NFIT] = t.y; d[D_DEVNULL] = 2.0 * u.x; d[D_SR] = u.y; d[D_DEVR] = 0.0;
        d[D_KKT] = 0.0;
        c[I_NWS] = 0; c[I_STOP] = -1; c[I_EVER] = 0; c[I_ITERS] = 0; c[I_DONE] = 0; c[I_DF] = 0;
    }
}

// ---- gradient -----------------------------------------------------------------------------------------------
constexpr int kGW = 4, kGFits = 64;                    // warps per CTA (8 genes each), fits per CTA

__global__ void __launch_bounds__(kGW * 32)
lasso_grad_kernel(const double *__restrict__ X, int32_t G, int64_t n_pad, int32_t fits, void *wsp, double lam2) {
    LassoWs s = lasso_ws(wsp, G, n_pad, fits);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j0 = (blockIdx.x * kGW + warp) * 8, f0 = blockIdx.y * kGFits;
    const int ja = j0 + (lane >> 2);
    const double *xa = X + (int64_t)min(ja, G - 1) * n_pad + (lane & 3);
    const double *rb[8];
    bool fb[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
        const int fr = f0 + t * 8 + (lane >> 2);
        fb[t] = fr < fits;
        rb[t] = s.R + (int64_t)(fb[t] ? fr : 0) * n_pad + (lane & 3);
    }
    double c[8][2];
#pragma unroll
    for (int t = 0; t < 8; ++t) c[t][0] = c[t][1] = 0.0;
    const bool aok = ja < G;
    for (int64_t kk = 0; kk < n_pad; kk += 4) {
        const double a = aok ? __ldg(xa + kk) : 0.0;
#pragma unroll
        for (int t = 0; t < 8; ++t) dmma_8x8x4(c[t], a, fb[t] ? rb[t][kk] : 0.0);
    }
    const int jo = j0 + (lane >> 2);
    if (jo >= G) return;
#pragma unroll
    for (int t = 0; t < 8; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int f = f0 + t * 8 + (lane & 3) * 2 + h;
            if (f >= fits) continue;
            const int64_t o = (int64_t)f * G + jo;
            const double *d = s.dsc + (int64_t)f * D_N;
            s.g[o] = -(c[t][h] - s.mu[o] * d[D_SR]) * s.isd[o] / d[D_NFIT] + lam2 * s.beta[o];
        }
}

// ---- lambda_max ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLT)
lasso_lmax_kernel(int32_t G, int64_t n_pad, int32_t fits, void *wsp, double adiv, double *out) {
    __shared__ double2 buf[2 * kLW];
    int par = 0;
    LassoWs s = lasso_ws(wsp, G, n_pad, fits);
    double m = 0.0;
    for (int j = threadIdx.x; j < G; j += kLT) m = fmax(m, fabs(s.g[j]));
    m = lmax(m, buf, par);
    if (threadIdx.x == 0) *out = m / adiv;
}

// ---- proximal Newton + coordinate descent -------------------------------------------------------------------
struct CdOut {
    int32_t *df, *n_iter;
    double *dev_ratio, *kkt;
    int16_t *entry;
    double *entry_abs, *path;
    int32_t *ctl;
};

// One sweep over list[0..m): returns max v d^2.  Every thread owns samples tid, tid + kLT, ...
__device__ double lasso_sweep(const double *__restrict__ X, int64_t n_pad, int n, const int32_t *list, int m,
                              const LassoWs &s, int64_t o, int64_t on, double inv_n, double l1, double l2, double sw,
                              double *b0, double2 *buf, int &par) {
    double dlx = 0.0;
    double *w = s.w + on, *r = s.r + on, *eta = s.eta + on, *beta = s.beta + o;
    for (int q = 0; q < m; ++q) {
        const int j = list[q];
        const double *xr = X + (int64_t)j * n_pad;
        const double mu = s.mu[o + j], isd = s.isd[o + j], b = beta[j];
        double a = 0.0, v = 0.0;
        for (int i = threadIdx.x; i < n; i += kLT) {
            const double z = (__ldg(xr + i) - mu) * isd, wz = w[i] * z;
            a = fma(wz, r[i], a);
            v = fma(wz, z, v);
        }
        const double2 t = lsum2(a, v, buf, par);
        const double vv = t.y * inv_n, u = fma(vv, b, t.x * inv_n);
        const double au = fabs(u) - l1;
        const double bn = au > 0.0 ? copysign(au, u) / (vv + l2) : 0.0;
        if (bn != b) {
            const double d = bn - b;
            for (int i = threadIdx.x; i < n; i += kLT) {
                const double z = (__ldg(xr + i) - mu) * isd;
                if (w[i] != 0.0) r[i] = fma(-d, z, r[i]);
                eta[i] = fma(d, z, eta[i]);
            }
            if (threadIdx.x == 0) beta[j] = bn;
            dlx = fmax(dlx, vv * d * d);
        }
    }
    double a = 0.0;
    for (int i = threadIdx.x; i < n; i += kLT) a += w[i] * r[i];
    const double2 t = lsum2(a, 0.0, buf, par);
    const double d0 = t.x / sw;
    if (d0 != 0.0) {
        for (int i = threadIdx.x; i < n; i += kLT) {
            if (w[i] != 0.0) r[i] -= d0;
            eta[i] += d0;
        }
        *b0 += d0;
        dlx = fmax(dlx, sw * inv_n * d0 * d0);
    }
    return dlx;
}

__global__ void __launch_bounds__(kLT)
lasso_cd_kernel(const double *__restrict__ X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *__restrict__ y,
                int32_t fits, void *wsp, int32_t k, double lam, double lam_prev, double alpha, int32_t round,
                CdOut out) {
    __shared__ double2 buf[2 * kLW];
    __shared__ int cnt[2 * kLW];
    int par = 0, cpar = 0;
    const int f = blockIdx.x;
    LassoWs s = lasso_ws(wsp, G, n_pad, fits);
    const int64_t o = (int64_t)f * G, on = (int64_t)f * n_pad, ol = (int64_t)f * G2V_LASSO_N_LAMBDA + k;
    double *d = s.dsc + (int64_t)f * D_N;
    int32_t *c = s.isc + (int64_t)f * I_N;
    int32_t *wl = s.wl + o, *al = s.al + o;
    uint8_t *inws = s.inws + o;
    const uint8_t *tr = s.tr + on;
    double *beta = s.beta + o, *eta = s.eta + on;
    const double l1 = lam * alpha, l2 = lam * (1.0 - alpha), inv_n = 1.0 / d[D_NFIT];
    if (c[I_STOP] >= 0) {                              // stopped: its last solution stands for this lambda
        if (round == 0 && threadIdx.x == 0) {
            out.df[ol] = c[I_DF]; out.dev_ratio[ol] = d[D_DEVR]; out.n_iter[ol] = 0; out.kkt[ol] = d[D_KKT];
        }
        return;
    }
    if (round > 0 && c[I_DONE]) return;
    int nws = c[I_NWS];
    if (round == 0) {
        for (int q = threadIdx.x; q < nws; q += kLT) s.bprev[o + wl[q]] = beta[wl[q]];
        for (int64_t i = threadIdx.x; i < n_pad; i += kLT) s.etap[on + i] = eta[i];
        __syncthreads();
        if (threadIdx.x == 0) { c[I_ITERS] = 0; c[I_DONE] = 0; d[D_B0P] = d[D_B0]; }
    }
    // certificate and working set
    const double thr = round == 0 ? alpha * (2.0 * lam - lam_prev) : l1;
    double viol = threadIdx.x == 0 ? fabs(d[D_SR] * inv_n) : 0.0;
    const double *g = s.g + o;
    for (int j0 = 0; j0 < G; j0 += kLT) {
        const int j = j0 + threadIdx.x;
        bool add = false;
        if (j < G && s.isd[o + j] != 0.0) {
            const double gj = g[j], b = beta[j];
            if (inws[j])
                viol = fmax(viol, b == 0.0 ? fmax(fabs(gj) - l1, 0.0) : fabs(gj + copysign(l1, b)));
            else {
                viol = fmax(viol, fmax(fabs(gj) - l1, 0.0));
                add = fabs(gj) > thr;
            }
        }
        int total;
        const int slot = lcompact(add, cnt, cpar, total);
        if (add) { wl[nws + slot] = j; inws[j] = 1; }
        nws += total;
    }
    viol = lmax(viol, buf, par);
    const int iters = c[I_ITERS];
    if (viol <= G2V_LASSO_EPS || iters >= kMaxNewton) {
        // finish lambda k
        double dv = 0.0;
        for (int i = threadIdx.x; i < n; i += kLT)
            if (tr[i]) dv += nll(eta[i], (double)y[i]);
        int dfl = 0, newl = 0;
        for (int q = threadIdx.x; q < nws; q += kLT) {
            const int j = wl[q];
            if (beta[j] != 0.0) { ++dfl; newl += out.entry[o + j] < 0; }
        }
        const double2 t = lsum2(dv, (double)dfl, buf, par);
        const double2 t2 = lsum2((double)newl, 0.0, buf, par);
        const int df = (int)t.y, nw = (int)t2.x;
        if (c[I_EVER] + nw > G2V_LASSO_MAX_ACTIVE) {   // glmnet's pmax: the path ends before this lambda
            for (int q = threadIdx.x; q < nws; q += kLT) beta[wl[q]] = s.bprev[o + wl[q]];
            for (int64_t i = threadIdx.x; i < n_pad; i += kLT) eta[i] = s.etap[on + i];
            if (threadIdx.x == 0) {
                d[D_B0] = d[D_B0P];
                c[I_STOP] = k;
                out.df[ol] = c[I_DF]; out.dev_ratio[ol] = d[D_DEVR]; out.n_iter[ol] = iters; out.kkt[ol] = d[D_KKT];
            }
        } else {
            for (int q = threadIdx.x; q < nws; q += kLT) {
                const int j = wl[q];
                if (beta[j] != 0.0 && out.entry[o + j] < 0) { out.entry[o + j] = (int16_t)k; out.entry_abs[o + j] = fabs(beta[j]); }
            }
            if (out.path && f == 0)
                for (int j = threadIdx.x; j <= G; j += kLT) out.path[(int64_t)k * (G + 1) + j] = j ? beta[j - 1] : d[D_B0];
            if (threadIdx.x == 0) {
                const double dr = 1.0 - 2.0 * t.x / d[D_DEVNULL], prev = d[D_DEVR];
                c[I_EVER] += nw; c[I_DF] = df; d[D_DEVR] = dr; d[D_KKT] = viol;
                out.df[ol] = df; out.dev_ratio[ol] = dr; out.n_iter[ol] = iters; out.kkt[ol] = viol;
                if (dr > 0.999 || (k >= 4 && dr - prev < 1e-5 * dr)) c[I_STOP] = k + 1;
            }
        }
        if (threadIdx.x == 0) { c[I_DONE] = 1; c[I_NWS] = nws; if (f == 0) out.ctl[1] = c[I_STOP]; }
        return;
    }
    // proximal Newton over the working set
    double *w = s.w + on, *r = s.r + on;
    double b0 = d[D_B0];
    int it = iters;
    while (it < kMaxNewton) {
        double swl = 0.0;
        for (int i = threadIdx.x; i < n; i += kLT) {
            double wi = 0.0, ri = 0.0;
            if (tr[i]) {
                const double p = sigmoid(eta[i]);
                wi = fmax(p * (1.0 - p), kWMin);
                ri = ((double)y[i] - p) / wi;
            }
            w[i] = wi; r[i] = ri; swl += wi;
        }
        const double sw = lsum2(swl, 0.0, buf, par).x;
        ++it;
        double first = 0.0;
        for (int sweep = 0; sweep < kMaxSweeps;) {
            const double dlx = lasso_sweep(X, n_pad, n, wl, nws, s, o, on, inv_n, l1, l2, sw, &b0, buf, par);
            ++sweep;
            if (sweep == 1) first = dlx;
            if (dlx < kTolCD) break;
            // the nonzero genes of the working set, in working-set order
            int m = 0;
            for (int q0 = 0; q0 < nws; q0 += kLT) {
                const int q = q0 + threadIdx.x;
                const bool nz = q < nws && beta[wl[q]] != 0.0;
                int total;
                const int slot = lcompact(nz, cnt, cpar, total);
                if (nz) al[m + slot] = wl[q];
                m += total;
            }
            __syncthreads();
            for (; sweep < kMaxSweeps; ++sweep)
                if (lasso_sweep(X, n_pad, n, al, m, s, o, on, inv_n, l1, l2, sw, &b0, buf, par) < kTolCD) break;
        }
        if (first < kTolCD) break;
    }
    __syncthreads();
    double sr = 0.0;
    for (int i = threadIdx.x; i < n; i += kLT) {
        const double ri = tr[i] ? (double)y[i] - sigmoid(eta[i]) : 0.0;
        s.R[on + i] = ri; sr += ri;
    }
    sr = lsum2(sr, 0.0, buf, par).x;
    if (threadIdx.x == 0) {
        d[D_B0] = b0; d[D_SR] = sr; c[I_ITERS] = it; c[I_NWS] = nws;
        atomicAdd(out.ctl, 1);
        if (f == 0) out.ctl[1] = c[I_STOP];
    }
}

// ---- held-out scores ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLT)
lasso_score_kernel(const uint8_t *__restrict__ y, const int8_t *__restrict__ fold, int32_t n, int64_t n_pad,
                   int32_t K, int32_t F, int32_t fit0, int32_t fits, void *wsp, int32_t G, int32_t k,
                   double *__restrict__ scores, double *__restrict__ dev) {
    const int f = blockIdx.x, gf = fit0 + f;
    if (gf == 0) return;
    LassoWs s = lasso_ws(wsp, G, n_pad, fits);
    const int rep = (gf - 1) / F, fo = (gf - 1) % F;
    const int8_t *frow = fold + (int64_t)rep * n;
    const double *eta = s.eta + (int64_t)f * n_pad;
    const int64_t base = ((int64_t)k * K + rep) * n;
    for (int i = threadIdx.x; i < n; i += kLT)
        if (frow[i] == fo) {
            const double e = eta[i], p = fmin(fmax(sigmoid(e), kPMin), 1.0 - kPMin);
            scores[base + i] = e;
            dev[base + i] = -2.0 * (y[i] ? log(p) : log(1.0 - p));
        }
}

}  // namespace g2v

using namespace g2v;

#define G2V_LASSO_CHECK(fn, G, n, n_pad, fits)                                                                    \
    do {                                                                                                         \
        G2V_REQUIRE((n) >= 3 && (n) <= G2V_SIG_MAX_SAMPLES, fn ": n = %d samples, must be in [3, %d]", (int)(n),  \
                    G2V_SIG_MAX_SAMPLES);                                                                        \
        G2V_REQUIRE((G) >= 1 && (G) <= G2V_LASSO_MAX_GENES, fn ": G = %d genes, must be in [1, %d]", (int)(G),    \
                    G2V_LASSO_MAX_GENES);                                                                        \
        G2V_REQUIRE((n_pad) >= (n) && (n_pad) % 4 == 0, fn ": n_pad = %lld, must be >= n and a multiple of 4",    \
                    (long long)(n_pad));                                                                         \
        G2V_REQUIRE((fits) >= 1 && (fits) <= 1 + G2V_SIG_MAX_REPEATS * G2V_SIG_MAX_FOLDS,                        \
                    fn ": fits = %d, must be in [1, %d]", (int)(fits), 1 + G2V_SIG_MAX_REPEATS * G2V_SIG_MAX_FOLDS); \
    } while (0)
#define G2V_LASSO_CHECK_SPLIT(fn, K, F, fit0, fits)                                                               \
    G2V_REQUIRE((K) >= 1 && (K) <= G2V_SIG_MAX_REPEATS && (F) >= 2 && (F) <= G2V_SIG_MAX_FOLDS && (fit0) >= 0 &&  \
                    (fit0) + (fits) <= 1 + (K) * (F),                                                            \
                fn ": K = %d, F = %d, fits %d + [0, %d) must be K in [1, %d], F in [2, %d], within 1 + K F",     \
                (int)(K), (int)(F), (int)(fit0), (int)(fits), G2V_SIG_MAX_REPEATS, G2V_SIG_MAX_FOLDS)

extern "C" size_t g2v_lasso_workspace_bytes(int32_t G, int64_t n_pad, int32_t fits) {
    if (G < 1 || G > G2V_LASSO_MAX_GENES || n_pad < 4 || n_pad > G2V_SIG_MAX_SAMPLES + 32 || fits < 1 ||
        fits > 1 + G2V_SIG_MAX_REPEATS * G2V_SIG_MAX_FOLDS)
        return 0;
    return lasso_ws_bytes(G, n_pad, fits);
}

extern "C" int g2v_lasso_standardise(const double *X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *y,
                                     const int8_t *fold, int32_t K, int32_t F, int32_t fit0, int32_t fits, void *ws,
                                     int16_t *entry, double *entry_abs, void *stream) {
    G2V_REQUIRE(X && y && fold && ws && entry && entry_abs, "g2v_lasso_standardise: null pointer");
    G2V_LASSO_CHECK("g2v_lasso_standardise", G, n, n_pad, fits);
    G2V_LASSO_CHECK_SPLIT("g2v_lasso_standardise", K, F, fit0, fits);
    lasso_std_kernel<<<(unsigned)fits, kLT, 0, (cudaStream_t)stream>>>(X, G, n, n_pad, y, fold, F, fit0, fits, ws,
                                                                       entry, entry_abs);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_lasso_grad(const double *X, int32_t G, int32_t n, int64_t n_pad, int32_t fits, void *ws,
                              double lam, double alpha, void *stream) {
    G2V_REQUIRE(X && ws, "g2v_lasso_grad: null pointer");
    G2V_LASSO_CHECK("g2v_lasso_grad", G, n, n_pad, fits);
    G2V_REQUIRE(lam >= 0.0 && alpha > 0.0 && alpha <= 1.0, "g2v_lasso_grad: lambda = %g, alpha = %g", lam, alpha);
    const dim3 grid((unsigned)((G + 8 * kGW - 1) / (8 * kGW)), (unsigned)((fits + kGFits - 1) / kGFits));
    lasso_grad_kernel<<<grid, kGW * 32, 0, (cudaStream_t)stream>>>(X, G, n_pad, fits, ws, lam * (1.0 - alpha));
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_lasso_lambda_max(int32_t G, int64_t n_pad, int32_t fits, void *ws, double alpha, double *lam_max,
                                    void *stream) {
    G2V_REQUIRE(ws && lam_max, "g2v_lasso_lambda_max: null pointer");
    G2V_REQUIRE(G >= 1 && G <= G2V_LASSO_MAX_GENES && fits >= 1 && alpha > 0.0 && alpha <= 1.0,
                "g2v_lasso_lambda_max: G = %d, fits = %d, alpha = %g", (int)G, (int)fits, alpha);
    lasso_lmax_kernel<<<1, kLT, 0, (cudaStream_t)stream>>>(G, n_pad, fits, ws, fmax(alpha, 1e-3), lam_max);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_lasso_cd(const double *X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *y, int32_t fits,
                            void *ws, int32_t k, double lam, double lam_prev, double alpha, int32_t round, int32_t *df,
                            double *dev_ratio, int32_t *n_iter, double *kkt, int16_t *entry, double *entry_abs,
                            double *path, int32_t *ctl, void *stream) {
    G2V_REQUIRE(X && y && ws && df && dev_ratio && n_iter && kkt && entry && entry_abs && ctl,
                "g2v_lasso_cd: null pointer");
    G2V_LASSO_CHECK("g2v_lasso_cd", G, n, n_pad, fits);
    G2V_REQUIRE(k >= 0 && k < G2V_LASSO_N_LAMBDA && round >= 0, "g2v_lasso_cd: lambda index %d, round %d", (int)k,
                (int)round);
    G2V_REQUIRE(lam > 0.0 && lam_prev >= lam && alpha > 0.0 && alpha <= 1.0,
                "g2v_lasso_cd: lambda = %g after %g, alpha = %g", lam, lam_prev, alpha);
    G2V_CUDA_OK(cudaMemsetAsync(ctl, 0, sizeof(int32_t), (cudaStream_t)stream));
    const CdOut out{df, n_iter, dev_ratio, kkt, entry, entry_abs, path, ctl};
    lasso_cd_kernel<<<(unsigned)fits, kLT, 0, (cudaStream_t)stream>>>(X, G, n, n_pad, y, fits, ws, k, lam, lam_prev,
                                                                      alpha, round, out);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}

extern "C" int g2v_lasso_score(const uint8_t *y, const int8_t *fold, int32_t n, int64_t n_pad, int32_t K, int32_t F,
                               int32_t fit0, int32_t fits, void *ws, int32_t G, int32_t k, double *scores,
                               double *dev, void *stream) {
    G2V_REQUIRE(y && fold && ws && scores && dev, "g2v_lasso_score: null pointer");
    G2V_LASSO_CHECK("g2v_lasso_score", G, n, n_pad, fits);
    G2V_LASSO_CHECK_SPLIT("g2v_lasso_score", K, F, fit0, fits);
    G2V_REQUIRE(k >= 0 && k < G2V_LASSO_N_LAMBDA, "g2v_lasso_score: lambda index %d", (int)k);
    lasso_score_kernel<<<(unsigned)fits, kLT, 0, (cudaStream_t)stream>>>(y, fold, n, n_pad, K, F, fit0, fits, ws, G,
                                                                         k, scores, dev);
    G2V_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
}
