/*
 * g2v_oracle.c -- CPU ORACLE for the two G2Vec hot paths.  TEST INFRASTRUCTURE ONLY.
 *
 * This file is the checker, never the product: only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  Nothing under
 * g2vec_b200/ links, imports or calls it.
 *
 * It restates, in plain scalar C, the algorithm of the reference
 *   /root/reference/G2Vec.py:324-352  generate_pathSet / generate_randomPath  (walks)
 *   /root/reference/G2Vec.py:217-286  compute_genetovec                        (CBOW)
 * on the sparse layouts the GPU path uses (CSR graph, CSR windows).
 *
 * Parity status:
 *   walks  -- the walk LOGIC (directed rows, every gene starts a walk, append-then-test,
 *             self-avoidance, <= L nodes, dead-end stop) is pinned bit-exact against the
 *             reference's own generate_pathSet through the legacy-stream mode in
 *             oracle/legacy.py (tests/test_oracle_pin.py, tests/golden/).  The Philox
 *             integer draw below replaces only `np.random.choice` (G2Vec.py:341), whose
 *             global MT19937 stream cannot be parallelised; it is compared with the
 *             reference statistically (tests/test_walk_statistics.py).
 *   CBOW   -- TensorFlow 1.x (unpinned ">=1.4", manual p.3) is absent from this image, so
 *             the reference's step 4 cannot be executed: "parity unpinned" against TF
 *             itself; anchored on the call site G2Vec.py:231-283, on TF1's published
 *             ApplyAdam formula and on the README accuracy trajectory.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

/* ------------------------------------------------------------------------------------
 * Philox4x32-10 exactly as curand defines it (curand_philox4x32_x.h: constants
 * 0xD2511F53 / 0xCD9E8D57, Weyl 0x9E3779B9 / 0xBB67AE85, 10 rounds).
 * ---------------------------------------------------------------------------------- */
static inline void philox_round(uint32_t c[4], const uint32_t k[2])
{
    uint64_t p0 = (uint64_t)0xD2511F53u * c[0];
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c[2];
    uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
    uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    uint32_t n0 = hi1 ^ c[1] ^ k[0];
    uint32_t n1 = lo1;
    uint32_t n2 = hi0 ^ c[3] ^ k[1];
    uint32_t n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}

void g2v_oracle_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4])
{
    uint32_t c[4] = {ctr[0], ctr[1], ctr[2], ctr[3]};
    uint32_t k[2] = {key[0], key[1]};
    for (int r = 0; r < 10; ++r) {
        philox_round(c, k);
        if (r < 9) { k[0] += 0x9E3779B9u; k[1] += 0xBB67AE85u; }
    }
    out[0] = c[0]; out[1] = c[1]; out[2] = c[2]; out[3] = c[3];
}

/* 64-bit draw number `s` of walker subsequence `subseq` under `seed`.
 * curand layout: key = (seed lo, seed hi); ctr = (k/4, 0, subseq lo, subseq hi) for 32-bit
 * word index k; draw s consumes words 2s (low half) and 2s+1 (high half). */
static inline uint64_t draw64(uint64_t seed, uint64_t subseq, uint32_t s)
{
    uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    uint32_t ctr[4] = {s >> 1, 0u, (uint32_t)subseq, (uint32_t)(subseq >> 32)};
    uint32_t w[4];
    g2v_oracle_philox4x32_10(ctr, key, w);
    uint32_t lo = w[2 * (s & 1u)], hi = w[2 * (s & 1u) + 1];
    return ((uint64_t)hi << 32) | lo;
}

uint64_t g2v_oracle_draw64(uint64_t seed, uint64_t subseq, uint32_t s) { return draw64(seed, subseq, s); }

/* ------------------------------------------------------------------------------------
 * Walks.  Follows G2Vec.py:328-346 step for step:
 *   path.append(cur)                         :332
 *   prob = row(cur); prob[path] = 0          :334-336   (row = OUT-edges, directed)
 *   if prob.sum() > 0: draw next             :338-341
 *   else: break                              :342-344
 * with at most L appended nodes (:331).  Walker id w = rep*V + src covers
 * `for step in range(iterations): for src in range(n_genes)` (:348-349).
 * The draw: T = sum of quantised weights of unvisited out-neighbours (uint64),
 * r = floor(x * T / 2^64) with x the 64-bit Philox draw, next = first neighbour in
 * ascending dest order whose inclusive prefix sum exceeds r (inverse CDF, the same rule
 * as np.random.choice's searchsorted(cdf, u, side='right'), G2Vec.py:341).
 * Output keeps VISIT ORDER (the reference sorts afterwards, :345); rows are padded
 * with -1.  Returns 0, or -1 on bad arguments.
 * ---------------------------------------------------------------------------------- */
int g2v_oracle_walks(const int32_t *rowptr, const int32_t *col, const uint32_t *qw,
                     int32_t V, int32_t L, uint64_t seed, uint32_t group,
                     int64_t walker_begin, int64_t walker_end, int64_t walker_stride,
                     int32_t *out_nodes, int32_t *out_len)
{
    if (V <= 0 || L <= 0 || walker_stride <= 0 || walker_begin < 0) return -1;
    uint8_t *visited = (uint8_t *)calloc((size_t)V, 1);
    if (!visited) return -1;
    int64_t slot = 0;
    for (int64_t w = walker_begin; w < walker_end; w += walker_stride, ++slot) {
        int32_t *path = out_nodes + slot * (int64_t)L;
        int32_t cur = (int32_t)(w % V);
        uint64_t subseq = ((uint64_t)group << 40) + (uint64_t)w;
        int32_t n = 0;
        for (int32_t s = 0; s < L; ++s) {
            path[n++] = cur;
            visited[cur] = 1;
            if (s == L - 1) break;      /* the reference's last draw is never appended */
            int32_t b = rowptr[cur], e = rowptr[cur + 1];
            uint64_t T = 0;
            for (int32_t j = b; j < e; ++j)
                if (!visited[col[j]]) T += qw[j];
            if (T == 0) break;          /* dead end */
            uint64_t x = draw64(seed, subseq, (uint32_t)s);
            uint64_t r = (uint64_t)(((unsigned __int128)x * T) >> 64);
            uint64_t acc = 0;
            int32_t nxt = -1;
            for (int32_t j = b; j < e; ++j) {
                if (visited[col[j]]) continue;
                acc += qw[j];
                if (acc > r) { nxt = col[j]; break; }
            }
            cur = nxt;                  /* always found: r < T */
        }
        for (int32_t i = 0; i < n; ++i) visited[path[i]] = 0;
        for (int32_t i = n; i < L; ++i) path[i] = -1;
        out_len[slot] = n;
    }
    free(visited);
    return 0;
}

/* ------------------------------------------------------------------------------------
 * CBOW.  One full-batch optimizer step of G2Vec.py:239-246 on CSR windows, float32
 * arithmetic in the order a scalar loop gives:
 *   H = X.W_ih   (SUM of the rows of the window's genes, :239)
 *   O = H.W_ho   (:240)
 *   cost = mean(max(x,0) - x z + log1p(exp(-|x|)))                       (:243)
 *   dO = (sigmoid(O) - Y) / N ; dW_ho = H^T dO ; dW_ih = X^T (dO W_ho^T)   (autodiff of :243)
 *   TF1 ApplyAdam: lr_t = lr sqrt(1-b2^t)/(1-b1^t); m += (g-m)(1-b1); v += (g^2-v)(1-b2);
 *                  var -= lr_t m / (sqrt(v) + eps)                       (:246)
 * `win` lists the training windows (indices into rowptr/label); n_total is the N of
 * the mean.  Gradients are written to g_ih [V*D] / g_ho [D] (overwritten).  If
 * apply_update != 0 the Adam step is applied with step number t (1-based).
 * Returns the mean loss through *loss_out and the number of windows whose prediction
 * (O > 0) equals the label through *n_correct (computed with the PRE-update weights).
 * ---------------------------------------------------------------------------------- */
static inline float sigmoidf_(float x)
{
    if (x >= 0.f) { float z = expf(-x); return 1.f / (1.f + z); }
    float z = expf(x);
    return z / (1.f + z);
}

int g2v_oracle_cbow_grad(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                         const int64_t *win, int64_t n_win, int64_t n_total,
                         const float *W_ih, const float *W_ho, int32_t V, int32_t D,
                         float *g_ih, float *g_ho, double *loss_out, int64_t *n_correct)
{
    (void)V;
    float *h = (float *)malloc(sizeof(float) * (size_t)D);
    if (!h) return -1;
    memset(g_ih, 0, sizeof(float) * (size_t)V * (size_t)D);
    memset(g_ho, 0, sizeof(float) * (size_t)D);
    double loss = 0.0;
    int64_t correct = 0;
    const float invN = 1.0f / (float)n_total;
    for (int64_t i = 0; i < n_win; ++i) {
        int64_t n = win[i];
        int32_t b = rowptr[n], e = rowptr[n + 1];
        for (int32_t d = 0; d < D; ++d) h[d] = 0.f;
        for (int32_t j = b; j < e; ++j) {
            const float *row = W_ih + (size_t)gene[j] * (size_t)D;
            for (int32_t d = 0; d < D; ++d) h[d] += row[d];
        }
        float o = 0.f;
        for (int32_t d = 0; d < D; ++d) o += h[d] * W_ho[d];
        float y = (float)label[n];
        loss += (double)(fmaxf(o, 0.f) - o * y + log1pf(expf(-fabsf(o))));
        correct += ((o > 0.f) == (label[n] != 0));
        float dO = (sigmoidf_(o) - y) * invN;
        for (int32_t d = 0; d < D; ++d) g_ho[d] += h[d] * dO;
        for (int32_t j = b; j < e; ++j) {
            float *grow = g_ih + (size_t)gene[j] * (size_t)D;
            for (int32_t d = 0; d < D; ++d) grow[d] += dO * W_ho[d];
        }
    }
    free(h);
    if (loss_out) *loss_out = loss / (double)n_total;
    if (n_correct) *n_correct = correct;
    return 0;
}

/* TF1 ApplyAdam on one flat parameter array (tensorflow/core/kernels/training_ops.cc,
 * ApplyAdam functor: alpha = lr*sqrt(1-beta2_power)/(1-beta1_power); m += (g-m)*(1-beta1);
 * v += (g*g-v)*(1-beta2); var -= (m*alpha)/(sqrt(v)+epsilon)). */
void g2v_oracle_adam(float *var, float *m, float *v, const float *g, int64_t n,
                     float lr, float beta1, float beta2, float eps, int32_t t)
{
    /* TF1 keeps beta1_power / beta2_power as float32 variables multiplied once per step
     * (AdamOptimizer._finish), i.e. beta^t by repeated float32 multiplication. */
    float b1p = 1.f, b2p = 1.f;
    for (int32_t i = 0; i < t; ++i) { b1p *= beta1; b2p *= beta2; }
    float alpha = lr * sqrtf(1.f - b2p) / (1.f - b1p);
    for (int64_t i = 0; i < n; ++i) {
        m[i] += (g[i] - m[i]) * (1.f - beta1);
        v[i] += (g[i] * g[i] - v[i]) * (1.f - beta2);
        var[i] -= (m[i] * alpha) / (sqrtf(v[i]) + eps);
    }
}

/* Plain SGD epilogue (the north_star's variant): var -= lr * g. */
void g2v_oracle_sgd(float *var, const float *g, int64_t n, float lr)
{
    for (int64_t i = 0; i < n; ++i) var[i] -= lr * g[i];
}

/* Accuracy of G2Vec.py:249-251 ((sigmoid(O) > 0.5) == Y  <=>  (O > 0) == Y) over the
 * listed windows; also returns the logits if o_out != NULL. */
int64_t g2v_oracle_cbow_eval(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                             const int64_t *win, int64_t n_win,
                             const float *W_ih, const float *W_ho, int32_t D, float *o_out)
{
    float *h = (float *)malloc(sizeof(float) * (size_t)D);
    int64_t correct = 0;
    for (int64_t i = 0; i < n_win; ++i) {
        int64_t n = win[i];
        for (int32_t d = 0; d < D; ++d) h[d] = 0.f;
        for (int32_t j = rowptr[n]; j < rowptr[n + 1]; ++j) {
            const float *row = W_ih + (size_t)gene[j] * (size_t)D;
            for (int32_t d = 0; d < D; ++d) h[d] += row[d];
        }
        float o = 0.f;
        for (int32_t d = 0; d < D; ++d) o += h[d] * W_ho[d];
        if (o_out) o_out[i] = o;
        correct += ((o > 0.f) == (label[n] != 0));
    }
    free(h);
    return correct;
}
