/*
 * g2vec_b200.h -- C ABI of libg2vec_b200.so: the two G2Vec hot paths as sm_90a CUDA.
 *
 * The reference (mathcom/G2Vec) has no FFI or plugin interface: its boundary for these
 * paths is two plain Python calls in main(),
 *     pathSet = generate_pathSet(adjMat, args.lenPath, args.numRepetition)     G2Vec.py:62
 *     genetovec['mat'] = compute_genetovec(pathList, n_genes, hidden, lr)      G2Vec.py:74
 * The entry points below are what a binding for those two call sites needs; the ctypes
 * binding that ships is g2vec_b200/_capi.py, and INTEGRATION.md shows the stub a
 * maintainer of the reference would add.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no exceptions, no torch types.
 *   - every function returns 0 on success, non-zero on failure; g2v_last_error() then
 *     returns a thread-local message.
 *   - `stream` is a cudaStream_t passed as void*; device entry points are asynchronous on
 *     it and never synchronise.  Buffers are owned by the caller.
 *   - `_host` entry points take HOST pointers, do their own device allocation and
 *     host<->device copies, and return after the result is back in host memory.
 *   - there is no CPU fallback: without a usable sm_90 device the calls fail.
 */
#ifndef G2VEC_B200_H
#define G2VEC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define G2V_ABI_VERSION 2

/* optimizer codes for g2v_cbow_update */
#define G2V_OPT_ADAM_TF1 0 /* tf.train.AdamOptimizer, G2Vec.py:246 (parity default) */
#define G2V_OPT_SGD 1      /* var -= lr * g (north_star variant) */

/* context reduction for the CBOW forward */
#define G2V_REDUCE_SUM 0  /* H = X.W_ih, G2Vec.py:239 (parity default) */
#define G2V_REDUCE_MEAN 1 /* H = X.W_ih / len(window) */

int g2v_abi_version(void);
const char *g2v_last_error(void);

/* Device facts (current device): SM count, compute capability, L2 bytes, and the number of
 * kernels this library has launched since load (bench.py's gpu_launches). */
int g2v_device_info(int32_t *sm_count, int32_t *cc_major, int32_t *cc_minor, int64_t *l2_bytes);
int64_t g2v_launch_count(void);

/* ---------------------------------------------------------------------------------------
 * HOT PATH 1 -- walk sampler.  Replaces generate_pathSet / generate_randomPath,
 * G2Vec.py:324-352, for the walkers  w = walker_begin + i*walker_stride < walker_end,
 * w = rep*V + src  (rep = G2Vec.py:348 `step`, src = :349).
 *
 *   rowptr [V+1], col [E] (ascending inside a row = dense row order), qw [E]: CSR of the
 *     group's directed adjacency (rows = out-edges, G2Vec.py:390) with weights quantised to
 *     integers, 1 <= qw <= 2^24  (q = rint(|PCC| * 2^16)).
 *   L: --lenPath, the maximum number of NODES of a path (G2Vec.py:331).  1 <= L <= 4096, and the
 *     per-CTA path + visited-set buffers must fit shared memory: always true for L <= 1365, and
 *     for any L <= 4096 while V <= ~90k (bitmap visited set); otherwise the call fails with a message.
 *   seed/group: Philox4x32-10 key and the high bits of the walker's subsequence
 *     (subsequence = group*2^40 + w, 64-bit draw s = words 2s,2s+1), so that any
 *     (walker, step) is addressable independently: results do not depend on sharding.
 *   out_nodes [n*L]: visit order of walker i in row i, padded with -1  (the reference
 *     sorts afterwards, G2Vec.py:345).  out_len [n]: nodes visited.  n = number of walkers.
 *   workspace: >= g2v_walk_workspace_bytes() bytes of device scratch (zeroed by the call).
 * ------------------------------------------------------------------------------------- */
size_t g2v_walk_workspace_bytes(void);
int g2v_walk_launch(const int32_t *rowptr, const int32_t *col, const uint32_t *qw, int32_t V,
                    int64_t E, int32_t L, uint64_t seed, uint32_t group, int64_t walker_begin,
                    int64_t walker_end, int64_t walker_stride, int32_t *out_nodes,
                    int32_t *out_len, void *workspace, void *stream);

/* Packed graph layouts (built once per graph; the graph is static across all repetitions, G2Vec.py:348-351).
 * g2v_walk_prepare turns the CSR arrays (device pointers) into
 *   rows  [V]  int32 pairs {begin, end} of each node's out-edges                (g2v_walk_packed_bytes: rows_bytes)
 *   edges      layout 1: uint32 pairs {col, qw}, rows starting at even indices: one 16-byte load brings two
 *              neighbours per lane;
 *              layout 2: uint32 col | (qw - 32768) << 16 [E] -- chosen when V <= 65535 and every
 *              32768 <= qw <= 65536 (weights |PCC| in [0.5, 1], G2Vec.py:389): one 8-byte load brings two
 *              neighbours per lane                                              (edges_bytes covers both)
 * and returns the layout chosen through *layout_out (a host int; the call synchronises the stream once).
 * g2v_walk_launch_packed is g2v_walk_launch on the packed graph.  With out_key != NULL it also performs
 * `path = tuple(sorted(path))` (G2Vec.py:345) in the same kernel: out_nodes rows are then SORTED ascending and
 * padded with INT32_MAX, and out_key [n] receives the 64-bit row key g2v_paths_canonicalise would compute. */
int g2v_walk_packed_bytes(int32_t V, int64_t E, size_t *rows_bytes, size_t *edges_bytes);
int g2v_walk_prepare(const int32_t *rowptr, const int32_t *col, const uint32_t *qw, int32_t V, int64_t E,
                     void *rows, void *edges, int32_t *layout_out, void *workspace, void *stream);
int g2v_walk_launch_packed(const void *rows, const void *edges, int32_t layout, int32_t V, int64_t E, int32_t L,
                           uint64_t seed, uint32_t group, int64_t walker_begin, int64_t walker_end,
                           int64_t walker_stride, int32_t *out_nodes, int32_t *out_len, int64_t *out_key,
                           void *workspace, void *stream);

/* Same, HOST pointers in and out (one device slab: copies in, packs, launches, copies back, frees). */
int g2v_walk_host(const int32_t *rowptr, const int32_t *col, const uint32_t *qw, int32_t V,
                  int64_t E, int32_t L, uint64_t seed, uint32_t group, int64_t walker_begin,
                  int64_t walker_end, int64_t walker_stride, int32_t *out_nodes,
                  int32_t *out_len);

/* node2vec's in-out bias (Grover & Leskovec 2016, parameter q).  A walker at v whose previous node is t weighs an
 * unvisited out-neighbour x of quantised weight qw as  qw * a_near  if the edge t -> x exists (x in t's CSR row)
 * and  qw * a_far  otherwise; step 0 has no previous node and uses qw.  The draw is unchanged: T = sum of the
 * effective weights (uint64), r = floor(x * T / 2^64), first neighbour in ascending order whose inclusive prefix
 * exceeds r.  1 <= a_near, a_far <= 256, else the call fails.  Equal multipliers scale every weight alike and give
 * the bits of the plain entry point (they run its kernels).  Arguments otherwise as their plain counterparts. */
int g2v_walk_launch_biased(const int32_t *rowptr, const int32_t *col, const uint32_t *qw, int32_t V,
                           int64_t E, int32_t L, uint64_t seed, uint32_t group, int64_t walker_begin,
                           int64_t walker_end, int64_t walker_stride, int32_t *out_nodes,
                           int32_t *out_len, uint32_t a_near, uint32_t a_far, void *workspace, void *stream);
int g2v_walk_launch_packed_biased(const void *rows, const void *edges, int32_t layout, int32_t V, int64_t E,
                                  int32_t L, uint64_t seed, uint32_t group, int64_t walker_begin,
                                  int64_t walker_end, int64_t walker_stride, int32_t *out_nodes, int32_t *out_len,
                                  int64_t *out_key, uint32_t a_near, uint32_t a_far, void *workspace, void *stream);
int g2v_walk_host_biased(const int32_t *rowptr, const int32_t *col, const uint32_t *qw, int32_t V,
                         int64_t E, int32_t L, uint64_t seed, uint32_t group, int64_t walker_begin,
                         int64_t walker_end, int64_t walker_stride, int32_t *out_nodes,
                         int32_t *out_len, uint32_t a_near, uint32_t a_far);

/* ---------------------------------------------------------------------------------------
 * HOT PATH 2 -- modified CBOW.  Replaces the TF1 graph of compute_genetovec,
 * G2Vec.py:231-251, one optimizer step at a time; the epoch loop and the early stop
 * (G2Vec.py:262-283) stay with the host (g2vec_b200/cbow.py).
 *
 * Windows (the rows of pathList, G2Vec.py:316-320) are CSR: rowptr [N+1], gene [nnz],
 * label [N] (0 good / 1 poor).  `win` (nullable) is a list of window indices (the shuffled
 * 80/20 split of G2Vec.py:219-222); NULL means windows win_begin..win_begin+n_win-1.
 * W_ih [V*D] row-major are the gene vectors; W_ho [D].
 *
 * g2v_cbow_fwdbwd: for every listed window, gather the rows of its genes, reduce (sum),
 *   logit o = h.W_ho, dO = (sigmoid(o) - y) * inv_n_total, then ADD  dO*W_ho into
 *   g_ih[gene,:] for each gene of the window and h*dO into g_ho.  Adds the BCE loss sum
 *   into *loss_sum (double) and the count of (o > 0) == y into *n_correct.  g_ih, g_ho,
 *   loss_sum, n_correct are ACCUMULATED (device memory; the caller or g2v_cbow_update zeroes).
 * g2v_cbow_update: optimizer epilogue over W_ih and W_ho from g_ih / g_ho (after the
 *   all-reduce when multi-GPU); zeroes g_ih / g_ho for the next step.  t = 1-based step.
 * g2v_cbow_eval: forward only; adds the count of correct predictions into *n_correct.
 * ------------------------------------------------------------------------------------- */
int g2v_cbow_fwdbwd(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                    const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total,
                    const float *W_ih, const float *W_ho, float *g_ih, float *g_ho,
                    double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                    void *stream);

/* g2v_cbow_fwdbwd_csc: the same step as g2v_cbow_fwdbwd over the WHOLE list win[0..n_win-1], with the list's
 * windows x genes incidence also given transposed (CSC over list positions: cscptr [V+1], csc_pos [nnz] =
 * positions i of the windows that contain the gene, as for g2v_cbow_r1_windows_csc).  The forward stores
 * dO*scale per list position in the scratch dO [n_win]; a second kernel then adds c[g]*W_ho into g_ih[g,:] once
 * per gene, c[g] = sum of dO over the gene's positions in a fixed order -- no floating-point atomics on g_ih.
 * Same accumulation semantics as g2v_cbow_fwdbwd (g_ih, g_ho, loss_sum, n_correct are added into); rows of
 * genes in no listed window are not touched.  csc_pos may be NULL only when nnz == 0 (every listed window is empty,
 * so every segment of cscptr is empty); g2v_cbow_fwdbwd_csc_det takes the same arguments with the same rule. */
int g2v_cbow_fwdbwd_csc(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                        const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                        const float *W_ho, const int32_t *cscptr, const int32_t *csc_pos, float *dO,
                        float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V,
                        int32_t D, int32_t reduce, void *stream);

/* g2v_cbow_fwd_do: the first half of g2v_cbow_fwdbwd_csc over win[0..n_win-1] (win may point into a longer list,
 * e.g. at the start of a mini-batch): the fused forward stores dO*scale per list position i in dO [n_win] and adds
 * into g_ho, loss_sum and n_correct as g2v_cbow_fwdbwd does.  Nothing is added into any gradient row. */
int g2v_cbow_fwd_do(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                    int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho, float *dO, float *g_ho,
                    double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce, void *stream);

/* g2v_cbow_lazy_adam: lazy (touched-row) TF1 Adam after g2v_cbow_fwd_do, as tf.contrib.opt.LazyAdamOptimizer applies
 * it to an embedding lookup.  rows [n_rows] = the distinct genes of the batch; the positions of gene rows[r] in the
 * batch are pos[segptr[r] .. segptr[r+1]) (indices into dO, in the order they are summed).  For each listed gene
 * W_ih/m_ih/v_ih[g,:] take one TF1 ApplyAdam step with gradient c*W_ho, c = the sum of dO over its positions and W_ho
 * the value before this call; every other row is left untouched.  Then W_ho/m_ho/v_ho take the dense step from g_ho,
 * and g_ho is zeroed.  Step size: alpha_dev as in g2v_cbow_update (device beta powers), else from t.  Two launches
 * (one when n_rows == 0). */
int g2v_cbow_lazy_adam(const int32_t *rows, const int32_t *segptr, const int32_t *pos, const float *dO,
                       int64_t n_rows, float *W_ih, float *m_ih, float *v_ih, float *W_ho, float *m_ho, float *v_ho,
                       float *g_ho, int32_t V, int32_t D, float lr, float beta1, float beta2, float eps, int32_t t,
                       const float *alpha_dev, void *stream);

/* Deterministic mode (DESIGN.md §4.13): the same results as g2v_cbow_fwdbwd_csc / g2v_cbow_fwd_do /
 * g2v_cbow_loop_tail, with every floating-point sum in a fixed order, so that the bits do not depend on the run or on
 * the launch grid.  The forward cuts the list into tiles of 64 positions, stores each tile's g_ho partial and loss in
 * `workspace` (g2v_cbow_det_workspace_bytes(n_win, D) bytes, device memory, contents not needed across calls), and a
 * second launch adds the tiles in a fixed order into g_ho and *loss_sum.  max_ctas > 0 caps the number of CTAs of
 * every launch (0 = the whole chip); the results are the same for every value.  Same accumulation semantics, `stopped`
 * and `carried` handling and launch counts plus one (the tile sum) as the forms they mirror; never synchronises.
 * g2v_cbow_batch_expand: the expansion of g2v_cbow_fwdbwd_csc on one batch's plan from g2v_cbow_batch_plan: for
 *   r < n_rows, g_ih[rows[r],:] += c * W_ho with c = the sum of dO over pos[segptr[r] .. segptr[r+1]) in a fixed
 *   order; rows must be distinct.  With g2v_cbow_fwd_do_det it replaces g2v_cbow_fwdbwd's scatter on a mini-batch.
 *   One launch (none when n_rows == 0). */
size_t g2v_cbow_det_workspace_bytes(int64_t n_win, int32_t D);
int g2v_cbow_fwdbwd_csc_det(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                            int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                            const int32_t *cscptr, const int32_t *csc_pos, float *dO, float *g_ih, float *g_ho,
                            double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                            void *workspace, int32_t max_ctas, void *stream);
int g2v_cbow_fwd_do_det(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                        int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho, float *dO, float *g_ho,
                        double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce, void *workspace,
                        int32_t max_ctas, void *stream);
int g2v_cbow_loop_tail_det(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                           const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                           float *dO, float *g_ho, int64_t *acc, int32_t V, int32_t D, int32_t reduce, void *workspace,
                           int32_t max_ctas, void *stream);
int g2v_cbow_batch_expand(const int32_t *rows, const int32_t *segptr, const int32_t *pos, const float *dO,
                          int64_t n_rows, const float *W_ho, float *g_ih, int32_t V, int32_t D, int32_t max_ctas,
                          void *stream);

/* Reshuffled mini-batch epochs (csrc/g2v_cbow_plan.cu, DESIGN.md §4.12).
 * g2v_cbow_epoch_order: out[i] = tr[P(rank + i*world)] for i < ceil((n - rank) / world): rank `rank`'s share of the
 *   epoch's list tr[P(0..n-1)].  P = P(seed, epoch, n) is a pseudo-random permutation of [0, n) (a 4-round Feistel
 *   network with Philox4x32-10 rounds, cycle-walked into [0, n); exact definition in DESIGN.md §4.12).  One launch.
 * g2v_cbow_batch_plan: the plan g2v_cbow_lazy_adam reads, for every batch k of B consecutive windows of the list
 *   win[0..n_win-1] (the last one shorter): the ascending distinct genes of the batch, rows[batch_rowptr[k] ..
 *   batch_rowptr[k+1]); segment pointers segptr (absolute into pos, segptr[S] = nnz, S = batch_rowptr[n_b]); the
 *   positions of each gene's windows relative to the batch start, ascending inside each segment, in pos.  nnz = the
 *   number of (window, gene) incidences of the list; rows [nnz], segptr [nnz + 1], pos [nnz], batch_rowptr
 *   [ceil(n_win / B) + 1]; workspace: g2v_cbow_batch_plan_workspace_bytes(n_win, nnz, B, V) bytes.  If the list has
 *   more than nnz incidences nothing is written except batch_rowptr[n_b] = -1.  Genes must lie in [0, V).  Never
 *   synchronises; 7 launches per wave of K = max(1, 2^22 / V) batches. */
int g2v_cbow_epoch_order(const int32_t *tr, int64_t n, uint64_t seed, int32_t epoch, int64_t rank, int64_t world,
                         int32_t *out, void *stream);
size_t g2v_cbow_batch_plan_workspace_bytes(int64_t n_win, int64_t nnz, int64_t B, int32_t V);
int g2v_cbow_batch_plan(const int32_t *rowptr, const int32_t *gene, const int32_t *win, int64_t n_win, int64_t nnz,
                        int64_t B, int32_t V, int32_t *rows, int32_t *segptr, int32_t *pos, int32_t *batch_rowptr,
                        void *workspace, void *stream);

int g2v_cbow_update(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                    float *g_ih, float *g_ho, int32_t V, int32_t D, int32_t optimizer, float lr,
                    float beta1, float beta2, float eps, int32_t t, const float *alpha_dev, void *stream);

/* Decoupled weight decay (DESIGN.md §4.18; TF1 DecoupledWeightDecayExtension, AdamW / SGDW): the *_wd entry points
 * take the arguments of their counterparts plus `weight_decay` (lambda) after `eps`, and apply
 *     w <- fl(w - fl(lambda * w))     (two separately rounded operations, never one FMA)
 * to every parameter element the step updates, before the unchanged Adam / SGD arithmetic on that value.  m and v are
 * not touched by the decay, the gradients are those of the weights before the step, and lambda is not scaled by the
 * learning rate.  lambda = 0 launches the same kernels as the counterpart (which is that call with 0), so the results
 * and the launch count are the counterpart's; lambda must be finite with 0 <= lambda < 1, else the call fails with
 * g2v_last_error() set and nothing launched.  Elements decayed:
 *   g2v_cbow_update_wd      every element of W_ih and W_ho;
 *   g2v_cbow_lazy_adam_wd   the listed rows of W_ih, each once, and all of W_ho; the other rows keep W, m and v;
 *   g2v_cbow_update_nvl_wd  rank r's slice (and the scalar tail on rank world-1), after the reduce and before the
 *                           step; the all-gather then delivers the decayed and updated values to every rank;
 *   g2v_cbow_r1_update_wd   every element of W_ih, rows with c[g] = 0 included (SGD too), and W_ho; g_ho = W_ih^T.c
 *                           uses W_ih before the decay. */
int g2v_cbow_update_wd(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                       float *g_ih, float *g_ho, int32_t V, int32_t D, int32_t optimizer, float lr,
                       float beta1, float beta2, float eps, float weight_decay, int32_t t, const float *alpha_dev,
                       void *stream);
int g2v_cbow_lazy_adam_wd(const int32_t *rows, const int32_t *segptr, const int32_t *pos, const float *dO,
                          int64_t n_rows, float *W_ih, float *m_ih, float *v_ih, float *W_ho, float *m_ho, float *v_ho,
                          float *g_ho, int32_t V, int32_t D, float lr, float beta1, float beta2, float eps,
                          float weight_decay, int32_t t, const float *alpha_dev, void *stream);
int g2v_cbow_update_nvl_wd(float *const *g_ptrs_dev, float *const *w_ptrs_dev, float *g_multicast, float *w_multicast,
                           float *m_flat, float *v_flat, int64_t n, int32_t rank, int32_t world, int32_t optimizer,
                           float lr, float beta1, float beta2, float eps, float weight_decay, int32_t t,
                           const float *alpha_dev, void *stream);
int g2v_cbow_r1_update_wd(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                          float *c, float *g_ho, float *s, int32_t V, int32_t D, int32_t optimizer,
                          float lr, float beta1, float beta2, float eps, float weight_decay, int32_t t,
                          const float *alpha_dev, void *stream);

/* Class weights of the training loss (DESIGN.md §4.20; Keras fit(class_weight=...)): the *_cw entry points take the
 * arguments of their counterparts plus the weights w0, w1 (labels 0 and 1) before the stream.  A window of label y
 * forms
 *     dO = fl(fl(fl(sigmoid(o) - y) * inv_n_total) * w_y)
 * (then the counterpart's * scale and everything after it, unchanged) and adds fl(w_y * l) to *loss_sum instead of
 * its BCE term l.  The correct count is not weighted.  With w0 = w1 = 1 both products are exact, so a *_cw call gives
 * the bits of its counterpart (on the fixed-order routes; the atomic ones reorder as their counterparts do).  The
 * weights must be finite and > 0, else the call fails with g2v_last_error() set and nothing launched.  The launches
 * are the counterpart's, with the class-weighted instantiations of the kernels that form dO. */
int g2v_cbow_fwdbwd_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                       int64_t win_begin, int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                       float *g_ih, float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D,
                       int32_t reduce, float w0, float w1, void *stream);
int g2v_cbow_fwdbwd_csc_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                           int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                           const int32_t *cscptr, const int32_t *csc_pos, float *dO, float *g_ih, float *g_ho,
                           double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce, float w0,
                           float w1, void *stream);
int g2v_cbow_fwd_do_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                       int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho, float *dO, float *g_ho,
                       double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce, float w0, float w1,
                       void *stream);
int g2v_cbow_fwdbwd_csc_det_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                               int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                               const int32_t *cscptr, const int32_t *csc_pos, float *dO, float *g_ih, float *g_ho,
                               double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                               void *workspace, int32_t max_ctas, float w0, float w1, void *stream);
int g2v_cbow_fwd_do_det_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                           int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho, float *dO,
                           float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                           void *workspace, int32_t max_ctas, float w0, float w1, void *stream);
int g2v_cbow_loop_tail_cw(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                          const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                          float *dO, float *g_ho, int64_t *acc, int32_t V, int32_t D, int32_t reduce, float w0,
                          float w1, void *stream);
int g2v_cbow_loop_tail_val_cw(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                              const int32_t *tr_win, int64_t n_tr, float inv_n_total, const int32_t *va_win,
                              int64_t n_va, const float *W_ih, const float *W_ho, float *st, float *dO, float *g_ho,
                              int64_t *acc, int32_t V, int32_t D, int32_t reduce, float w0, float w1, void *stream);
int g2v_cbow_loop_tail_det_cw(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                              const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih,
                              const float *W_ho, float *dO, float *g_ho, int64_t *acc, int32_t V, int32_t D,
                              int32_t reduce, void *workspace, int32_t max_ctas, float w0, float w1, void *stream);
int g2v_cbow_fwdbwd_slabs_cw(const int32_t *gene, const uint8_t *label, const int32_t *win, int64_t win_begin,
                             int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho, float *g_ih,
                             float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                             int32_t n_slabs, void *workspace, float w0, float w1, void *stream);
int g2v_cbow_r1_windows_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                           int64_t win_begin, int64_t n_win, float inv_n_total, const float *s, float *c,
                           double *loss_sum, int64_t *n_correct, int32_t V, int32_t reduce, float w0, float w1,
                           void *stream);
int g2v_cbow_r1_windows_csc_cw(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                               int64_t n_win, float inv_n_total, const float *s, const int32_t *cscptr,
                               const int32_t *csc_pos, float *dO, float *c, double *loss_sum, int64_t *n_correct,
                               int32_t V, int32_t reduce, float w0, float w1, void *stream);

/* Multi-GPU optimizer epilogue fused with the gradient exchange (one process per GPU, one node): replaces
 * ncclAllReduce(gradient) + g2v_cbow_update.  All buffers are flat [W_ih (V*D) | W_ho (D)] = n floats, the gradient
 * and the parameters in symmetric memory (same size on every rank, peer-mapped): g_ptrs_dev / w_ptrs_dev are DEVICE
 * arrays of `world` pointers (entry r = rank r's buffer as seen from this rank); g_multicast / w_multicast are the
 * NVLS multicast addresses of the same buffers, or both NULL (then peer loads/stores are used).  Rank r reduces the
 * slice r of every rank's gradient (multimem.ld_reduce or peer loads), zeroes it everywhere, applies TF1 Adam / SGD
 * to slice r of its m / v / parameters, and stores the new parameters into every rank's buffer.  The caller must
 * place a cross-GPU barrier before the call (all gradients complete) and after it (all parameters delivered).
 * Slice r is the float4 range [r*c, min(n/4, (r+1)*c)) with c = ceil((n/4) / world) -- empty for the ranks past
 * n/4 -- and the scalar tail [4*floor(n/4), n) belongs to rank world-1.  m_flat / v_flat are n floats per rank, of
 * which the call reads and writes only slice r: across steps each rank's m / v hold only its own slice, so `world`
 * and the partition must stay the same for the whole run.  On the peer path rank r adds the gradients to 0 in the
 * rank order r, r+1, ..., r-1 (mod world) on its float4 slice and 0, 1, ..., world-1 on the tail. */
int g2v_cbow_update_nvl(float *const *g_ptrs_dev, float *const *w_ptrs_dev, float *g_multicast, float *w_multicast,
                        float *m_flat, float *v_flat, int64_t n, int32_t rank, int32_t world, int32_t optimizer,
                        float lr, float beta1, float beta2, float eps, int32_t t, const float *alpha_dev, void *stream);

/* Device-resident Adam step state -- TF1 keeps beta1^t / beta2^t as variables (AdamOptimizer's
 * beta1_power / beta2_power, G2Vec.py:246).  state = {beta1^t, beta2^t, alpha_t, unused}, initialised to
 * {1, 1, 0, 0}; g2v_cbow_adam_tick advances it by one step on the device.  Passing the same pointer as
 * `alpha_dev` to g2v_cbow_update / g2v_cbow_r1_update (else NULL: alpha is computed on the host from t)
 * makes every launch of a training step independent of host-side values, so the whole step can be captured
 * once in a CUDA graph and replayed (g2vec_b200/cbow.py). */
int g2v_cbow_adam_tick(float *state, float lr, float beta1, float beta2, void *stream);
/* g2v_cbow_adam_tick with the learning rate read from *lr_dev on the device (the rate of g2v_cbow_lr_plateau's state):
 * the same arithmetic, so an unchanged rate gives g2v_cbow_adam_tick's bits.  Tests the loop's `stopped` word as
 * g2v_cbow_adam_tick does. */
int g2v_cbow_adam_tick_lr(float *state, const float *lr_dev, float beta1, float beta2, void *stream);

int g2v_cbow_eval(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                  const int32_t *win, int64_t win_begin, int64_t n_win, const float *W_ih,
                  const float *W_ho, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                  void *stream);

/* g2v_cbow_eval_certified: adds into *n_correct the same count as g2v_cbow_eval, for every input, mostly without
 * gathering rows (DESIGN.md §4.16).  A first launch writes st [2*V floats, device scratch] = {s[g], t[g]} per gene,
 * s = W_ih.W_ho and t[g] = sum_d |W_ih[g,d] W_ho[d]|; the second takes each window's prediction from the collapsed
 * logit scale * sum_{g in n} s[g] where a float32 error bound shows it has the sign of g2v_cbow_eval's logit, and
 * computes that logit by g2v_cbow_eval's own row gather for every other window (empty ones included).  Admits the D
 * range of g2v_cbow_eval.  Test arguments: force_gather != 0 sends every window to the row gather; n_gathered
 * (nullable) is added the number of windows that took it.  Both launches test the loop's `stopped` word; never
 * synchronises. */
int g2v_cbow_eval_certified(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                            const int32_t *win, int64_t win_begin, int64_t n_win, const float *W_ih,
                            const float *W_ho, float *st, int64_t *n_correct, int64_t *n_gathered, int32_t V,
                            int32_t D, int32_t reduce, int32_t force_gather, void *stream);

/* ---------------------------------------------------------------------------------------
 * Device-side control of the training loop (SURVEY.md 8f-4; G2Vec.py:262-283), so that several iterations of
 * the reference's loop can be enqueued -- or replayed as ONE CUDA graph -- without a host decision in between.
 *   ctl  [8] int64 in device memory: {stopped, step, stop_step, before_val, max_steps, early_stop, carried, queue}
 *        g2v_cbow_loop_init sets {0, 0, -1, -1, max_steps, early_stop, 0, 0}.
 *   g2v_cbow_loop_attach(ctl): from now on every CBOW kernel launched by THIS host thread first reads
 *        ctl.stopped and returns at once if it is set (attach(NULL) detaches); the forward of
 *        g2v_cbow_fwdbwd_csc also returns at once while ctl.carried is set (its per-gene expansion still runs).
 *   g2v_cbow_loop_begin: unless stopped, copies W_ih [n floats] into `snapshot` (nullable) -- the weights the
 *        reference would return if this step's validation accuracy drops (:283,:286) -- and zeroes acc[0..3];
 *        if ctl.carried is set, acc[0..1] take the carried loss and count acc[4..5] instead, which are zeroed.
 *   g2v_cbow_loop_tail: the training-accuracy pass of a step (after the update and the validation pass) that is
 *        also the next step's forward -- valid because nothing changes the weights or the training list in
 *        between.  It runs g2v_cbow_fwd_do over the training list win[0..n_win-1] for which the caller prepared
 *        g2v_cbow_fwdbwd_csc's transposed incidence: dO [n_win] per list position, g_ho += sum h*dO (the update
 *        has just zeroed it), loss sum into acc[4] (f64 bits), correct count into acc[5]; then, unless stopped,
 *        acc[3] += acc[5] (the step's ACC[tr]) and ctl.carried = 1.  acc is then int64 [6]: the carry slots lie
 *        outside acc[1..3], which a multi-GPU step sums over the ranks.  Two launches.
 *   g2v_cbow_loop_decide: unless stopped, stores acc[0..3] (loss-sum bits, pre-update train correct, validation
 *        correct, train correct) in hist[step*4 ..] (acc == NULL: they are there already, see below), applies `if acc_val < before_acc_val: break` (:276) on the
 *        validation count, else before_val = count (:280); stops after max_steps; step += 1.
 * The host reads ctl / hist whenever it wants to print (every 5th step, :269) instead of after every step.
 * ------------------------------------------------------------------------------------- */
int g2v_cbow_loop_init(int64_t *ctl, int64_t max_steps, int32_t early_stop, void *stream);
int g2v_cbow_loop_attach(const int64_t *ctl);
int g2v_cbow_loop_begin(const int64_t *ctl, int64_t *acc, const float *W_ih, float *snapshot, int64_t n, void *stream);
int g2v_cbow_loop_tail(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                       const int32_t *win, int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho,
                       float *dO, float *g_ho, int64_t *acc, int32_t V, int32_t D, int32_t reduce, void *stream);
/* g2v_cbow_loop_tail_val (DESIGN.md §4.32): the validation pass g2v_cbow_eval_certified(va_win[0..n_va-1]) into
 * acc[2] and the tail pass g2v_cbow_loop_tail(tr_win[0..n_tr-1]) in one window launch, after st's own launch: the same
 * validation count, the same dO and acc[5]; g_ho and acc[4] differ only by the order of their atomics.  Warps take
 * validation groups of four windows, then training windows, from the counter in ctl[7], which the launch leaves at 0
 * (g2v_cbow_loop_init sets it so).  D = 128, 256 or 512.  Both window launches and the carry test `stopped`. */
int g2v_cbow_loop_tail_val(int64_t *ctl, const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                           const int32_t *tr_win, int64_t n_tr, float inv_n_total, const int32_t *va_win, int64_t n_va,
                           const float *W_ih, const float *W_ho, float *st, float *dO, float *g_ho, int64_t *acc,
                           int32_t V, int32_t D, int32_t reduce, void *stream);
int g2v_cbow_loop_decide(int64_t *ctl, const int64_t *acc, int64_t *hist, void *stream);
/* Early stopping with patience (DESIGN.md §4.15): the loop keeps the weights of its best step instead of a snapshot.
 *   best [4] int64 in device memory: {patience, best_step, bad_steps, improved}; the caller sets {K, -1, 0, 0}
 *        after g2v_cbow_loop_init (K >= 1).  ctl.before_val then holds the best validation count so far.
 *   g2v_cbow_loop_decide_best: in place of g2v_cbow_loop_decide (same acc / hist forms).  If stopped, clears
 *        `improved` and returns.  Else records the counters, and a validation count >= the best so far makes this
 *        step the best (improved = 1, bad_steps = 0); a lower count adds one bad step (improved = 0), and with
 *        ctl.early_stop set the K-th bad step in a row stops the loop with stop_step = step.  Stops after max_steps;
 *        step += 1.  With K = 1 it decides exactly as g2v_cbow_loop_decide.
 *   g2v_cbow_loop_keep_best: after it, copies W_ih [n floats] into `result` if `improved`.  It does not test
 *        ctl.stopped (the step that reaches max_steps may be the best one), so `result` ends as W_ih of best_step.
 * Pass snapshot = NULL to g2v_cbow_loop_begin on this path.  Neither call depends on a host value that changes between
 * steps or synchronises, so both are captured in the loop's CUDA graphs. */
int g2v_cbow_loop_decide_best(int64_t *ctl, int64_t *best, const int64_t *acc, int64_t *hist, void *stream);
int g2v_cbow_loop_keep_best(const int64_t *best, const float *W_ih, float *result, int64_t n, void *stream);
/* Reduce-on-plateau learning rate (DESIGN.md §4.17): Keras ReduceLROnPlateau(mode="max", min_delta=0, cooldown=0) on
 * the integer validation count of each step, decided on the device.
 *   state in device memory, int64 x 8 then float32 x (4 + cap):
 *        {K, best, wait, n_reductions, steps, cap, -, -}, then {lr, factor, min_lr, -, rate[0 .. cap-1]}.
 *        The caller sets {K, -1, 0, 0, 0, cap, 0, 0} and {lr, factor, min_lr, 0} (K >= 1, 0 < factor < 1,
 *        min_lr >= 0); the rate lives at byte offset 64 and is what g2v_cbow_adam_tick_lr reads.
 *   g2v_cbow_lr_plateau: for every step s not yet decided, v = counts[s * stride]; rate[s] = lr (if s < cap: the rate
 *        step s trained with); then if v > best: best = v, wait = 0 (a tie is no improvement), else wait += 1 and when
 *        wait >= K: if lr > min_lr, lr = max(float32(lr * factor), min_lr) and n_reductions += 1; wait = 0.
 *        The steps it decides are steps .. *n_decided - 1, and exactly one step if n_decided is NULL; steps is then
 *        advanced past them.  One kernel for both loops:
 *        - device loop: after g2v_cbow_loop_decide[_best], counts = hist + 2, stride = 4, n_decided = &ctl.step.  The
 *          decision reads the count that the loop's decision just recorded (summed over the ranks on every exchange),
 *          and the no-op steps after a stop decide nothing, so it is captured in the loop's CUDA graphs;
 *        - host-driven loop: after the all-reduce of acc[1..3], counts = acc + 2, stride = 0, n_decided = NULL.
 *        It does not test the loop's `stopped` word.  One launch of one thread, never synchronises. */
int g2v_cbow_lr_plateau(int64_t *state, const int64_t *counts, int64_t stride, const int64_t *n_decided, void *stream);
/* Multi-GPU, hist in symmetric memory (zero-initialised, same size on every rank): add this rank's acc[1..3] into
 * hist[step][1..3] of every rank (multimem.red through hist_multicast, or system-scope atomics on hist_ptrs_dev);
 * after a cross-GPU barrier call g2v_cbow_loop_decide with acc == NULL, which then decides on the summed counters
 * already in hist[step].  Replaces the all_reduce of the counters. */
int g2v_cbow_loop_counters_nvl(const int64_t *ctl, const int64_t *acc, int64_t *const *hist_ptrs_dev,
                               int64_t *hist_multicast, int32_t world, void *stream);

/* Validation-loss monitor (DESIGN.md §4.19): the early-stop and reduce-on-plateau rules decided on the validation
 * loss instead of the validation count.
 *   g2v_cbow_val_loss: adds into *q_sum  Q = sum over windows n of the list of q_n = rint(min(l_n, 64) * 2^24), with
 *        l_n = max(z,0) - z*y + log1p(exp(-|z|)) in float64 (64 when z is not finite) and the collapsed logit
 *        z = scale_n * sum_{g in n} s[g] in float32 (scale_n = 1 for REDUCE_SUM, 1/len for REDUCE_MEAN).  s[g] is read at
 *        s[g * s_stride]: s_stride = 2 on the st = {s, t} that g2v_cbow_eval_certified or g2v_cbow_st_prepare wrote,
 *        1 on the rank-1 model's s.  The sum over g is taken in one fixed order per window (8 lanes, lane k adding
 *        genes k, k+8, ... of the window, then a shuffle tree 4, 2, 1), so Q is the same integer for any launch grid,
 *        any order of the windows and any split of the list (the parts' Q add up to the whole's).  q_n <= 2^30 and
 *        n_win < 2^32, so Q < 2^62 never overflows.  Tests the loop's `stopped` word; one launch, never synchronises.
 *   g2v_cbow_st_prepare: the first launch of g2v_cbow_eval_certified alone (st = {s, t} per gene, 2*V floats), for a
 *        list whose count came from another route (the gene slabs).  Tests the loop's `stopped` word.
 *   The monitored score of a step is 2^62 - Q (non-negative, higher is better), so the loop's sentinels (-1) and
 *   g2v_cbow_lr_plateau (counts = score, stride = 1) apply to it unchanged.
 *   g2v_cbow_loop_decide_score / g2v_cbow_loop_decide_best_score: g2v_cbow_loop_decide / g2v_cbow_loop_decide_best
 *        (same ctl, best, acc, hist forms) deciding on score[step] = 2^62 - Q instead of the validation count.
 *        q != NULL: Q = *q (summed over the ranks), which is then zeroed for the next step; q == NULL: score[step]
 *        holds the Q g2v_cbow_loop_score_nvl added.  score[step] is left holding the score.
 *   g2v_cbow_loop_score_nvl: unless stopped, adds *q into element offset + step of every rank's symmetric buffer
 *        (multimem.red through multicast, else system-scope atomics on ptrs_dev) and zeroes *q; a cross-GPU barrier
 *        then precedes the decision with q == NULL on score = buffer + offset. */
int g2v_cbow_val_loss(const int32_t *rowptr, const int32_t *gene, const uint8_t *label, const int32_t *win,
                      int64_t win_begin, int64_t n_win, const float *s, int32_t s_stride, uint64_t *q_sum, int32_t V,
                      int32_t reduce, void *stream);
int g2v_cbow_st_prepare(const float *W_ih, const float *W_ho, float *st, int32_t V, int32_t D, void *stream);
int g2v_cbow_loop_decide_score(int64_t *ctl, const int64_t *acc, int64_t *hist, uint64_t *q, int64_t *score,
                               void *stream);
int g2v_cbow_loop_decide_best_score(int64_t *ctl, int64_t *best, const int64_t *acc, int64_t *hist, uint64_t *q,
                                    int64_t *score, void *stream);
int g2v_cbow_loop_score_nvl(const int64_t *ctl, uint64_t *q, int64_t *const *ptrs_dev, int64_t *multicast,
                            int64_t offset, int32_t world, void *stream);

/* ---------------------------------------------------------------------------------------
 * HOT PATH 2 for tables larger than the L2 (csrc/g2v_cbow_slab.cu): the same step as g2v_cbow_fwdbwd /
 * g2v_cbow_eval, processed gene slab by gene slab so that the gathered rows and the gradient rows stay
 * L2-resident.  Needs windows whose gene lists are strictly ascending (tuple(sorted(path)), G2Vec.py:345).
 *
 * g2v_cbow_slab_plan: number of slabs for a [V, D] table on the current device (1 = the table fits the L2,
 *   or D is not 128/256/512: use g2v_cbow_fwdbwd_csc / g2v_cbow_fwdbwd).
 * g2v_cbow_slab_workspace_bytes / g2v_cbow_slab_setup: per window list (win/win_begin/n_win as in
 *   g2v_cbow_fwdbwd; the list is static across steps, G2Vec.py:262-264), records where each window's sorted gene
 *   list crosses the slab boundaries.  Synchronises the stream once; fails on an unsorted window.
 * g2v_cbow_fwdbwd_slabs / g2v_cbow_eval_slabs: same accumulation semantics as g2v_cbow_fwdbwd / g2v_cbow_eval,
 *   for the list the workspace was set up with.
 * ------------------------------------------------------------------------------------- */
int g2v_cbow_slab_plan(int32_t V, int32_t D, int32_t *n_slabs);
size_t g2v_cbow_slab_workspace_bytes(int64_t n_win, int32_t D, int32_t n_slabs);
int g2v_cbow_slab_setup(const int32_t *rowptr, const int32_t *gene, const int32_t *win, int64_t win_begin,
                        int64_t n_win, int32_t V, int32_t n_slabs, void *workspace, void *stream);
int g2v_cbow_fwdbwd_slabs(const int32_t *gene, const uint8_t *label, const int32_t *win, int64_t win_begin,
                          int64_t n_win, float inv_n_total, const float *W_ih, const float *W_ho, float *g_ih,
                          float *g_ho, double *loss_sum, int64_t *n_correct, int32_t V, int32_t D, int32_t reduce,
                          int32_t n_slabs, void *workspace, void *stream);
int g2v_cbow_eval_slabs(const int32_t *gene, const uint8_t *label, const int32_t *win, int64_t win_begin,
                        int64_t n_win, const float *W_ih, const float *W_ho, int64_t *n_correct, int32_t V,
                        int32_t D, int32_t reduce, int32_t n_slabs, void *workspace, void *stream);

/* One full-batch step from HOST buffers: uploads the windows and the parameters/optimizer
 * state, runs fwdbwd + update, downloads the updated parameters/state, the loss sum and the
 * correct count (of the pre-update forward).  m/v may be NULL for SGD. */
int g2v_cbow_step_host(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                       int64_t n_win, int64_t nnz, float *W_ih, float *W_ho, float *m_ih,
                       float *v_ih, float *m_ho, float *v_ho, int32_t V, int32_t D,
                       int32_t optimizer, int32_t reduce, float lr, float beta1, float beta2,
                       float eps, int32_t t, double *loss_sum, int64_t *n_correct);

/* ---------------------------------------------------------------------------------------
 * HOT PATH 2, collapsed ("rank-1") form -- SURVEY.md 8f-3.  The reference's model is linear
 * (G2Vec.py:239-240: O = (X.W_ih).W_ho), so with  s = W_ih.W_ho [V]  and  c = X^T.dO [V]
 * the same step is  o = sum_{g in window} s[g];  dW_ih[g,:] = c[g]*W_ho;  dW_ho = W_ih^T.c.
 * Same results up to float32 reassociation; 4-byte scalars per (window, gene) instead of
 * D-wide rows, and a 4*V-byte all-reduce (of c) instead of 4*V*D bytes.
 *
 * g2v_cbow_r1_prepare: s[g] = <W_ih[g,:], W_ho>.
 * g2v_cbow_r1_windows: forward over the listed windows from s; if c != NULL also the backward:
 *   c[gene] += dO for every gene of the window, loss sum and pre-update correct count
 *   accumulated as in g2v_cbow_fwdbwd.  c == NULL: accuracy pass only (g2v_cbow_eval).
 * g2v_cbow_r1_update: optimizer epilogue from c (after its all-reduce when multi-GPU): per row
 *   g = c[g]*W_ho and g_ho += c[g]*W_ih[g,:] (old W_ih), TF1 Adam / SGD on W_ih, then on W_ho,
 *   zeroes c, and refreshes s for the updated parameters.  g_ho: scratch of
 *   g2v_cbow_r1_scratch_bytes(D) bytes (per-block partial sums of W_ih^T.c, reduced in a fixed
 *   order: no floating-point atomics anywhere in this call).
 * ------------------------------------------------------------------------------------- */
int g2v_cbow_r1_prepare(const float *W_ih, const float *W_ho, float *s, int32_t V, int32_t D,
                        void *stream);
int g2v_cbow_r1_windows(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                        const int32_t *win, int64_t win_begin, int64_t n_win, float inv_n_total,
                        const float *s, float *c, double *loss_sum, int64_t *n_correct, int32_t V,
                        int32_t reduce, void *stream);
/* Deterministic backward: the list's windows x genes incidence is also given transposed (CSC over list
 * positions: cscptr [V+1], csc_pos [nnz] = positions i in 0..n_win-1 of the windows that contain the gene).
 * dO [n_win] is scratch; c[g] += sum of dO over the gene's positions with a fixed reduction order, so
 * the step is bit-reproducible (no floating-point atomics). */
int g2v_cbow_r1_windows_csc(const int32_t *rowptr, const int32_t *gene, const uint8_t *label,
                            const int32_t *win, int64_t n_win, float inv_n_total, const float *s,
                            const int32_t *cscptr, const int32_t *csc_pos, float *dO, float *c,
                            double *loss_sum, int64_t *n_correct, int32_t V, int32_t reduce, void *stream);
size_t g2v_cbow_r1_scratch_bytes(int32_t D);
int g2v_cbow_r1_update(float *W_ih, float *W_ho, float *m_ih, float *v_ih, float *m_ho, float *v_ho,
                       float *c, float *g_ho, float *s, int32_t V, int32_t D, int32_t optimizer,
                       float lr, float beta1, float beta2, float eps, int32_t t, const float *alpha_dev,
                       void *stream);

/* ---------------------------------------------------------------------------------------
 * Upstream of the walks -- edge weighting (SURVEY.md 8f-1).  Replaces construct_adjMat /
 * compute_PCC, G2Vec.py:354-391, for one patient group.
 * g2v_pcc_zscore: expr [S*V] sample-major (rows = the group's samples, G2Vec.py:378) ->
 *   z [V*S] gene-major z-scores (population std; 0 for zero-variance genes, :359,366-367).
 * g2v_pcc_edge_weights: w[e] = |mean_s z[src[e]][s] * z[dst[e]][s]|  (G2Vec.py:362-365,385).
 * The > 0.5 threshold (:389) and the CSR assembly are done by the caller.
 * ------------------------------------------------------------------------------------- */
int g2v_pcc_zscore(const float *expr, int32_t S, int32_t V, float *z, void *stream);
int g2v_pcc_edge_weights(const float *z, int32_t S, int32_t V, const int32_t *src, const int32_t *dst,
                         int64_t E, float *w, void *stream);

/* Spearman and biweight-midcorrelation edge weights (DESIGN.md §4.22).  g2v_corr_transform writes, like
 * g2v_pcc_zscore, a gene-major z [V*S] from the sample-major expr [S*V] (z must not overlap expr), with
 * mean_s z[a][s] * z[b][s] = the coefficient, so g2v_pcc_edge_weights turns z into the weights unchanged:
 *   G2V_CORR_SPEARMAN  z = the Pearson z-score (population std; 0 for a constant gene) of the average ranks
 *                      r_i = (#{x < x_i} + #{x <= x_i} + 1) / 2, -0.0 tying with +0.0;
 *   G2V_CORR_BICOR     med = median(x) (mean of the two middle values for even S), mad = median(|x - med|); if
 *                      mad > 0: u = (x - med) / (9 mad), t = (x - med)(1 - u^2)^2 for |u| < 1 else 0,
 *                      z = t sqrt(S) / ||t||; if mad = 0: the bits g2v_pcc_zscore gives the gene.
 * Double arithmetic, float32 z; the bits do not depend on the run or on the launch.  1 <= S <= G2V_CORR_MAX_SAMPLES
 * and V >= 1, else the call fails with nothing launched.  Two launches, never synchronises. */
#define G2V_CORR_SPEARMAN 1
#define G2V_CORR_BICOR 2
#define G2V_CORR_MAX_SAMPLES 32768
int g2v_corr_transform(const float *expr, int32_t S, int32_t V, int32_t method, float *z, void *stream);

/* ---------------------------------------------------------------------------------------
 * Label-permutation test of the gene t statistics (DESIGN.md §4.24; g2vec_b200/perm.py does the host side).
 * n samples (3 <= n <= G2V_PERM_MAX_SAMPLES), S_pad = a multiple of 32 with n <= S_pad <= G2V_PERM_MAX_SAMPLES;
 * padding bytes are 0.  Permutations are numbered b = 1 .. B, B <= G2V_PERM_MAX_PERMUTATIONS.
 * g2v_perm_labels: M [n_b * S_pad] u8, row r = permutation b = b_begin + 1 + r of the indicator obs [n] (0/1):
 *   Fisher-Yates from obs, for i = n-1 down to 1: j = hi64(draw64(seed, 2^63 + b, n-1-i) * (i+1)), swap i and j
 *   (draw64 = the walk sampler's Philox4x32-10 stream).  A row depends only on (obs, seed, b): chunks of one
 *   sequence of calls give the rows of one big call.
 * g2v_perm_sums: A [n_b * G] int64 = M . q, exact.  q [G][S_pad] reaches the device as three byte planes,
 *   planes = {h [G*S_pad] s8, m [G*S_pad] u8, l [G*S_pad] u8} back to back, q = 2^16 h + 2^8 m + l, each gene's
 *   samples contiguous; |q| <= 2^22.  INT8 tensor cores (mma.sync m16n8k32), int64 only in the epilogue.
 * g2v_perm_tally: per row of A, N_j = n A_j - k Q_j and rho_j = N_j^2 / W_j (float64, 0 when W_j = 0);
 *   count[j] += |N_j| >= absN_obs[j];  count_maxt[j] += (max over j' >= j of rho_j') >= rho_obs[j].
 *   Integer atomics only; the counts do not depend on the grid or on how the rows are chunked.
 * Out-of-range sizes fail with nothing launched.  One launch each, never synchronises. */
#define G2V_PERM_MAX_SAMPLES 32768
#define G2V_PERM_MAX_PERMUTATIONS (1 << 24)
int g2v_perm_labels(const uint8_t *obs, int32_t n, int32_t S_pad, uint64_t seed, int64_t b_begin, int64_t n_b,
                    uint8_t *M, void *stream);
int g2v_perm_sums(const uint8_t *M, const uint8_t *planes, int64_t n_b, int32_t S_pad, int32_t G, int64_t *A,
                  void *stream);
int g2v_perm_tally(const int64_t *A, int64_t n_b, int32_t G, int32_t n, int32_t k, const int64_t *Q, const double *W,
                   const int64_t *absN_obs, const double *rho_obs, int64_t *count, int64_t *count_maxt, void *stream);

/* ---------------------------------------------------------------------------------------
 * Exact cosine K nearest genes of every gene (DESIGN.md §4.25; g2vec_b200/neighbors.py does the host side).
 * W [m][D] float32 row-major, 2 <= m <= G2V_NBR_MAX_GENES, D >= 1, every value finite; 1 <= K <= min(G2V_NBR_MAX_K,
 * m - 1).  Everything in IEEE float64:
 *   dot_ij = ((0 + W_i0 W_j0) + W_i1 W_j1) + ... + W_i(D-1) W_j(D-1)   (a chain of fma in ascending d, from +0);
 *   n_i = dot_ii;  inv_i = 1 / sqrt(n_i) (correctly rounded), 0 when n_i = 0;
 *   s_ij = (dot_ij * inv_i) * inv_j, +0 when either norm is 0.
 * The neighbours of i are the K genes j != i with the largest s_ij, ordered by s_ij descending, equal values by j
 * ascending: idx [m][K] int32 and sim [m][K] float64, the same bits whatever the grid or the split.
 * g2v_nbr_splits: the number of column splits of g2v_nbr_partial for m genes on the current device (a function of m
 *   and the SM count only); 0 on error.  The partial lists take splits * m * K entries of each type.
 * g2v_nbr_norms: inv [m].
 * g2v_nbr_partial: per split y and row i, the list of row i over split y's column range at [(y * m + i) * K], padded
 *   with j = -1, s = -inf when the range holds fewer than K genes.  With one split the lists are the result: pass idx
 *   and sim as part_idx and part_sim.
 * g2v_nbr_merge: splits > 1 (must equal g2v_nbr_splits(m)) partial lists -> idx, sim.
 * Out-of-range sizes fail with nothing launched.  One launch each, never synchronises. */
#define G2V_NBR_MAX_K 64
#define G2V_NBR_MAX_GENES (1 << 30)
int32_t g2v_nbr_splits(int64_t m);
int g2v_nbr_norms(const float *W, int64_t m, int32_t D, double *inv, void *stream);
int g2v_nbr_partial(const float *W, const double *inv, int64_t m, int32_t D, int32_t K, int32_t *part_idx,
                    double *part_sim, void *stream);
int g2v_nbr_merge(const int32_t *part_idx, const double *part_sim, int32_t splits, int64_t m, int32_t K, int32_t *idx,
                  double *sim, void *stream);

/* ---------------------------------------------------------------------------------------
 * Best-of-R k-means (k = 3) restarts of the L-groups (DESIGN.md §4.26; g2vec_b200/kmeans.py does the host side).
 * W [n][D] float32 row-major, 3 <= n <= G2V_KM_MAX_GENES, D >= 1, every value finite; x_i = (double) W_i.
 * dist(i, c) = the float64 chain acc = acc + t * t, t = x_id - c_d, d ascending from +0, every operation rounded
 * separately (no fma).  A chunk holds R' <= G2V_KM_MAX_RESTARTS restarts in slots 0 .. R'-1; slot s is restart
 * r_begin + s, whose seeding draws come from draw64(seed, 2^62 + r_begin + s, t).  Per slot: centres [3][D] double at
 * [s * 3 * D], labels [n] int8 and mind [n] double at [s * n], flags (bit c: cluster c holds a row, bit 3: a label
 * changed), state (0 running, 1 done).  `active` lists the n_active slots a launch works on.  Sums run in blocks of
 * G2V_KM_BLOCK consecutive rows (nb = ceil(n / G2V_KM_BLOCK)): psum [R'][nb][3][D] double, pcnt [R'][nb][3] int32,
 * pin [R'][nb] double.
 * g2v_km_assign: kc in [1, 3] centres; mind_i = min over c < kc of dist(i, c).  With kc = 3 also labels_i = the argmin
 *   (ties: the lower c) and the flags (integer atomics; the caller zeroes them once, g2v_km_update resets them).
 * g2v_km_seed: k-means++ pick t in [0, 2] of every slot 0 .. R'-1 (t > 0 reads mind of the first t centres): writes
 *   seeds [s * 3 + t] (a row) and centre t = x of that row.
 * g2v_km_blocks: per active slot and block, the chain of x over the block's rows of each cluster, the counts and the
 *   chain of mind.
 * g2v_km_update: per active slot, one Lloyd decision at iteration it (1-based) of max_iter: stop (state = 1, inertia,
 *   n_iter = it) when it == max_iter or (it > 1, no label changed and no cluster empty); otherwise the new centres
 *   (block chains / count) with each empty cluster, in ascending c, moved to a distinct row of largest mind (ties:
 *   the lowest row).  Resets the slot's flags.
 * g2v_km_contingency: table [R'][3][3] int64 += #{i : labels_si = a, best_i = b} (the caller zeroes it).
 * g2v_km_agree: count [n] int32 += #{s < R' : perm[s][labels_si] = best_i}, perm [R'][3] int8.
 * Out-of-range sizes fail with nothing launched.  One launch each, never synchronises; no floating-point atomics. */
#define G2V_KM_MAX_GENES (1 << 30)
#define G2V_KM_MAX_RESTARTS 1024
#define G2V_KM_BLOCK 256
int g2v_km_assign(const float *W, int64_t n, int32_t D, const double *centres, int32_t kc, const int32_t *active,
                  int32_t n_active, int8_t *labels, double *mind, int32_t *flags, void *stream);
int g2v_km_seed(const float *W, int64_t n, int32_t D, const double *mind, uint64_t seed, int64_t r_begin, int32_t t,
                int32_t n_slots, double *centres, int32_t *seeds, void *stream);
int g2v_km_blocks(const float *W, const int8_t *labels, const double *mind, int64_t n, int32_t D,
                  const int32_t *active, int32_t n_active, double *psum, int32_t *pcnt, double *pin, void *stream);
int g2v_km_update(const float *W, const double *mind, const double *psum, const int32_t *pcnt, const double *pin,
                  int64_t n, int32_t D, const int32_t *active, int32_t n_active, int32_t it, int32_t max_iter,
                  int32_t *flags, double *centres, int32_t *state, double *inertia, int32_t *n_iter, void *stream);
int g2v_km_contingency(const int8_t *labels, const int8_t *best, int64_t n, int32_t n_slots, int64_t *table,
                       void *stream);
int g2v_km_agree(const int8_t *labels, const int8_t *best, const int8_t *perm, int64_t n, int32_t n_slots,
                 int32_t *count, void *stream);

/* ---------------------------------------------------------------------------------------
 * Exact 2-D t-SNE of the gene vectors (DESIGN.md §4.27; g2vec_b200/tsne.py does the host side).
 * W [m][D] float32 row-major, 2 <= m <= G2V_TSNE_MAX_GENES, D >= 1, every value finite; x_i = (double) W_i.
 * P [m][m] double: first d, then the conditional affinities c, then the joint P.  Y, u, gains [m][2] double.
 * nb = ceil(m / G2V_TSNE_BLOCK); ws: g2v_tsne_workspace_bytes(m) bytes (0 for an m out of range), laid out as the
 * block partials [nb][5][m], the row chains [5][m] and the row-block chains of Z [nb].
 * g2v_tsne_dist: d_ij = the float64 chain acc = acc + t * t, t = x_id - x_jd, d ascending from +0, every operation
 *   rounded separately (no fma); d_ji has the bits of d_ij and d_ii = +0.
 * g2v_tsne_affinity: per row i, scikit-learn's perplexity bisection on the row of d (1 <= perplexity < m, at most 100
 *   evaluations, tolerance float32(1e-5) on |H - log perplexity|, a row sum of 0 taken as float32(1e-8), j = i left
 *   out); writes beta [m] double (the beta the row was computed from), steps [m] int32 (the 0-based evaluation that
 *   met the tolerance, 100 if none did) and overwrites the row with c_ij = exp(-d_ij beta_i) / S_i, c_ii = 0.
 * g2v_tsne_symmetrize: in place P_ij = (c_ij + c_ji) / (2m); P is symmetric bit for bit and P_ii = 0.
 * g2v_tsne_grad: per row i and column block b, the chains over the block's j != i (ascending) of w = 1 / (1 + d),
 *   p_ij w t_c and w^2 t_c, t_c = y_ic - y_jc, d = t_0 t_0 + t_1 t_1, into the block partials of ws.
 * g2v_tsne_update: iteration it >= 0 from the partials of g2v_tsne_grad at the current Y: per row the chains of the
 *   block partials, Z = the chain of Z_i in blocks of 256 rows, g = 4 ((alpha A) - (R / Z)), then scikit-learn's gains
 *   (+0.2 / *0.8, at least 0.01), momentum and step with learning rate eta > 0 (alpha = 12, momentum 0.5 for it < 250,
 *   else 1 and 0.8; u and the gains start over at 0 and 1 at it = 0 and it = 250).
 * g2v_tsne_kl: kl [1] double = sum over i != j of p_ij log(max(p_ij, eps) / max(w_ij / Z, eps)) at Y, in a fixed
 *   order (overwrites ws).
 * Out-of-range sizes fail with nothing launched.  Never synchronises; no atomics, no tensor cores. */
#define G2V_TSNE_MAX_GENES 32768
#define G2V_TSNE_BLOCK 256
size_t g2v_tsne_workspace_bytes(int64_t m);
int g2v_tsne_dist(const float *W, int64_t m, int32_t D, double *P, void *stream);
int g2v_tsne_affinity(double *P, int64_t m, double perplexity, double *beta, int32_t *steps, void *stream);
int g2v_tsne_symmetrize(double *P, int64_t m, void *stream);
int g2v_tsne_grad(const double *P, const double *Y, int64_t m, double *ws, void *stream);
int g2v_tsne_update(double *ws, int64_t m, int32_t it, double eta, double *Y, double *u, double *gains, void *stream);
int g2v_tsne_kl(const double *P, const double *Y, int64_t m, double *ws, double *kl, void *stream);

/* ---------------------------------------------------------------------------------------
 * Phenotype-permutation gene-set enrichment (GSEA) of the good / poor contrast (DESIGN.md §4.28; g2vec_b200/gsea.py
 * does the host side).  A row is one labelling (the observed one, or a permutation from g2v_perm_labels) with its
 * exact sums A [n_b][G] from g2v_perm_sums over the genes in their input order; n, k, Q, W as for g2v_perm_tally, and
 * s = +1 when the selected group is label 1, -1 when it is label 0.  2 <= G <= G2V_GSEA_MAX_GENES, 1 <= n_b <=
 * G2V_GSEA_MAX_ROWS with n_b * G < 2^31.
 * g2v_gsea_keys: per row and gene N = n A - k Q, r = (double)(s N) / sqrt(W) (+0 when W = 0), rq = rint(r 2^32);
 *   u [n_b][G] = |rq| and key [n_b][G] = ((2^32 - rq) << 20) | g: ascending keys order a row by rq descending, ties
 *   by gene ascending.
 * g2v_gsea_rank: pos [n_b][G] int32 = the 0-based rank of each gene in its row's key order.  workspace:
 *   g2v_gsea_rank_workspace_bytes(n_b, G) bytes of device scratch (0 for sizes out of range).
 * g2v_gsea_es: es [n_b][n_sets] = the enrichment score of every set in every row.  The sets are CSR over the genes:
 *   set_ptr [n_sets + 1], set_gene [set_ptr[n_sets]] (distinct genes per set); max_k >= the largest set, 1 <= max_k
 *   <= min(G2V_GSEA_MAX_SET_SIZE, G - 1).  With the members' ranks sorted, p_1 < ... < p_k, their weights u_j,
 *   S_j = u_1 + ... + u_j (exact), N_R = S_k and m_j = p_j - (j - 1):
 *     D+ = max(0, max_j (S_j / N_R - m_j / (G - k))),  D- = min(0, min_j (S_(j-1) / N_R - m_j / (G - k))),
 *   each term three correctly rounded float64 operations; ES = D+ if D+ >= -D-, else D-; +0 when N_R = 0.
 * g2v_gsea_norm: es [B][n_sets] of the permutations and es_obs [n_sets] of the observed labelling -> per set
 *   mean_pos = the mean of the es >= 0 and mean_neg = the mean of |es| over es < 0 (float64 sums in b order; NaN when
 *   empty), nes_obs = es_obs / mean_pos (es_obs >= 0) or es_obs / mean_neg, NaN when that side is empty; nes [B][n_sets]
 *   = each es over the mean of its own side, or NaN for the whole column of a set whose nes_obs is NaN; counts
 *   [3][n_sets] int64 = #{b: es >= 0}, #{b: es < 0} and #{b: es >= es_obs} (es_obs >= 0) or #{b: es <= es_obs}.
 *   B * n_sets <= G2V_GSEA_MAX_ES.
 * Out-of-range sizes fail with nothing launched.  Never synchronises; no floating-point atomics. */
#define G2V_GSEA_MAX_GENES (1 << 20)
#define G2V_GSEA_MAX_ROWS 65535
#define G2V_GSEA_MAX_SETS (1 << 28)
#define G2V_GSEA_MAX_SET_SIZE 4096
#define G2V_GSEA_MAX_PERMUTATIONS (1 << 20)
#define G2V_GSEA_MAX_ES (1 << 28)
int g2v_gsea_keys(const int64_t *A, int64_t n_b, int32_t G, int32_t n, int32_t k, int32_t s, const int64_t *Q,
                  const double *W, uint64_t *key, uint64_t *u, void *stream);
size_t g2v_gsea_rank_workspace_bytes(int64_t n_b, int32_t G);
int g2v_gsea_rank(const uint64_t *key, int64_t n_b, int32_t G, int32_t *pos, void *workspace, size_t workspace_bytes,
                  void *stream);
int g2v_gsea_es(const int32_t *pos, const uint64_t *u, int64_t n_b, int32_t G, const int32_t *set_ptr,
                const int32_t *set_gene, int32_t n_sets, int32_t max_k, double *es, void *stream);
int g2v_gsea_norm(const double *es, int64_t B, int32_t n_sets, const double *es_obs, double *nes, double *mean_pos,
                  double *mean_neg, double *nes_obs, int64_t *counts, void *stream);

/* ---------------------------------------------------------------------------------------
 * Cross-validated prediction of the good / poor label from a gene signature (DESIGN.md §4.29; g2vec_b200/signature.py
 * does the host side).  n samples (3 <= n <= G2V_SIG_MAX_SAMPLES) with y [n] in {0, 1}; K repeats (1 <= K <=
 * G2V_SIG_MAX_REPEATS) of stratified F-fold splits (2 <= F <= G2V_SIG_MAX_FOLDS); signatures of p sorted distinct gene
 * indices (1 <= p <= min(G2V_SIG_MAX_SIZE, G)).  A fit is (signature s, repeat k, fold f), numbered (s K + k) F + f.
 * g2v_sig_folds: fold [K][n] int8.  For repeat k and class c the class's samples in ascending order are Fisher-Yates
 *   shuffled (draw s swaps position m-1-s with umulhi(draw64(seed, 2^61 + 2k + c, s), m - s)); the sample at shuffled
 *   position t goes to fold t mod F.  F <= n / 2 (the caller keeps F <= min(n0, n1)).
 * g2v_sig_draw: genes [count][p] int32 for random signatures r = r_begin .. r_begin + count - 1 (1 <= r <=
 *   G2V_SIG_MAX_RANDOM): Floyd's sampling with u_t = draw64(seed, 2^61 + 2^40 + r, t), j = G - p + t,
 *   v = umulhi(u_t, j + 1), v if new else j; sorted ascending.
 * g2v_sig_fit: one fit per CTA.  X [G][n_pad] float64 (gene-major, n_pad >= n); genes [n_sig][p].  Per fit, on the
 *   samples outside fold f: each feature standardised by the training mean and population SD (mu = the value, SD = 1
 *   for a feature whose training values are all equal), then the ridge logistic loss sum log(1 + e^eta) - y eta +
 *   |beta|^2 / 2 (intercept unpenalised) minimised by damped Newton from 0: Cholesky solve of H d = g, Armijo halving
 *   (at most 40) with constant 1e-4, stop after the step with max |t d| <= 1e-10, at most 100 iterations.
 *   scores [n_sig][K][n] = the out-of-fold logit of every sample; n_iter and converged [n_sig * K * F]; beta
 *   [beta_rows][K][F][p + 1] (intercept first) for the first beta_rows signatures (beta may be NULL when 0).
 *   g2v_sig_fit_smem_bytes(p): the fit kernel's dynamic shared memory (0 for p out of range).
 * g2v_sig_auc: per fit over its test fold, auc = (2 #{pos > neg} + #{pos == neg}) / (2 n_pos n_neg) and acc =
 *   #{(score > 0) == y} / n_test, from exact integer counts.  cap >= the largest test fold (shared memory of cap
 *   doubles); a fold larger than cap gets NaN.
 * n_sig K F <= G2V_SIG_MAX_FITS.  Out-of-range sizes fail with nothing launched.  Never synchronises; no floating-point
 * atomics. */
#define G2V_SIG_MAX_SAMPLES 32768
#define G2V_SIG_MAX_SIZE 128
#define G2V_SIG_MAX_FOLDS 100
#define G2V_SIG_MAX_REPEATS 100
#define G2V_SIG_MAX_RANDOM 65536
#define G2V_SIG_MAX_FITS (1 << 24)
int g2v_sig_folds(const uint8_t *y, int32_t n, int32_t K, int32_t F, uint64_t seed, int8_t *fold, void *stream);
int g2v_sig_draw(int32_t G, int32_t p, uint64_t seed, int64_t r_begin, int64_t count, int32_t *genes, void *stream);
size_t g2v_sig_fit_smem_bytes(int32_t p);
int g2v_sig_fit(const double *X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *y, const int8_t *fold, int32_t K,
                int32_t F, const int32_t *genes, int32_t n_sig, int32_t p, double *scores, int32_t *n_iter,
                uint8_t *converged, double *beta, int32_t beta_rows, void *stream);
int g2v_sig_auc(const double *scores, const uint8_t *y, const int8_t *fold, int32_t n, int32_t K, int32_t F,
                int32_t n_sig, int32_t cap, double *auc, double *acc, void *stream);

/* ---------------------------------------------------------------------------------------
 * Cross-validated survival prediction from a gene signature: ridge Cox regression (DESIGN.md §4.33;
 * g2vec_b200/survival_cv.py does the host side).  The sizes are bounded as for g2v_sig_*: 3 <= n <=
 * G2V_SIG_MAX_SAMPLES, 1 <= K <= G2V_SIG_MAX_REPEATS, 2 <= F <= min(G2V_SIG_MAX_FOLDS, n / 2), 1 <= p <=
 * min(G2V_SIG_MAX_SIZE, G), 1 <= n_sig and n_sig K F <= G2V_SIG_MAX_FITS.  Samples are in time positions (time
 * descending, ties by sample index); flags [n] uint8 per position: bit 0 event, bit 1 last position of its time group.
 * fold [K][n] int8 over the positions (g2v_sig_folds with y = the event bits).  A fit is (s, k, f), numbered
 * (s K + k) F + f.
 * g2v_cox_fit: one fit per CTA.  X [G][n_pad] float64 (gene-major over the positions, n_pad >= n); genes [n_sig][p].
 *   Per fit, on the positions outside fold f: each feature standardised as g2v_sig_fit does (no intercept), then the
 *   Breslow negative log partial likelihood plus |beta|^2 / 2 minimised by g2v_sig_fit's damped Newton.  ell
 *   [n_sig * K * F][n] float64 is scratch.  scores [n_sig][K][n] = the out-of-fold eta of every position; n_iter and
 *   converged [n_sig * K * F]; beta [beta_rows][K][F][p] for the first beta_rows signatures (beta may be NULL when
 *   0).  g2v_cox_fit_smem_bytes(p): the fit kernel's dynamic shared memory (0 for p out of range).
 * g2v_cox_concordance: counts [n_sig * K * F][3] int64 over the test fold of each fit: the pairs (i, j) with
 *   grp[i] > grp[j] (grp [n] int32: the time group of each position, numbered in descending time) and i an event, and
 *   of those the ones with score_i > score_j and score_i == score_j.  A test fold of at most cap positions (0 <= cap
 *   <= min(n, G2V_COX_MAX_STAGED)) is staged in cap * 12 bytes of shared memory; a larger one is read from global
 *   memory.
 * Out-of-range sizes fail with nothing launched.  Never synchronises; no floating-point atomics. */
#define G2V_COX_MAX_STAGED 18432
size_t g2v_cox_fit_smem_bytes(int32_t p);
int g2v_cox_fit(const double *X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *flags, const int8_t *fold,
                int32_t K, int32_t F, const int32_t *genes, int32_t n_sig, int32_t p, double *ell, double *scores,
                int32_t *n_iter, uint8_t *converged, double *beta, int32_t beta_rows, void *stream);
int g2v_cox_concordance(const double *scores, const uint8_t *flags, const int32_t *grp, const int8_t *fold, int32_t n,
                        int32_t K, int32_t F, int32_t n_sig, int32_t cap, int64_t *counts, void *stream);

/* ---------------------------------------------------------------------------------------
 * Label-permutation test of differential co-expression for every network pair (DESIGN.md §4.30; g2vec_b200/diffcoex.py
 * does the host side).  A row is one labelling: an indicator [S_pad] u8 of its selected samples (g2v_perm_labels'
 * rows, or the all-ones and observed rows), padding 0.  q [G][S_pad] int32, gene-major, |q| <= 2^16, padding 0.
 * Pairs e = 0 .. E-1 are (pair_i[e], pair_j[e]), genes in [0, G).  1 <= n_b <= G2V_DCX_MAX_ROWS, 1 <= E <=
 * G2V_DCX_MAX_PAIRS, S_pad a multiple of 32 in [32, G2V_DCX_MAX_SAMPLES].
 * g2v_dcx_sums: S[r][e] = sum_s M[r][s] q[pair_i[e]][s] q[pair_j[e]][s], exact (FP64 mma.sync m8n8k4, every partial
 *   sum an integer <= 2^47).  Exactly one of P and D is given:
 *   P [n_b][E] int64: the sums (A .. P_tot, n and k unused; pairs (g, g) give sum_s q_g^2);
 *   D [n_b][E] float64: every row has k selected samples of n (4 <= k <= n - 4); group 1 = the selected samples, group
 *     2 = the others, with A [n_b][G] (g2v_perm_sums' sums of q), Bq [n_b][G] (sums of q^2), and the all-sample totals
 *     A_tot, B_tot [G] and P_tot [E] giving group 2 by subtraction.  Per group (size m): C = m P - A_i A_j and
 *     V_g = m B_g - A_g^2 (int64, exact), r = ll2double(C) / sqrt(ll2double(V_i) * ll2double(V_j)) clamped to [-1, 1],
 *     0 when V_i or V_j is 0; D = 0 when r1 = r2, else |r2 - r1| / (1 - r1 r2), every operation correctly rounded.
 * g2v_dcx_tally: per row of D, count[e] += D[e] >= D_obs[e];  count_maxt[e] += (max over e' >= e of D[e']) >=
 *   D_obs[e].  Integer atomics only; the counts do not depend on the grid or on how the rows are chunked.
 * Out-of-range sizes fail with nothing launched.  One launch each, never synchronises. */
#define G2V_DCX_MAX_SAMPLES 32768
#define G2V_DCX_MAX_ROWS (1 << 20)
#define G2V_DCX_MAX_PAIRS (1 << 26)
int g2v_dcx_sums(const uint8_t *M, int64_t n_b, int32_t S_pad, const int32_t *q, int32_t G, const int32_t *pair_i,
                 const int32_t *pair_j, int64_t E, int32_t n, int32_t k, const int64_t *A, const int64_t *Bq,
                 const int64_t *A_tot, const int64_t *B_tot, const int64_t *P_tot, int64_t *P, double *D,
                 void *stream);
int g2v_dcx_tally(const double *D, int64_t n_b, int64_t E, const double *D_obs, int64_t *count, int64_t *count_maxt,
                  void *stream);

/* ---------------------------------------------------------------------------------------
 * Network-propagated gene scores with a label-permutation test, NetRank (DESIGN.md §4.35; g2vec_b200/netrank.py does
 * the host side).  A labelling is the observed one or a row of g2v_perm_labels, with its exact sums A [n_b][G] from
 * g2v_perm_sums over the genes in their input order; n, k, Q, W as for g2v_perm_tally.  Columns: S and x are gene-major
 * [G][ld] float64, column b = labelling b of the launch, 1 <= n_b <= ld <= G2V_NR_MAX_ROWS.  1 <= G <=
 * G2V_NR_MAX_GENES.  The network is CSR over the genes: rowptr [G + 1] and col [rowptr[G]] int32, each row's
 * neighbours ascending; w [G] float64 = 1 / deg (any value for a gene without neighbours).
 * g2v_nr_seed: S[g][b] = sqrt(rho), rho = (double) N * (double) N / W[g] with N = n A[b][g] - k Q[g] (0 when W = 0).
 * g2v_nr_step: one power iteration on the columns c0 .. c0 + n_cols - 1: for every gene j (rows [G] int32 lists each
 *   gene once, in the order the warps take them), acc = +0, then acc = acc + x_in[i][b] * w[i] over the neighbours i
 *   of j in CSR order, and x_out[j][b] = (1 - d) * S[j][b] + d * acc, with 1 - d computed on the host, every operation
 *   correctly rounded (no fma).  0 <= d <= G2V_NR_MAX_DAMPING; x_in may be S, x_out must be neither.
 * g2v_nr_tile_cols: the columns of a tile whose S and two x buffers fit in half the L2 of the current device (a
 *   multiple of 32, at least 32); 0 for G out of range.
 * g2v_nr_tally: count [G] int64 += #{b < n_b : x[j][b] >= score_obs[j]} (integer adds, one warp per gene).
 * Out-of-range sizes fail with nothing launched.  One launch each, never synchronises; no floating-point atomics. */
#define G2V_NR_MAX_GENES (1 << 24)
#define G2V_NR_MAX_ROWS (1 << 20)
#define G2V_NR_MAX_DAMPING 0.95
int g2v_nr_seed(const int64_t *A, int64_t n_b, int32_t G, int32_t n, int32_t k, const int64_t *Q, const double *W,
                double *S, int64_t ld, void *stream);
int g2v_nr_step(const int32_t *rowptr, const int32_t *col, const double *w, const int32_t *rows, const double *S,
                const double *x_in, double *x_out, int32_t G, int64_t ld, int64_t c0, int64_t n_cols, double damping,
                void *stream);
int64_t g2v_nr_tile_cols(int32_t G);
int g2v_nr_tally(const double *x, int32_t G, int64_t n_b, int64_t ld, const double *score_obs, int64_t *count,
                 void *stream);

/* ---------------------------------------------------------------------------------------
 * Cross-validated lasso / elastic-net logistic regression over every gene, the glmnet path (DESIGN.md §4.37;
 * g2vec_b200/lasso.py does the host side).  n samples (3 <= n <= G2V_SIG_MAX_SAMPLES) with y [n] in {0, 1}, X [G][n_pad]
 * float64 gene-major (n_pad >= n, a multiple of 4), fold [K][n] from g2v_sig_folds.  Global fit 0 uses every sample,
 * fit 1 + k F + f the samples outside fold f of repeat k; a launch covers fits fit0 .. fit0 + fits - 1 (a chunk) whose
 * state lives in ws (g2v_lasso_workspace_bytes(G, n_pad, fits) bytes, 0 for sizes out of range).  Per fit and lambda
 * the objective is  -(1/n_fit) sum [y eta - log(1 + e^eta)] + lambda [alpha |beta|_1 + (1 - alpha)/2 |beta|^2],
 * eta = b0 + z^T beta, z each gene standardised over the fit's training samples (population SD; a constant gene gets
 * z = 0 and never enters), b0 unpenalised, 0 < alpha <= 1.
 * g2v_lasso_standardise: the standardisation, the null model and a cleared state; entry [fits][G] int16 = -1 and
 *   entry_abs [fits][G] = 0 (both offset to the chunk's first fit).
 * g2v_lasso_grad: the gradient of the smooth part of every fit of the chunk at its current solution (one DGEMM on the
 *   FP64 tensor cores).  g2v_lasso_lambda_max: lam_max [1] (device) = max_j |g_j| / max(alpha, 1e-3) of the chunk's
 *   first fit (call it after standardise and one grad).
 * g2v_lasso_cd: round r of lambda index k (lam_prev = lambda_{k-1}, lambda_0 at k = 0).  Per fit not yet done: the
 *   largest KKT violation of the current solution (|g_0|, |g_j| - lambda alpha at beta_j = 0, |g_j + lambda alpha
 *   sign beta_j| otherwise); at most G2V_LASSO_EPS, or after 100 Newton steps at this lambda, the fit records lambda k:
 *   df, dev_ratio, n_iter, kkt [fits][G2V_LASSO_N_LAMBDA] at [f][k], entry / entry_abs of genes entering, path [k][G + 1]
 *   (intercept then beta of the chunk's first fit, may be NULL) and its stop rules; else it extends its working set (the sequential strong
 *   rule at r = 0, KKT violators after) and runs proximal Newton with coordinate descent.  ctl [2] int32: ctl[0] = the
 *   fits still pending after the call, ctl[1] = the chunk's first fit's path length once it stopped (-1 before).  A fit
 *   whose ever-active genes would exceed G2V_LASSO_MAX_ACTIVE keeps its previous solution and stops with path length
 *   k; one whose deviance ratio exceeds 0.999, or at k >= 4 rose by less than 1e-5 of itself, stops with k + 1.  A
 *   stopped fit reports its last solution at later lambdas.
 * g2v_lasso_score: for each fold fit of the chunk and each sample i of its test fold, scores [L][K][n] at [k][rep][i] =
 *   eta_i and dev the binomial deviance -2 log p(y_i) with p clamped to [1e-5, 1 - 1e-5].
 * Out-of-range sizes fail with nothing launched.  Never synchronises; no floating-point atomics. */
#define G2V_LASSO_N_LAMBDA 100
#define G2V_LASSO_MAX_ACTIVE 512
#define G2V_LASSO_MAX_GENES (1 << 20)
#define G2V_LASSO_EPS 1e-7
size_t g2v_lasso_workspace_bytes(int32_t G, int64_t n_pad, int32_t fits);
int g2v_lasso_standardise(const double *X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *y, const int8_t *fold,
                          int32_t K, int32_t F, int32_t fit0, int32_t fits, void *ws, int16_t *entry,
                          double *entry_abs, void *stream);
int g2v_lasso_grad(const double *X, int32_t G, int32_t n, int64_t n_pad, int32_t fits, void *ws, double lam,
                   double alpha, void *stream);
int g2v_lasso_lambda_max(int32_t G, int64_t n_pad, int32_t fits, void *ws, double alpha, double *lam_max,
                         void *stream);
int g2v_lasso_cd(const double *X, int32_t G, int32_t n, int64_t n_pad, const uint8_t *y, int32_t fits, void *ws,
                 int32_t k, double lam, double lam_prev, double alpha, int32_t round, int32_t *df, double *dev_ratio,
                 int32_t *n_iter, double *kkt, int16_t *entry, double *entry_abs, double *path, int32_t *ctl,
                 void *stream);
int g2v_lasso_score(const uint8_t *y, const int8_t *fold, int32_t n, int64_t n_pad, int32_t K, int32_t F, int32_t fit0,
                    int32_t fits, void *ws, int32_t G, int32_t k, double *scores, double *dev, void *stream);

/* ---------------------------------------------------------------------------------------
 * Permutation Cox score test of every gene against survival (DESIGN.md §4.31; g2vec_b200/survival.py does the host
 * side).  n samples (3 <= n <= G2V_SURV_MAX_SAMPLES) with survival records; the time order lists them by time
 * descending and slot [n] int32 is its inverse (slot[s] = the time position of sample s).  Permutations are numbered
 * b = 1 .. B, B <= G2V_SURV_MAX_PERMUTATIONS.
 * g2v_surv_rows: idx [n_b][n] uint16, row r = permutation b = b_begin + 1 + r: pi_b is Fisher-Yates on the identity
 *   with the draws of g2v_perm_labels' row b (for i = n-1 down to 1: j = hi64(draw64(seed, 2^63 + b, n-1-i) * (i+1)),
 *   swap i and j), and idx[slot[pi_b(s)]] = s: sample s's expression meets sample pi_b(s)'s record.  A row depends
 *   only on (slot, seed, b).
 * g2v_surv_scores: T [n_b][G] float64 from q [n][G] int32 (sample-major, |q| <= 2^16) and the rows idx [n_b][n] (the
 *   time order itself is the observed row).  flags [n] u8 per time position: bit 0 = an event, bit 1 = the last
 *   position of its group of equal times; a, c [n] float64 at the group ends: a = 1 / S0, c = d / (S0 S0) with S0 =
 *   the position + 1 and d the group's events.  Scanning the positions p = 0 .. n-1 with x = q[idx[r][p]][g]:
 *   S1 += x, S2 += x^2, and over the group's events E1 += x, d += 1 (exact int64); at the end of a group with d > 0,
 *   num_u = S0 E1 - d S1, num_v = S0 S2 - S1^2, U = U + ll2double(num_u) * a[p], V = V + ll2double(num_v) * c[p]
 *   (each operation correctly rounded, from U = V = +0); then T = (U * U) / V, 0 when V = 0.  UV (may be NULL):
 *   [2][n_b][G] float64, U then V.
 * Out-of-range sizes fail with nothing launched.  One launch each, never synchronises; no floating-point atomics.
 * The counts of T >= T_obs are g2v_dcx_tally's (E = G, the genes in rank order). */
#define G2V_SURV_MAX_SAMPLES 32768
#define G2V_SURV_MAX_PERMUTATIONS (1 << 20)
#define G2V_SURV_MAX_GENES (1 << 20)
int g2v_surv_rows(const int32_t *slot, int32_t n, uint64_t seed, int64_t b_begin, int64_t n_b, uint16_t *idx,
                  void *stream);
int g2v_surv_scores(const int32_t *q, int32_t n, int32_t G, const uint16_t *idx, int64_t n_b, const uint8_t *flags,
                    const double *a, const double *c, double *T, double *UV, void *stream);

/* ---------------------------------------------------------------------------------------
 * Between the two hot paths (SURVEY.md 8f-2): `tuple(sorted(path))` into a set (G2Vec.py:345,351) and
 * the removal of paths common to both groups (G2Vec.py:313).
 * g2v_paths_canonicalise: row i of nodes [n*L] (-1 or INT32_MAX padded) -> sorted [n*L] ascending with
 *   INT32_MAX padding, and a non-negative 64-bit key per row (equal rows => equal keys).
 * g2v_paths_mark: rows visited in key order (key_sorted[i] = key[perm[i]], ascending).  group == NULL:
 *   flag[i] = 1 iff row perm[i] is the first occurrence of its content (set semantics, exact: rows of a key
 *   run are compared in full).  group != NULL (0/1 per row): flag[i] = 1 iff no row of the other group has
 *   the same content (the row survives `pathSet - commonPath`).
 * ------------------------------------------------------------------------------------- */
int g2v_paths_canonicalise(const int32_t *nodes, int64_t n, int32_t L, int32_t *sorted, int64_t *key,
                           void *stream);
int g2v_paths_mark(const int32_t *rows, const int64_t *key_sorted, const int64_t *perm, const uint8_t *group,
                   int64_t n, int32_t L, uint8_t *flag, void *stream);

/* ---------------------------------------------------------------------------------------
 * Between the two hot paths, sort-free form (SURVEY.md 8f-2): from the canonical rows of BOTH groups (sorted,
 * INT32_MAX padded, with their 64-bit keys and lengths -- what g2v_walk_launch_packed writes with out_key) to the
 * trainer's input: `pathSet.add` (G2Vec.py:351), `pathSet - commonPath` (:313), the rows of integrate_pathSet
 * (:316-320) as CSR windows, and count_geneFreq (:288-308).
 * g2v_paths_set_select: keep[i] = 1 iff row i is the first occurrence of its content in its group (group[i] in
 *   {0,1}; NULL = one group) and no row of the other group has the same content.  totals (device, 3 x int64) =
 *   {rows kept, their total length, key collisions}; if collisions != 0 two different contents shared a key and the
 *   caller must use the exact sort-based functions above instead (never observed; ~n^2/2^64).
 * g2v_paths_set_emit: the kept rows in input order as CSR windows (rowptr [kept+1], gene [nnz], label [kept] = the
 *   row's group) and, if freq/code are given, code[g] = 0 / 1 / 2 / -1: more good paths / more poor / tie / gene in
 *   no kept path (freq: 2*V int32 scratch).  Synchronises the stream.
 * workspace: g2v_paths_set_workspace_bytes(n) bytes, the same buffer for both calls.
 * ------------------------------------------------------------------------------------- */
size_t g2v_paths_set_workspace_bytes(int64_t n);
int g2v_paths_set_select(const int32_t *rows, const int64_t *key, const uint8_t *group, const int32_t *len, int64_t n,
                         int32_t L, void *workspace, uint8_t *keep, int64_t *totals, void *stream);
int g2v_paths_set_emit(const int32_t *rows, const uint8_t *group, const int32_t *len, const uint8_t *keep, int64_t n,
                       int32_t L, int32_t V, const void *workspace, int64_t kept, int64_t nnz, int32_t *rowptr,
                       int32_t *gene, uint8_t *label, int32_t *freq, int8_t *code, void *stream);

/* ---------------------------------------------------------------------------------------
 * Test hooks (used by tests/ only): 64-bit draws 0..n-1 of one walker subsequence from the
 * kernel's own Philox, and the same words from curand's Philox4_32_10 generator
 * (curand_init(seed, subsequence, 0)), to prove the stream is curand-compatible.
 * ------------------------------------------------------------------------------------- */
/* Measurement hook: (mode 0) read / (mode 1) red.add a constant into the rows idx[0..n_idx) of a [*, D] float
 * table, D a multiple of 128 -- the memory operations of the CBOW kernels without the arithmetic; bench.py times it
 * on an L2-resident table to get the L2 ceiling the fused kernel is compared with.  sink: >= 1024 floats. */
int g2v_test_l2_rows(const float *table, float *grad, const int32_t *idx, int64_t n_idx, int32_t D, int32_t mode,
                     float *sink, void *stream);
int g2v_test_draws(uint64_t seed, uint64_t subsequence, int32_t n, uint64_t *out_dev, void *stream);
int g2v_test_curand_draws(uint64_t seed, uint64_t subsequence, int32_t n, uint64_t *out_dev,
                          void *stream);

#ifdef __cplusplus
}
#endif
#endif /* G2VEC_B200_H */
