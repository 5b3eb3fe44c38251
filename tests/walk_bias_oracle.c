/*
 * walk_bias_oracle.c -- scalar C restatement of the walk sampler with node2vec's in-out bias.  TEST INFRASTRUCTURE.
 *
 * The walk of oracle/g2v_oracle.c (g2v_oracle_walks: append, self-avoidance, <= L nodes, dead-end stop, one Philox
 * draw per step at draw index s) with one change at steps s >= 1, where the walker at v came from t: an unvisited
 * out-neighbour x of v weighs qw * a_near if x is in t's CSR row (the edge t -> x exists) and qw * a_far otherwise.
 * T = sum of the effective weights (uint64), r = floor(x * T / 2^64), next = first neighbour in ascending order whose
 * inclusive prefix exceeds r.  Step 0 has no previous node and uses qw.  Returns 0, or -1 on bad arguments.
 */
#include <stdint.h>
#include <stdlib.h>

static inline void philox_round(uint32_t c[4], const uint32_t k[2])
{
    uint64_t p0 = (uint64_t)0xD2511F53u * c[0];
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c[2];
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k[0];
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k[1];
    uint32_t n3 = (uint32_t)p0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}

/* 64-bit draw s of subsequence `subseq` (curand Philox4x32-10 layout, as g2v_oracle.c) */
static uint64_t draw64(uint64_t seed, uint64_t subseq, uint32_t s)
{
    uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    uint32_t c[4] = {s >> 1, 0u, (uint32_t)subseq, (uint32_t)(subseq >> 32)};
    for (int r = 0; r < 10; ++r) {
        philox_round(c, k);
        if (r < 9) { k[0] += 0x9E3779B9u; k[1] += 0xBB67AE85u; }
    }
    uint32_t lo = c[2 * (s & 1u)], hi = c[2 * (s & 1u) + 1];
    return ((uint64_t)hi << 32) | lo;
}

/* x in the ascending row [b, e) of col? */
static int in_row(const int32_t *col, int32_t b, int32_t e, int32_t x)
{
    for (int32_t j = b; j < e; ++j)
        if (col[j] == x) return 1;
    return 0;
}

int walk_bias_oracle_walks(const int32_t *rowptr, const int32_t *col, const uint32_t *qw,
                           int32_t V, int32_t L, uint64_t seed, uint32_t group,
                           int64_t walker_begin, int64_t walker_end, int64_t walker_stride,
                           uint32_t a_near, uint32_t a_far, int32_t *out_nodes, int32_t *out_len)
{
    if (V <= 0 || L <= 0 || walker_stride <= 0 || walker_begin < 0) return -1;
    if (a_near < 1 || a_near > 256 || a_far < 1 || a_far > 256) return -1;
    uint8_t *visited = (uint8_t *)calloc((size_t)V, 1);
    if (!visited) return -1;
    int64_t slot = 0;
    for (int64_t w = walker_begin; w < walker_end; w += walker_stride, ++slot) {
        int32_t *path = out_nodes + slot * (int64_t)L;
        int32_t cur = (int32_t)(w % V), prev = -1;
        uint64_t subseq = ((uint64_t)group << 40) + (uint64_t)w;
        int32_t n = 0;
        for (int32_t s = 0; s < L; ++s) {
            path[n++] = cur;
            visited[cur] = 1;
            if (s == L - 1) break;
            int32_t b = rowptr[cur], e = rowptr[cur + 1];
            uint64_t T = 0;
            for (int32_t j = b; j < e; ++j) {
                if (visited[col[j]]) continue;
                uint64_t m = prev < 0 ? 1 : in_row(col, rowptr[prev], rowptr[prev + 1], col[j]) ? a_near : a_far;
                T += (uint64_t)qw[j] * m;
            }
            if (T == 0) break;
            uint64_t x = draw64(seed, subseq, (uint32_t)s);
            uint64_t r = (uint64_t)(((unsigned __int128)x * T) >> 64);
            uint64_t acc = 0;
            int32_t nxt = -1;
            for (int32_t j = b; j < e; ++j) {
                if (visited[col[j]]) continue;
                uint64_t m = prev < 0 ? 1 : in_row(col, rowptr[prev], rowptr[prev + 1], col[j]) ? a_near : a_far;
                acc += (uint64_t)qw[j] * m;
                if (acc > r) { nxt = col[j]; break; }
            }
            prev = cur;
            cur = nxt;
        }
        for (int32_t i = 0; i < n; ++i) visited[path[i]] = 0;
        for (int32_t i = n; i < L; ++i) path[i] = -1;
        out_len[slot] = n;
    }
    free(visited);
    return 0;
}
