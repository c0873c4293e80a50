/*
 * cornac_oracle.c -- CPU restatement of the reference's BPR / MF / score hot path.
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load this library.
 * The product (cornac_b200/) never links, imports or calls anything in oracle/.
 *
 * Parity status: PINNED.  The reference's own tests hold no golden vectors for
 * trained BPR/MF parameters (SURVEY.md 8c), so this restatement is pinned
 *   (1) against tests/cornac/utils/test_fastdot.py:26-37 (known answers), and
 *   (2) against outputs of the UNMODIFIED compiled reference (baseline/_ref,
 *       built by baseline/build_ref.sh) committed as .npz fixtures under tests/golden/ by
 *       tests/golden/make_golden.py and checked by tests/test_oracle_golden.py.
 *
 * Every function cites the reference file:line it follows (paths relative to
 * the reference root).  Arithmetic is written out in scalar f32 with
 * -ffp-contract=off so the operation order is exactly the one in the .pyx
 * source; the compiled reference uses -O3 -ffast-math (setup.py:130-137), so
 * agreement with it is to ~1e-7 relative, not bit-for-bit.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORA_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------- */
/* A1: boost::random::mt19937 (external/boost/random/mersenne_twister.hpp:623)
 * = the standard MT19937: init_genrand seeding, tempered 32-bit outputs.     */
typedef struct {
    uint32_t mt[624];
    int idx;
} ora_mt19937;

ORA_API void ora_mt_seed(ora_mt19937 *g, uint32_t seed)
{
    g->mt[0] = seed;
    for (int i = 1; i < 624; ++i)
        g->mt[i] = 1812433253u * (g->mt[i - 1] ^ (g->mt[i - 1] >> 30)) + (uint32_t)i;
    g->idx = 624;
}

static void ora_mt_twist(ora_mt19937 *g)
{
    uint32_t *mt = g->mt;
    for (int i = 0; i < 624; ++i) {
        uint32_t y = (mt[i] & 0x80000000u) | (mt[(i + 1) % 624] & 0x7fffffffu);
        uint32_t v = mt[(i + 397) % 624] ^ (y >> 1);
        if (y & 1u) v ^= 0x9908b0dfu;
        mt[i] = v;
    }
    g->idx = 0;
}

ORA_API uint32_t ora_mt_next(ora_mt19937 *g)
{
    if (g->idx >= 624) ora_mt_twist(g);
    uint32_t y = g->mt[g->idx++];
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}

/* A1: boost::random::uniform_int_distribution<long>(0, hi)(mt19937&)
 * (external/boost/random/uniform_int_distribution.hpp:49-228), min_value = 0,
 * brange = 0xFFFFFFFF.  Returns a value in [0, hi] INCLUSIVE and consumes a
 * data-dependent number of engine outputs.                                    */
ORA_API uint64_t ora_boost_uniform_u64(ora_mt19937 *g, uint64_t range)
{
    const uint64_t brange = 0xFFFFFFFFull;
    if (range == 0) return 0;                                   /* :65-66  */
    if (range == brange) return (uint64_t)ora_mt_next(g);       /* :67-71  */
    if (range < brange) {                                       /* :192-226 */
        uint32_t r32 = (uint32_t)range;
        uint32_t bucket = 0xFFFFFFFFu / (r32 + 1u);
        if (0xFFFFFFFFu % (r32 + 1u) == r32) ++bucket;
        for (;;) {
            uint32_t r = ora_mt_next(g) / bucket;
            if (r <= r32) return r;
        }
    }
    /* brange < range: concatenate base-2^32 digits with rejection (:72-176) */
    for (;;) {
        uint64_t limit;
        if (range == UINT64_MAX) {
            limit = range / (brange + 1);
            if (range % (brange + 1) == brange) ++limit;
        } else {
            limit = (range + 1) / (brange + 1);
        }
        uint64_t result = 0, mult = 1;
        int done = 0;
        while (mult <= limit) {
            result += (uint64_t)ora_mt_next(g) * mult;
            if (mult * brange == range - mult + 1) { done = 1; break; }
            mult *= brange + 1;
        }
        if (done) return result;
        uint64_t inc = ora_boost_uniform_u64(g, range / mult);
        if (UINT64_MAX / mult < inc) continue;
        inc *= mult;
        result += inc;
        if (result < inc) continue;
        if (result > range) continue;
        return result;
    }
}

/* Fill `out[n]` with n consecutive draws from [0, hi]; state carries on. */
ORA_API void ora_boost_uniform_fill(ora_mt19937 *g, int64_t hi, int64_t n, int64_t *out)
{
    for (int64_t s = 0; s < n; ++s) out[s] = (int64_t)ora_boost_uniform_u64(g, (uint64_t)hi);
}

/* ------------------------------------------------------------------------- */
/* A2: has_non_zero (cornac/models/bpr/recom_bpr.pyx:46-51):
 * std::binary_search over the user's sorted CSR row.                          */
static inline int ora_has_non_zero(const int32_t *indptr, const int32_t *indices,
                                   int64_t row, int32_t col)
{
    int64_t lo = indptr[row], hi = indptr[row + 1];
    while (lo < hi) {                       /* lower_bound */
        int64_t mid = lo + ((hi - lo) >> 1);
        if (indices[mid] < col) lo = mid + 1; else hi = mid;
    }
    return lo < indptr[row + 1] && indices[lo] == col;
}

/* One BPR triplet update, exactly the body of the prange loop in
 * BPR._fit_sgd (cornac/models/bpr/recom_bpr.pyx:241-267).  Returns 1 when the
 * sample was skipped, else 0; *correct is incremented when z < .5.            */
static int ora_mmmf_one(const int32_t *indptr, const int32_t *indices, int64_t u, int32_t i_id, int32_t j_id,
                        float *U, float *V, float *B, int k, float lr, float reg, int64_t *correct);

static inline int ora_bpr_one(const int32_t *indptr, const int32_t *indices,
                              int64_t u, int32_t i_id, int32_t j_id,
                              float *U, float *V, float *B, int k,
                              float lr, float reg, int use_bias, int64_t *correct)
{
    if (use_bias == 2) return ora_mmmf_one(indptr, indices, u, i_id, j_id, U, V, B, k, lr, reg, correct);
    if (ora_has_non_zero(indptr, indices, u, j_id)) return 1;      /* :241-243 */
    float *user = U + (size_t)u * k, *item_i = V + (size_t)i_id * k, *item_j = V + (size_t)j_id * k;
    float score = B[i_id] - B[j_id];                                /* :249 */
    for (int f = 0; f < k; ++f)                                     /* :250-251 */
        score = score + user[f] * (item_i[f] - item_j[f]);
    float z = (float)(1.0 / (1.0 + exp((double)score)));            /* :252 (libc double exp) */
    if (z < .5f) ++*correct;                                        /* :254-255 */
    for (int f = 0; f < k; ++f) {                                   /* :258-262 */
        float temp = user[f];
        user[f] += lr * (z * (item_i[f] - item_j[f]) - reg * user[f]);
        item_i[f] += lr * (z * temp - reg * item_i[f]);
        item_j[f] += lr * (-z * temp - reg * item_j[f]);
    }
    if (use_bias) {                                                 /* :265-267 */
        B[i_id] += lr * (z - reg * B[i_id]);
        B[j_id] += lr * (-z - reg * B[j_id]);
    }
    return 0;
}

/* MMMF variant of the loop body (cornac/models/mmmf/recom_mmmf.pyx:129-154): hinge instead of the
 * logistic loss -- a pair that is already ranked correctly (score > 0) is counted and left alone,
 * otherwise the update of BPR with z = 1; the item biases are always trained.  Selected by passing
 * use_bias == 2 to the epoch functions.                                                        */
static int ora_mmmf_one(const int32_t *indptr, const int32_t *indices, int64_t u, int32_t i_id, int32_t j_id,
                        float *U, float *V, float *B, int k, float lr, float reg, int64_t *correct)
{
    if (ora_has_non_zero(indptr, indices, u, j_id)) return 1;      /* :125-127 */
    float *user = U + (size_t)u * k, *item_i = V + (size_t)i_id * k, *item_j = V + (size_t)j_id * k;
    float score = B[i_id] - B[j_id];                                /* :133 */
    for (int f = 0; f < k; ++f)
        score = score + user[f] * (item_i[f] - item_j[f]);
    if (score > 0) { ++*correct; return 0; }                        /* :137-139 */
    for (int f = 0; f < k; ++f) {                                   /* :142-146 */
        float temp = user[f];
        user[f] += lr * (item_i[f] - item_j[f] - reg * user[f]);
        item_i[f] += lr * (temp - reg * item_i[f]);
        item_j[f] += lr * (-temp - reg * item_j[f]);
    }
    B[i_id] += lr * (1 - reg * B[i_id]);                            /* :149-150 */
    B[j_id] += lr * (-1 - reg * B[j_id]);
    return 0;
}

/* A4: one epoch of BPR._fit_sgd with num_threads = 1 (the seeded,
 * deterministic configuration, recom_bpr.pyx:132-133): nnz iterations, each
 * drawing i_index from rng_pos in [0, nnz-1] and j_index from rng_neg in
 * [0, n_neg-1] (both draws happen even when the sample is then skipped,
 * :235-243).  neg_item_ids = arange(num_items) (:186) so j_id = j_index.
 * Optional trace_i / trace_j (length nnz) record the drawn stream.            */
ORA_API void ora_bpr_fit_sgd(ora_mt19937 *rng_pos, ora_mt19937 *rng_neg,
                             int64_t nnz, int64_t n_neg,
                             const int32_t *user_ids, const int32_t *item_ids,
                             const int32_t *indptr,
                             float *U, float *V, float *B, int k,
                             float lr, float reg, int use_bias,
                             int64_t *correct, int64_t *skipped,
                             int64_t *trace_i, int32_t *trace_j)
{
    int64_t c = 0, sk = 0;
    for (int64_t s = 0; s < nnz; ++s) {
        int64_t i_index = (int64_t)ora_boost_uniform_u64(rng_pos, (uint64_t)(nnz - 1));
        int32_t i_id = item_ids[i_index];
        int32_t j_id = (int32_t)ora_boost_uniform_u64(rng_neg, (uint64_t)(n_neg - 1));
        if (trace_i) trace_i[s] = i_index;
        if (trace_j) trace_j[s] = j_id;
        sk += ora_bpr_one(indptr, item_ids, user_ids[i_index], i_id, j_id, U, V, B, k,
                          lr, reg, use_bias, &c);
    }
    *correct = c;
    *skipped = sk;
}

/* WBPR epoch (cornac/models/bpr/recom_wbpr.pyx:125-136): the same _fit_sgd loop called with
 * rng_neg = rng_pos (ONE shared mt19937, so each sample consumes "pos draw, then neg draw" from
 * the same stream) and neg_item_ids = X.indices, i.e. negatives are drawn in proportion to
 * item popularity: j_id = item_ids[j_index], j_index uniform over [0, nnz-1].              */
ORA_API void ora_wbpr_fit_sgd(ora_mt19937 *rng, int64_t nnz,
                              const int32_t *user_ids, const int32_t *item_ids, const int32_t *indptr,
                              float *U, float *V, float *B, int k,
                              float lr, float reg, int use_bias,
                              int64_t *correct, int64_t *skipped,
                              int64_t *trace_i, int32_t *trace_j)
{
    int64_t c = 0, sk = 0;
    for (int64_t s = 0; s < nnz; ++s) {
        int64_t i_index = (int64_t)ora_boost_uniform_u64(rng, (uint64_t)(nnz - 1));
        int64_t j_index = (int64_t)ora_boost_uniform_u64(rng, (uint64_t)(nnz - 1));
        int32_t j_id = item_ids[j_index];
        if (trace_i) trace_i[s] = i_index;
        if (trace_j) trace_j[s] = j_id;
        sk += ora_bpr_one(indptr, item_ids, user_ids[i_index], item_ids[i_index], j_id, U, V, B, k,
                          lr, reg, use_bias, &c);
    }
    *correct = c;
    *skipped = sk;
}

/* Same loop body driven by an explicit (i_index, j_id) stream, sequentially.
 * Used to check the GPU replay kernel on arbitrary streams.                   */
ORA_API void ora_bpr_replay(const int64_t *i_index, const int32_t *j_ids, int64_t n,
                            const int32_t *user_ids, const int32_t *item_ids,
                            const int32_t *indptr,
                            float *U, float *V, float *B, int k,
                            float lr, float reg, int use_bias,
                            int64_t *correct, int64_t *skipped)
{
    int64_t c = 0, sk = 0;
    for (int64_t s = 0; s < n; ++s) {
        int64_t ii = i_index[s];
        sk += ora_bpr_one(indptr, item_ids, user_ids[ii], item_ids[ii], j_ids[s], U, V, B, k,
                          lr, reg, use_bias, &c);
    }
    *correct = c;
    *skipped = sk;
}

/* ------------------------------------------------------------------------- */
/* f3: VEBPR (cornac/models/bpr/recom_vebpr.pyx).  One sample of the prange loop of
 * VEBPR._fit_sgd_viewloss (:239-335); v_id < 0 = the user has no viewed item (the BPR fall-back
 * branch, :246-275).  The expressions are the .pyx expressions with the .pyx types: `floating` = float,
 * the literals 1.0 / 50.0 are doubles, so (1.0 - alpha) * ... is evaluated in double like in the
 * generated C.  No item biases.  Returns 1 when skipped.                                         */
static inline float ora_clip50(float x)
{
    if (x > 50.0) x = 50.0; else if (x < -50.0) x = -50.0;        /* :258-261, :296-309 */
    return x;
}

static int ora_vebpr_one(const int32_t *indptr, const int32_t *indices,
                         const int32_t *view_indptr, const int32_t *view_indices,
                         int64_t u, int32_t i_id, int32_t v_id, int32_t j_id,
                         float *U, float *V, int k, float lr, float reg, float alpha, int64_t *correct)
{
    float *user = U + (size_t)u * k, *item_i = V + (size_t)i_id * k, *item_j = V + (size_t)j_id * k;
    if (v_id < 0) {                                                 /* :246-275 */
        if (ora_has_non_zero(indptr, indices, u, j_id)) return 1;
        float x_uij = 0.0;
        for (int f = 0; f < k; ++f) x_uij = x_uij + user[f] * (item_i[f] - item_j[f]);
        x_uij = ora_clip50(x_uij);
        float delta_ij = 1.0 / (1.0 + exp(x_uij));
        if (delta_ij < 0.5) ++*correct;
        for (int f = 0; f < k; ++f) {
            float u_old = user[f], i_old = item_i[f], j_old = item_j[f];
            user[f] -= lr * (-delta_ij * (i_old - j_old) + reg * u_old);
            item_i[f] -= lr * (-delta_ij * u_old + reg * i_old);
            item_j[f] -= lr * (delta_ij * u_old + reg * j_old);
        }
        return 0;
    }
    if (ora_has_non_zero(indptr, indices, u, j_id) || ora_has_non_zero(view_indptr, view_indices, u, j_id))
        return 1;                                                   /* :281-285 */
    float *item_v = V + (size_t)v_id * k;
    float x_uij = 0.0, x_uiv = 0.0, x_uvj = 0.0;
    for (int f = 0; f < k; ++f) {                                   /* :292-295 */
        x_uij = x_uij + user[f] * (item_i[f] - item_j[f]);
        x_uiv = x_uiv + user[f] * (item_i[f] - item_v[f]);
        x_uvj = x_uvj + user[f] * (item_v[f] - item_j[f]);
    }
    x_uij = ora_clip50(x_uij); x_uiv = ora_clip50(x_uiv); x_uvj = ora_clip50(x_uvj);
    float delta_ij = 1.0 / (1.0 + exp(x_uij));                      /* :312-314 */
    float delta_iv = 1.0 / (1.0 + exp(x_uiv));
    float delta_vj = 1.0 / (1.0 + exp(x_uvj));
    if (delta_ij < 0.5 && delta_iv < 0.5 && delta_vj < 0.5) ++*correct;
    for (int f = 0; f < k; ++f) {                                   /* :321-335 */
        float u_old = user[f], i_old = item_i[f], v_old = item_v[f], j_old = item_j[f];
        user[f] -= lr * (-delta_ij * (i_old - j_old) - alpha * delta_iv * (i_old - v_old)
                         - (1.0 - alpha) * delta_vj * (v_old - j_old) + reg * u_old);
        item_i[f] -= lr * (-delta_ij * u_old - alpha * delta_iv * u_old + reg * i_old);
        item_v[f] -= lr * (alpha * delta_iv * u_old - (1.0 - alpha) * delta_vj * u_old + reg * v_old);
        item_j[f] -= lr * (delta_ij * u_old + (1.0 - alpha) * delta_vj * u_old + reg * j_old);
    }
    return 0;
}

/* One epoch of VEBPR._fit_sgd_viewloss with num_threads = 1: three mt19937 streams (pos in [0, nnz-1], view and
 * neg in [0, n_items-1], :198-200); the view stream is consumed only for users WITH viewed items, the neg
 * stream always (:240-280).  trace_* (optional, length nnz) record (i_index, v_id or -1, j_id).            */
ORA_API void ora_vebpr_fit_sgd(ora_mt19937 *rng_pos, ora_mt19937 *rng_view, ora_mt19937 *rng_neg,
                               int64_t nnz, int64_t n_items,
                               const int32_t *user_ids, const int32_t *item_ids, const int32_t *indptr,
                               const int32_t *view_item_ids, const int32_t *view_indptr,
                               float *U, float *V, int k, float lr, float reg, float alpha,
                               int64_t *correct, int64_t *skipped,
                               int64_t *trace_i, int32_t *trace_v, int32_t *trace_j)
{
    int64_t c = 0, sk = 0;
    for (int64_t s = 0; s < nnz; ++s) {
        int64_t i_index = (int64_t)(ora_boost_uniform_u64(rng_pos, (uint64_t)(nnz - 1)) % (uint64_t)nnz);   /* :240 */
        int64_t u = user_ids[i_index];
        int32_t num_view = view_indptr[u + 1] - view_indptr[u];      /* view_count, :196 */
        int32_t v_id = -1;
        if (num_view > 0) {                                         /* :277-278 */
            int64_t v_index = view_indptr[u] + (int64_t)(ora_boost_uniform_u64(rng_view, (uint64_t)(n_items - 1)) % (uint64_t)num_view);
            v_id = view_item_ids[v_index];
        }
        int32_t j_id = (int32_t)ora_boost_uniform_u64(rng_neg, (uint64_t)(n_items - 1));      /* :250 / :279 */
        if (trace_i) trace_i[s] = i_index;
        if (trace_v) trace_v[s] = v_id;
        if (trace_j) trace_j[s] = j_id;
        sk += ora_vebpr_one(indptr, item_ids, view_indptr, view_item_ids, u, item_ids[i_index], v_id, j_id,
                            U, V, k, lr, reg, alpha, &c);
    }
    *correct = c;
    *skipped = sk;
}

ORA_API void ora_vebpr_replay(const int64_t *i_index, const int32_t *v_ids, const int32_t *j_ids, int64_t n,
                              const int32_t *user_ids, const int32_t *item_ids, const int32_t *indptr,
                              const int32_t *view_item_ids, const int32_t *view_indptr,
                              float *U, float *V, int k, float lr, float reg, float alpha,
                              int64_t *correct, int64_t *skipped)
{
    int64_t c = 0, sk = 0;
    for (int64_t s = 0; s < n; ++s) {
        int64_t ii = i_index[s];
        sk += ora_vebpr_one(indptr, item_ids, view_indptr, view_item_ids, user_ids[ii], item_ids[ii], v_ids[s], j_ids[s],
                            U, V, k, lr, reg, alpha, &c);
    }
    *correct = c;
    *skipped = sk;
}

/* ------------------------------------------------------------------------- */
/* f3: SBPR (cornac/models/sbpr/recom_sbpr.pyx).  One sample of SBPR._fit_sgd (:225-298).
 * k_index = the sampled position in the user's social-item list (social_indptr[u] + floor(k_rand * n_social));
 * k_id = social_item_ids[k_index] is read even when the user has NO social item (:231-233) -- then it is some
 * other user's entry (or, past the end of the array, undefined in the reference: here -1 = never equal to j).
 * A user WITH social items whose position is past the end (k_index == n_social_total, which the float position
 * reaches for the last such user once num_items >= 2^24 - 1) has no third item either: the BPR branch, as the kernels.
 * Returns 1 when skipped (:238-240).                                                                  */
static int ora_sbpr_one(const int32_t *indptr, const int32_t *indices, int64_t u, int32_t i_id, int32_t j_id,
                        int64_t k_index, int32_t n_social, const int32_t *social_item_ids,
                        const int32_t *social_item_counts, int64_t n_social_total,
                        float *U, float *V, float *B, int k, float lr, float lbd_u, float lbd_v, float lbd_b, int use_bias)
{
    int32_t k_id = (k_index >= 0 && k_index < n_social_total) ? social_item_ids[k_index] : -1;
    if (ora_has_non_zero(indptr, indices, u, j_id) || j_id == k_id) return 1;
    float *user = U + (size_t)u * k, *item_i = V + (size_t)i_id * k, *item_j = V + (size_t)j_id * k;
    if (n_social == 0 || k_id < 0) {                                /* :247-265: BPR, biases always trained */
        float score = B[i_id] - B[j_id];
        for (int f = 0; f < k; ++f) score = score + user[f] * (item_i[f] - item_j[f]);
        float z = 1.0 / (1.0 + exp(score));
        for (int f = 0; f < k; ++f) {
            float u_temp = user[f];
            user[f] += lr * (z * (item_i[f] - item_j[f]) - lbd_u * user[f]);
            item_i[f] += lr * (z * u_temp - lbd_v * item_i[f]);
            item_j[f] += lr * (-z * u_temp - lbd_v * item_j[f]);
        }
        B[i_id] += lr * (z - lbd_b * B[i_id]);
        B[j_id] += lr * (-z - lbd_b * B[j_id]);
        return 0;
    }
    float *item_k = V + (size_t)k_id * k;                           /* :269-297: SBPR-2 */
    float score_ik = B[i_id] - B[k_id];
    float score_kj = B[k_id] - B[j_id];
    for (int f = 0; f < k; ++f) {
        score_ik = score_ik + user[f] * (item_i[f] - item_k[f]);
        score_kj = score_kj + user[f] * (item_k[f] - item_j[f]);
    }
    float s_uk = 1.0 / (1.0 + social_item_counts[k_index]);
    float z_ik = 1.0 / (1.0 + exp(score_ik * s_uk));
    float z_kj = 1.0 / (1.0 + exp(score_kj));
    for (int f = 0; f < k; ++f) {
        float u_temp = user[f];
        user[f] += lr * (z_ik * (item_i[f] - item_k[f]) * s_uk + z_kj * (item_k[f] - item_j[f]) - lbd_u * user[f]);
        item_i[f] += lr * (z_ik * u_temp * s_uk - lbd_v * item_i[f]);
        item_j[f] += lr * (-z_kj * u_temp - lbd_v * item_j[f]);
        item_k[f] += lr * (z_kj * u_temp - z_ik * u_temp * s_uk - lbd_v * item_k[f]);
    }
    if (use_bias) {
        B[i_id] += lr * (z_ik * s_uk - lbd_b * B[i_id]);
        B[j_id] += lr * (-z_kj - lbd_b * B[j_id]);
        B[k_id] += lr * (z_kj - z_ik * s_uk - lbd_b * B[k_id]);
    }
    return 0;
}

/* position of the sampled social item: social_indptr[u] + (int)floor(k_rand * n_social), k_rand = (float)draw / (float)num_items
 * (recom_sbpr.pyx:229-232; float product, libm floor on its promotion to double).  The reference is BUILT with -O3 -ffast-math
 * (setup.py:130-137): gcc hoists the loop-invariant 1 / (float)num_items out of the sample loop and MULTIPLIES, which rounds
 * differently from the division for about one draw in four (e.g. 20 / 100 * 5 -> 1, 20 * (1/100) * 5 -> 0).  The fixture
 * tests/golden/sbpr_mid_k16.npz (compiled reference) is reproduced by the reciprocal form only (checked both), so that is
 * what the oracle -- and the product -- compute.                                                                        */
static inline int64_t ora_sbpr_k_index(const int32_t *social_indptr, int64_t u, uint64_t draw, int64_t num_items)
{
    int32_t n_social = social_indptr[u + 1] - social_indptr[u];
    volatile float inv_items = 1.0f / ((float)num_items);
    float k_rand = ((float)(long)draw) * inv_items;
    return (int64_t)social_indptr[u] + (int)floor(k_rand * n_social);
}

/* One epoch of SBPR._fit_sgd with num_threads = 1: i_index from rng_pos in [0, nnz-1]; j_id, then the draw behind
 * k_rand, both from rng_neg in [0, num_items-1] (:225-230).  trace_k records k_index.                           */
ORA_API void ora_sbpr_fit_sgd(ora_mt19937 *rng_pos, ora_mt19937 *rng_neg, int64_t nnz, int64_t num_items,
                              const int32_t *user_ids, const int32_t *item_ids, const int32_t *indptr,
                              const int32_t *social_item_ids, const int32_t *social_item_counts,
                              const int32_t *social_indptr, int64_t n_social_total,
                              float *U, float *V, float *B, int k,
                              float lr, float lbd_u, float lbd_v, float lbd_b, int use_bias,
                              int64_t *skipped, int64_t *trace_i, int32_t *trace_j, int64_t *trace_k)
{
    int64_t sk = 0;
    for (int64_t s = 0; s < nnz; ++s) {
        int64_t i_index = (int64_t)ora_boost_uniform_u64(rng_pos, (uint64_t)(nnz - 1));
        int64_t u = user_ids[i_index];
        int32_t j_id = (int32_t)ora_boost_uniform_u64(rng_neg, (uint64_t)(num_items - 1));
        uint64_t kd = ora_boost_uniform_u64(rng_neg, (uint64_t)(num_items - 1));
        int64_t k_index = ora_sbpr_k_index(social_indptr, u, kd, num_items);
        if (trace_i) trace_i[s] = i_index;
        if (trace_j) trace_j[s] = j_id;
        if (trace_k) trace_k[s] = k_index;
        sk += ora_sbpr_one(indptr, item_ids, u, item_ids[i_index], j_id, k_index,
                           social_indptr[u + 1] - social_indptr[u], social_item_ids, social_item_counts, n_social_total,
                           U, V, B, k, lr, lbd_u, lbd_v, lbd_b, use_bias);
    }
    *skipped = sk;
}

ORA_API void ora_sbpr_replay(const int64_t *i_index, const int32_t *j_ids, const int64_t *k_index, int64_t n,
                             const int32_t *user_ids, const int32_t *item_ids, const int32_t *indptr,
                             const int32_t *social_item_ids, const int32_t *social_item_counts,
                             const int32_t *social_indptr, int64_t n_social_total,
                             float *U, float *V, float *B, int k,
                             float lr, float lbd_u, float lbd_v, float lbd_b, int use_bias, int64_t *skipped)
{
    int64_t sk = 0;
    for (int64_t s = 0; s < n; ++s) {
        int64_t ii = i_index[s], u = user_ids[ii];
        sk += ora_sbpr_one(indptr, item_ids, u, item_ids[ii], j_ids[s], k_index[s],
                           social_indptr[u + 1] - social_indptr[u], social_item_ids, social_item_counts, n_social_total,
                           U, V, B, k, lr, lbd_u, lbd_v, lbd_b, use_bias);
    }
    *skipped = sk;
}

/* Multi-threaded Hogwild port of the same epoch (`prange(schedule='guided')`
 * with one mt19937 pair per thread, recom_bpr.pyx:54-62,231-234).  Only used
 * as the "port" CPU baseline when baseline/_ref is unavailable; racy by design. */
ORA_API void ora_bpr_fit_sgd_omp(const uint32_t *seeds_pos, const uint32_t *seeds_neg, int n_threads,
                                 int64_t nnz, int64_t n_neg,
                                 const int32_t *user_ids, const int32_t *item_ids,
                                 const int32_t *indptr,
                                 float *U, float *V, float *B, int k,
                                 float lr, float reg, int use_bias,
                                 int64_t *correct, int64_t *skipped)
{
    int64_t c = 0, sk = 0;
#ifdef _OPENMP
#pragma omp parallel num_threads(n_threads) reduction(+ : c, sk)
#endif
    {
        int tid = 0;
#ifdef _OPENMP
        tid = omp_get_thread_num();
#endif
        ora_mt19937 gp, gn;
        ora_mt_seed(&gp, seeds_pos[tid]);
        ora_mt_seed(&gn, seeds_neg[tid]);
#ifdef _OPENMP
#pragma omp for schedule(guided)
#endif
        for (int64_t s = 0; s < nnz; ++s) {
            int64_t ii = (int64_t)ora_boost_uniform_u64(&gp, (uint64_t)(nnz - 1));
            int32_t j = (int32_t)ora_boost_uniform_u64(&gn, (uint64_t)(n_neg - 1));
            sk += ora_bpr_one(indptr, item_ids, user_ids[ii], item_ids[ii], j, U, V, B, k,
                              lr, reg, use_bias, &c);
        }
    }
    *correct = c;
    *skipped = sk;
}

/* ------------------------------------------------------------------------- */
/* A6: one epoch of backend_cpu.fit_sgd (cornac/models/mf/backend_cpu.pyx:58-83)
 * over the ratings in stored order; returns the epoch's 0.5 * sum(err^2)
 * exactly as the f32 `loss` accumulator does (:72, :85).                      */
ORA_API float ora_mf_epoch(const int64_t *rid, const int64_t *cid, const float *val, int64_t n,
                           float *U, float *V, float *Bu, float *Bi, int k,
                           float lr, float reg, float mu, int use_bias)
{
    float loss = 0.f;
    for (int64_t j = 0; j < n; ++j) {
        int64_t u = rid[j], i = cid[j];
        float r = val[j];
        float *user = U + (size_t)u * k, *item = V + (size_t)i * k;
        float r_pred = mu + Bu[u] + Bi[i];                          /* :67 */
        for (int f = 0; f < k; ++f) r_pred = r_pred + user[f] * item[f];   /* :68-69 */
        float error = r - r_pred;                                   /* :71 */
        loss += error * error;                                      /* :72 */
        for (int f = 0; f < k; ++f) {                               /* :75-78 */
            float u_f = user[f], i_f = item[f];
            user[f] += lr * (error * i_f - reg * u_f);
            item[f] += lr * (error * u_f - reg * i_f);
        }
        if (use_bias) {                                             /* :81-83 */
            Bu[u] += lr * (error - reg * Bu[u]);
            Bi[i] += lr * (error - reg * Bi[i]);
        }
    }
    return 0.5f * loss;
}

/* Hogwild multi-thread port (prange schedule='static', backend_cpu.pyx:62). */
ORA_API float ora_mf_epoch_omp(const int64_t *rid, const int64_t *cid, const float *val, int64_t n,
                               float *U, float *V, float *Bu, float *Bi, int k,
                               float lr, float reg, float mu, int use_bias, int n_threads)
{
    float loss = 0.f;
#ifdef _OPENMP
#pragma omp parallel for schedule(static) num_threads(n_threads) reduction(+ : loss)
#endif
    for (int64_t j = 0; j < n; ++j) {
        int64_t u = rid[j], i = cid[j];
        float r = val[j];
        float *user = U + (size_t)u * k, *item = V + (size_t)i * k;
        float r_pred = mu + Bu[u] + Bi[i];
        for (int f = 0; f < k; ++f) r_pred = r_pred + user[f] * item[f];
        float error = r - r_pred;
        loss += error * error;
        for (int f = 0; f < k; ++f) {
            float u_f = user[f], i_f = item[f];
            user[f] += lr * (error * i_f - reg * u_f);
            item[f] += lr * (error * u_f - reg * i_f);
        }
        if (use_bias) {
            Bu[u] += lr * (error - reg * Bu[u]);
            Bi[i] += lr * (error - reg * Bi[i]);
        }
    }
    return 0.5f * loss;
}

/* ------------------------------------------------------------------------- */
/* A8/A9: fast_dot (cornac/utils/fast_dot.pyx:40-43): out[i] += sdot(vec, mat[i]).
 *
 * The reference delegates the k-length dot to BLAS `sdot` (scipy's bundled
 * OpenBLAS), whose summation order is unspecified.  The restatement DEFINES
 * it: products and partial sums in f64 in index order f = 0..k-1 (every f32
 * product is exact in f64), rounded once to f32, then added to out[i] in f32.
 * That is the correctly rounded dot for all practical inputs, agrees with any
 * f32 BLAS order to ~k*2^-24 relative, and is what the GPU path reproduces
 * bit-for-bit.                                                                */
ORA_API void ora_fast_dot(const float *vec, const float *mat, int64_t n_rows, int k, float *out)
{
    for (int64_t i = 0; i < n_rows; ++i) {
        const float *row = mat + (size_t)i * k;
        double acc = 0.0;
        for (int f = 0; f < k; ++f) acc += (double)vec[f] * (double)row[f];
        out[i] = out[i] + (float)acc;
    }
}

/* Batched scores for the rank path: for each query user q,
 *   out[q, i] = (item_base[i] + user_off[q]) + dot(Uq[q], V[i])
 * which is BPR.score (recom_bpr.pyx:290-293: item_base = B, user_off = 0) and
 * MF.score (mf/recom_mf.py:272-278: item_base = mu + Bi, user_off = Bu[u]).   */
ORA_API void ora_score_batch(const float *Uq, int64_t n_q, const float *V, int64_t n_items, int k,
                             const float *item_base, const float *user_off, float *out)
{
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
    for (int64_t q = 0; q < n_q; ++q) {
        const float *u = Uq + (size_t)q * k;
        float *o = out + (size_t)q * n_items;
        float uo = user_off ? user_off[q] : 0.f;
        for (int64_t i = 0; i < n_items; ++i) {
            const float *row = V + (size_t)i * k;
            double acc = 0.0;
            for (int f = 0; f < k; ++f) acc += (double)u[f] * (double)row[f];
            float base = item_base ? item_base[i] : 0.f;
            o[i] = (base + uo) + (float)acc;
        }
    }
}

/* A10 restated as a TOTAL order: top-k of `scores[n]` among the candidates
 * that are not excluded, ordered by (score descending, item id ascending).
 * numpy's argpartition/argsort used by Recommender.rank
 * (cornac/models/recommender.py:521-528) leave the order of exact ties
 * unspecified; the restatement fixes it so ids can be compared bit-for-bit.
 * excl (sorted ascending, may be NULL) lists item ids removed from the
 * candidate set.  Writes min(topk, #candidates) entries, pads ids with -1.    */
typedef struct { float s; int32_t id; } ora_pair;
static int ora_pair_cmp(const void *a, const void *b)
{
    const ora_pair *x = (const ora_pair *)a, *y = (const ora_pair *)b;
    if (x->s > y->s) return -1;
    if (x->s < y->s) return 1;
    return (x->id > y->id) - (x->id < y->id);
}
ORA_API int64_t ora_topk(const float *scores, int64_t n, const int32_t *excl, int64_t n_excl,
                         int topk, int32_t *out_ids, float *out_scores)
{
    ora_pair *buf = (ora_pair *)malloc(sizeof(ora_pair) * (size_t)(n > 0 ? n : 1));
    int64_t m = 0, e = 0;
    for (int64_t i = 0; i < n; ++i) {
        while (e < n_excl && excl[e] < i) ++e;
        if (e < n_excl && excl[e] == i) continue;
        buf[m].s = scores[i];
        buf[m].id = (int32_t)i;
        ++m;
    }
    qsort(buf, (size_t)m, sizeof(ora_pair), ora_pair_cmp);
    int64_t w = m < topk ? m : topk;
    for (int64_t t = 0; t < w; ++t) { out_ids[t] = buf[t].id; out_scores[t] = buf[t].s; }
    for (int64_t t = w; t < topk; ++t) { out_ids[t] = -1; out_scores[t] = -INFINITY; }
    free(buf);
    return w;
}

ORA_API int ora_num_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
