/*
 * b200cornac.h -- C ABI of libb200cornac.so: the H100 (sm_90a) implementation of
 * Cornac's embedding train-and-rank hot path (BPR / MF SGD, per-user score + rank).
 *
 * The reference has no C ABI for this path: its kernels are Cython `def`/`cpdef`
 * functions taking typed memoryviews (paths relative to the reference root):
 *     BPR._fit_sgd             cornac/models/bpr/recom_bpr.pyx:208-269
 *     RNGVector                cornac/models/bpr/recom_bpr.pyx:54-62 (+ recom_bpr.pxd:26-41)
 *     backend_cpu.fit_sgd      cornac/models/mf/backend_cpu.pyx:35-97
 *     fast_dot                 cornac/utils/fast_dot.pyx:40-43
 *     Recommender.rank         cornac/models/recommender.py:476-530
 * Each entry point below names the reference interface it replaces.  The Python
 * plug-in classes in cornac_b200/ (same constructor arguments as the reference's
 * BPR / MF) call these through ctypes; see INTEGRATION.md for the binding.
 *
 * Conventions
 *  - plain C types only; every pointer documented "device" is a CUDA device pointer
 *    (row-major, contiguous), every pointer documented "host" is ordinary host memory;
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *  - calls are asynchronous on `stream` unless stated otherwise and never allocate
 *    device memory; scratch comes in through explicit workspace arguments;
 *  - return value: 0 = ok, otherwise a B200_ERR_* code; b200_last_error() returns the
 *    message of the calling thread's last failure;
 *  - there is NO CPU fallback anywhere in this library.
 */
#ifndef B200CORNAC_H_
#define B200CORNAC_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_API __attribute__((visibility("default")))

#define B200_OK 0
#define B200_ERR_INVALID 1   /* bad argument (message says which) */
#define B200_ERR_CUDA 2      /* a CUDA runtime call or kernel launch failed */
#define B200_ERR_UNSUPPORTED 3

/* flags for the SGD epochs */
#define B200_SGD_ATOMIC 1u   /* scatter with red.global.add.f32 (no lost updates) instead of plain stores */
#define B200_SGD_EXACT_EXP 2u /* z = 1/(1+exp(double)) like the reference instead of the fast f32 path */
#define B200_BPR_NEG_WEIGHTED 8u /* WBPR (recom_wbpr.pyx:125-136): j = item of a uniformly drawn INTERACTION */
#define B200_BPR_LOSS_HINGE 16u  /* MMMF (cornac/models/mmmf/recom_mmmf.pyx:129-154): hinge loss, biases always trained */
#define B200_SGD_UNBOUNDED 4u /* do not cap the number of concurrently running samples (see b200_bpr_epoch) */
#define B200_BPR_DETERMINISTIC 64u /* rounds of at most 16384 samples that read the factors as the previous round left them;
                                   * a round's updates are summed exactly (fixed point) and applied once: the epoch's result
                                   * depends on the arguments only, not on thread timing (B200_SGD_ATOMIC is then implied) */
#define B200_BPR_BLOCKED 32u /* cache-blocked sample ORDER (same per-epoch law, see b200_bpr_block_plan): the epoch visits the
                              * interaction list window by window and the items block by block so that the rows in use stay in
                              * the L2; a no-op for matrices whose factors already fit (plan 1 x 1) */

B200_API const char* b200_last_error(void);
B200_API int b200_abi_version(void);
/* Number of CUDA kernels this library has launched in the calling process so far (all entry points, all
 * streams): what bench.py reports as `gpu_launches` around its timed region. */
B200_API int64_t b200_kernel_launches(void);
/* multiProcessorCount / compute capability of the current device (host call). */
B200_API int b200_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------
 * BPR, throughput mode.
 *
 * b200_bpr_prepare: analogue of BPR._prepare_data (recom_bpr.pyx:154-161).  Turns the CSR
 * training matrix into the two device structures the epoch kernel gathers from:
 *   pairs  device int32[nnz, 2]  (user, item) of every stored interaction, CSR order
 *                                (= the reference's user_ids[] and X.indices[] interleaved);
 *   table  device uint64[table_slots], table_slots = b200_bpr_table_slots(nnz): an
 *                                open-addressing hash set of (user << 32 | item) with 4-slot
 *                                buckets, answering has_non_zero(u, j) (recom_bpr.pyx:46-51)
 *                                with one 32-byte gather instead of a binary search.
 *   indptr device int32[n_users+1], indices device int32[nnz] (train_set.matrix).           */
B200_API int64_t b200_bpr_table_slots(int64_t nnz);
B200_API int b200_bpr_prepare(const int32_t* indptr, const int32_t* indices, int64_t n_users, int64_t nnz,
                              int32_t* pairs, uint64_t* table, int64_t table_slots, void* stream);

/* b200_bpr_epoch replaces one call of BPR._fit_sgd (recom_bpr.pyx:208-269) run Hogwild
 * over all cores: `n_samples` triplets, each drawing i_index uniformly from [0, nnz) and j
 * uniformly from [0, n_neg) ON DEVICE (Philox4x32-10 keyed by `seed`, counter =
 * (sample_base + s, epoch)), skipping (not redrawing) a sample when user u already has
 * item j (recom_bpr.pyx:241-243), otherwise applying the update of recom_bpr.pyx:249-267
 * to U[u], V[i], V[j], B[i], B[j].  Updates are scattered with red.global.add (B200_SGD_ATOMIC,
 * no lost updates; recommended) or plain stores (the reference's racy
 * Hogwild).  At most min(n_users, n_neg)/4 samples run concurrently so that small matrices
 * are not trained from hopelessly stale rows (B200_SGD_UNBOUNDED lifts the cap).
 *   U device f32[*, k], V device f32[*, k], B device f32[*]
 *   stats   device int64[2]: {correct, skipped} are ADDED to it (caller zeroes)           */
B200_API int b200_bpr_epoch(const int32_t* pairs, const uint64_t* table, int64_t table_slots,
                            int64_t nnz, int64_t n_users, int64_t n_neg, int64_t n_samples,
                            float* U, float* V, float* B, int k,
                            float lr, float reg, int use_bias,
                            uint64_t seed, uint64_t epoch, uint64_t sample_base,
                            unsigned flags, int64_t* stats, void* stream);

/* The plan of the cache-blocked order for a factor matrix pair: windows of the interaction list (user side) and blocks
 * of the items such that one window's user rows and one block's item rows stay L2-resident.  Sample s of an epoch
 * (s = sample_base + local index) belongs to run (s / ceil(nnz / (windows * blocks))) mod (windows * blocks); run
 * (w, b) draws i_index uniformly from the w-th window of [0, nnz) and j uniformly from item block (b + epoch) mod blocks:
 * every interaction is still drawn once per epoch in expectation and every negative is uniform over the items,
 * independently of the interaction (the law of recom_bpr.pyx:237-239); only the ORDER of the epoch's triplets changes. */
B200_API int b200_bpr_block_plan(int64_t n_users, int64_t n_neg, int k, uint32_t* n_windows, uint32_t* n_blocks);

/* The sample law of b200_bpr_epoch, evaluated on the HOST (no CUDA): writes, for
 * s = 0..n-1, the i_index and j_id that sample `sample_base + s` of `epoch` draws.  Lets a
 * caller replay / audit the exact stream the throughput kernel consumed.
 *   out_i_index host int64[n], out_j_id host int32[n]                                      */
B200_API int b200_bpr_draw_host(uint64_t seed, uint64_t epoch, uint64_t sample_base, int64_t n,
                                int64_t nnz, int64_t n_neg, int64_t* out_i_index, int32_t* out_j_id);
/* the same for an epoch run with B200_BPR_BLOCKED under the plan (n_windows, n_blocks) of b200_bpr_block_plan */
B200_API int b200_bpr_draw_host2(uint64_t seed, uint64_t epoch, uint64_t sample_base, int64_t n,
                                 int64_t nnz, int64_t n_neg, uint32_t n_windows, uint32_t n_blocks,
                                 int64_t* out_i_index, int32_t* out_j_id);

/* BPR, parity mode.  Applies an explicit sample stream (i_index[s], j_id[s]),
 * s = 0..n_samples-1, with the SAME RESULT AS APPLYING IT SEQUENTIALLY in stream order,
 * i.e. the seeded single-thread reference (recom_bpr.pyx:132-133).  The stream normally
 * comes from b200_mt_sampler_* below.  flags: B200_BPR_LOSS_HINGE selects the MMMF loop body.
 *   i_index device int64[n_samples], j_id device int32[n_samples]                          */
B200_API int b200_bpr_epoch_replay(const int64_t* i_index, const int32_t* j_id, int64_t n_samples,
                                   const int32_t* indptr, const int32_t* indices, const int32_t* coo_row,
                                   float* U, float* V, float* B, int k,
                                   float lr, float reg, int use_bias, unsigned flags,
                                   int64_t* stats, void* stream);

/* The same with the row counts of U and V given (n_users x k, n_items x k, B n_items): when the whole model fits the
 * shared memory of one SM (ML-100K sized problems) the epoch runs on an on-chip copy of the factors.  Same result. */
B200_API int b200_bpr_epoch_replay2(const int64_t* i_index, const int32_t* j_id, int64_t n_samples,
                                    const int32_t* indptr, const int32_t* indices, const int32_t* coo_row,
                                    int64_t n_users, int64_t n_items,
                                    float* U, float* V, float* B, int k,
                                    float lr, float reg, int use_bias, unsigned flags,
                                    int64_t* stats, void* stream);

/* Host-side restatement of RNGVector (recom_bpr.pyx:54-62): boost::random::mt19937 seeded
 * with `seed` + boost::random::uniform_int_distribution<long>(0, hi).  Pure host code, no
 * CUDA.  `fill` writes n consecutive draws from [0, hi] INCLUSIVE into host memory.        */
typedef struct b200_mt_sampler b200_mt_sampler;
B200_API b200_mt_sampler* b200_mt_sampler_create(uint32_t seed);
B200_API void b200_mt_sampler_destroy(b200_mt_sampler* s);
B200_API int b200_mt_sampler_fill_i64(b200_mt_sampler* s, int64_t hi, int64_t n, int64_t* out_host);
B200_API int b200_mt_sampler_fill_i32(b200_mt_sampler* s, int64_t hi, int64_t n, int32_t* out_host);

/* ------------------------------------------------------------------------------------
 * BPR siblings with a third item per sample (SURVEY.md 8(f)-3), csrc/bprx.cu.  Common arguments:
 *   indptr / indices  device int32 CSR of the (purchase) interactions, rows sorted;  coo_row device int32[nnz] = row of
 *                     every interaction (BPR._prepare_data, recom_bpr.pyx:154-161)
 *   stats             device int64[2], accumulated: [0] correct (VEBPR only), [1] skipped
 *   *_epoch           one Hogwild epoch of n_samples samples drawn on the device (Philox keyed by seed, epoch) in the
 *                     reference's law; scatter with red.global.add
 *   *_epoch_replay    an explicit sample stream (device arrays, from *_draw_host) applied with the SERIAL result, arithmetic
 *                     in the reference's operation order and types: trained factors match the seeded single-thread
 *                     reference within 1e-4
 *   *_draw_host       (host, no CUDA) the seeded streams in the reference's RNG order; all pointers are HOST pointers
 *
 * VEBPR: replaces VEBPR._fit_sgd_viewloss (bpr/recom_vebpr.pyx:214-337).  view_indptr / view_indices = CSR of the
 * "viewed but not purchased" matrix (PurchaseViewDataset.view_matrix, sorted rows, same shape as the purchase matrix);
 * v_id = the sampled viewed item, -1 for a user without viewed items (BPR fall-back branch).  No item biases.        */
B200_API int b200_vebpr_epoch(const int32_t* indptr, const int32_t* indices, const int32_t* coo_row, int64_t n_users,
                              int64_t n_items, int64_t nnz, const int32_t* view_indptr, const int32_t* view_indices,
                              float* U, float* V, int k, float lr, float reg, float alpha, uint64_t seed, uint64_t epoch,
                              int64_t n_samples, int64_t* stats, void* stream);
B200_API int b200_vebpr_epoch_replay(const int64_t* i_index, const int32_t* v_id, const int32_t* j_id, int64_t n_samples,
                                     const int32_t* indptr, const int32_t* indices, const int32_t* coo_row,
                                     const int32_t* view_indptr, const int32_t* view_indices,
                                     float* U, float* V, int k, float lr, float reg, float alpha, int64_t* stats, void* stream);
B200_API int b200_vebpr_draw_host(b200_mt_sampler* pos, b200_mt_sampler* view, b200_mt_sampler* neg, int64_t nnz, int64_t n_items,
                                  const int32_t* coo_row, const int32_t* view_indptr, const int32_t* view_indices,
                                  int64_t n_samples, int64_t* i_index_out, int32_t* v_id_out, int32_t* j_id_out);
/* SBPR: replaces SBPR._fit_sgd (sbpr/recom_sbpr.pyx:193-300).  social_indptr / social_item_ids / social_item_counts =
 * the output of SBPR._prepare_social_data (:119-145): per user the items her friends have and she has not, and how many
 * friends have each; n_social = len(social_item_ids).  k_index = the sampled POSITION in social_item_ids (the entry is
 * read, and compared with j, also for users without social items, as in the reference; positions past the end compare
 * unequal).  lambda_u / lambda_v / lambda_b regularise users / items / biases; use_bias gates the bias updates of the
 * SBPR-2 branch only (the BPR fall-back branch always trains them, :263-264).                                        */
B200_API int b200_sbpr_epoch(const int32_t* indptr, const int32_t* indices, const int32_t* coo_row, int64_t n_users,
                             int64_t n_items, int64_t nnz, const int32_t* social_indptr, const int32_t* social_item_ids,
                             const int32_t* social_item_counts, int64_t n_social,
                             float* U, float* V, float* B, int k, float lr, float lambda_u, float lambda_v, float lambda_b,
                             int use_bias, uint64_t seed, uint64_t epoch, int64_t n_samples, int64_t* stats, void* stream);
B200_API int b200_sbpr_epoch_replay(const int64_t* i_index, const int32_t* j_id, const int64_t* k_index, int64_t n_samples,
                                    const int32_t* indptr, const int32_t* indices, const int32_t* coo_row,
                                    const int32_t* social_indptr, const int32_t* social_item_ids,
                                    const int32_t* social_item_counts, int64_t n_social,
                                    float* U, float* V, float* B, int k, float lr, float lambda_u, float lambda_v, float lambda_b,
                                    int use_bias, int64_t* stats, void* stream);
B200_API int b200_sbpr_draw_host(b200_mt_sampler* pos, b200_mt_sampler* neg, int64_t nnz, int64_t n_items,
                                 const int32_t* coo_row, const int32_t* social_indptr, int64_t n_samples,
                                 int64_t* i_index_out, int32_t* j_id_out, int64_t* k_index_out);

/* ------------------------------------------------------------------------------------
 * MF.  Replaces one epoch of backend_cpu.fit_sgd (mf/backend_cpu.pyx:58-83).
 *   rid, cid device int64[n] (the reference's INT64_t layout) or int32[n] when ids_are_i32
 *   val device f32[n]; U f32[n_users,k]; V f32[n_items,k]; Bu f32[n_users], Bi f32[n_items]
 *   ordered = 1: ratings are applied with the same result as the stored-order sequential
 *                loop (seeded reference); ordered = 0: Hogwild over the whole GPU.
 *   loss device f32[1]: receives sum(err^2) of the epoch (caller multiplies by 0.5,
 *                backend_cpu.pyx:85); it is overwritten, not accumulated.
 *   k = 0: the bias-only model -- one epoch of BaselineOnly._fit_sgd
 *                (baseline_only/recom_bo.pyx:121-131: r_pred = mu + Bu[u] + Bi[i]); U and V are
 *                not read and may be NULL, n_users / n_items are then given explicitly.     */
B200_API int b200_mf_epoch(const void* rid, const void* cid, const float* val, int64_t n, int ids_are_i32,
                           int64_t n_users, int64_t n_items, float* U, float* V, float* Bu, float* Bi, int k,
                           float lr, float reg, float mu, int use_bias, int ordered,
                           unsigned flags, float* loss, void* stream);

/* ------------------------------------------------------------------------------------
 * WMF.  One optimisation step of the reference's TensorFlow-1 graph (cornac/models/wmf/wmf.py:34-55, fed by
 * cornac/models/wmf/recom_wmf.py:186-199) for a mini-batch of `b` item ids:
 *   loss = sum(C (R_b - U V_b^T)^2) + lambda_u |U|^2/2 + lambda_v |V_b|^2/2,  C = a_conf where R_b != 0 else b_conf;
 *   gradients clipped elementwise to [-5, 5]; Adam with TF-1 semantics (dense step on U; the sparse step on V decays
 *   the moments of ALL rows and moves ALL rows).  The caller advances the beta powers and passes
 *   lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t).
 *   csc_indptr / csc_rows / csc_vals  device int32[n_items+1] / int32[nnz] / f32[nnz]: train_set.csc_matrix
 *                (user indices sorted within a column); ids device int32[b], distinct
 *   U f32[n_users,k], V f32[n_items,k] and their Adam slots mU, vU, mV, vV (same shapes), all device, updated in place
 *   slot_of      device int32[n_items], all -1 on entry and on exit (scratch: item -> position in the batch)
 *   gV_scratch   device f32[b*k]; loss device f64[1]: receives the batch loss                                          */
B200_API int b200_wmf_step(const int32_t* csc_indptr, const int32_t* csc_rows, const float* csc_vals,
                           const int32_t* ids, int b, int64_t n_users, int64_t n_items, int k,
                           float* U, float* V, float* mU, float* vU, float* mV, float* vV,
                           float a_conf, float b_conf, float lambda_u, float lambda_v,
                           float lr_t, float beta1, float beta2, float epsilon,
                           int32_t* slot_of, float* gV_scratch, double* loss, void* stream);

/* ------------------------------------------------------------------------------------
 * Neighbourhood models (UserKNN / ItemKNN, cornac/models/knn).  CSR inputs are int32 indptr / indices with f64 data.
 *
 * Replaces compute_similarity (cornac/models/knn/similarity.pyx:51-105) followed by the amplify map of recom_knn.py:48-55:
 * out = the dense symmetric f64 [n, n] cosine similarity of the n rows of the weight matrix, bit-identical to the compiled
 * reference for amplify == 1 (ordered sums, every product and sum rounded, denominator sqrt(D1 * D2)).
 *   row_*      the weight matrix (n rows, n_cols columns), entries of a row in the order the reference visits them
 *   col_*      its transpose (n_cols rows), indices ascending within each row
 *   order      device int32[n], a permutation of the rows (the order the CTAs take them in; heaviest first)
 *   amplify    w -> sign(w) |w|^amplify on every non-zero similarity (1 = none)
 *   workspace  device scratch of b200_knn_similarity_workspace_bytes(n) bytes (0 = none needed, may be NULL)        */
B200_API int64_t b200_knn_similarity_workspace_bytes(int64_t n);
B200_API int b200_knn_similarity(int64_t n, const int32_t* row_indptr, const int32_t* row_indices, const double* row_data,
                                 int64_t n_cols, const int32_t* col_indptr, const int32_t* col_indices, const double* col_data,
                                 const int32_t* order, double amplify, void* workspace, double* out, void* stream);

/* The csr_matrix(sim_mat) step of compute_similarity (similarity.pyx:102) in two passes: counts[r] = non-zeros of row r of
 * the dense [n, n] matrix; the caller turns the counts into indptr (int32 [n+1]) and b200_knn_compact writes the column
 * indices (ascending) and values of every row.                                                                           */
B200_API int b200_knn_row_nnz(int64_t n, const double* sim, int32_t* counts, void* stream);
B200_API int b200_knn_compact(int64_t n, const double* sim, const int32_t* indptr, int32_t* indices, double* data, void* stream);

/* Replaces compute_score (similarity.pyx:154-201, SparseNeighbors / TopK of similarity.h:15-89) for a batch of users:
 * out[q, i] = mean[users[q]] + sum(w v) / (sum |w| + 1e-8) over the k neighbours the reference keeps (candidates in
 * descending neighbour index; after the first k, one is kept only if its weight is strictly greater than the smallest kept
 * weight, and it replaces the smallest kept (weight, value) pair).  out is device f64 [n_q, n_items].
 *   b200_knn_score_items (ItemKNN.score): ui_* = the user-item matrix, sim = dense [n_items, n_items]; candidates of (u, i)
 *     are the items j with ui[u,j] != 0 and sim[i,j] != 0, weight sim[i,j], value ui[u,j].
 *   b200_knn_score_users (UserKNN.score): iu_* = the item-user matrix, sim = dense [n_users, n_users]; candidates of (u, i)
 *     are the users v in row i of iu with sim[u,v] != 0, weight sim[u,v], value iu[i,v].
 *   workspace  device scratch of b200_knn_score_workspace_bytes(n_q, n_stage, k) bytes, n_stage = n_users for
 *              b200_knn_score_users and 0 for b200_knn_score_items (0 bytes = none needed, may be NULL)              */
B200_API int64_t b200_knn_score_workspace_bytes(int64_t n_q, int64_t n_stage, int k);
B200_API int b200_knn_score_items(const int64_t* users, int64_t n_q, int64_t n_items, const int32_t* ui_indptr,
                                  const int32_t* ui_indices, const double* ui_data, const double* sim, const double* mean,
                                  int k, void* workspace, double* out, void* stream);
B200_API int b200_knn_score_users(const int64_t* users, int64_t n_q, int64_t n_users, int64_t n_items,
                                  const int32_t* iu_indptr, const int32_t* iu_indices, const double* iu_data,
                                  const double* sim, const double* mean, int k, void* workspace, double* out, void* stream);

/* ------------------------------------------------------------------------------------
 * PMF (cornac/models/pmf/cython/pmf.pyx:55-173: pmf_linear / pmf_non_linear), SGD with RMSProp over the ratings in
 * stored order, in f64.  Rating r must see every earlier update of its user row and of its item row; two ratings that
 * share no row commute exactly.  level(r) = 1 + max(level of the previous rating of the same user, level of the previous
 * rating of the same item): the ratings of one level touch pairwise disjoint rows, so applying the levels in turn, in
 * any order inside a level, gives the serial loop's result bit for bit.
 *
 * b200_pmf_schedule (HOST): the level schedule of the ratings (uid, iid: host int32[nnz], stored order).
 *   order       host int32[nnz]: the stored index of each scheduled slot, level-major, stored order inside a level
 *   level_ptr   host int32[nnz + 1] (capacity): level l is slots [level_ptr[l], level_ptr[l+1])
 *   n_levels    host int32: number of levels (0 when nnz == 0)
 *
 * b200_pmf_fit: n_epochs epochs of pmf_linear (variant B200_PMF_LINEAR) or pmf_non_linear (B200_PMF_NON_LINEAR) in one
 * launch (one CTA walking the levels, a barrier between consecutive levels).
 *   uid, iid, rat   device int32 / int32 / f32 [nnz], already permuted into schedule order (x[order[slot]])
 *   level_ptr       device int32[n_levels + 1]
 *   U, V            device f64 [n_users, k] / [n_items, k], updated in place
 *   cache_u/v       device f64, same shapes: the RMSProp caches (zero at the start of a fit, kept across calls)
 *   lambda_reg, learning_rate, gamma   f32, as the reference's C `float` parameters (used in f64 expressions)
 *   loss            device f64 [n_epochs, nnz] or NULL: loss[e, order[slot]] = e*e + lambda_reg*(|U[u]|^2 + |V[i]|^2)
 *                   of that rating in epoch e; summing a row in stored order gives the reference's loss[epoch]
 *   order           device int32[nnz]; read only when loss != NULL
 * Calling it twice with n_epochs = a and b is the same as calling it once with a + b.
 *
 * b200_pmf_sigmoid: out[j] = the reference's sigmoid(z[j]) (pmf.pyx:27-37; C++ resolves exp(float) to expf) as the
 * fit kernel evaluates it, for device f32 z / out [n].                                                                  */
#define B200_PMF_LINEAR 0
#define B200_PMF_NON_LINEAR 1
B200_API int b200_pmf_schedule(const int32_t* uid, const int32_t* iid, int64_t nnz, int64_t n_users, int64_t n_items,
                               int32_t* order, int32_t* level_ptr, int32_t* n_levels);
B200_API int b200_pmf_fit(int variant, const int32_t* uid, const int32_t* iid, const float* rat, const int32_t* level_ptr,
                          int32_t n_levels, int64_t nnz, int k, double* U, double* V, double* cache_u, double* cache_v,
                          int n_epochs, float lambda_reg, float learning_rate, float gamma, double* loss,
                          const int32_t* order, void* stream);
B200_API int b200_pmf_sigmoid(const float* z, int64_t n, float* out, void* stream);

/* ------------------------------------------------------------------------------------
 * SoRec (cornac/models/sorec/cython/sorec.pyx:40-147) and MCF (cornac/models/mcf/cython/mcf.pyx:43-148): per epoch
 * the non-linear PMF update (pmf_non_linear's element steps, in f64) over the n_edges graph edges in stored order, then
 * over the n_ratings ratings.  The epoch is one stream of n_edges + n_ratings updates (edges first) that each touch two
 * rows of U [n_users, k], V [n_items, k] and Z: SoRec's edge (i, j) updates U[i] and Z[j] (Z is [n_users, k]) with the
 * step lambda_c * learning_rate rounded to f32, MCF's updates V[i] and Z[j] (Z is [n_items, k]) with learning_rate; a
 * rating (u, i) updates U[u] and V[i].  With the three matrices in one row space, the level rule of b200_pmf_schedule
 * applies unchanged to the mixed stream.
 *
 * b200_cofactor_schedule (HOST): net_a, net_b host int32[n_edges] (user ids for SoRec, item ids for MCF), uid, iid host
 * int32[n_ratings], all in stored order.
 *   order       host int32[n_edges + n_ratings]: the stored index of each slot (edges [0, n_edges), rating r at
 *               n_edges + r), level-major, stored order inside a level
 *   level_ptr   host int32[n_edges + n_ratings + 1] (capacity); n_levels host int32
 *
 * b200_cofactor_fit: n_epochs epochs in one launch (one CTA walking the levels, a barrier between consecutive levels).
 *   a_id, b_id, val device int32 / int32 / f32 [n_edges + n_ratings] in schedule order: the two row ids (within their
 *                   matrices) and the target of each slot
 *   is_edge         device uint8 [n_edges + n_ratings]: 1 for an edge slot, 0 for a rating slot
 *   U, V, Z         device f64, updated in place; cache_u/v/z the RMSProp caches, same shapes (zero at the start of a
 *                   fit, kept across calls).  A cache belongs to its matrix: both passes step SoRec's cache_u, MCF's cache_v
 *   lambda_c        f32, SoRec only (ignored for MCF); lambda_reg (MCF's lamda), learning_rate, gamma f32
 *   loss            device f64 [n_epochs, n_edges + n_ratings] or NULL: each update's loss term at its stored index;
 *                   summing a row in stored order gives the reference's loss[epoch]
 *   order           device int32[n_edges + n_ratings]; read only when loss != NULL
 * Calling it twice with n_epochs = a and b is the same as calling it once with a + b.                                  */
#define B200_COFACTOR_SOREC 0
#define B200_COFACTOR_MCF 1
B200_API int b200_cofactor_schedule(int variant, const int32_t* net_a, const int32_t* net_b, int64_t n_edges,
                                    const int32_t* uid, const int32_t* iid, int64_t n_ratings, int64_t n_users,
                                    int64_t n_items, int32_t* order, int32_t* level_ptr, int32_t* n_levels);
B200_API int b200_cofactor_fit(int variant, const int32_t* a_id, const int32_t* b_id, const float* val,
                               const uint8_t* is_edge, const int32_t* level_ptr, int32_t n_levels, int64_t n_edges,
                               int64_t n_ratings, int k, double* U, double* V, double* Z, double* cache_u, double* cache_v,
                               double* cache_z, int n_epochs, float lambda_c, float lambda_reg, float learning_rate,
                               float gamma, double* loss, const int32_t* order, void* stream);

/* ------------------------------------------------------------------------------------
 * A sparse matrix (n_rows x n_cols, nnz stored entries) as NMF, HPF, C2PF and EFM take it, all on the device:
 *   p##ptr, p##idx, p##row, p##val       the CSR int32[n_rows + 1] / int32[nnz] / int32[nnz] / T[nnz]: the row offsets,
 *                                        then the column, row and value of each entry
 *   p##cptr, p##crow, p##cpos, p##cval   its stable CSC transpose int32[n_cols + 1] / int32[nnz] / int32[nnz] / T[nnz]:
 *                                        the column offsets, then the row, CSR index and value of each CSC entry
 *
 * b200_csc_map (HOST): checks a CSR (indptr int32[n_rows + 1] from 0 to nnz, never decreasing; indices int32[nnz] in
 *   [0, n_cols)) and builds its stable CSC position map: csc_ptr int32[n_cols + 1] (column c is CSC entries
 *   [csc_ptr[c], csc_ptr[c+1])) and csc_pos int32[nnz] (the CSR index of each CSC entry, stored order inside a column). */
#define B200_SPARSE(p, T)                                                                                              \
    const int32_t *p##ptr, const int32_t *p##idx, const int32_t *p##row, const T *p##val, int64_t p##nnz,              \
        const int32_t *p##cptr, const int32_t *p##crow, const int32_t *p##cpos, const T *p##cval
B200_API int b200_csc_map(const int32_t* indptr, const int32_t* indices, int64_t n_rows, int64_t n_cols, int64_t nnz,
                          int32_t* csc_ptr, int32_t* csc_pos);

/* ------------------------------------------------------------------------------------
 * NMF (cornac/models/nmf/recom_nmf.pyx:182-267), multiplicative updates in plain IEEE f32, bit-identical to the
 * reference's serial loop.  Per epoch: a pass over the ratings in stored (CSR) order computes each prediction rp and,
 * with use_bias, steps the biases; then U and V are updated element-wise from ordered sums over each user's row and each
 * item's column (r * other factor and rp * other factor), the item sums reading the U the epoch started with.
 *
 * b200_nmf_fit: n_epochs epochs; calling it twice with a and b epochs is the same as calling it once with a + b.
 *   r_*                       the ratings, B200_SPARSE of f32 (n_users x n_items)
 *   item_order                device int32[n_items]: items by decreasing number of ratings (ties by id), the order
 *                             columns are launched in
 *   s_uid, s_iid, s_rat, s_pos, level_ptr, n_levels   with use_bias (else NULL / 0): the ratings in the level order of
 *                             b200_pmf_schedule (applied to the stored order), s_pos = their stored indices
 *   U, V, Bu, Bi              device f32 [n_users, k] / [n_items, k] / [n_users] / [n_items], updated in place; Bu and
 *                             Bi enter every prediction and are trained only when use_bias
 *   rp                        device f32 [nnz] workspace (the predictions of the last epoch on return)
 *   U_work                    device f32 [n_users, k] workspace, not aliasing U
 *   mu, learning_rate, lambda_*   f32, as the reference's `floating` locals
 *   loss                      device f64 [n_epochs] or NULL: += sum err^2 + lambda_u |U|^2 + lambda_v |V|^2 per epoch,
 *                             summed in f64 in no fixed order (a progress figure; not the reference's f32 sum)      */
B200_API int b200_nmf_fit(int64_t n_users, int64_t n_items, B200_SPARSE(r_, float), const int32_t* item_order,
                          const int32_t* s_uid, const int32_t* s_iid,
                          const float* s_rat, const int32_t* s_pos, const int32_t* level_ptr, int32_t n_levels, int k,
                          float* U, float* V, float* Bu, float* Bi, float* rp, float* U_work, int n_epochs, float mu,
                          float learning_rate, float lambda_u, float lambda_v, float lambda_bu, float lambda_bi,
                          int use_bias, double* loss, void* stream);

/* ------------------------------------------------------------------------------------
 * EASE (cornac/models/ease/recom_ease.py:57-126): G = X^T X + lamb I, P = G^-1, B = P / -diag(P) with B[j,j] = 0 (and
 * negatives to 0 under posB), score(u) = X[u, :] . B.
 *
 * b200_ease_gram: out = the dense f64 [n, n] X^T X with lamb added to the diagonal, bit-identical to scipy's
 *   X.T.dot(X).toarray() + lamb: every entry is the sum over users in ascending order of X[u,a] * X[u,b], each product
 *   and sum rounded.  Arguments as b200_knn_similarity with row_* = X^T (items x users, users ascending in each row) and
 *   col_* = X (users x items, items ascending); workspace of b200_ease_gram_workspace_bytes(n) bytes (0 = none needed).
 *
 * b200_spd_inverse: A (device f64 [n, n], row-major, lower triangle read) is replaced by its inverse, exactly symmetric,
 *   through a blocked Cholesky factorisation on the FP64 tensor cores.  The result repeats bit for bit from run to run.
 *   phases: B200_SPD_ALL, or the bits of the phases to run (in this order; each needs the ones before it):
 *     B200_SPD_POTRF  A = L L^T, L in the lower triangle
 *     B200_SPD_TRTRI  Z = L^-T in the upper triangle (the diagonal blocks' lower parts keep stale values)
 *     B200_SPD_LAUUM  A = Z Z^T = A^-1, both triangles
 *   info       device int: 0, or (set by B200_SPD_POTRF) the first column j + 1 whose pivot is not a positive finite number
 *              -- A is then not positive definite and its contents are undefined
 *   workspace  device scratch of b200_spd_inverse_workspace_bytes(n) bytes, kept between the phases of one inverse
 *
 * b200_ease_weights: P (device f64 [n, n]) is replaced by B, element by element as numpy's expression (the diagonal of P
 *   is saved to diag_workspace, device f64 [n], first).
 *
 * b200_ease_score: out[q, :] = X[users[q], :] . B (device f64 [n_q, n_items]), bit-identical to scipy's sparse row times
 *   dense matrix: acc = +0.0, then acc = acc + x * B[i, :] for the stored (i, x) of the row in stored order, no FMA.
 *   indptr / indices / data: the CSR of X (int32, int32, f64); B device f64 [n_items, n_items].                          */
#define B200_SPD_POTRF 1
#define B200_SPD_TRTRI 2
#define B200_SPD_LAUUM 4
#define B200_SPD_ALL 7
B200_API int64_t b200_ease_gram_workspace_bytes(int64_t n);
B200_API int b200_ease_gram(int64_t n, const int32_t* row_indptr, const int32_t* row_indices, const double* row_data,
                            int64_t n_cols, const int32_t* col_indptr, const int32_t* col_indices, const double* col_data,
                            const int32_t* order, double lamb, void* workspace, double* out, void* stream);
B200_API int64_t b200_spd_inverse_workspace_bytes(int64_t n);
B200_API int b200_spd_inverse(int64_t n, double* A, void* workspace, int* info, int phases, void* stream);
B200_API int b200_ease_weights(int64_t n, double* P, double* diag_workspace, int posB, void* stream);
B200_API int b200_ease_score(const int64_t* users, int64_t n_q, int64_t n_items, const int32_t* indptr,
                             const int32_t* indices, const double* data, const double* B, double* out, void* stream);

/* ------------------------------------------------------------------------------------
 * HPF / PF (cornac/models/hpf/cpp/cpp_hpf.cpp:139-275): the variational fit of (hierarchical) Poisson factorisation in
 * f64, in the reference's update order.  hierarchical != 0 is hpf_cpp (K_r and T_r updated), 0 is pf_cpp (they stay).
 * Every product, sum and quotient of the update is rounded on its own (no FMA) in the reference's order, so
 * b200_hpf_update is a fixed function of its inputs; the expectations use CUDA's exp / log and a Cephes digamma.
 *
 * The ratings r_*: B200_SPARSE of f64 (n_users x n_items, no explicit zeros), items ascending in each row.
 * The state, device f64, updated in place: Gs, Gr [n_users, k]; Ls, Lr [n_items, k]; Kr [n_users]; Tr [n_items].
 * work: device scratch of b200_hpf_workspace_bytes(n_users, n_items, nnz, k) bytes.
 *
 * b200_hpf_expect: out[t] = exp(digamma(shape[t]) - log(rate[t])), where a term whose argument is <= 0 (or NaN) is
 *   dropped, and out[t] = 0 when both are: the reference's sparse expectation matrices store positive entries only.
 * b200_hpf_update: one iteration from given expectations Lt [n_users, k] and Lb [n_items, k] (device f64): G_s, G_r,
 *   (HPF) K_r, then L_s, L_r, (HPF) T_r.
 * b200_hpf_fit: max_iter iterations (expectations + update), enqueued without a host synchronisation.  With
 *   hierarchical it first sets K_r and T_r from the state, as hpf_cpp does before its loop; those are the values an
 *   iteration leaves, so two calls of a and b iterations equal one call of a + b.                                       */
B200_API int64_t b200_hpf_workspace_bytes(int64_t n_users, int64_t n_items, int64_t nnz, int k);
B200_API int b200_hpf_expect(const double* shape, const double* rate, int64_t n, double* out, void* stream);
B200_API int b200_hpf_update(int hierarchical, int64_t n_users, int64_t n_items, int k, B200_SPARSE(r_, double),
                             const double* Lt, const double* Lb, double* Gs, double* Gr, double* Ls, double* Lr, double* Kr,
                             double* Tr, double* work, void* stream);
B200_API int b200_hpf_fit(int hierarchical, int64_t n_users, int64_t n_items, int k, B200_SPARSE(r_, double), double* Gs,
                          double* Gr, double* Ls, double* Lr, double* Kr, double* Tr, int max_iter, double* work,
                          void* stream);

/* ------------------------------------------------------------------------------------
 * C2PF (cornac/models/c2pf/cpp/cpp_c2pf.cpp): the variational fit of Collaborative Context Poisson Factorization in f64,
 * in the reference's update order.  variant 0 is c2pf_cpp, 1 tc2pf_cpp (L2 is L: L2s, L2r, L2b are ignored), 2 rc2pf_cpp
 * (no L: Ls, Lr, Lb are ignored).  Arithmetic and expectations as for HPF above.
 *
 * The ratings are HPF's arrays.  The context graph is a symmetric n_items x n_items pattern with n_edges stored entries:
 *   c_ptr, c_row, c_col      device CSC int32[n_items + 1] / int32[n_edges] / int32[n_edges] (the column of each entry),
 *                            rows ascending in each column
 *   c_mir                    device int32[n_edges]: the position of (i, r) for the entry (r, i)
 *   util                     device f64[n_items]: the column sums of the graph's values (read by variant 0 only)
 * State (device f64, updated in place): Gs, Gr [n_users, k]; Ls, Lr, L2s, L2r [n_items, k]; L3s, L3r [n_edges] in CSC
 * order; T3r [n_items] (ones for variants 1 and 2, which never write it).  (at, bt) is the kappa prior of the call.
 * work: device scratch of b200_c2pf_workspace_bytes(n_users, n_items, nnz, n_edges, k) bytes.
 *
 * b200_c2pf_update: one iteration from the expectations Lt [n_users, k], Lb, L2b, Lb2 [n_items, k], L3b [n_edges], which
 *   are replaced by those the iteration computes.  Each given_* that is not NULL is taken in place of the expectation the
 *   iteration would compute at that point; with all four given the state is a fixed function of the inputs.
 * b200_c2pf_fit: one call of the reference's fit: (variant 0) T3r from the state, the expectations, then n_iter
 *   iterations, enqueued without a host synchronisation.  Two calls of a and b iterations with the same (at, bt) equal
 *   one call of a + b.                                                                                                 */
#define B200_C2PF_PARAMS                                                                                               \
    int variant, int64_t n_users, int64_t n_items, int k, B200_SPARSE(r_, double), int64_t n_edges,                    \
        const int32_t *c_ptr, const int32_t *c_row, const int32_t *c_col, const int32_t *c_mir, const double *util,    \
        double at, double bt, double *Gs, double *Gr, double *Ls, double *Lr, double *L2s, double *L2r, double *L3s,   \
        double *L3r, double *T3r
B200_API int64_t b200_c2pf_workspace_bytes(int64_t n_users, int64_t n_items, int64_t nnz, int64_t n_edges, int k);
B200_API int b200_c2pf_update(B200_C2PF_PARAMS, double* Lt, double* Lb, double* L2b, double* L3b, double* Lb2,
                              const double* given_Lt, const double* given_Lb, const double* given_L2b,
                              const double* given_L3b, double* work, void* stream);
B200_API int b200_c2pf_fit(B200_C2PF_PARAMS, int n_iter, double* work, void* stream);

/* ------------------------------------------------------------------------------------
 * EFM (cornac/models/efm/recom_efm.pyx:268-353), multiplicative updates in plain IEEE f32 over the ratings A
 * (n_users x n_items), the user aspect attentions X (n_users x n_aspects) and the item aspect qualities Y
 * (n_items x n_aspects).  The predictions are the defined dot (f64 sum in index order of the exact f32 products, rounded
 * once to f32; the A prediction f32(U1.U2) + f32(H1.H2)); everything else is the reference's f32 arithmetic and order,
 * so the fit is bit-identical to oracle/efm_oracle.c.  Every accumulator reads the factors the iteration started with.
 *
 * b200_efm_fit: n_iter iterations; two calls of a and b iterations equal one call of a + b.  B200_EFM_DATA, all device:
 *   a_*, x_*, y_*  the matrices A, X and Y, each a B200_SPARSE of f32
 *   item_order    int32[n_items]: the order item rows are launched in (longest chains first)
 *   aspect_order  int32[n_aspects]: the order aspect rows are launched in (longest chains first)
 * U1 [n_users, E], U2 [n_items, E], V [n_aspects, E], H1 [n_users, L], H2 [n_items, L]: device f32, updated in place.
 * work: device f32 workspace of (n_users + n_items) * (E + L) + n_aspects * E floats; pred: device f32
 * [a_nnz + x_nnz + y_nnz] (the last iteration's predictions on return).  lambda_*: f32, as the reference's `floating`
 * locals.  loss: device f64 [n_iter] or NULL: += the reference's loss terms of each iteration, summed in f64 in no fixed
 * order.
 *
 * b200_efm_queries: the query vector of each user users[q] (device int64[n_q]) for the aspect-weighted rank:
 *   X_[a] = dot(U1[u], V[a]) (the defined dot); a_0..a_{m-1} the m = min(N, n_aspects) aspects of largest X_ (ties: the
 *   smaller id first); with c = alpha / (N * rating_scale) and beta = 1 - alpha in f64,
 *   Q[q, f] = f32(c * sum_t X_[a_t] V[a_t, f] + beta U1[u, f]) for f < E and Q[q, E + f] = f32(beta H1[u, f]) for f < L,
 *   every f64 product and sum rounded separately, the sum over t ascending.  Q: device f32 [n_q, E + L].  Then
 *   Q[q] . [U2 | H2][i] is, up to rounding, alpha * explicit(u, i) + (1 - alpha) * score(u, i): the row the reference's
 *   rank() orders.                                                                                                      */
#define B200_EFM_DATA                                                                                                   \
    B200_SPARSE(a_, float), B200_SPARSE(x_, float), B200_SPARSE(y_, float), const int32_t *item_order,                  \
        const int32_t *aspect_order, int64_t n_users, int64_t n_items, int64_t n_aspects
B200_API int b200_efm_fit(B200_EFM_DATA, int E, int L, float* U1, float* U2, float* V, float* H1, float* H2, float* work,
                          float* pred, int n_iter, float lambda_x, float lambda_y, float lambda_u, float lambda_h,
                          float lambda_v, double* loss, void* stream);
B200_API int b200_efm_queries(const int64_t* users, int64_t n_q, const float* U1, const float* H1, const float* V,
                              int64_t n_aspects, int E, int L, int num_most_cared, double alpha, double rating_scale,
                              float* Q, void* stream);

/* ------------------------------------------------------------------------------------
 * Scores.  Replaces `out = base; fast_dot(U[u], V, out)` (fast_dot.pyx:40-43 as used by
 * BPR.score recom_bpr.pyx:290-293 and MF.score mf/recom_mf.py:272-278) for a BATCH of
 * query users:  out[q, i] = (item_base[i] + user_off[q]) + dot(U[user_idx[q]], V[i]).
 * The dot is accumulated in f64 in index order and rounded once to f32 (the defined
 * summation order shared with the oracle), so results are reproducible bit-for-bit.
 *   user_idx device int64[n_q] (NULL = rows 0..n_q-1 of U); item_base, user_off may be NULL
 *   out device f32[n_q, n_items]                                                            */
B200_API int b200_score_batch(const float* U, const int64_t* user_idx, int64_t n_q,
                              const float* V, int64_t n_items, int k,
                              const float* item_base, const float* user_off,
                              float* out, void* stream);

/* One user: out[i] = (item_base[i] + user_off) + dot(U[user_idx], V[i]) -- one call of fast_dot as BPR.score / MF.score
 * make it (fast_dot.pyx:25-43; user_off = mu + Bu[u] for MF, 0 for BPR).  Same arithmetic as b200_score_batch.          */
B200_API int b200_score(const float* U, int64_t user_idx, const float* V, int64_t n_items, int k,
                        const float* item_base, float user_off, float* out, void* stream);

/* Top-k of precomputed score rows.  Replaces the argpartition/argsort of
 * Recommender.rank (recommender.py:521-528) with a TOTAL order (score desc, id asc).
 *   scores device f32[n_q, n_items]; excl_indptr device int64[n_q+1] / excl_indices device
 *   int32 (sorted per row) list item ids removed from row q's candidates (NULL = none);
 *   out_ids device int32[n_q, topk] (-1 padded), out_scores device f32[n_q, topk].         */
B200_API int b200_topk_rows(const float* scores, int64_t n_q, int64_t n_items,
                            const int64_t* excl_indptr, const int32_t* excl_indices,
                            int topk, int32_t* out_ids, float* out_scores, void* stream);

/* f64 scores of a batch of users, as PMF.score(u) defines them (cornac/models/pmf/recom_pmf.py:215-216, V.dot(U[u])):
 *   out[q, i] = sum_f U[user_idx[q], f] * V[i, f]   in f64, f ascending, every product and every sum rounded on its own
 *   (no FMA), so the result is a fixed function of the inputs.
 *   user_idx device int64[n_q] (NULL = rows 0..n_q-1 of U); out device f64[n_q, n_items]                               */
B200_API int b200_score_batch_f64(const double* U, const int64_t* user_idx, int64_t n_q, const double* V, int64_t n_items,
                                  int k, double* out, void* stream);

/* b200_topk_rows over f64 score rows: the same exclusion-aware radix select (over 64-bit keys) and the same total order
 * (score desc, id asc).  Rows must be NaN-free.  out_scores device f64[n_q, topk].                                      */
B200_API int b200_topk_rows_f64(const double* scores, int64_t n_q, int64_t n_items,
                                const int64_t* excl_indptr, const int32_t* excl_indices,
                                int topk, int32_t* out_ids, double* out_scores, void* stream);

/* Fused rank: scores (as b200_score_batch) + exclusion + top-k (as b200_topk_rows) for a
 * batch of users without materialising the [n_q, n_items] score matrix.  Tensor-core
 * (wgmma) candidate pass + exact f64 re-score of the candidates; ids and scores are
 * identical to b200_score_batch followed by b200_topk_rows.
 *   workspace: device scratch of b200_rank_topk_workspace_bytes(...) bytes.                */
B200_API int64_t b200_rank_topk_workspace_bytes(int64_t n_q, int64_t n_items, int k, int topk);
B200_API int b200_rank_topk(const float* U, const int64_t* user_idx, int64_t n_q,
                            const float* V, int64_t n_items, int k,
                            const float* item_base, const float* user_off,
                            const int64_t* excl_indptr, const int32_t* excl_indices,
                            int topk, int32_t* out_ids, float* out_scores,
                            void* workspace, int64_t workspace_bytes, void* stream);

/* The item side of the fused rank, packed once: fp16 tile images of V (with the item base folded in) and the scaling
 * scalars.  V and item_base are constant across an evaluation / a serving session, so a caller that ranks many batches
 * builds this once (b200_rank_pack_items, ~0.4 ms at 1 M items x k = 128) and passes it to b200_rank_topk_packed, which
 * then skips the two passes over V every b200_rank_topk call makes.  The caller owns the buffer and must rebuild it
 * whenever V or item_base change (e.g. after a training epoch).  b200_rank_items_bytes returns 0 for shapes the
 * tensor-core pass does not take (then pass packed_items = NULL).
 *   packed device, 128-byte aligned, b200_rank_items_bytes(n_items, k) bytes                                              */
B200_API int64_t b200_rank_items_bytes(int64_t n_items, int k);
B200_API int b200_rank_pack_items(const float* V, int64_t n_items, int k, const float* item_base,
                                  void* packed, int64_t packed_bytes, void* stream);
B200_API int b200_rank_topk_packed(const float* U, const int64_t* user_idx, int64_t n_q,
                                   const float* V, int64_t n_items, int k,
                                   const float* item_base, const float* user_off,
                                   const int64_t* excl_indptr, const int32_t* excl_indices,
                                   int topk, int32_t* out_ids, float* out_scores,
                                   const void* packed_items, void* workspace, int64_t workspace_bytes, void* stream);

/* Validation hook of the tensor-core pass: dense APPROXIMATE scores (operands scaled by powers of
 * two and rounded to fp16, f32 accumulation, + item_base, scaled back) as the candidate pass of
 * b200_rank_topk sees them; padding items (>= n_items) read -inf.
 *   out device f32[ceil(n_q/128)*128, ceil(n_items/256)*256] row-major; workspace as above. */
B200_API int b200_rank_tc_debug_scores(const float* U, int64_t n_q, const float* V, int64_t n_items, int k,
                                       const float* item_base, float* out, int64_t out_elems,
                                       void* workspace, int64_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * Top-k ranking metrics of a batch of ranked lists (the metric half of the per-user loop of
 * `ranking_eval`, cornac/eval_methods/base_method.py:200-220, for the metrics that only read
 * pd_rank[:k]: cornac/metrics/ranking.py:67-123 NDCG, :126-178 NCRR, :240-275 MeasureAtK ->
 * HitRatio / Precision / Recall / FMeasure).  A hit is `ids[q, r] in positives of user q`.
 *   ids          device int32[n_q, ids_stride], the first `topk` of each row are the ranked
 *                list (b200_rank_topk output; -1 = padding, never a hit)
 *   user_idx     device int64[n_q] row of the positives CSR for list q (NULL = q)
 *   pos_indptr / pos_indices  device int64[.] / int32[.] CSR of the test positives, ids sorted
 *                per row; every listed user must have >= 1 positive (base_method.py:180-182)
 *   metric_kind / metric_k    device int32[n_metrics]: B200_METRIC_* and its k (1 <= k)
 *   out          device f64[n_metrics, n_q]: the value metric.compute() returns for each user */
#define B200_METRIC_NDCG 0
#define B200_METRIC_PRECISION 1
#define B200_METRIC_RECALL 2
#define B200_METRIC_FMEASURE 3
#define B200_METRIC_HIT 4
#define B200_METRIC_NCRR 5
B200_API int b200_topk_metrics(const int32_t* ids, int64_t n_q, int topk, int64_t ids_stride,
                               const int64_t* user_idx, const int64_t* pos_indptr, const int32_t* pos_indices,
                               const int32_t* metric_kind, const int32_t* metric_k, int n_metrics,
                               double* out, void* stream);

/* The counts behind the full-vector ranking metrics of the same loop -- AUC (cornac/metrics/ranking.py:473-485), MAP
 * (:522-525), MRR (:213-222) -- for a batch of users whose score rows are on the device (b200_score_batch output):
 *   scores       device f32[n_q, n_items]; MODIFIED: the entries listed in excl_* are overwritten with NaN (not candidates)
 *   excl_indptr / excl_indices   device int64[n_q+1] / int32: per ROW q, the item ids that are not candidates (NULL = none)
 *   user_idx / pos_indptr / pos_indices   as for b200_topk_metrics: the test positives of row q are row user_idx[q] of the CSR
 *   less         device int64, indexed like pos_indices: number of candidates of the user scoring strictly BELOW that positive
 *   pos_score    device f32, indexed like pos_indices: the positive's score
 *   n_cand       device int64[n_q]: candidates of the user (items minus exclusions)
 *   before_first device int64[n_q]: candidates ranked ahead of the user's best positive in the total order
 *                (score desc, id asc) -> MRR = 1 / (1 + before_first)
 * From these: rank_p = n_cand - less_p (rankdata "max"), AUC = sum_p (less_p - #{positives below p}) / (|P| (n_cand - |P|)). */
B200_API int b200_rank_counts(float* scores, int64_t n_q, int64_t n_items,
                              const int64_t* excl_indptr, const int32_t* excl_indices,
                              const int64_t* user_idx, const int64_t* pos_indptr, const int32_t* pos_indices,
                              int64_t* less, float* pos_score, int64_t* n_cand, int64_t* before_first, void* stream);

/* ------------------------------------------------------------------------------------
 * MTER (cornac/models/mter/recom_mter.pyx:434-675): the seeded fit, bit-identical to the reference's serial f32 loop
 * given the same draws.  Shapes: U [n_users, d1], I [n_items, d2], A [n_aspects + 1, d3],
 * O [n_opinions, d4], G1 [d1, d2, d3], G2 [d1, d3, d4], G3 [d2, d3, d4], row-major device f32.
 *
 * b200_mter_fit: n_iter iterations in one cooperative launch; two calls of a and b iterations equal one call of a + b.
 *   X / YU / YI       the three sentiment tensors: f32 values and int32 index arrays of n_x / n_yu / n_yi entries
 *   indptr, indices   the CSR of the ratings (sorted columns), rrow the row of each entry, rval the f32 rating of
 *                     the entry's exact (user, item) pair: the BPR skip / sign rule
 *   draws             int32 [n_iter][3 n_el + 2 n_bpr]: per iteration the uia, uao, iao draws (n_el each), then the
 *                     pos and neg draws (n_bpr each), as the reference's five RNGVector streams give them; unused (may
 *                     be NULL) with B200_MTER_PHILOX
 *   flags             0: the exact mode.  B200_MTER_PHILOX: draw k of iteration iter0 + it is Philox4x32-10 of
 *                     (k, iteration) with key `seed`, reduced to [0, n) (bias <= n / 2^64), the reference's uniform law.
 *                     B200_MTER_UNORDERED: the rows' gradients are summed per sample with f32 atomics (no fixed order;
 *                     the result can differ from run to run by rounding) instead of the reference's ordered chains.
 *                     Seeded fits use 0; unseeded fits both flags (the reference defines no order without a seed)
 *   params, sgrad     host arrays of 7 device pointers in the order U, I, A, O, G1, G2, G3: the parameters and their
 *                     AdaGrad sums, updated in place (the reference's del_*_reg is reset every iteration: no state)
 *   work              device, b200_mter_workspace_bytes(...) bytes, zero before the first call; the fit leaves the
 *                     part that must be zero (del and the row owners) zero
 *   phase_ns          device u64[4] or NULL: += the nanoseconds of the phases (predictions, owners + stored terms,
 *                     gradients, AdaGrad) as block 0 sees them
 *   lr, lambda_*      f32, as the reference's `floating` locals
 *   counts            device u64[2]: += correct, skipped over the call's iterations
 *   losses            device f64[2] or NULL: += the squared errors and the BPR log-likelihood terms, summed in f64 in
 *                     no fixed order (the reference's figures are f32 sums)
 *
 * b200_mter_queries: Q [n_users, d2] = the rank query of every user: M[p, q] = f32(sum_r G1[p, q, r] a_last[r]) and
 *   Q[u, q] = f32(sum_p U[u, p] M[p, q]), each an f64 sum in index order of exact products.  Q . I[i] is score(u)[i]
 *   up to rounding.                                                                                                    */
#define B200_MTER_UNORDERED 1
#define B200_MTER_PHILOX 2
B200_API int64_t b200_mter_workspace_bytes(int64_t n_users, int64_t n_items, int64_t n_aspects, int64_t n_opinions,
                                           int d1, int d2, int d3, int d4, int n_el, int n_bpr);
B200_API int b200_mter_fit(int64_t n_users, int64_t n_items, int64_t n_aspects, int64_t n_opinions, int d1, int d2,
                           int d3, int d4, const float* X, const int32_t* X_u, const int32_t* X_i, const int32_t* X_a,
                           int64_t n_x, const float* YU, const int32_t* YU_u, const int32_t* YU_a, const int32_t* YU_o,
                           int64_t n_yu, const float* YI, const int32_t* YI_i, const int32_t* YI_a, const int32_t* YI_o,
                           int64_t n_yi, const int32_t* indptr, const int32_t* indices, const int32_t* rrow,
                           const float* rval, int64_t nnz, int n_el, int n_bpr, int n_iter, const int32_t* draws,
                           float* const* params, float* const* sgrad, void* work, float lr, float lambda_reg,
                           float lambda_bpr, int flags, uint64_t seed, uint64_t iter0, unsigned long long* counts,
                           double* losses, unsigned long long* phase_ns, void* stream);
B200_API int b200_mter_queries(const float* U, int64_t n_users, const float* G1, const float* a_last, int d1, int d2,
                               int d3, float* Q, void* stream);

/* ------------------------------------------------------------------------------------
 * ComparERSub (cornac/models/comparer/recom_comparer_sub.pyx:487-806): MTER plus a third sample phase over the
 * comparative pairs (user, earlier item, later item, aspect) of the user's purchase history.
 *
 * b200_comparer_sub_fit: b200_mter_fit's fit and arguments (b200_mter_fit is the case n_pair = 0), plus
 *   p_user, p_earlier, p_later, p_aspect   int32 [n_plist]: the pair list, in the reference's order
 *   n_pair            pair samples per iteration (>= 0; n_plist > 0 when n_pair > 0)
 *   draws             int32 [n_iter][3 n_el + 2 n_bpr + n_pair]: b200_mter_fit's draws of an iteration, then the
 *                     n_pair draws of the pair stream
 *   lambda_d          f32, the weight of the pair terms
 *   work              device, b200_comparer_sub_workspace_bytes(...) bytes, zero before the first call
 *   counts            device u64[3]: += correct, skipped, aspect_correct (pairs whose later item scores higher)
 *   losses            device f64[3] or NULL: += loss, bpr_loss, aspect_bpr_loss
 * A pair sample's terms follow the BPR samples' in every accumulator chain; within a sample with earlier == later the
 * I row takes -v then +v for every term, as the reference's statements do.
 *
 * b200_comparer_rank_rows: out [n_q, n_items] f32, the rank rows of users[0..n_q) over items [0, n_items):
 *   ts3[i, a] = sum_q I[i, q] sum_r (sum_p G1[p, q, r] U[u, p]) A[a, r] for a <= n_aspects, and
 *   out[i] = f32(alpha * mean(the n_top largest ts3[i, a < n_aspects]) + (1 - alpha) * ts3[i, n_aspects]),
 *   every sum in f64 in index order and one rounding at the end (0 < n_top <= n_aspects < 1024).                       */
B200_API int64_t b200_comparer_sub_workspace_bytes(int64_t n_users, int64_t n_items, int64_t n_aspects,
                                                   int64_t n_opinions, int d1, int d2, int d3, int d4, int n_el,
                                                   int n_bpr, int n_pair);
B200_API int b200_comparer_sub_fit(int64_t n_users, int64_t n_items, int64_t n_aspects, int64_t n_opinions, int d1,
                                   int d2, int d3, int d4, const float* X, const int32_t* X_u, const int32_t* X_i,
                                   const int32_t* X_a, int64_t n_x, const float* YU, const int32_t* YU_u,
                                   const int32_t* YU_a, const int32_t* YU_o, int64_t n_yu, const float* YI,
                                   const int32_t* YI_i, const int32_t* YI_a, const int32_t* YI_o, int64_t n_yi,
                                   const int32_t* indptr, const int32_t* indices, const int32_t* rrow,
                                   const float* rval, int64_t nnz, const int32_t* p_user, const int32_t* p_earlier,
                                   const int32_t* p_later, const int32_t* p_aspect, int64_t n_plist, int n_el,
                                   int n_bpr, int n_pair, int n_iter, const int32_t* draws, float* const* params,
                                   float* const* sgrad, void* work, float lr, float lambda_reg, float lambda_bpr,
                                   float lambda_d, int flags, uint64_t seed, uint64_t iter0, unsigned long long* counts,
                                   double* losses, unsigned long long* phase_ns, void* stream);
B200_API int b200_comparer_rank_rows(const float* U, const float* I, const float* A, const float* G1,
                                     const int64_t* users, int64_t n_q, int64_t n_items, int d1, int d2, int d3,
                                     int64_t n_aspects, int n_top, double alpha, float* out, void* stream);

/* ------------------------------------------------------------------------------------
 * LRPPM (cornac/models/lrppm/recom_lrppm.pyx:356-560): the fit, bit-identical to the reference's compiled float loop
 * given the same draws, and its aspect-mixed rank rows.  Shapes: U [n_users, k], I [n_items, k], UA and IA
 * [n_aspects, k], row-major device f32.
 *
 * b200_lrppm_fit: up to n_iter iterations in one cooperative launch.  It stops after the first iteration in which every
 *   element of U, I, UA and IA is numpy-isclose (rtol 1e-5, atol 1e-8, in f32) to its value before that iteration, as
 *   the reference's convergence test does.  Two calls of a and b iterations equal one call of a + b unless the first
 *   call stops early.
 *   r_u, r_i, r_val   int32 / f32 [n_r]: the train set's (user, item, rating) triples (the `pos` stream draws them)
 *   x_u, x_i, x_a     int32 [n_x]: the review triples (user, item, aspect) in the reference's order, x_l f32 [n_x] their
 *                     weight 1 / (cnt (n_aspects - cnt))
 *   akeys             int32 [n_akeys]: sorted distinct get_key3(u, i, a) of the triples, in C int with two's-complement
 *                     wrap (the skip test: a ranking sample is skipped when get_key3(u, i, a_j) is among them)
 *   rkeys, rvals      int32 / f32 [n_rkeys]: sorted distinct get_key(u, i) of the ratings and the value the reference's
 *                     IntFloatDict keeps for each (the last); an absent key reads 0
 *   draws             int32 [n_iter][n_samples + 2 n_ranking_samples]: per iteration the pos, pos_uia and neg_uia
 *                     draws; unused (may be NULL) with B200_LRPPM_PHILOX, which draws Philox4x32-10 of
 *                     (draw, iter0 + it) with key `seed` on the device under the same uniform law
 *   params            host array of 4 device pointers U, I, UA, IA, updated in place
 *   work              device, b200_lrppm_workspace_bytes(...) bytes, zero before the first call; the fit leaves it so
 *   lr, reg, ld       f32, as the reference's `floating` locals
 *   counts            device u64[4]: += correct, skipped, iterations run; counts[3] = 1 when the fit converged
 *   losses            device f64[3] or NULL: += loss, ranking_loss, r_loss, summed in f64 in no fixed order
 *   phase_ns          device u64[3] or NULL: += the nanoseconds of the phases (predictions, del chains, dense step)
 *
 * b200_lrppm_rank_rows: out [n_q, n_items] f64, the rank rows of users[0..n_q) over items [0, n_items):
 *   s[i, a] = f32(f32(f32(UA[a] . U[u]) + f32(I[i] . IA[a])) + f32(I[i] . U[u])), each dot an f64 index-order sum,
 *   out[i] = alpha rating_scale (sum over the n_top largest s[i, :] of s q[i, a]) / n_top
 *            + f32(f32(1 - alpha) f32(I[i] . U[u]))
 *   q: the item x aspect quality CSR (f64, sorted or not; an absent entry is 0).  At a tie at the n_top-th place the
 *   smaller aspect ids are taken.  0 < n_top <= n_aspects <= 1024.                                                    */
#define B200_LRPPM_PHILOX 1
B200_API int64_t b200_lrppm_workspace_bytes(int64_t n_users, int64_t n_items, int64_t n_aspects, int k, int n_samples,
                                            int n_ranking_samples);
B200_API int b200_lrppm_fit(int64_t n_users, int64_t n_items, int64_t n_aspects, int k, const int32_t* r_u,
                            const int32_t* r_i, const float* r_val, int64_t n_r, const int32_t* x_u, const int32_t* x_i,
                            const int32_t* x_a, const float* x_l, int64_t n_x, const int32_t* akeys, int64_t n_akeys,
                            const int32_t* rkeys, const float* rvals, int64_t n_rkeys, int n_samples,
                            int n_ranking_samples, int n_iter, const int32_t* draws, float* const* params, void* work,
                            float lr, float reg, float ld, int flags, uint64_t seed, uint64_t iter0,
                            unsigned long long* counts, double* losses, unsigned long long* phase_ns, void* stream);
B200_API int b200_lrppm_rank_rows(const float* U, const float* I, const float* UA, const float* IA,
                                  const int32_t* q_indptr, const int32_t* q_indices, const double* q_data,
                                  const int64_t* users, int64_t n_q, int64_t n_items, int k, int64_t n_aspects,
                                  int n_top, double alpha, double rating_scale, double* out, void* stream);

/* ------------------------------------------------------------------------------------
 * Multi-GPU item-factor exchange (no reference counterpart: the reference is a single
 * process).  Each rank trains its user shard against a replica of V / B; at the epoch
 * boundary   b200_delta_make:  delta[i] = x[i] - snapshot[i]
 * the caller all-reduces (sum) `delta` over NCCL, then
 *            b200_delta_apply: x[i] = snapshot[i] + delta[i];  snapshot[i] = x[i]
 * so every replica ends the epoch with x_start + sum over ranks of the local changes -- or, the default of the Python layer,
 * x_start + (sum of the changes) / (number of ranks that changed the element): the caller also all-reduces the indicator
 * (delta != 0) and divides.  The plain sum is the single-process step count only while the ranks change different rows; a row
 * every rank trains (a popular item) moves `world` times too far and the epochs oscillate with growing amplitude from 4 ranks
 * on (tools/sim_localsgd.py: pairwise accuracy 0.81 -> 0.30 at 4 ranks); the mean over the ranks that changed an element is a
 * convex combination of their local results: stable at any world size, equal to the sum where one rank alone touched it.   */
B200_API int b200_delta_make(const float* x, const float* snapshot, float* delta, int64_t n, void* stream);
B200_API int b200_delta_apply(float* x, float* snapshot, const float* delta, int64_t n, void* stream);

/* The same exchange as ONE kernel over NVLink peer memory (one process per GPU, replicas mapped into each other with
 * CUDA IPC): rank r owns the slice b200_item_exchange_slice(r, world, n) of the vector, reads that slice of EVERY
 * replica over NVLink, forms  snapshot + sum_r (x_r - snapshot)  in rank order (deterministic, bit-equal everywhere) and
 * stores it into every replica and into its snapshot -- delta, reduce-scatter, apply and all-gather fused; each byte
 * crosses NVLink once per direction and there is no delta buffer.
 *   b200_ipc_export   (host) 64-byte CUDA IPC handle of the allocation containing dev_ptr + the pointer's offset in it
 *   b200_ipc_open     (host) map a peer's exported allocation; returns the peer pointer (peer access enabled lazily)
 *   x_peers / flag_peers  host arrays of `world` DEVICE pointers: every rank's replica (f32[n]) and flag buffer
 *                     (u32[32], zeroed once by its owner before the first exchange), own pointers at [rank]
 *   snapshot_slice    device f32[hi - lo]: the epoch-start values of the owned slice (= the replica's after each exchange)
 *   seq               1, 2, 3, ... : the same value on every rank for the same exchange
 *   mean_touched      1: snapshot + (sum_r d_r) / #{r : d_r != 0} per element (see above; the default of the Python layer); 0: the sum
 * Every rank must call it once per exchange; the kernel returns when all peers have finished writing this rank's
 * replica.  A peer that never arrives sets flag word [17] after ~4 s instead of hanging the GPU. */
B200_API int b200_ipc_export(const void* dev_ptr, void* handle64_out, int64_t* offset_out);
B200_API int b200_ipc_open(const void* handle64, int64_t offset, void** mapped_out);
B200_API int b200_ipc_close(void* mapped, int64_t offset);
B200_API int b200_item_exchange_slice(int rank, int world, int64_t n, int64_t* lo_out, int64_t* hi_out);
B200_API int b200_item_exchange(int rank, int world, void* const* x_peers, void* const* flag_peers, float* snapshot_slice,
                                int64_t n, uint32_t seq, int mean_touched, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200CORNAC_H_ */
