// BPR siblings whose samples touch a THIRD item row: VEBPR and SBPR (SURVEY.md 8(f)-3), sm_90a.
//
//   VEBPR  cornac/models/bpr/recom_vebpr.pyx:214-337  (u, i = purchased, v = viewed but not purchased, j = negative):
//          three pairwise logistic terms i>j, i>v, v>j (weights 1, alpha, 1 - alpha), scores clipped to +-50, no item
//          biases; users without viewed items fall back to the plain BPR triplet (:246-275).
//   SBPR   cornac/models/sbpr/recom_sbpr.pyx:193-300  (u, i, k = item a friend has and u has not, j = negative):
//          SBPR-2: i >_{s_uk} k and k > j with s_uk = 1 / (1 + #friends having k); users without social items fall back
//          to BPR (:247-265); separate regularisers for users / items / biases.
//
// Same two modes as bpr.cu:
//   * tri_hogwild_kernel  throughput mode: one sample per G-lane group, on-device Philox sampling in the reference's law
//     (positive uniform over interactions, negative uniform over items, third item uniform over the user's viewed /
//     social items), membership tests by binary search in the user's sorted CSR rows (the extra rows of these models
//     are short), four rows gathered with 128-bit L2-only loads, dots by group shuffles, red.global.add scatter;
//   * tri_replay_window_kernel  parity mode: an explicit sample stream (drawn on the host by b200_vebpr_draw_host /
//     b200_sbpr_draw_host in the reference's RNG order) applied with the serial result: 32-sample windows, one sample
//     per warp, a sample runs once no earlier pending sample of the window shares its user row or one of its item
//     rows; unfused arithmetic in the reference's operation order and types (the .pyx expressions mix float
//     variables with the double literal 1.0: (1.0 - alpha) * ... is evaluated in double, as in the generated C).
// HBM / L2-bound gather-scatter work: no tensor cores by design.
#include <math.h>

#include "sgd_common.cuh"

namespace b200 {

enum { KIND_VEBPR = 0, KIND_SBPR = 1 };

struct TriParams {
    const int32_t* __restrict__ indptr;       // purchases: CSR (sorted rows) + COO row of every interaction
    const int32_t* __restrict__ indices;
    const int32_t* __restrict__ coo_row;
    const int32_t* __restrict__ aux_indptr;   // VEBPR: view CSR; SBPR: social_indptr
    const int32_t* __restrict__ aux_items;    // VEBPR: view item ids (sorted rows); SBPR: social_item_ids
    const int32_t* __restrict__ aux_counts;   // SBPR: social_item_counts (VEBPR: null)
    int64_t n_items, nnz, n_aux;
    float* U;
    float* V;
    float* B;                                  // SBPR only
    int k, n_units;
    float lr, reg_u, reg_v, reg_b, alpha;
    int use_bias;
    // throughput mode
    uint64_t seed, epoch;
    int64_t n_samples;
    // parity mode: the sample stream
    const int64_t* __restrict__ i_index;
    const int32_t* __restrict__ j_id;
    const int32_t* __restrict__ v_id;          // VEBPR: viewed item or -1
    const int64_t* __restrict__ k_index;       // SBPR: position in social_item_ids
    unsigned long long* stats;                 // [0] correct (VEBPR), [1] skipped
};

__device__ __forceinline__ float sigmoid_neg_fast(float x) { return __frcp_rn(1.f + __expf(x)); }     // 1 / (1 + e^x)

// One resolved sample: rows to touch and whether it is skipped.  t < 0: no third item (the BPR fall-back branches).
struct TriSample {
    int32_t u, i, j, t;
    int32_t t_count;       // SBPR: social_item_counts[k_index]
    bool skip;
};

// ---------------------------------------------------------------------------------------
// Throughput mode
template <int G, int NPL, bool VEC, int KIND>
__global__ void __launch_bounds__(256) tri_hogwild_kernel(const TriParams p)
{
    constexpr int GPB = 256 / G;
    const int lg = threadIdx.x % G;
    const int64_t gid = (int64_t)blockIdx.x * GPB + threadIdx.x / G;
    const int64_t n_groups = (int64_t)gridDim.x * GPB;
    const size_t k = (size_t)p.k;
    const float inv_items = 1.0f / (float)p.n_items;
    unsigned n_correct = 0, n_skipped = 0;
    using Frag = RowFrag<NPL, VEC>;
    constexpr int N = NPL * Frag::W;
    for (int64_t s = gid; s < p.n_samples; s += n_groups) {
        // every lane of the group resolves the same sample (pure function of (seed, epoch, s): no broadcast needed)
        const Philox4 r = philox4x32_10((uint32_t)s, (uint32_t)((uint64_t)s >> 32), (uint32_t)p.epoch, 0x7813u + KIND,
                                        (uint32_t)p.seed, (uint32_t)(p.seed >> 32));
        const int64_t ii = (int64_t)range64(r.x, r.y, (uint64_t)p.nnz);
        TriSample m;
        m.j = (int32_t)mulhi32(r.z, (uint32_t)p.n_items);
        const uint32_t d3 = mulhi32(r.w, (uint32_t)p.n_items);              // the third draw, uniform over [0, n_items)
        m.u = __ldg(p.coo_row + ii);
        m.i = __ldg(p.indices + ii);
        const int32_t a_lo = __ldg(p.aux_indptr + m.u), a_hi = __ldg(p.aux_indptr + m.u + 1);
        const int32_t n_aux_u = a_hi - a_lo;
        m.t = -1; m.t_count = 0;
        m.skip = row_contains(p.indices, __ldg(p.indptr + m.u), __ldg(p.indptr + m.u + 1), m.j);
        if (KIND == KIND_VEBPR) {
            if (n_aux_u > 0) {                                               // recom_vebpr.pyx:277-285
                m.t = __ldg(p.aux_items + a_lo + (int32_t)(d3 % (uint32_t)n_aux_u));
                m.skip = m.skip || row_contains(p.aux_items, a_lo, a_hi, m.j);
            }
        } else {
            // recom_sbpr.pyx:229-240: the entry at the sampled position is read -- and compared with j -- even for a user
            // without social items (then it belongs to a later user; past the end of the array: nothing to compare).  The
            // position can equal a_hi (fl(d3 * fl(1 / n_items)) rounds to 1 once n_items >= 2^24 - 1): the next user's
            // entry and count, as the reference reads them, or -- for the last user -- no entry: the BPR fall-back.
            const int64_t kidx = (int64_t)a_lo + (int)floorf(((float)d3 * inv_items) * (float)n_aux_u);
            const bool in_array = kidx < p.n_aux;
            const int32_t kid = in_array ? __ldg(p.aux_items + kidx) : -1;
            m.skip = m.skip || (m.j == kid);
            if (n_aux_u > 0 && in_array) { m.t = kid; m.t_count = __ldg(p.aux_counts + kidx); }
        }
        if (m.skip) { ++n_skipped; continue; }

        float* pu = p.U + (size_t)m.u * k;
        float* pi = p.V + (size_t)m.i * k;
        float* pj = p.V + (size_t)m.j * k;
        float* pt = p.V + (size_t)(m.t < 0 ? m.j : m.t) * k;                // harmless address when there is no third item
        Frag fu, fi, fj, ft;
        row_load<G, NPL, VEC>(fu, pu, lg, p.n_units);
        row_load<G, NPL, VEC>(fi, pi, lg, p.n_units);
        row_load<G, NPL, VEC>(fj, pj, lg, p.n_units);
        if (m.t >= 0) row_load<G, NPL, VEC>(ft, pt, lg, p.n_units);
        const float lr = p.lr;
        if (KIND == KIND_VEBPR) {
            const float reg = p.reg_u;
            if (m.t < 0) {
                float x = 0.f;
#pragma unroll
                for (int e = 0; e < N; ++e) x = fmaf(fu.v[e], fi.v[e] - fj.v[e], x);
                x = fminf(fmaxf(group_sum<G>(x), -50.f), 50.f);
                const float d = sigmoid_neg_fast(x);
                n_correct += (lg == 0 && d < .5f);
                Frag du, di, dj;
#pragma unroll
                for (int e = 0; e < N; ++e) {
                    const float u = fu.v[e], vi = fi.v[e], vj = fj.v[e];
                    du.v[e] = -lr * (-d * (vi - vj) + reg * u);
                    di.v[e] = -lr * (-d * u + reg * vi);
                    dj.v[e] = -lr * (d * u + reg * vj);
                }
                row_red_add<G, NPL, VEC>(du, pu, lg, p.n_units);
                row_red_add<G, NPL, VEC>(di, pi, lg, p.n_units);
                row_red_add<G, NPL, VEC>(dj, pj, lg, p.n_units);
            } else {
                float xij = 0.f, xiv = 0.f, xvj = 0.f;
#pragma unroll
                for (int e = 0; e < N; ++e) {
                    xij = fmaf(fu.v[e], fi.v[e] - fj.v[e], xij);
                    xiv = fmaf(fu.v[e], fi.v[e] - ft.v[e], xiv);
                    xvj = fmaf(fu.v[e], ft.v[e] - fj.v[e], xvj);
                }
                xij = fminf(fmaxf(group_sum<G>(xij), -50.f), 50.f);
                xiv = fminf(fmaxf(group_sum<G>(xiv), -50.f), 50.f);
                xvj = fminf(fmaxf(group_sum<G>(xvj), -50.f), 50.f);
                const float dij = sigmoid_neg_fast(xij), div_ = sigmoid_neg_fast(xiv), dvj = sigmoid_neg_fast(xvj);
                n_correct += (lg == 0 && dij < .5f && div_ < .5f && dvj < .5f);
                const float a = p.alpha * div_, b = (1.f - p.alpha) * dvj;
                Frag du, di, dj, dv;
#pragma unroll
                for (int e = 0; e < N; ++e) {
                    const float u = fu.v[e], vi = fi.v[e], vj = fj.v[e], vv = ft.v[e];
                    du.v[e] = -lr * (-dij * (vi - vj) - a * (vi - vv) - b * (vv - vj) + reg * u);
                    di.v[e] = -lr * (-dij * u - a * u + reg * vi);
                    dv.v[e] = -lr * (a * u - b * u + reg * vv);
                    dj.v[e] = -lr * (dij * u + b * u + reg * vj);
                }
                row_red_add<G, NPL, VEC>(du, pu, lg, p.n_units);
                row_red_add<G, NPL, VEC>(di, pi, lg, p.n_units);
                row_red_add<G, NPL, VEC>(dv, pt, lg, p.n_units);
                row_red_add<G, NPL, VEC>(dj, pj, lg, p.n_units);
            }
        } else {
            const float bi = __ldcg(p.B + m.i), bj = __ldcg(p.B + m.j);
            if (m.t < 0) {                                                   // plain BPR, biases always trained (:247-265)
                float x = 0.f;
#pragma unroll
                for (int e = 0; e < N; ++e) x = fmaf(fu.v[e], fi.v[e] - fj.v[e], x);
                const float z = sigmoid_neg_fast(bi - bj + group_sum<G>(x));
                Frag du, di, dj;
#pragma unroll
                for (int e = 0; e < N; ++e) {
                    const float u = fu.v[e], vi = fi.v[e], vj = fj.v[e];
                    du.v[e] = lr * (z * (vi - vj) - p.reg_u * u);
                    di.v[e] = lr * (z * u - p.reg_v * vi);
                    dj.v[e] = lr * (-z * u - p.reg_v * vj);
                }
                row_red_add<G, NPL, VEC>(du, pu, lg, p.n_units);
                row_red_add<G, NPL, VEC>(di, pi, lg, p.n_units);
                row_red_add<G, NPL, VEC>(dj, pj, lg, p.n_units);
                if (lg == 0) {
                    red_add_f32(p.B + m.i, lr * (z - p.reg_b * bi));
                    red_add_f32(p.B + m.j, lr * (-z - p.reg_b * bj));
                }
            } else {                                                         // SBPR-2 (:269-297)
                const float bk = __ldcg(p.B + m.t);
                float xik = 0.f, xkj = 0.f;
#pragma unroll
                for (int e = 0; e < N; ++e) {
                    xik = fmaf(fu.v[e], fi.v[e] - ft.v[e], xik);
                    xkj = fmaf(fu.v[e], ft.v[e] - fj.v[e], xkj);
                }
                const float s_uk = 1.f / (1.f + (float)m.t_count);
                const float zik = sigmoid_neg_fast((bi - bk + group_sum<G>(xik)) * s_uk) * s_uk;     // z_ik * s_uk everywhere below
                const float zkj = sigmoid_neg_fast(bk - bj + group_sum<G>(xkj));
                Frag du, di, dj, dk;
#pragma unroll
                for (int e = 0; e < N; ++e) {
                    const float u = fu.v[e], vi = fi.v[e], vj = fj.v[e], vk = ft.v[e];
                    du.v[e] = lr * (zik * (vi - vk) + zkj * (vk - vj) - p.reg_u * u);
                    di.v[e] = lr * (zik * u - p.reg_v * vi);
                    dj.v[e] = lr * (-zkj * u - p.reg_v * vj);
                    dk.v[e] = lr * (zkj * u - zik * u - p.reg_v * vk);
                }
                row_red_add<G, NPL, VEC>(du, pu, lg, p.n_units);
                row_red_add<G, NPL, VEC>(di, pi, lg, p.n_units);
                row_red_add<G, NPL, VEC>(dj, pj, lg, p.n_units);
                row_red_add<G, NPL, VEC>(dk, pt, lg, p.n_units);
                if (p.use_bias && lg == 0) {
                    red_add_f32(p.B + m.i, lr * (zik - p.reg_b * bi));
                    red_add_f32(p.B + m.j, lr * (-zkj - p.reg_b * bj));
                    red_add_f32(p.B + m.t, lr * (zkj - zik - p.reg_b * bk));
                }
            }
        }
    }
    // one count per group (lane 0 of the group), reduced per warp
    const unsigned c = __reduce_add_sync(0xffffffffu, n_correct);
    const unsigned sk = __reduce_add_sync(0xffffffffu, lg == 0 ? n_skipped : 0u);
    if ((threadIdx.x & 31) == 0) {
        if (c) atomicAdd(p.stats + 0, (unsigned long long)c);
        if (sk) atomicAdd(p.stats + 1, (unsigned long long)sk);
    }
}

// ---------------------------------------------------------------------------------------
// Parity mode.  The update of one sample by one warp, lane-strided over the factors, in the reference's operation order.
__device__ __forceinline__ float sig_exact(float x) { return (float)(1.0 / (1.0 + exp((double)x))); }
__device__ __forceinline__ float clip50(float x) { return x > 50.0f ? 50.0f : (x < -50.0f ? -50.0f : x); }

// float a - lr * (double expression): the reference's `row[f] -= lr * (<mixed float / double>)` is evaluated in double
__device__ __forceinline__ float sub_lr_d(float a, float lr, double e) { return (float)((double)a - (double)lr * e); }

template <int KIND>
__device__ __forceinline__ void tri_apply_exact(const TriParams& p, const TriSample& m, int lane, unsigned long long& n_correct)
{
    const size_t k = (size_t)p.k;
    float* pu = p.U + (size_t)m.u * k;
    float* pi = p.V + (size_t)m.i * k;
    float* pj = p.V + (size_t)m.j * k;
    float* pt = p.V + (size_t)(m.t < 0 ? m.j : m.t) * k;
    const float lr = p.lr;
    if (KIND == KIND_VEBPR) {
        const float reg = p.reg_u, alpha = p.alpha;
        if (m.t < 0) {                                                       // recom_vebpr.pyx:255-275
            float part = 0.f;
            for (int f = lane; f < p.k; f += 32)
                part = __fadd_rn(part, __fmul_rn(__ldcg(pu + f), __fsub_rn(__ldcg(pi + f), __ldcg(pj + f))));
            const float d = sig_exact(clip50(group_sum<32>(part)));
            n_correct += (d < .5f);
            for (int f = lane; f < p.k; f += 32) {
                const float u = __ldcg(pu + f), vi = __ldcg(pi + f), vj = __ldcg(pj + f);
                __stcg(pu + f, __fsub_rn(u, __fmul_rn(lr, __fadd_rn(__fmul_rn(-d, __fsub_rn(vi, vj)), __fmul_rn(reg, u)))));
                __stcg(pi + f, __fsub_rn(vi, __fmul_rn(lr, __fadd_rn(__fmul_rn(-d, u), __fmul_rn(reg, vi)))));
                __stcg(pj + f, __fsub_rn(vj, __fmul_rn(lr, __fadd_rn(__fmul_rn(d, u), __fmul_rn(reg, vj)))));
            }
            return;
        }
        float xij = 0.f, xiv = 0.f, xvj = 0.f;                               // :289-295
        for (int f = lane; f < p.k; f += 32) {
            const float u = __ldcg(pu + f), vi = __ldcg(pi + f), vj = __ldcg(pj + f), vv = __ldcg(pt + f);
            xij = __fadd_rn(xij, __fmul_rn(u, __fsub_rn(vi, vj)));
            xiv = __fadd_rn(xiv, __fmul_rn(u, __fsub_rn(vi, vv)));
            xvj = __fadd_rn(xvj, __fmul_rn(u, __fsub_rn(vv, vj)));
        }
        const float dij = sig_exact(clip50(group_sum<32>(xij)));
        const float div_ = sig_exact(clip50(group_sum<32>(xiv)));
        const float dvj = sig_exact(clip50(group_sum<32>(xvj)));
        n_correct += (dij < .5f && div_ < .5f && dvj < .5f);
        const double one_m_alpha = 1.0 - (double)alpha;                      // (1.0 - alpha): a double in the reference
        const float a_div = __fmul_rn(alpha, div_);                          // alpha * delta_iv (float)
        const double b_dvj = one_m_alpha * (double)dvj;                      // (1.0 - alpha) * delta_vj (double)
        for (int f = lane; f < p.k; f += 32) {                               // :321-335
            const float u = __ldcg(pu + f), vi = __ldcg(pi + f), vj = __ldcg(pj + f), vv = __ldcg(pt + f);
            const float t12 = __fsub_rn(__fmul_rn(-dij, __fsub_rn(vi, vj)), __fmul_rn(a_div, __fsub_rn(vi, vv)));
            const double eu = ((double)t12 - b_dvj * (double)__fsub_rn(vv, vj)) + (double)__fmul_rn(reg, u);
            __stcg(pu + f, sub_lr_d(u, lr, eu));
            const float ei = __fadd_rn(__fsub_rn(__fmul_rn(-dij, u), __fmul_rn(a_div, u)), __fmul_rn(reg, vi));
            __stcg(pi + f, __fsub_rn(vi, __fmul_rn(lr, ei)));
            const double ev = ((double)__fmul_rn(a_div, u) - b_dvj * (double)u) + (double)__fmul_rn(reg, vv);
            __stcg(pt + f, sub_lr_d(vv, lr, ev));
            const double ej = ((double)__fmul_rn(dij, u) + b_dvj * (double)u) + (double)__fmul_rn(reg, vj);
            __stcg(pj + f, sub_lr_d(vj, lr, ej));
        }
    } else {
        const float bi = __ldcg(p.B + m.i), bj = __ldcg(p.B + m.j);
        if (m.t < 0) {                                                       // recom_sbpr.pyx:247-265
            float part = 0.f;
            for (int f = lane; f < p.k; f += 32)
                part = __fadd_rn(part, __fmul_rn(__ldcg(pu + f), __fsub_rn(__ldcg(pi + f), __ldcg(pj + f))));
            const float z = sig_exact(__fadd_rn(__fsub_rn(bi, bj), group_sum<32>(part)));
            for (int f = lane; f < p.k; f += 32) {
                const float u = __ldcg(pu + f), vi = __ldcg(pi + f), vj = __ldcg(pj + f);
                __stcg(pu + f, __fadd_rn(u, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, __fsub_rn(vi, vj)), __fmul_rn(p.reg_u, u)))));
                __stcg(pi + f, __fadd_rn(vi, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, u), __fmul_rn(p.reg_v, vi)))));
                __stcg(pj + f, __fadd_rn(vj, __fmul_rn(lr, __fsub_rn(__fmul_rn(-z, u), __fmul_rn(p.reg_v, vj)))));
            }
            if (lane == 0) {                                                 // biases: not gated by use_bias in this branch
                __stcg(p.B + m.i, __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(z, __fmul_rn(p.reg_b, bi)))));
                __stcg(p.B + m.j, __fadd_rn(bj, __fmul_rn(lr, __fsub_rn(-z, __fmul_rn(p.reg_b, bj)))));
            }
            return;
        }
        const float bk = __ldcg(p.B + m.t);                                  // :269-297
        float xik = 0.f, xkj = 0.f;
        for (int f = lane; f < p.k; f += 32) {
            const float u = __ldcg(pu + f), vi = __ldcg(pi + f), vj = __ldcg(pj + f), vk = __ldcg(pt + f);
            xik = __fadd_rn(xik, __fmul_rn(u, __fsub_rn(vi, vk)));
            xkj = __fadd_rn(xkj, __fmul_rn(u, __fsub_rn(vk, vj)));
        }
        const float score_ik = __fadd_rn(__fsub_rn(bi, bk), group_sum<32>(xik));
        const float score_kj = __fadd_rn(__fsub_rn(bk, bj), group_sum<32>(xkj));
        const float s_uk = (float)(1.0 / (1.0 + (double)m.t_count));
        const float zik = sig_exact(__fmul_rn(score_ik, s_uk));
        const float zkj = sig_exact(score_kj);
        // k can be i: a position at the end of the list reads the next user's entry, which may be one of u's own items.
        // The reference then updates item_k / B[k] from the values item_i / B[i] have just been given.
        const bool k_is_i = m.t == m.i;
        for (int f = lane; f < p.k; f += 32) {
            const float u = __ldcg(pu + f), vi = __ldcg(pi + f), vj = __ldcg(pj + f), vk0 = __ldcg(pt + f);
            const float eu = __fsub_rn(__fadd_rn(__fmul_rn(__fmul_rn(zik, __fsub_rn(vi, vk0)), s_uk), __fmul_rn(zkj, __fsub_rn(vk0, vj))),
                                       __fmul_rn(p.reg_u, u));
            __stcg(pu + f, __fadd_rn(u, __fmul_rn(lr, eu)));
            const float vi_new = __fadd_rn(vi, __fmul_rn(lr, __fsub_rn(__fmul_rn(__fmul_rn(zik, u), s_uk), __fmul_rn(p.reg_v, vi))));
            __stcg(pi + f, vi_new);
            __stcg(pj + f, __fadd_rn(vj, __fmul_rn(lr, __fsub_rn(__fmul_rn(-zkj, u), __fmul_rn(p.reg_v, vj)))));
            const float vk = k_is_i ? vi_new : vk0;
            const float ek = __fsub_rn(__fsub_rn(__fmul_rn(zkj, u), __fmul_rn(__fmul_rn(zik, u), s_uk)), __fmul_rn(p.reg_v, vk));
            __stcg(pt + f, __fadd_rn(vk, __fmul_rn(lr, ek)));
        }
        if (p.use_bias && lane == 0) {
            const float bi_new = __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(__fmul_rn(zik, s_uk), __fmul_rn(p.reg_b, bi))));
            __stcg(p.B + m.i, bi_new);
            __stcg(p.B + m.j, __fadd_rn(bj, __fmul_rn(lr, __fsub_rn(-zkj, __fmul_rn(p.reg_b, bj)))));
            const float bk_cur = k_is_i ? bi_new : bk;
            __stcg(p.B + m.t, __fadd_rn(bk_cur, __fmul_rn(lr, __fsub_rn(__fsub_rn(zkj, __fmul_rn(zik, s_uk)), __fmul_rn(p.reg_b, bk_cur)))));
        }
    }
}

// metadata of stream entry s (read-only inputs: order-free)
template <int KIND>
__device__ __forceinline__ TriSample tri_resolve_stream(const TriParams& p, int64_t s)
{
    TriSample m;
    const int64_t ii = p.i_index[s];
    m.j = p.j_id[s];
    m.u = __ldg(p.coo_row + ii);
    m.i = __ldg(p.indices + ii);
    m.t = -1; m.t_count = 0;
    m.skip = row_contains(p.indices, __ldg(p.indptr + m.u), __ldg(p.indptr + m.u + 1), m.j);
    if (KIND == KIND_VEBPR) {
        m.t = p.v_id[s];
        if (m.t >= 0) m.skip = m.skip || row_contains(p.aux_items, __ldg(p.aux_indptr + m.u), __ldg(p.aux_indptr + m.u + 1), m.j);
    } else {
        const int64_t kidx = p.k_index[s];
        const bool in_array = kidx >= 0 && kidx < p.n_aux;
        const int32_t kid = in_array ? __ldg(p.aux_items + kidx) : -1;
        m.skip = m.skip || (m.j == kid);
        if (__ldg(p.aux_indptr + m.u + 1) > __ldg(p.aux_indptr + m.u) && in_array) { m.t = kid; m.t_count = __ldg(p.aux_counts + kidx); }
    }
    return m;
}

template <int KIND>
__global__ void __launch_bounds__(1024) tri_replay_window_kernel(const TriParams p)
{
    __shared__ int m_u[1024], m_i[1024], m_j[1024], m_t[1024], m_c[1024];
    __shared__ unsigned char m_todo[1024];
    __shared__ int s_u[32], s_i[32], s_j[32], s_t[32], s_pending[32];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long n_correct = 0, n_skipped = 0;
    for (int64_t base0 = 0; base0 < p.n_samples; base0 += 1024) {
        __syncthreads();
        {   // resolve 1024 samples at once, one per thread
            const int64_t s = base0 + threadIdx.x;
            TriSample m;
            m.u = m.i = m.j = 0; m.t = -1; m.t_count = 0; m.skip = true;
            if (s < p.n_samples) {
                m = tri_resolve_stream<KIND>(p, s);
                if (m.skip) ++n_skipped;
            }
            m_u[threadIdx.x] = m.u; m_i[threadIdx.x] = m.i; m_j[threadIdx.x] = m.j; m_t[threadIdx.x] = m.t;
            m_c[threadIdx.x] = m.t_count; m_todo[threadIdx.x] = m.skip ? 0 : 1;
        }
        __syncthreads();
        const int n_win = (int)min((int64_t)32, (p.n_samples - base0 + 31) / 32);
        for (int win = 0; win < n_win; ++win) {
            const int slot = win * 32 + w;
            TriSample m;
            m.u = m_u[slot]; m.i = m_i[slot]; m.j = m_j[slot]; m.t = m_t[slot]; m.t_count = m_c[slot]; m.skip = false;
            bool todo = m_todo[slot] != 0;
            __syncthreads();                        // previous window fully retired
            if (lane == 0) { s_u[w] = m.u; s_i[w] = m.i; s_j[w] = m.j; s_t[w] = m.t; s_pending[w] = todo ? 1 : 0; }
            for (;;) {
                if (!__syncthreads_or(todo)) break;
                bool run = false;
                if (todo) {
                    bool conflict = false;
                    if (lane < w && s_pending[lane]) {        // an earlier pending sample sharing the user row or an item row
                        const int ou = s_u[lane], oi = s_i[lane], oj = s_j[lane], ot = s_t[lane];
                        conflict = (ou == m.u) | (oi == m.i) | (oi == m.j) | (oj == m.i) | (oj == m.j);
                        if (m.t >= 0) conflict |= (oi == m.t) | (oj == m.t);
                        if (ot >= 0) conflict |= (ot == m.i) | (ot == m.j) | (ot == m.t);
                    }
                    run = !__any_sync(0xffffffffu, conflict);
                }
                __syncthreads();                    // everybody has read the snapshot of s_pending
                if (run) {
                    tri_apply_exact<KIND>(p, m, lane, n_correct);
                    todo = false;
                    if (lane == 0) s_pending[w] = 0;
                }
            }
        }
    }
    const unsigned long long sk = __reduce_add_sync(0xffffffffu, (unsigned)n_skipped);
    if (lane == 0) {
        if (KIND == KIND_VEBPR) atomicAdd(p.stats + 0, n_correct);
        atomicAdd(p.stats + 1, sk);
    }
}

// ---------------------------------------------------------------------------------------
template <int G, int NPL, bool VEC, int KIND>
static int launch_tri_hogwild(const TriParams& p, int64_t n_users, cudaStream_t st)
{
    constexpr int GPB = 256 / G;
    int occ = 1;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, tri_hogwild_kernel<G, NPL, VEC, KIND>, 256, 0));
    if (occ < 1) occ = 1;
    int64_t blocks = (int64_t)sm_count() * occ;
    // staleness cap (as b200_bpr_epoch): at most min(n_users, n_items) / 4 samples in flight
    int64_t cap = (n_users < p.n_items ? n_users : p.n_items) / 4;
    if (cap < 1) cap = 1;
    const int64_t cap_blocks = (cap + GPB - 1) / GPB;
    if (blocks > cap_blocks) blocks = cap_blocks;
    const int64_t need = (p.n_samples + GPB - 1) / GPB;
    if (blocks > need) blocks = need;
    if (blocks < 1) blocks = 1;
    ::b200::count_launch();
    tri_hogwild_kernel<G, NPL, VEC, KIND><<<(unsigned)blocks, 256, 0, st>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

template <int KIND>
static int tri_hogwild(const TriParams& p, int64_t n_users, cudaStream_t st)
{
    const RowLayout L = pick_layout(p.k);
    B200_REQUIRE(L.npl <= (L.vec ? 4 : 4), "k=%d is not supported by the VEBPR / SBPR kernels (k <= 512 with k %% 4 == 0, else k <= 128)", p.k);
#define CALL(G_, NPL_, VEC_)                                                                  \
    do {                                                                                      \
        if (NPL_ <= 4) return launch_tri_hogwild<G_, (NPL_ <= 4 ? NPL_ : 4), VEC_, KIND>(p, n_users, st); \
        ::b200::set_error("unsupported factor width");                                       \
        return B200_ERR_UNSUPPORTED;                                                          \
    } while (0)
    B200_DISPATCH_LAYOUT(L, CALL);
#undef CALL
    return B200_OK;
}

}  // namespace b200

using namespace b200;

static int check_common(const char* who, const void* indptr, const void* indices, const void* coo_row, const void* U, const void* V,
                        const void* stats, int k)
{
    B200_REQUIRE(indptr && indices && coo_row && U && V && stats, "%s: null pointer argument", who);
    B200_REQUIRE(k >= 1, "%s: k=%d", who, k);
    return B200_OK;
}

extern "C" int b200_vebpr_epoch(const int32_t* indptr, const int32_t* indices, const int32_t* coo_row, int64_t n_users,
                                int64_t n_items, int64_t nnz, const int32_t* view_indptr, const int32_t* view_indices,
                                float* U, float* V, int k, float lr, float reg, float alpha, uint64_t seed, uint64_t epoch,
                                int64_t n_samples, int64_t* stats, void* stream)
{
    int rc = check_common("b200_vebpr_epoch", indptr, indices, coo_row, U, V, stats, k);
    if (rc) return rc;
    B200_REQUIRE(view_indptr, "b200_vebpr_epoch: null view_indptr");
    B200_REQUIRE(n_items >= 1 && n_items < (1ll << 31) && nnz >= 1, "b200_vebpr_epoch: n_items=%lld nnz=%lld", (long long)n_items, (long long)nnz);
    if (n_samples <= 0) return B200_OK;
    TriParams p = {};
    p.indptr = indptr; p.indices = indices; p.coo_row = coo_row;
    p.aux_indptr = view_indptr; p.aux_items = view_indices; p.aux_counts = nullptr;
    p.n_items = n_items; p.nnz = nnz; p.n_aux = 0;
    p.U = U; p.V = V; p.B = nullptr; p.k = k; p.n_units = pick_layout(k).n_units;
    p.lr = lr; p.reg_u = reg; p.reg_v = reg; p.reg_b = 0.f; p.alpha = alpha; p.use_bias = 0;
    p.seed = seed; p.epoch = epoch; p.n_samples = n_samples;
    p.stats = reinterpret_cast<unsigned long long*>(stats);
    return tri_hogwild<KIND_VEBPR>(p, n_users, (cudaStream_t)stream);
}

extern "C" int b200_vebpr_epoch_replay(const int64_t* i_index, const int32_t* v_id, const int32_t* j_id, int64_t n_samples,
                                       const int32_t* indptr, const int32_t* indices, const int32_t* coo_row,
                                       const int32_t* view_indptr, const int32_t* view_indices,
                                       float* U, float* V, int k, float lr, float reg, float alpha, int64_t* stats, void* stream)
{
    int rc = check_common("b200_vebpr_epoch_replay", indptr, indices, coo_row, U, V, stats, k);
    if (rc) return rc;
    B200_REQUIRE(i_index && v_id && j_id && view_indptr, "b200_vebpr_epoch_replay: null pointer argument");
    if (n_samples <= 0) return B200_OK;
    TriParams p = {};
    p.indptr = indptr; p.indices = indices; p.coo_row = coo_row;
    p.aux_indptr = view_indptr; p.aux_items = view_indices;
    p.U = U; p.V = V; p.k = k; p.lr = lr; p.reg_u = reg; p.reg_v = reg; p.alpha = alpha;
    p.n_samples = n_samples; p.i_index = i_index; p.j_id = j_id; p.v_id = v_id;
    p.stats = reinterpret_cast<unsigned long long*>(stats);
    ::b200::count_launch();
    tri_replay_window_kernel<KIND_VEBPR><<<1, 1024, 0, (cudaStream_t)stream>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_sbpr_epoch(const int32_t* indptr, const int32_t* indices, const int32_t* coo_row, int64_t n_users,
                               int64_t n_items, int64_t nnz, const int32_t* social_indptr, const int32_t* social_item_ids,
                               const int32_t* social_item_counts, int64_t n_social,
                               float* U, float* V, float* B, int k, float lr, float lambda_u, float lambda_v, float lambda_b,
                               int use_bias, uint64_t seed, uint64_t epoch, int64_t n_samples, int64_t* stats, void* stream)
{
    int rc = check_common("b200_sbpr_epoch", indptr, indices, coo_row, U, V, stats, k);
    if (rc) return rc;
    B200_REQUIRE(B && social_indptr && (n_social == 0 || (social_item_ids && social_item_counts)), "b200_sbpr_epoch: null pointer argument");
    B200_REQUIRE(n_items >= 1 && n_items < (1ll << 31) && nnz >= 1, "b200_sbpr_epoch: n_items=%lld nnz=%lld", (long long)n_items, (long long)nnz);
    if (n_samples <= 0) return B200_OK;
    TriParams p = {};
    p.indptr = indptr; p.indices = indices; p.coo_row = coo_row;
    p.aux_indptr = social_indptr; p.aux_items = social_item_ids; p.aux_counts = social_item_counts;
    p.n_items = n_items; p.nnz = nnz; p.n_aux = n_social;
    p.U = U; p.V = V; p.B = B; p.k = k; p.n_units = pick_layout(k).n_units;
    p.lr = lr; p.reg_u = lambda_u; p.reg_v = lambda_v; p.reg_b = lambda_b; p.use_bias = use_bias;
    p.seed = seed; p.epoch = epoch; p.n_samples = n_samples;
    p.stats = reinterpret_cast<unsigned long long*>(stats);
    return tri_hogwild<KIND_SBPR>(p, n_users, (cudaStream_t)stream);
}

extern "C" int b200_sbpr_epoch_replay(const int64_t* i_index, const int32_t* j_id, const int64_t* k_index, int64_t n_samples,
                                      const int32_t* indptr, const int32_t* indices, const int32_t* coo_row,
                                      const int32_t* social_indptr, const int32_t* social_item_ids,
                                      const int32_t* social_item_counts, int64_t n_social,
                                      float* U, float* V, float* B, int k, float lr, float lambda_u, float lambda_v, float lambda_b,
                                      int use_bias, int64_t* stats, void* stream)
{
    int rc = check_common("b200_sbpr_epoch_replay", indptr, indices, coo_row, U, V, stats, k);
    if (rc) return rc;
    B200_REQUIRE(i_index && j_id && k_index && B && social_indptr && (n_social == 0 || (social_item_ids && social_item_counts)),
                 "b200_sbpr_epoch_replay: null pointer argument");
    if (n_samples <= 0) return B200_OK;
    TriParams p = {};
    p.indptr = indptr; p.indices = indices; p.coo_row = coo_row;
    p.aux_indptr = social_indptr; p.aux_items = social_item_ids; p.aux_counts = social_item_counts; p.n_aux = n_social;
    p.U = U; p.V = V; p.B = B; p.k = k; p.lr = lr; p.reg_u = lambda_u; p.reg_v = lambda_v; p.reg_b = lambda_b; p.use_bias = use_bias;
    p.n_samples = n_samples; p.i_index = i_index; p.j_id = j_id; p.k_index = k_index;
    p.stats = reinterpret_cast<unsigned long long*>(stats);
    ::b200::count_launch();
    tri_replay_window_kernel<KIND_SBPR><<<1, 1024, 0, (cudaStream_t)stream>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
