// MTER (cornac/models/mter/recom_mter.pyx:434-675) for sm_90a: the seeded fit, bit-identical to the reference's serial
// float loop given the same sample draws, and the rank queries of the device scoring path.
//
// One iteration of the reference reads the parameters it started with everywhere and writes them only in its final
// AdaGrad step, so it splits into independent chains:
//   phase 1  the predictions: one f32 chain of d1*d2*d3 terms per element sample, two per BPR sample (the two lanes of
//            a pair compute score(i) and score(j) side by side and swap them); the sample's coefficient
//            (2 (pred - score), or lambda_bpr z s) and the ids it touches.
//   phase 2  which (matrix, row) each touch slot is the first to name: that slot owns the row's accumulator.
//   phase 3  every accumulator element as one ordered f32 chain over the samples that touch it, in the reference's
//            order (element samples: uia, uao, iao terms; then the BPR samples; (i, j, k) order inside a sample): a
//            thread per core-tensor element and per (owned row, column).  The result goes to a dense `del` buffer.
//   phase 4  the dense AdaGrad step over every parameter, which also clears `del` for the next iteration.
// The phases are separated by grid-wide barriers of one cooperative launch, so a call of n iterations is one launch.
// Every f32 operation is an explicitly rounded __f*_rn intrinsic (no contraction into FMA), in the reference's grouping:
// products left to right.  The BPR weight uses glibc's expf (expf.cuh), as the compiled reference does.
#include "common.cuh"
#include "expf.cuh"

#include <cooperative_groups.h>

#include <algorithm>

namespace cg = cooperative_groups;

namespace b200 {

constexpr int MTER_THREADS = 256;
enum { M_U = 0, M_I, M_A, M_O, M_G1, M_G2, M_G3, M_N };

struct MterArgs {
    int64_t n_users, n_items, n_aspects, n_opinions;
    int d1, d2, d3, d4;
    const float* X;
    const int32_t *X_u, *X_i, *X_a;
    const float* YU;
    const int32_t *YU_u, *YU_a, *YU_o;
    const float* YI;
    const int32_t *YI_i, *YI_a, *YI_o;
    const int32_t *indptr, *indices, *rrow;
    const float* rval;
    int n_el, n_bpr, n_iter;
    const int32_t* draws;
    float* P[M_N];
    float* S[M_N];
    float* D[M_N];
    int64_t cnt[M_N];
    float* coef;       // [3 n_el + n_bpr]: 2 (pred - score) of each element sample, then del_bpr of each BPR sample
    int32_t* ids;      // [9 n_el + 4 n_bpr]: (u, i, a), (u, a, o), (i, a, o) per element sample, (u, i, j, live) per BPR
    int64_t* keys;     // [9 n_el + 4 n_bpr]: matrix << 40 | row of every touch slot
    uint8_t* owner;    // [9 n_el + 4 n_bpr]
    float lr, ld_reg, ld_bpr;
    int core_smem;
    unsigned long long* counts;   // += correct, skipped
    double* losses;               // += loss, bpr_loss (f64)
    int32_t* first;               // per (matrix, row): n_slots - (first slot naming it), 0 when unnamed
    int64_t row_off[4];           // offset of U, I, A, O rows in `first`
    float* aterms;                // [d3][aterm_stride]: the BPR terms of the A[n_aspects] chain, in chain order
    int64_t aterm_stride;
    int unordered, philox;        // B200_MTER_UNORDERED, B200_MTER_PHILOX
    uint32_t key0, key1;
    uint64_t iter0;
    int64_t n_x, n_yu, n_yi, nnz;
    unsigned long long* phase_ns; // += device time of each phase (block 0's view), or NULL
};

__device__ __forceinline__ float mul4(float a, float b, float c, float d)
{
    return __fmul_rn(__fmul_rn(__fmul_rn(a, b), c), d);
}

// sum over (p, q, r) of G[p, q, r] * x[p] * y[q] * w[r]: the reference's get_score, one serial f32 chain
__device__ float score3(const float* G, int n1, int n2, int n3, const float* x, const float* y, const float* w)
{
    float s = 0.f;
    for (int p = 0; p < n1; ++p)
        for (int q = 0; q < n2; ++q) {
            const float* g = G + ((int64_t)p * n2 + q) * n3;
            for (int r = 0; r < n3; ++r) s = __fadd_rn(s, __fmul_rn(__fmul_rn(__fmul_rn(g[r], x[p]), y[q]), w[r]));
        }
    return s;
}

// has_non_zero + the position: CSR columns are sorted
__device__ int64_t find_col(const int32_t* indptr, const int32_t* indices, int32_t r, int32_t c)
{
    int64_t lo = indptr[r], hi = indptr[r + 1];
    const int64_t end = hi;
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo) / 2;
        if (indices[mid] < c) lo = mid + 1;
        else hi = mid;
    }
    return (lo < end && indices[lo] == c) ? lo : -1;
}

// draw k of this iteration: the caller's stream, or Philox4x32-10 of (k, iteration) reduced to [0, n)
__device__ __forceinline__ int64_t mter_draw(const MterArgs& a, const int32_t* dr, int it, int64_t k, int64_t n)
{
    if (!a.philox) return dr[k];
    const uint64_t itg = a.iter0 + (uint64_t)it;
    const Philox4 r = philox4x32_10((uint32_t)k, (uint32_t)itg, (uint32_t)(itg >> 32), 0x4d544552u, a.key0, a.key1);
    return (int64_t)range64(r.x, r.y, (uint64_t)n);
}

__device__ __forceinline__ int64_t key_index(const MterArgs& a, int64_t key)
{
    return a.row_off[key >> 40] + (key & ((1ll << 40) - 1));
}

__device__ __forceinline__ int mat_cols(const MterArgs& a, int m)
{
    return m == M_U ? a.d1 : m == M_I ? a.d2 : m == M_A ? a.d3 : a.d4;
}

// phase 1: predictions, coefficients, ids and touch keys of one iteration
__device__ void mter_predict(const MterArgs& a, const int32_t* dr, int it, const float* G1, const float* G2,
                             const float* G3)
{
    const int64_t n_slots = 9ll * a.n_el + 4ll * a.n_bpr;
    const int n_el = a.n_el, n_bpr = a.n_bpr;
    const int d1 = a.d1, d2 = a.d2, d3 = a.d3, d4 = a.d4;
    const float *U = a.P[M_U], *I = a.P[M_I], *A = a.P[M_A], *O = a.P[M_O];
    const float* An = A + a.n_aspects * d3;
    const int64_t total = 2ll * n_bpr + 3ll * n_el;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t* keys_bpr = a.keys + 9ll * n_el;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += stride) {
        if (w < 2ll * n_bpr) {
            const int t = (int)(w >> 1), side = (int)(w & 1);
            const int64_t idx = mter_draw(a, dr, it, 3ll * n_el + t, a.nnz);
            const int32_t u = a.rrow[idx], i = a.indices[idx];
            const int32_t j = (int32_t)mter_draw(a, dr, it, 3ll * n_el + n_bpr + t, a.n_items);
            float s = 1.f;
            bool skip = false;
            const int64_t jp = find_col(a.indptr, a.indices, u, j);
            if (jp >= 0) {
                const float is = a.rval[idx], js = a.rval[jp];
                if (is == js) skip = true;
                else if (is < js) s = -1.f;
            }
            float sc = 0.f;
            if (!skip) sc = score3(G1, d1, d2, d3, U + (int64_t)u * d1, I + (int64_t)(side ? j : i) * d2, An);
            const unsigned pair = 3u << (threadIdx.x & 30);
            const float other = __shfl_xor_sync(pair, sc, 1);
            if (side == 0) {
                int32_t* id = a.ids + 9ll * n_el + 4ll * t;
                id[0] = u; id[1] = i; id[2] = j; id[3] = skip ? 0 : 1;
                keys_bpr[4ll * t + 0] = ((int64_t)M_U << 40) | u;
                keys_bpr[4ll * t + 1] = ((int64_t)M_I << 40) | i;
                keys_bpr[4ll * t + 2] = ((int64_t)M_I << 40) | j;
                keys_bpr[4ll * t + 3] = ((int64_t)M_A << 40) | a.n_aspects;
                if (!a.unordered)
                    for (int k = 0; k < 4; ++k)
                        atomicMax(a.first + key_index(a, keys_bpr[4ll * t + k]), (int32_t)(n_slots - (9ll * n_el + 4ll * t + k)));
                if (skip) {
                    a.coef[3 * n_el + t] = 0.f;
                    atomicAdd(a.counts + 1, 1ull);     // its slots may own a row: the row's chain then sums no term
                } else {
                    const float pred = __fmul_rn(__fsub_rn(sc, other), s);
                    const float z = __double2float_rn(__ddiv_rn(1.0, __dadd_rn(1.0, (double)glibc_expf(pred))));
                    if ((double)z < 0.5) atomicAdd(a.counts + 0, 1ull);
                    a.coef[3 * n_el + t] = __fmul_rn(__fmul_rn(a.ld_bpr, z), s);
                    if (a.losses) atomicAdd(a.losses + 1, log(1.0 / (1.0 + (double)glibc_expf(-pred))));
                }
            }
        } else {
            const int64_t e = w - 2ll * n_bpr;
            const int kind = (int)(e / n_el), t = (int)(e % n_el);
            const int64_t idx = mter_draw(a, dr, it, (int64_t)kind * n_el + t, kind == 0 ? a.n_x : kind == 1 ? a.n_yu : a.n_yi);
            int32_t x, y, zz;
            float score, pred;
            int64_t k0, k1, k2;
            if (kind == 0) {
                x = a.X_u[idx]; y = a.X_i[idx]; zz = a.X_a[idx]; score = a.X[idx];
                pred = score3(G1, d1, d2, d3, U + (int64_t)x * d1, I + (int64_t)y * d2, A + (int64_t)zz * d3);
                k0 = (int64_t)M_U << 40 | x; k1 = (int64_t)M_I << 40 | y; k2 = (int64_t)M_A << 40 | zz;
            } else if (kind == 1) {
                x = a.YU_u[idx]; y = a.YU_a[idx]; zz = a.YU_o[idx]; score = a.YU[idx];
                pred = score3(G2, d1, d3, d4, U + (int64_t)x * d1, A + (int64_t)y * d3, O + (int64_t)zz * d4);
                k0 = (int64_t)M_U << 40 | x; k1 = (int64_t)M_A << 40 | y; k2 = (int64_t)M_O << 40 | zz;
            } else {
                x = a.YI_i[idx]; y = a.YI_a[idx]; zz = a.YI_o[idx]; score = a.YI[idx];
                pred = score3(G3, d2, d3, d4, I + (int64_t)x * d2, A + (int64_t)y * d3, O + (int64_t)zz * d4);
                k0 = (int64_t)M_I << 40 | x; k1 = (int64_t)M_A << 40 | y; k2 = (int64_t)M_O << 40 | zz;
            }
            const float diff = __fsub_rn(pred, score);
            a.coef[kind * n_el + t] = __fmul_rn(2.f, diff);      // (float)(2.0 * diff) is exact either way
            int32_t* id = a.ids + 3ll * (kind * n_el + t);
            id[0] = x; id[1] = y; id[2] = zz;
            int64_t* k = a.keys + 3ll * (kind * n_el + t);
            k[0] = k0; k[1] = k1; k[2] = k2;
            if (!a.unordered)
                for (int q = 0; q < 3; ++q)
                    atomicMax(a.first + key_index(a, k[q]), (int32_t)(n_slots - (3ll * (kind * n_el + t) + q)));
            if (a.losses) atomicAdd(a.losses, (double)__fmul_rn(diff, diff));
        }
    }
}

// phase 2: slot s owns its row when it is the first slot naming it (the largest n_slots - s of phase 1's atomicMax);
// and every term of the longest chain, A[n_aspects]'s BPR part, stored in chain order so that phase 3 only adds
__device__ void mter_owners(const MterArgs& a, const float* G1)
{
    const int64_t n_slots = 9ll * a.n_el + 4ll * a.n_bpr;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (int64_t s = gtid; s < n_slots; s += stride)
        a.owner[s] = a.first[key_index(a, a.keys[s])] == (int32_t)(n_slots - s);
    const int d1 = a.d1, d2 = a.d2, d3 = a.d3, n_el = a.n_el;
    const int64_t pq = (int64_t)d1 * d2, per_c = (int64_t)a.n_bpr * pq;
    const float *U = a.P[M_U], *I = a.P[M_I];
    for (int64_t w = gtid; w < per_c * d3; w += stride) {
        const int c = (int)(w / per_c);
        const int64_t e = w - c * per_c;
        const int t = (int)(e / pq), p = (int)(e % pq) / d2, q = (int)(e % d2);
        const int32_t* id = a.ids + 9ll * n_el + 4ll * t;
        float v = 0.f;                 // a skipped sample: acc - (+0) == acc for every acc
        if (id[3]) {
            const float db = a.coef[3 * n_el + t];
            v = mul4(db, G1[(p * d2 + q) * d3 + c], U[(int64_t)id[0] * d1 + p],
                     __fsub_rn(I[(int64_t)id[1] * d2 + q], I[(int64_t)id[2] * d2 + q]));
        }
        a.aterms[c * a.aterm_stride + e] = v;
    }
}

// phase 3, rows: accumulator element (m, row, c) as the reference's loops build it
__device__ float row_chain(const MterArgs& a, const float* G1, const float* G2, const float* G3, int m, int32_t row, int c)
{
    const int n_el = a.n_el, n_bpr = a.n_bpr;
    const int d1 = a.d1, d2 = a.d2, d3 = a.d3, d4 = a.d4;
    const float *U = a.P[M_U], *I = a.P[M_I], *A = a.P[M_A], *O = a.P[M_O];
    float acc = 0.f;
    for (int t = 0; t < n_el; ++t) {
        {   // user item aspect: G1 (d1, d2, d3) against U[u], I[i], A[a]
            const int32_t* id = a.ids + 3ll * t;
            const int32_t u = id[0], i = id[1], as = id[2];
            const float ds = a.coef[t];
            const float *Ur = U + (int64_t)u * d1, *Ir = I + (int64_t)i * d2, *Ar = A + (int64_t)as * d3;
            if (m == M_U && u == row)
                for (int q = 0; q < d2; ++q)
                    for (int r = 0; r < d3; ++r) acc = __fadd_rn(acc, mul4(ds, G1[(c * d2 + q) * d3 + r], Ir[q], Ar[r]));
            if (m == M_I && i == row)
                for (int p = 0; p < d1; ++p)
                    for (int r = 0; r < d3; ++r) acc = __fadd_rn(acc, mul4(ds, G1[(p * d2 + c) * d3 + r], Ur[p], Ar[r]));
            if (m == M_A && as == row)
                for (int p = 0; p < d1; ++p)
                    for (int q = 0; q < d2; ++q) acc = __fadd_rn(acc, mul4(ds, G1[(p * d2 + q) * d3 + c], Ur[p], Ir[q]));
        }
        {   // user aspect opinion: G2 (d1, d3, d4) against U[u], A[a], O[o]
            const int32_t* id = a.ids + 3ll * (n_el + t);
            const int32_t u = id[0], as = id[1], o = id[2];
            const float ds = a.coef[n_el + t];
            const float *Ur = U + (int64_t)u * d1, *Ar = A + (int64_t)as * d3, *Or = O + (int64_t)o * d4;
            if (m == M_U && u == row)
                for (int q = 0; q < d3; ++q)
                    for (int r = 0; r < d4; ++r) acc = __fadd_rn(acc, mul4(ds, G2[(c * d3 + q) * d4 + r], Ar[q], Or[r]));
            if (m == M_A && as == row)
                for (int p = 0; p < d1; ++p)
                    for (int r = 0; r < d4; ++r) acc = __fadd_rn(acc, mul4(ds, G2[(p * d3 + c) * d4 + r], Ur[p], Or[r]));
            if (m == M_O && o == row)
                for (int p = 0; p < d1; ++p)
                    for (int q = 0; q < d3; ++q) acc = __fadd_rn(acc, mul4(ds, G2[(p * d3 + q) * d4 + c], Ur[p], Ar[q]));
        }
        {   // item aspect opinion: G3 (d2, d3, d4) against I[i], A[a], O[o]
            const int32_t* id = a.ids + 3ll * (2 * n_el + t);
            const int32_t i = id[0], as = id[1], o = id[2];
            const float ds = a.coef[2 * n_el + t];
            const float *Ir = I + (int64_t)i * d2, *Ar = A + (int64_t)as * d3, *Or = O + (int64_t)o * d4;
            if (m == M_I && i == row)
                for (int q = 0; q < d3; ++q)
                    for (int r = 0; r < d4; ++r) acc = __fadd_rn(acc, mul4(ds, G3[(c * d3 + q) * d4 + r], Ar[q], Or[r]));
            if (m == M_A && as == row)
                for (int p = 0; p < d2; ++p)
                    for (int r = 0; r < d4; ++r) acc = __fadd_rn(acc, mul4(ds, G3[(p * d3 + c) * d4 + r], Ir[p], Or[r]));
            if (m == M_O && o == row)
                for (int p = 0; p < d2; ++p)
                    for (int q = 0; q < d3; ++q) acc = __fadd_rn(acc, mul4(ds, G3[(p * d3 + q) * d4 + c], Ir[p], Ar[q]));
        }
    }
    if (m == M_O) return acc;
    if (m == M_A) {
        if (row != a.n_aspects) return acc;
        // the stored terms of phase 2, subtracted in order: only the adds are serial here
        const float* tp = a.aterms + (int64_t)c * a.aterm_stride;
        const int64_t n = (int64_t)n_bpr * d1 * d2, n4 = n / 4;
        const float4* t4 = reinterpret_cast<const float4*>(tp);
        constexpr int BATCH = 16;           // loads in flight: the L2 latency is hidden behind the previous adds
        int64_t k = 0;
        for (; k + BATCH <= n4; k += BATCH) {
            float4 v[BATCH];
#pragma unroll
            for (int b = 0; b < BATCH; ++b) v[b] = t4[k + b];
#pragma unroll
            for (int b = 0; b < BATCH; ++b)
                acc = __fsub_rn(__fsub_rn(__fsub_rn(__fsub_rn(acc, v[b].x), v[b].y), v[b].z), v[b].w);
        }
        for (; k < n4; ++k) {
            const float4 v = t4[k];
            acc = __fsub_rn(__fsub_rn(__fsub_rn(__fsub_rn(acc, v.x), v.y), v.z), v.w);
        }
        for (int64_t k = n4 * 4; k < n; ++k) acc = __fsub_rn(acc, tp[k]);
        return acc;
    }
    const float* An = A + a.n_aspects * d3;
    for (int t = 0; t < n_bpr; ++t) {
        const int32_t* id = a.ids + 9ll * n_el + 4ll * t;
        if (!id[3]) continue;
        const int32_t u = id[0], i = id[1], j = id[2];
        const float db = a.coef[3 * n_el + t];
        const float *Ur = U + (int64_t)u * d1, *Ii = I + (int64_t)i * d2, *Ij = I + (int64_t)j * d2;
        if (m == M_U && u == row)
            for (int q = 0; q < d2; ++q) {
                const float iij = __fsub_rn(Ii[q], Ij[q]);
                for (int r = 0; r < d3; ++r) acc = __fsub_rn(acc, mul4(db, G1[(c * d2 + q) * d3 + r], iij, An[r]));
            }
        if (m == M_I && (i == row || j == row)) {
            for (int p = 0; p < d1; ++p)
                for (int r = 0; r < d3; ++r) {
                    const float v = mul4(db, G1[(p * d2 + c) * d3 + r], Ur[p], An[r]);
                    acc = i == row ? __fsub_rn(acc, v) : __fadd_rn(acc, v);
                }
        }
    }
    return acc;
}

// phase 3, cores: element e of G1, G2 or G3
__device__ float core_chain(const MterArgs& a, int g, int e)
{
    const int n_el = a.n_el, n_bpr = a.n_bpr;
    const int d1 = a.d1, d2 = a.d2, d3 = a.d3, d4 = a.d4;
    const float *U = a.P[M_U], *I = a.P[M_I], *A = a.P[M_A], *O = a.P[M_O];
    float acc = 0.f;
    if (g == 0) {
        const int p = e / (d2 * d3), q = (e / d3) % d2, r = e % d3;
        for (int t = 0; t < n_el; ++t) {
            const int32_t* id = a.ids + 3ll * t;
            acc = __fadd_rn(acc, mul4(a.coef[t], U[(int64_t)id[0] * d1 + p], I[(int64_t)id[1] * d2 + q],
                                      A[(int64_t)id[2] * d3 + r]));
        }
        const float an = A[a.n_aspects * d3 + r];
        for (int t = 0; t < n_bpr; ++t) {
            const int32_t* id = a.ids + 9ll * n_el + 4ll * t;
            if (!id[3]) continue;
            const float iij = __fsub_rn(I[(int64_t)id[1] * d2 + q], I[(int64_t)id[2] * d2 + q]);
            acc = __fsub_rn(acc, mul4(a.coef[3 * n_el + t], U[(int64_t)id[0] * d1 + p], iij, an));
        }
    } else if (g == 1) {
        const int p = e / (d3 * d4), q = (e / d4) % d3, r = e % d4;
        for (int t = 0; t < n_el; ++t) {
            const int32_t* id = a.ids + 3ll * (n_el + t);
            acc = __fadd_rn(acc, mul4(a.coef[n_el + t], U[(int64_t)id[0] * d1 + p], A[(int64_t)id[1] * d3 + q],
                                      O[(int64_t)id[2] * d4 + r]));
        }
    } else {
        const int p = e / (d3 * d4), q = (e / d4) % d3, r = e % d4;
        for (int t = 0; t < n_el; ++t) {
            const int32_t* id = a.ids + 3ll * (2 * n_el + t);
            acc = __fadd_rn(acc, mul4(a.coef[2 * n_el + t], I[(int64_t)id[0] * d2 + p], A[(int64_t)id[1] * d3 + q],
                                      O[(int64_t)id[2] * d4 + r]));
        }
    }
    return acc;
}

__device__ void mter_gradients(const MterArgs& a, const float* G1, const float* G2, const float* G3)
{
    const int64_t nG1 = a.cnt[M_G1], nG2 = a.cnt[M_G2], nG3 = a.cnt[M_G3];
    const int dmax = max(max(a.d1, a.d2), max(a.d3, a.d4));
    const int64_t n_slots = 9ll * a.n_el + 4ll * a.n_bpr;
    const int64_t n_row_items = n_slots * dmax;
    const int64_t total = n_row_items + nG1 + nG2 + nG3;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += stride) {
        if (w < n_row_items) {
            // the BPR slots (and so the aspect row every BPR sample touches, the longest chain) come first
            const int64_t s = (w / dmax + 9ll * a.n_el) % n_slots;
            const int c = (int)(w % dmax);
            if (!a.owner[s]) continue;
            const int64_t key = a.keys[s];
            if (c == 0) a.first[key_index(a, key)] = 0;        // cleared for the next iteration
            const int m = (int)(key >> 40);
            const int32_t row = (int32_t)(key & ((1ll << 40) - 1));
            if (c >= mat_cols(a, m)) continue;
            a.D[m][(int64_t)row * mat_cols(a, m) + c] = row_chain(a, G1, G2, G3, m, row, c);
        } else {
            int64_t e = w - n_row_items;
            int g = 0;
            if (e >= nG1) { e -= nG1; g = 1; if (e >= nG2) { e -= nG2; g = 2; } }
            a.D[M_G1 + g][e] = core_chain(a, g, (int)e);
        }
    }
}

// phase 4: the reference's dense AdaGrad step (recom_mter.pyx:611-673) on every element; clears del
__device__ void mter_adagrad(const MterArgs& a)
{
    const float eps = 1e-9f;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int m = 0; m < M_N; ++m) {
        float *x = a.P[m], *sg = a.S[m], *del = a.D[m];
        for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < a.cnt[m]; e += stride) {
            const float d = del[e];
            const float xv = x[e];
            float reg = 0.f;
            if (d != 0.0f) {
                reg = __fadd_rn(d, __fmul_rn(a.ld_reg, xv));
                del[e] = 0.f;
            }
            const float s = __fadd_rn(sg[e], __fadd_rn(eps, __fmul_rn(reg, reg)));
            sg[e] = s;
            float nx = __double2float_rn(
                __dsub_rn((double)xv, __dmul_rn(__ddiv_rn((double)a.lr, (double)__fsqrt_rn(s)), (double)reg)));
            if (nx < 0) nx = 0;
            x[e] = nx;
        }
    }
}

// Unordered mode, phase 3: the core elements as in the exact mode (each a short chain over the samples), and one warp
// per sample adding its row gradients with atomics: for a sample (x, y, w) of core G and weight c,
// dx[p] += c sum_qr G[p,q,r] y[q] w[r], dy[q] += c sum_pr G[p,q,r] x[p] w[r], dw[r] += c sum_pq G[p,q,r] x[p] y[q]
// (a BPR sample: x = U[u], y = I[i] - I[j], w = A[n_aspects], c = -del_bpr, and I[j] takes -dy).  f32 atomics: the
// sums are not in a fixed order, so the result can differ from run to run by rounding.
__device__ void sample_rows(const float* G, int n1, int n2, int n3, const float* x, const float* y, const float* y2,
                            const float* w, float c, float* dx, float* dy, float* dy2, float* dw, int lane)
{
    auto yv = [&](int q) { return y2 ? y[q] - y2[q] : y[q]; };
    for (int o = lane; o < n1 + n2 + n3; o += 32) {
        float sum = 0.f;
        if (o < n1) {
            for (int q = 0; q < n2; ++q) {
                const float yq = yv(q);
                for (int r = 0; r < n3; ++r) sum += G[(o * n2 + q) * n3 + r] * yq * w[r];
            }
            atomicAdd(dx + o, c * sum);
        } else if (o < n1 + n2) {
            const int q = o - n1;
            for (int p = 0; p < n1; ++p)
                for (int r = 0; r < n3; ++r) sum += G[(p * n2 + q) * n3 + r] * x[p] * w[r];
            atomicAdd(dy + q, c * sum);
            if (dy2) atomicAdd(dy2 + q, -c * sum);
        } else {
            const int r = o - n1 - n2;
            for (int p = 0; p < n1; ++p)
                for (int q = 0; q < n2; ++q) sum += G[(p * n2 + q) * n3 + r] * x[p] * yv(q);
            atomicAdd(dw + r, c * sum);
        }
    }
}

__device__ void mter_gradients_unordered(const MterArgs& a, const float* G1, const float* G2, const float* G3)
{
    const int64_t nG1 = a.cnt[M_G1], nG2 = a.cnt[M_G2], nG3 = a.cnt[M_G3];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (int64_t e = gtid; e < nG1 + nG2 + nG3; e += stride) {
        int64_t f = e;
        int g = 0;
        if (f >= nG1) { f -= nG1; g = 1; if (f >= nG2) { f -= nG2; g = 2; } }
        a.D[M_G1 + g][f] = core_chain(a, g, (int)f);
    }
    const int d1 = a.d1, d2 = a.d2, d3 = a.d3, d4 = a.d4, n_el = a.n_el;
    const float *U = a.P[M_U], *I = a.P[M_I], *A = a.P[M_A], *O = a.P[M_O];
    float *dU = a.D[M_U], *dI = a.D[M_I], *dA = a.D[M_A], *dO = a.D[M_O];
    const int lane = threadIdx.x & 31;
    const int64_t n_samples = 3ll * n_el + a.n_bpr;
    for (int64_t sm = gtid >> 5; sm < n_samples; sm += stride >> 5) {
        const float c = a.coef[sm];
        if (sm < 3ll * n_el) {
            const int32_t* id = a.ids + 3 * sm;
            const int kind = (int)(sm / n_el);
            if (kind == 0)
                sample_rows(G1, d1, d2, d3, U + (int64_t)id[0] * d1, I + (int64_t)id[1] * d2, nullptr,
                            A + (int64_t)id[2] * d3, c, dU + (int64_t)id[0] * d1, dI + (int64_t)id[1] * d2, nullptr,
                            dA + (int64_t)id[2] * d3, lane);
            else if (kind == 1)
                sample_rows(G2, d1, d3, d4, U + (int64_t)id[0] * d1, A + (int64_t)id[1] * d3, nullptr,
                            O + (int64_t)id[2] * d4, c, dU + (int64_t)id[0] * d1, dA + (int64_t)id[1] * d3, nullptr,
                            dO + (int64_t)id[2] * d4, lane);
            else
                sample_rows(G3, d2, d3, d4, I + (int64_t)id[0] * d2, A + (int64_t)id[1] * d3, nullptr,
                            O + (int64_t)id[2] * d4, c, dI + (int64_t)id[0] * d2, dA + (int64_t)id[1] * d3, nullptr,
                            dO + (int64_t)id[2] * d4, lane);
        } else {
            const int32_t* id = a.ids + 9ll * n_el + 4ll * (sm - 3ll * n_el);
            if (!id[3]) continue;
            sample_rows(G1, d1, d2, d3, U + (int64_t)id[0] * d1, I + (int64_t)id[1] * d2, I + (int64_t)id[2] * d2,
                        A + a.n_aspects * d3, -c, dU + (int64_t)id[0] * d1, dI + (int64_t)id[1] * d2,
                        dI + (int64_t)id[2] * d2, dA + a.n_aspects * d3, lane);
        }
    }
}

__device__ __forceinline__ uint64_t global_ns()
{
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__global__ void __launch_bounds__(MTER_THREADS) mter_fit_kernel(MterArgs a)
{
    extern __shared__ float sh_core[];
    cg::grid_group grid = cg::this_grid();
    const int64_t per_iter = 3ll * a.n_el + 2ll * a.n_bpr;
    const int64_t nG1 = a.cnt[M_G1], nG2 = a.cnt[M_G2], nG3 = a.cnt[M_G3];
    const float *G1 = a.P[M_G1], *G2 = a.P[M_G2], *G3 = a.P[M_G3];
    if (a.core_smem) {
        G1 = sh_core;
        G2 = sh_core + nG1;
        G3 = sh_core + nG1 + nG2;
    }
    const bool timer = a.phase_ns && blockIdx.x == 0 && threadIdx.x == 0;
    uint64_t t0 = timer ? global_ns() : 0;
    auto mark = [&](int k) {
        if (timer) {
            const uint64_t t1 = global_ns();
            a.phase_ns[k] += t1 - t0;
            t0 = t1;
        }
    };
    for (int it = 0; it < a.n_iter; ++it) {
        if (a.core_smem) {      // the cores as this iteration starts (phase 4 of the last one wrote them)
            for (int64_t e = threadIdx.x; e < nG1 + nG2 + nG3; e += blockDim.x)
                sh_core[e] = e < nG1 ? a.P[M_G1][e] : e < nG1 + nG2 ? a.P[M_G2][e - nG1] : a.P[M_G3][e - nG1 - nG2];
            __syncthreads();
        }
        mter_predict(a, a.draws + (a.philox ? 0 : per_iter * it), it, G1, G2, G3);
        grid.sync();
        mark(0);
        if (a.unordered) {
            mter_gradients_unordered(a, G1, G2, G3);
        } else {
            mter_owners(a, G1);
            grid.sync();
            mark(1);
            mter_gradients(a, G1, G2, G3);
        }
        grid.sync();
        mark(2);
        mter_adagrad(a);
        grid.sync();
        mark(3);
    }
}

// rank queries: M[p, q] = f32(sum_r G1[p, q, r] a[r]), Q[u, q] = f32(sum_p U[u, p] M[p, q]); f64 sums in index order
__global__ void __launch_bounds__(MTER_THREADS) mter_queries_kernel(const float* __restrict__ U, int64_t n_users,
                                                                    const float* __restrict__ G1,
                                                                    const float* __restrict__ a_last, int d1, int d2,
                                                                    int d3, float* __restrict__ Q)
{
    extern __shared__ float sh_m[];
    for (int e = threadIdx.x; e < d1 * d2; e += blockDim.x) {
        double s = 0.0;
        for (int r = 0; r < d3; ++r) s = __dadd_rn(s, __dmul_rn((double)G1[(int64_t)e * d3 + r], (double)a_last[r]));
        sh_m[e] = __double2float_rn(s);
    }
    __syncthreads();
    const int64_t n = n_users * d2;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t u = w / d2;
        const int q = (int)(w % d2);
        double s = 0.0;
        for (int p = 0; p < d1; ++p) s = __dadd_rn(s, __dmul_rn((double)U[u * d1 + p], (double)sh_m[p * d2 + q]));
        Q[w] = __double2float_rn(s);
    }
}

}  // namespace b200

using namespace b200;

static int64_t mter_counts(int64_t n_users, int64_t n_items, int64_t n_aspects, int64_t n_opinions, int d1, int d2,
                           int d3, int d4, int64_t* cnt)
{
    cnt[M_U] = n_users * d1;
    cnt[M_I] = n_items * d2;
    cnt[M_A] = (n_aspects + 1) * d3;
    cnt[M_O] = n_opinions * d4;
    cnt[M_G1] = (int64_t)d1 * d2 * d3;
    cnt[M_G2] = (int64_t)d1 * d3 * d4;
    cnt[M_G3] = (int64_t)d2 * d3 * d4;
    int64_t t = 0;
    for (int m = 0; m < M_N; ++m) t += cnt[m];
    return t;
}

// The workspace: del (f32 per parameter) and `first` (int32 per row) lead and must be zero between calls; then the
// per-iteration sample buffers and the stored terms of the A[n_aspects] chain.
struct MterLayout {
    int64_t del, first, coef, ids, keys, owner, aterms, total, aterm_stride, rows;
};

static MterLayout mter_layout(int64_t n_users, int64_t n_items, int64_t n_aspects, int64_t n_opinions, int d1, int d2,
                              int d3, int d4, int n_el, int n_bpr)
{
    int64_t cnt[M_N];
    const int64_t params = mter_counts(n_users, n_items, n_aspects, n_opinions, d1, d2, d3, d4, cnt);
    const int64_t slots = 9ll * n_el + 4ll * n_bpr;
    auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
    MterLayout l{};
    l.rows = n_users + n_items + n_aspects + 1 + n_opinions;
    l.aterm_stride = ((int64_t)n_bpr * d1 * d2 + 3) / 4 * 4;
    l.del = 0;
    l.first = l.del + up(4 * params);
    l.coef = l.first + up(4 * l.rows);
    l.ids = l.coef + up(4 * (3ll * n_el + n_bpr));
    l.keys = l.ids + up(4 * slots);
    l.owner = l.keys + up(8 * slots);
    l.aterms = l.owner + up(slots);
    l.total = l.aterms + up(4 * l.aterm_stride * d3);
    return l;
}

extern "C" int64_t b200_mter_workspace_bytes(int64_t n_users, int64_t n_items, int64_t n_aspects, int64_t n_opinions,
                                             int d1, int d2, int d3, int d4, int n_el, int n_bpr)
{
    return mter_layout(n_users, n_items, n_aspects, n_opinions, d1, d2, d3, d4, n_el, n_bpr).total;
}

extern "C" int b200_mter_fit(int64_t n_users, int64_t n_items, int64_t n_aspects, int64_t n_opinions, int d1, int d2,
                             int d3, int d4, const float* X, const int32_t* X_u, const int32_t* X_i, const int32_t* X_a,
                             int64_t n_x, const float* YU, const int32_t* YU_u, const int32_t* YU_a,
                             const int32_t* YU_o, int64_t n_yu, const float* YI, const int32_t* YI_i,
                             const int32_t* YI_a, const int32_t* YI_o, int64_t n_yi, const int32_t* indptr,
                             const int32_t* indices, const int32_t* rrow, const float* rval, int64_t nnz, int n_el,
                             int n_bpr, int n_iter, const int32_t* draws, float* const* params, float* const* sgrad,
                             void* work, float lr, float lambda_reg, float lambda_bpr, int flags, uint64_t seed,
                             uint64_t iter0, unsigned long long* counts, double* losses, unsigned long long* phase_ns,
                             void* stream)
{
    B200_REQUIRE(n_users > 0 && n_items > 0 && n_aspects >= 0 && n_opinions > 0 && d1 > 0 && d2 > 0 && d3 > 0 &&
                     d4 > 0 && n_el > 0 && n_bpr > 0 && n_iter >= 0 && nnz > 0 && n_x > 0 && n_yu > 0 && n_yi > 0,
                 "b200_mter_fit: bad sizes (users %lld items %lld aspects %lld opinions %lld factors %d/%d/%d/%d "
                 "samples %d/%d iterations %d ratings %lld tensors %lld/%lld/%lld)",
                 (long long)n_users, (long long)n_items, (long long)n_aspects, (long long)n_opinions, d1, d2, d3, d4,
                 n_el, n_bpr, n_iter, (long long)nnz, (long long)n_x, (long long)n_yu, (long long)n_yi);
    B200_REQUIRE(n_aspects + 1 < (1ll << 31) && n_users < (1ll << 31) && n_items < (1ll << 31) &&
                     n_opinions < (1ll << 31) && nnz < (1ll << 31) && 9ll * n_el + 4ll * n_bpr < (1ll << 31),
                 "b200_mter_fit: sizes beyond int32 ids");
    B200_REQUIRE(X && X_u && X_i && X_a && YU && YU_u && YU_a && YU_o && YI && YI_i && YI_a && YI_o && indptr &&
                     indices && rrow && rval && params && sgrad && work && counts,
                 "b200_mter_fit: null pointer argument");
    B200_REQUIRE((flags & ~(B200_MTER_UNORDERED | B200_MTER_PHILOX)) == 0, "b200_mter_fit: unknown flags %d", flags);
    if (n_iter == 0) return B200_OK;
    B200_REQUIRE(draws || (flags & B200_MTER_PHILOX), "b200_mter_fit: null draws");
    MterArgs a{};
    a.n_users = n_users; a.n_items = n_items; a.n_aspects = n_aspects; a.n_opinions = n_opinions;
    a.d1 = d1; a.d2 = d2; a.d3 = d3; a.d4 = d4;
    a.X = X; a.X_u = X_u; a.X_i = X_i; a.X_a = X_a;
    a.YU = YU; a.YU_u = YU_u; a.YU_a = YU_a; a.YU_o = YU_o;
    a.YI = YI; a.YI_i = YI_i; a.YI_a = YI_a; a.YI_o = YI_o;
    a.indptr = indptr; a.indices = indices; a.rrow = rrow; a.rval = rval;
    a.n_el = n_el; a.n_bpr = n_bpr; a.n_iter = n_iter; a.draws = draws;
    mter_counts(n_users, n_items, n_aspects, n_opinions, d1, d2, d3, d4, a.cnt);
    for (int m = 0; m < M_N; ++m) {
        a.P[m] = params[m];
        a.S[m] = sgrad[m];
        B200_REQUIRE(a.P[m] && a.S[m], "b200_mter_fit: null parameter or AdaGrad state %d", m);
    }
    const MterLayout l = mter_layout(n_users, n_items, n_aspects, n_opinions, d1, d2, d3, d4, n_el, n_bpr);
    char* w = (char*)work;
    float* del = (float*)(w + l.del);
    for (int m = 0; m < M_N; ++m) {
        a.D[m] = del;
        del += a.cnt[m];
    }
    a.first = (int32_t*)(w + l.first);
    a.coef = (float*)(w + l.coef);
    a.ids = (int32_t*)(w + l.ids);
    a.keys = (int64_t*)(w + l.keys);
    a.owner = (uint8_t*)(w + l.owner);
    a.aterms = (float*)(w + l.aterms);
    a.aterm_stride = l.aterm_stride;
    a.row_off[0] = 0;
    a.row_off[1] = n_users;
    a.row_off[2] = n_users + n_items;
    a.row_off[3] = n_users + n_items + n_aspects + 1;
    a.unordered = (flags & B200_MTER_UNORDERED) != 0;
    a.philox = (flags & B200_MTER_PHILOX) != 0;
    a.key0 = (uint32_t)seed;
    a.key1 = (uint32_t)(seed >> 32);
    a.iter0 = iter0;
    a.n_x = n_x; a.n_yu = n_yu; a.n_yi = n_yi; a.nnz = nnz;
    a.phase_ns = phase_ns;
    a.lr = lr; a.ld_reg = lambda_reg; a.ld_bpr = lambda_bpr;
    a.counts = counts; a.losses = losses;

    int dev = 0;
    B200_CUDA(cudaGetDevice(&dev));
    int smem_max = 0;
    B200_CUDA(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    const int64_t core_bytes = 4 * (a.cnt[M_G1] + a.cnt[M_G2] + a.cnt[M_G3]);
    a.core_smem = core_bytes <= smem_max - 1024;
    const size_t smem = a.core_smem ? (size_t)core_bytes : 0;
    B200_CUDA(cudaFuncSetAttribute(mter_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mter_fit_kernel, MTER_THREADS, smem));
    B200_REQUIRE(per_sm > 0, "b200_mter_fit: the fit kernel does not fit on an SM");
    const int blocks = sm_count() * per_sm;
    void* kargs[] = {&a};
    count_launch();
    B200_CUDA(cudaLaunchCooperativeKernel((const void*)mter_fit_kernel, dim3(blocks), dim3(MTER_THREADS), kargs, smem,
                                          (cudaStream_t)stream));
    return B200_OK;
}

extern "C" int b200_mter_queries(const float* U, int64_t n_users, const float* G1, const float* a_last, int d1, int d2,
                                 int d3, float* Q, void* stream)
{
    B200_REQUIRE(n_users >= 0 && d1 > 0 && d2 > 0 && d3 > 0 && (int64_t)d1 * d2 * 4 <= 48 * 1024,
                 "b200_mter_queries: bad sizes n_users=%lld d=%d/%d/%d", (long long)n_users, d1, d2, d3);
    B200_REQUIRE(U && G1 && a_last && Q, "b200_mter_queries: null pointer argument");
    if (n_users == 0) return B200_OK;
    const int64_t n = n_users * d2;
    const int blocks = (int)std::min<int64_t>((n + MTER_THREADS - 1) / MTER_THREADS, 4ll * sm_count());
    count_launch();
    mter_queries_kernel<<<blocks, MTER_THREADS, (size_t)d1 * d2 * 4, (cudaStream_t)stream>>>(U, n_users, G1, a_last, d1,
                                                                                             d2, d3, Q);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
