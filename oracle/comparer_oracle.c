/* TEST INFRASTRUCTURE (not product code).
 *
 * Serial restatement of ComparERSub._fit_mter (cornac/models/comparer/recom_comparer_sub.pyx:487-760) in its float
 * specialisation with one thread (the reference forces one thread when a seed is given), statement for statement in
 * source order: oracle/mter_oracle.c's MTER loop plus the third phase over the comparative pairs.  The sample indices
 * are inputs: draw t of iteration it of each stream is stream[it * n + t], as the six RNGVector streams (uia, uao, iao,
 * pair, pos, neg) give them; a skipped BPR sample still has its two draws.
 *
 * Pair phase:  pred = score(u, later, a) - score(u, earlier, a);  z = (float)(1.0 / (1.0 + (double)expf(pred)));
 *   del_aspect_bpr = lambda_d * z;  for (i, j, k): a_ji = I[later, j] - I[earlier, j];
 *   del_g1 -= d * U * a_ji * A[a];  del_u -= d * G1 * a_ji * A[a];  del_i[later] -= d * G1 * U * A[a];
 *   del_i[earlier] += d * G1 * U * A[a];  del_a[a] -= d * G1 * U * a_ji.
 *
 * Arithmetic as the generated C++ (recom_mter.cpp) spells it, no FMA (-ffp-contract=off):
 *   products left to right in f32 (((c * a) * b) * d); the prediction a serial f32 chain in (i, j, k) order;
 *   del_sqerror = (float)(2.0 * (pred - score));   z = (float)(1.0 / (1.0 + (double)expf(pred)));
 *   del_bpr = (ld_bpr * z) * (float)s;   bpr term = log(1.0 / (1.0 + (double)expf(-pred))) added to the f32 sum in f64;
 *   AdaGrad: reg = del + ld_reg * x where del != 0 (else 0: the reference resets del_*_reg every call),
 *            sgrad += eps + reg * reg,   x = (float)((double)x - ((double)lr / (double)sqrtf(sgrad)) * (double)reg),
 *            x = 0 if x < 0.
 * Shapes: U[n_users, d1], I[n_items, d2], A[n_aspects + 1, d3], O[n_opinions, d4], G1[d1, d2, d3], G2[d1, d3, d4],
 * G3[d2, d3, d4], row-major f32.  The BPR data: the CSR (indptr, indices) of the ratings with sorted columns, `rrow` the
 * row of each CSR entry, and `rval` the f32 rating of the exact (user, item) pair (the last value a repeated pair has).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define EXPORT __attribute__((visibility("default")))

static float score3(const float* G, int64_t d1, int64_t d2, int64_t d3, const float* a, const float* b, const float* c)
{
    float s = 0.f;
    for (int64_t i = 0; i < d1; ++i)
        for (int64_t j = 0; j < d2; ++j)
            for (int64_t k = 0; k < d3; ++k) s = s + G[(i * d2 + j) * d3 + k] * a[i] * b[j] * c[k];
    return s;
}

/* position of column c in CSR row r, or -1 (binary search over sorted columns, as std::binary_search) */
static int64_t find(const int32_t* indptr, const int32_t* indices, int32_t r, int32_t c)
{
    int64_t lo = indptr[r], hi = indptr[r + 1];
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo) / 2;
        if (indices[mid] < c) lo = mid + 1;
        else hi = mid;
    }
    return (lo < indptr[r + 1] && indices[lo] == c) ? lo : -1;
}

static void adagrad(float* x, float* sg, const float* del, int64_t n, float lr, float ld_reg)
{
    const float eps = 1e-9f;
    for (int64_t t = 0; t < n; ++t) {
        float reg = 0.f;
        if (del[t] != 0.0f) reg = del[t] + ld_reg * x[t];
        sg[t] += eps + reg * reg;
        x[t] = (float)((double)x[t] - ((double)lr / (double)sqrtf(sg[t])) * (double)reg);
        if (x[t] < 0) x[t] = 0;
    }
}

EXPORT int comparer_sub_fit(int64_t n_users, int64_t n_items, int64_t n_aspects, int64_t n_opinions, int64_t d1, int64_t d2,
                    int64_t d3, int64_t d4,
                    const float* X, const int32_t* X_u, const int32_t* X_i, const int32_t* X_a,
                    const float* YU, const int32_t* YU_u, const int32_t* YU_a, const int32_t* YU_o,
                    const float* YI, const int32_t* YI_i, const int32_t* YI_a, const int32_t* YI_o,
                    const int32_t* indptr, const int32_t* indices, const int32_t* rrow, const float* rval,
                    const int32_t* p_u, const int32_t* p_e, const int32_t* p_l, const int32_t* p_a,
                    int64_t n_el, int64_t n_bpr, int64_t n_pair, int64_t n_iter,
                    const int64_t* d_uia, const int64_t* d_uao, const int64_t* d_iao, const int64_t* d_pair,
                    const int64_t* d_pos, const int64_t* d_neg,
                    float* U, float* I, float* A, float* O, float* G1, float* G2, float* G3,
                    float* sU, float* sI, float* sA, float* sO, float* sG1, float* sG2, float* sG3,
                    float lr, float ld_reg, float ld_bpr, float ld_d,
                    int64_t* correct_out, int64_t* skipped_out, float* loss_out, float* bpr_loss_out,
                    int64_t* aspect_correct_out)
{
    const int64_t nU = n_users * d1, nI = n_items * d2, nA = (n_aspects + 1) * d3, nO = n_opinions * d4;
    const int64_t nG1 = d1 * d2 * d3, nG2 = d1 * d3 * d4, nG3 = d2 * d3 * d4;
    float* buf = (float*)calloc((size_t)(nU + nI + nA + nO + nG1 + nG2 + nG3), sizeof(float));
    if (!buf) return 1;
    float *du = buf, *di = du + nU, *da = di + nI, *dO = da + nA, *dg1 = dO + nO, *dg2 = dg1 + nG1, *dg3 = dg2 + nG2;
    const float* An = A + n_aspects * d3;
    for (int64_t it = 0; it < n_iter; ++it) {
        memset(buf, 0, sizeof(float) * (size_t)(nU + nI + nA + nO + nG1 + nG2 + nG3));
        int64_t correct = 0, skipped = 0, aspect_correct = 0;
        float loss = 0.f, bpr_loss = 0.f;
        for (int64_t t = 0; t < n_el; ++t) {
            int64_t idx = d_uia[it * n_el + t];
            {
                const int64_t u = X_u[idx], i = X_i[idx], a = X_a[idx];
                const float* Ur = U + u * d1; const float* Ir = I + i * d2; const float* Ar = A + a * d3;
                const float score = X[idx];
                const float pred = score3(G1, d1, d2, d3, Ur, Ir, Ar);
                loss = loss + (pred - score) * (pred - score);
                const float ds = (float)(2.0 * (double)(pred - score));
                for (int64_t p = 0; p < d1; ++p)
                    for (int64_t q = 0; q < d2; ++q)
                        for (int64_t r = 0; r < d3; ++r) {
                            const float g = G1[(p * d2 + q) * d3 + r];
                            dg1[(p * d2 + q) * d3 + r] += ds * Ur[p] * Ir[q] * Ar[r];
                            du[u * d1 + p] += ds * g * Ir[q] * Ar[r];
                            di[i * d2 + q] += ds * g * Ur[p] * Ar[r];
                            da[a * d3 + r] += ds * g * Ur[p] * Ir[q];
                        }
            }
            idx = d_uao[it * n_el + t];
            {
                const int64_t u = YU_u[idx], a = YU_a[idx], o = YU_o[idx];
                const float* Ur = U + u * d1; const float* Ar = A + a * d3; const float* Or = O + o * d4;
                const float score = YU[idx];
                const float pred = score3(G2, d1, d3, d4, Ur, Ar, Or);
                loss = loss + (pred - score) * (pred - score);
                const float ds = (float)(2.0 * (double)(pred - score));
                for (int64_t p = 0; p < d1; ++p)
                    for (int64_t q = 0; q < d3; ++q)
                        for (int64_t r = 0; r < d4; ++r) {
                            const float g = G2[(p * d3 + q) * d4 + r];
                            dg2[(p * d3 + q) * d4 + r] += ds * Ur[p] * Ar[q] * Or[r];
                            du[u * d1 + p] += ds * g * Ar[q] * Or[r];
                            da[a * d3 + q] += ds * g * Ur[p] * Or[r];
                            dO[o * d4 + r] += ds * g * Ur[p] * Ar[q];
                        }
            }
            idx = d_iao[it * n_el + t];
            {
                const int64_t i = YI_i[idx], a = YI_a[idx], o = YI_o[idx];
                const float* Ir = I + i * d2; const float* Ar = A + a * d3; const float* Or = O + o * d4;
                const float score = YI[idx];
                const float pred = score3(G3, d2, d3, d4, Ir, Ar, Or);
                loss = loss + (pred - score) * (pred - score);
                const float ds = (float)(2.0 * (double)(pred - score));
                for (int64_t p = 0; p < d2; ++p)
                    for (int64_t q = 0; q < d3; ++q)
                        for (int64_t r = 0; r < d4; ++r) {
                            const float g = G3[(p * d3 + q) * d4 + r];
                            dg3[(p * d3 + q) * d4 + r] += ds * Ir[p] * Ar[q] * Or[r];
                            di[i * d2 + p] += ds * g * Ar[q] * Or[r];
                            da[a * d3 + q] += ds * g * Ir[p] * Or[r];
                            dO[o * d4 + r] += ds * g * Ir[p] * Ar[q];
                        }
            }
        }
        for (int64_t t = 0; t < n_bpr; ++t) {
            const int64_t idx = d_pos[it * n_bpr + t];
            const int32_t u = rrow[idx], i = indices[idx];
            const int32_t j = (int32_t)d_neg[it * n_bpr + t];
            float s = 1.f;
            const int64_t jp = find(indptr, indices, u, j);
            if (jp >= 0) {
                const float is = rval[idx], js = rval[jp];
                if (is == js) { ++skipped; continue; }
                if (is < js) s = -1.f;
            }
            const float* Ur = U + (int64_t)u * d1; const float* Ii = I + (int64_t)i * d2; const float* Ij = I + (int64_t)j * d2;
            const float pred = (score3(G1, d1, d2, d3, Ur, Ii, An) - score3(G1, d1, d2, d3, Ur, Ij, An)) * s;
            const float z = (float)(1.0 / (1.0 + (double)expf(pred)));
            if (z < .5) ++correct;
            const float db = (ld_bpr * z) * s;
            bpr_loss = (float)((double)bpr_loss + log(1.0 / (1.0 + (double)expf(-pred))));
            for (int64_t p = 0; p < d1; ++p)
                for (int64_t q = 0; q < d2; ++q) {
                    const float iij = Ii[q] - Ij[q];
                    for (int64_t r = 0; r < d3; ++r) {
                        const float g = G1[(p * d2 + q) * d3 + r];
                        dg1[(p * d2 + q) * d3 + r] -= db * Ur[p] * iij * An[r];
                        du[(int64_t)u * d1 + p] -= db * g * iij * An[r];
                        di[(int64_t)i * d2 + q] -= db * g * Ur[p] * An[r];
                        di[(int64_t)j * d2 + q] += db * g * Ur[p] * An[r];
                        da[n_aspects * d3 + r] -= db * g * Ur[p] * iij;
                    }
                }
        }
        for (int64_t t = 0; t < n_pair; ++t) {
            const int64_t idx = d_pair[it * n_pair + t];
            const int64_t u = p_u[idx], e = p_e[idx], l = p_l[idx], a = p_a[idx];
            const float* Ur = U + u * d1; const float* Ie = I + e * d2; const float* Il = I + l * d2;
            const float* Ar = A + a * d3;
            const float pred = score3(G1, d1, d2, d3, Ur, Il, Ar) - score3(G1, d1, d2, d3, Ur, Ie, Ar);
            const float z = (float)(1.0 / (1.0 + (double)expf(pred)));
            if (z < .5) ++aspect_correct;
            const float dp = ld_d * z;
            for (int64_t p = 0; p < d1; ++p)
                for (int64_t q = 0; q < d2; ++q) {
                    const float aji = Il[q] - Ie[q];
                    for (int64_t r = 0; r < d3; ++r) {
                        const float g = G1[(p * d2 + q) * d3 + r];
                        dg1[(p * d2 + q) * d3 + r] -= dp * Ur[p] * aji * Ar[r];
                        du[u * d1 + p] -= dp * g * aji * Ar[r];
                        di[l * d2 + q] -= dp * g * Ur[p] * Ar[r];
                        di[e * d2 + q] += dp * g * Ur[p] * Ar[r];
                        da[a * d3 + r] -= dp * g * Ur[p] * aji;
                    }
                }
        }
        adagrad(U, sU, du, nU, lr, ld_reg);
        adagrad(G1, sG1, dg1, nG1, lr, ld_reg);
        adagrad(G2, sG2, dg2, nG2, lr, ld_reg);
        adagrad(I, sI, di, nI, lr, ld_reg);
        adagrad(G3, sG3, dg3, nG3, lr, ld_reg);
        adagrad(A, sA, da, nA, lr, ld_reg);
        adagrad(O, sO, dO, nO, lr, ld_reg);
        correct_out[it] = correct;
        skipped_out[it] = skipped;
        loss_out[it] = loss;
        bpr_loss_out[it] = bpr_loss;
        aspect_correct_out[it] = aspect_correct;
    }
    free(buf);
    return 0;
}
