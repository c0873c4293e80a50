/* TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A serial restatement of LRPPM._fit (cornac/models/lrppm/recom_lrppm.pyx:356-482) and of the convergence test of
 * LRPPM.fit (:316-346), given the three streams' draws.  It restates the float specialisation AS COMPILED
 * (gcc -O3 -ffast-math, x86-64 SSE2, no FMA), not the source's arithmetic.  From the disassembly of the reference's
 * recom_lrppm extension (the int / float instance of `_fit`):
 *   (1) the rating dot r_pred = sum_k U[u, k] I[i, k] is a serial mulss / addss chain from 0 in k order, in both loops;
 *   (2) get_score is vectorised over pairs of k (unpcklps loads, addps / mulps over 2 lanes): lane k % 2 adds
 *       (UA[a, k] + I[i, k]) * U[u, k] + IA[a, k] * I[i, k]; then shufps $0xe5 and addss add the lanes; with k odd a
 *       scalar tail adds (s + IA I) + (UA + I) U.  For k <= 3 (cmpl $0x2 on k - 1) only the scalar code runs, whose
 *       three statements group as (s + IA I) + (UA + I) U, (s + (UA + I) U) + IA I and s + ((UA + I) U + IA I);
 *   (3) exp(pred) is a call to expf; z = (float)(1.0 / (1.0 + (double)expf(pred))) (addsd, divsd, cvtsd2ss); the
 *       only exp / log kept in double are the loss's;
 *   (4) del_rating = (float)(2.0 * (double)l_ui * (double)(score - r_pred)): one rounding, which equals the f32
 *       product (2 l_ui) (score - r_pred);
 *   (5) the clamp `if x < 0: x = 0` is maxss(x, 0) with 0 as the source operand: NaN and -0.0 become +0.0;
 *   (6) `if del != 0` is comiss + jne for U, I and IA, whose fall-through only clamps, so a NaN del only clamps; for UA
 *       it is comiss + je around the reg term alone, so a NaN del still subtracts lr * del (and the clamp gives 0);
 *   (7) get_key (recom_mter.pyx:42-43) is lea / imul in 32 bits, then a floor halving: C int with two's-complement
 *       wrap.
 * The dict lookups are binary searches in sorted key arrays (akeys: the skip set; rkeys / rvals: the rating dict with
 * the value it keeps; an absent rating key reads 0, as operator[] inserts 0).
 * glibc's expf is called here through libm, as the reference calls it. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define EXPORT __attribute__((visibility("default")))

static int32_t lr_key(int32_t i, int32_t j)
{
    const uint32_t s = (uint32_t)i + (uint32_t)j;
    const int32_t p = (int32_t)(s * (s + 1u));
    return (int32_t)((uint32_t)(p >> 1) + (uint32_t)j);
}

EXPORT void lrppm_keys(int64_t n, const int32_t* a, const int32_t* b, int32_t* out)
{
    for (int64_t t = 0; t < n; ++t) out[t] = lr_key(a[t], b[t]);
}

static int64_t find(const int32_t* keys, int64_t n, int32_t key)
{
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo) / 2;
        if (keys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return (lo < n && keys[lo] == key) ? lo : -1;
}

static float dot_serial(const float* x, const float* y, int k)
{
    float s = 0.f;
    for (int f = 0; f < k; ++f) s = s + x[f] * y[f];
    return s;
}

static float score_k(const float* U, const float* I, const float* UA, const float* IA, int k)
{
#define T(f) ((UA[f] + I[f]) * U[f])
#define W(f) (IA[f] * I[f])
    float s = 0.f;
    if (k > 3) {
        float l0 = 0.f, l1 = 0.f;
        int f = 0;
        for (; f + 1 < k; f += 2) {
            l0 = l0 + (T(f) + W(f));
            l1 = l1 + (T(f + 1) + W(f + 1));
        }
        s = l1 + l0;
        if (f < k) s = (s + W(f)) + T(f);
        return s;
    }
    if (k > 0) s = (s + W(0)) + T(0);
    if (k > 1) s = (s + T(1)) + W(1);
    if (k > 2) s = s + (T(2) + W(2));
    return s;
#undef T
#undef W
}

static float clamp0(float x) { return x > 0.f ? x : 0.f; }

/* numpy 2 isclose(x, y) of f32 arrays */
static int isclose_f32(float x, float y)
{
    const float tol = 1e-8f + 1e-5f * fabsf(y);
    return (fabsf(x - y) <= tol && isfinite(y)) || x == y;
}

EXPORT void lrppm_isclose(int64_t n, const float* x, const float* y, uint8_t* out)
{
    for (int64_t t = 0; t < n; ++t) out[t] = (uint8_t)isclose_f32(x[t], y[t]);
}

/* Up to n_iter iterations; returns the number run (it stops after the first one that changed nothing: *converged = 1).
 * Per iteration: correct, skipped (int64) and loss, ranking_loss, r_loss (the reference's f32 sums). */
EXPORT int64_t lrppm_fit(int64_t n_users, int64_t n_items, int64_t n_aspects, int k, const int32_t* r_u,
                         const int32_t* r_i, const float* r_val, const int32_t* x_u, const int32_t* x_i,
                         const int32_t* x_a, const float* x_l, const int32_t* akeys, int64_t n_akeys,
                         const int32_t* rkeys, const float* rvals, int64_t n_rkeys, int n_s, int n_rank, int n_iter,
                         const int64_t* pos, const int64_t* pos_uia, const int64_t* neg_uia, float* U, float* I,
                         float* UA, float* IA, float lr, float reg, float ld, int64_t* correct, int64_t* skipped,
                         float* loss, float* ranking_loss, float* r_loss, int* converged)
{
    float* del[4];
    float* x[4] = {U, I, UA, IA};
    const int64_t rows[4] = {n_users, n_items, n_aspects, n_aspects};
    int64_t total = 0;
    for (int m = 0; m < 4; ++m) total += rows[m] * k;
    float* buf = (float*)calloc((size_t)total * 2, sizeof(float));
    if (!buf) return -1;
    float* prev = buf + total;
    int64_t off = 0;
    for (int m = 0; m < 4; ++m) {
        del[m] = buf + off;
        off += rows[m] * k;
    }
    *converged = 0;
    int64_t it = 0;
    for (; it < n_iter; ++it) {
        off = 0;
        for (int m = 0; m < 4; ++m) {
            memcpy(prev + off, x[m], sizeof(float) * rows[m] * k);
            off += rows[m] * k;
        }
        memset(buf, 0, sizeof(float) * total);
        int64_t c = 0, sk = 0;
        float lo = 0.f, rl = 0.f, rr = 0.f;
        for (int t = 0; t < n_s; ++t) {
            const int64_t idx = pos[it * n_s + t];
            const int32_t u = r_u[idx], i = r_i[idx];
            const float score = r_val[idx];
            const float rp = dot_serial(U + (int64_t)u * k, I + (int64_t)i * k, k);
            const float dsq = 2.f * (rp - score);
            lo += (score - rp) * (score - rp);
            for (int f = 0; f < k; ++f) {
                del[0][(int64_t)u * k + f] += dsq * I[(int64_t)i * k + f];
                del[1][(int64_t)i * k + f] += dsq * U[(int64_t)u * k + f];
            }
        }
        for (int t = 0; t < n_rank; ++t) {
            const int64_t idx = pos_uia[it * n_rank + t];
            const int32_t u = x_u[idx], i = x_i[idx], a = x_a[idx];
            const int32_t aj = (int32_t)neg_uia[it * n_rank + t];
            if (find(akeys, n_akeys, lr_key(lr_key(u, i), aj)) >= 0) {
                ++sk;
                continue;
            }
            const float *Uu = U + (int64_t)u * k, *Ii = I + (int64_t)i * k;
            const float pred = score_k(Uu, Ii, UA + (int64_t)a * k, IA + (int64_t)a * k, k) -
                               score_k(Uu, Ii, UA + (int64_t)aj * k, IA + (int64_t)aj * k, k);
            const float z = (float)(1.0 / (1.0 + (double)expf(pred)));
            if (z < 0.5f) ++c;
            const float dr = ld * z;
            rl = (float)((double)rl + (double)ld * log(1.0 / (1.0 + (double)expf(-pred))));
            for (int f = 0; f < k; ++f) {
                del[0][(int64_t)u * k + f] -= dr * (UA[(int64_t)a * k + f] - UA[(int64_t)aj * k + f]);
                del[1][(int64_t)i * k + f] -= dr * (IA[(int64_t)a * k + f] - IA[(int64_t)aj * k + f]);
                del[2][(int64_t)a * k + f] -= dr * Uu[f];
                del[2][(int64_t)aj * k + f] += dr * Uu[f];
                del[3][(int64_t)a * k + f] -= dr * Ii[f];
                del[3][(int64_t)aj * k + f] += dr * Ii[f];
            }
            const float rp = dot_serial(Uu, Ii, k);
            const int64_t kp = find(rkeys, n_rkeys, lr_key(u, i));
            const float score = kp >= 0 ? rvals[kp] : 0.f;
            const float l = x_l[idx];
            const float diff = score - rp;
            const float dt = (float)(2.0 * (double)l * (double)diff);
            rr += l * diff * diff;
            for (int f = 0; f < k; ++f) {
                del[0][(int64_t)u * k + f] += dt * Ii[f];
                del[1][(int64_t)i * k + f] += dt * Uu[f];
            }
        }
        for (int m = 0; m < 4; ++m)
            for (int64_t e = 0; e < rows[m] * k; ++e) {
                float d = del[m][e];
                if (d != 0.f && !isnan(d)) {
                    d += reg * x[m][e];
                    x[m][e] = clamp0(x[m][e] - lr * d);
                } else if (m == 2) {
                    x[m][e] = clamp0(x[m][e] - lr * d);
                } else {
                    x[m][e] = clamp0(x[m][e]);
                }
            }
        correct[it] = c;
        skipped[it] = sk;
        loss[it] = lo;
        ranking_loss[it] = rl;
        r_loss[it] = rr;
        int same = 1;
        off = 0;
        for (int m = 0; m < 4 && same; ++m) {
            for (int64_t e = 0; e < rows[m] * k; ++e)
                if (!isclose_f32(x[m][e], prev[off + e])) {
                    same = 0;
                    break;
                }
            off += rows[m] * k;
        }
        if (same) {
            *converged = 1;
            ++it;
            break;
        }
    }
    free(buf);
    return it;
}
