/* TEST INFRASTRUCTURE: a scalar C restatement of the reference EFM fit (cornac/models/efm/recom_efm.pyx:268-353) and of
 * the query vectors of the device rank (b200_efm_queries), the oracle the GPU is compared with.
 *
 * The reference extension is built with no extra flags (setup.py:205-210): no -fopenmp, so the prange loops run serially,
 * and every `floating` is a C float.  Its sqrt of a float expression is the float overload (the module is C++).  This file
 * is compiled -O2 -ffp-contract=off so that no multiply-add is fused either.  Each statement below is the reference's, in
 * its order, except the BLAS sdot, whose order is unspecified: dot() DEFINES it as the f64 sum in index order of the
 * exact f32 products, rounded once to f32 (as ora_fast_dot does). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

static float dot(const float* a, const float* b, int n)
{
    double acc = 0.0;
    for (int f = 0; f < n; ++f) acc += (double)a[f] * (double)b[f];
    return (float)acc;
}

/* n_iter iterations over A (a_uid, a_iid, a_val; nA entries in CSR order), X (x_uid, x_aid, x_val) and Y (y_iid, y_aid,
 * y_val).  U1 [n_users, E], U2 [n_items, E], V [n_aspects, E], H1 [n_users, L], H2 [n_items, L] are updated in place.
 * Returns 0, or -1 when out of memory. */
API int efm_fit(int64_t nA, const int32_t* a_uid, const int32_t* a_iid, const float* a_val, const int32_t* a_user_counts,
                const int32_t* a_item_counts, int64_t nX, const int32_t* x_uid, const int32_t* x_aid, const float* x_val,
                const int32_t* x_user_counts, const int32_t* x_aspect_counts, int64_t nY, const int32_t* y_iid,
                const int32_t* y_aid, const float* y_val, const int32_t* y_item_counts, const int32_t* y_aspect_counts,
                int64_t n_users, int64_t n_items, int64_t n_aspects, int E, int L, float* U1, float* U2, float* V,
                float* H1, float* H2, int n_iter, float lambda_x, float lambda_y, float lambda_u, float lambda_h,
                float lambda_v)
{
    const float eps = 1e-9;
    const size_t s1 = (size_t)n_users * E + 1, s2 = (size_t)n_items * E + 1, sv = (size_t)n_aspects * E + 1;
    const size_t h1 = (size_t)n_users * L + 1, h2 = (size_t)n_items * L + 1;
    float* U1n = malloc(sizeof(float) * s1);
    float* U1d = malloc(sizeof(float) * s1);
    float* U2n = malloc(sizeof(float) * s2);
    float* U2d = malloc(sizeof(float) * s2);
    float* Vn = malloc(sizeof(float) * sv);
    float* Vd = malloc(sizeof(float) * sv);
    float* H1n = malloc(sizeof(float) * h1);
    float* H1d = malloc(sizeof(float) * h1);
    float* H2n = malloc(sizeof(float) * h2);
    float* H2d = malloc(sizeof(float) * h2);
    int rc = 0;
    if (!U1n || !U1d || !U2n || !U2d || !Vn || !Vd || !H1n || !H1d || !H2n || !H2d) {
        rc = -1;
        goto done;
    }
    for (int t = 0; t < n_iter; ++t) {
        memset(U1n, 0, sizeof(float) * s1), memset(U1d, 0, sizeof(float) * s1);
        memset(U2n, 0, sizeof(float) * s2), memset(U2d, 0, sizeof(float) * s2);
        memset(Vn, 0, sizeof(float) * sv), memset(Vd, 0, sizeof(float) * sv);
        memset(H1n, 0, sizeof(float) * h1), memset(H1d, 0, sizeof(float) * h1);
        memset(H2n, 0, sizeof(float) * h2), memset(H2d, 0, sizeof(float) * h2);
        for (int64_t idx = 0; idx < nA; ++idx) {                        /* recom_efm.pyx:283-300 */
            const int64_t i = a_uid[idx], j = a_iid[idx];
            const float prediction = dot(U1 + i * E, U2 + j * E, E) + dot(H1 + i * L, H2 + j * L, L);
            const float score = a_val[idx];
            for (int k = 0; k < E; ++k) {
                U1n[i * E + k] += score * U2[j * E + k];
                U1d[i * E + k] += prediction * U2[j * E + k];
                U2n[j * E + k] += score * U1[i * E + k];
                U2d[j * E + k] += prediction * U1[i * E + k];
            }
            for (int k = 0; k < L; ++k) {
                H1n[i * L + k] += score * H2[j * L + k];
                H1d[i * L + k] += prediction * H2[j * L + k];
                H2n[j * L + k] += score * H1[i * L + k];
                H2d[j * L + k] += prediction * H1[i * L + k];
            }
        }
        for (int64_t idx = 0; idx < nX; ++idx) {                        /* :302-312 */
            const int64_t i = x_uid[idx], j = x_aid[idx];
            const float prediction = dot(U1 + i * E, V + j * E, E);
            const float score = x_val[idx];
            for (int k = 0; k < E; ++k) {
                Vn[j * E + k] += lambda_x * score * U1[i * E + k];
                Vd[j * E + k] += lambda_x * prediction * U1[i * E + k];
                U1n[i * E + k] += lambda_x * score * V[j * E + k];
                U1d[i * E + k] += lambda_x * prediction * V[j * E + k];
            }
        }
        for (int64_t idx = 0; idx < nY; ++idx) {                        /* :314-324 */
            const int64_t i = y_iid[idx], j = y_aid[idx];
            const float prediction = dot(U2 + i * E, V + j * E, E);
            const float score = y_val[idx];
            for (int k = 0; k < E; ++k) {
                Vn[j * E + k] += lambda_y * score * U2[i * E + k];
                Vd[j * E + k] += lambda_y * prediction * U2[i * E + k];
                U2n[i * E + k] += lambda_y * score * V[j * E + k];
                U2d[i * E + k] += lambda_y * prediction * V[j * E + k];
            }
        }
        for (int64_t i = 0; i < n_aspects; ++i)                         /* :326-331 */
            for (int j = 0; j < E; ++j) {
                Vd[i * E + j] += (x_aspect_counts[i] + y_aspect_counts[i]) * lambda_v * V[i * E + j] + eps;
                V[i * E + j] *= sqrtf(Vn[i * E + j] / Vd[i * E + j]);
            }
        for (int64_t i = 0; i < n_users; ++i) {                         /* :333-342 */
            for (int j = 0; j < E; ++j) {
                U1d[i * E + j] += (a_user_counts[i] + x_user_counts[i]) * lambda_u * U1[i * E + j] + eps;
                U1[i * E + j] *= sqrtf(U1n[i * E + j] / U1d[i * E + j]);
            }
            for (int j = 0; j < L; ++j) {
                H1d[i * L + j] += a_user_counts[i] * lambda_h * H1[i * L + j] + eps;
                H1[i * L + j] *= sqrtf(H1n[i * L + j] / H1d[i * L + j]);
            }
        }
        for (int64_t i = 0; i < n_items; ++i) {                         /* :344-353 */
            for (int j = 0; j < E; ++j) {
                U2d[i * E + j] += (a_item_counts[i] + y_item_counts[i]) * lambda_u * U2[i * E + j] + eps;
                U2[i * E + j] *= sqrtf(U2n[i * E + j] / U2d[i * E + j]);
            }
            for (int j = 0; j < L; ++j) {
                H2d[i * L + j] += a_item_counts[i] * lambda_h * H2[i * L + j] + eps;
                H2[i * L + j] *= sqrtf(H2n[i * L + j] / H2d[i * L + j]);
            }
        }
    }
done:
    free(U1n), free(U1d), free(U2n), free(U2d), free(Vn), free(Vd), free(H1n), free(H1d), free(H2n), free(H2d);
    return rc;
}

/* b200_efm_queries: for each user users[q], X_[a] = dot(U1[u], V[a]); the m = min(N, n_aspects) aspects of largest X_
 * (ties: smaller id first), chosen one at a time; Q[q, f] = f32(c * sum_t X_[a_t] V[a_t, f] + beta U1[u, f]) (f < E),
 * Q[q, E + f] = f32(beta H1[u, f]), with c = alpha / (N * rating_scale) and beta = 1 - alpha in f64.  Returns 0, or -1
 * when out of memory. */
API int efm_queries(const int64_t* users, int64_t n_q, const float* U1, const float* H1, const float* V,
                    int64_t n_aspects, int E, int L, int N, double alpha, double rating_scale, float* Q)
{
    const int64_t m = N < n_aspects ? N : n_aspects;
    float* xs = malloc(sizeof(float) * (size_t)(n_aspects + 1));
    int64_t* top = malloc(sizeof(int64_t) * (size_t)(m + 1));
    char* taken = malloc((size_t)(n_aspects + 1));
    if (!xs || !top || !taken) {
        free(xs), free(top), free(taken);
        return -1;
    }
    const double c = alpha / ((double)N * rating_scale);
    const double beta = 1.0 - alpha;
    for (int64_t q = 0; q < n_q; ++q) {
        const int64_t u = users[q];
        for (int64_t a = 0; a < n_aspects; ++a) xs[a] = dot(U1 + u * E, V + a * E, E), taken[a] = 0;
        for (int64_t t = 0; t < m; ++t) {
            int64_t best = -1;
            for (int64_t a = 0; a < n_aspects; ++a)
                if (!taken[a] && (best < 0 || xs[a] > xs[best])) best = a;
            top[t] = best;
            taken[best] = 1;
        }
        float* out = Q + q * (E + L);
        for (int f = 0; f < E; ++f) {
            double s = 0.0;
            for (int64_t t = 0; t < m; ++t) s = s + (double)xs[top[t]] * (double)V[top[t] * E + f];
            out[f] = (float)(c * s + beta * (double)U1[u * E + f]);
        }
        for (int f = 0; f < L; ++f) out[E + f] = (float)(beta * (double)H1[u * L + f]);
    }
    free(xs), free(top), free(taken);
    return 0;
}
