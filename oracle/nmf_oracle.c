/* TEST INFRASTRUCTURE: a scalar C restatement of the reference NMF fit (cornac/models/nmf/recom_nmf.pyx:182-267), the
 * oracle the GPU fit is compared with where the compiled reference is not available.
 *
 * The reference extension is built with Python's default flags (no -fopenmp, no -ffast-math): the prange loops run
 * serially and every `floating` is a C float.  This file is compiled -O2 -ffp-contract=off so that no multiply-add is
 * fused either.  Each statement below is the reference's, in its order. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

/* n_epochs epochs over the ratings (rid, cid, val) in stored order.  U [n_users, k], V [n_items, k], Bu, Bi are updated
 * in place; Bu / Bi change only when use_bias, but always enter the prediction.  Returns 0, or -1 when out of memory. */
API int nmf_fit(const int32_t* rid, const int32_t* cid, const float* val, int64_t nnz, int64_t n_users, int64_t n_items,
                const int32_t* user_counts, const int32_t* item_counts, int k, float* U, float* V, float* Bu, float* Bi,
                int n_epochs, float mu, float lr, float lambda_u, float lambda_v, float lambda_bu, float lambda_bi,
                int use_bias)
{
    const float eps = 1e-9;
    float* Un = malloc(sizeof(float) * (size_t)(n_users * k + 1));
    float* Ud = malloc(sizeof(float) * (size_t)(n_users * k + 1));
    float* Vn = malloc(sizeof(float) * (size_t)(n_items * k + 1));
    float* Vd = malloc(sizeof(float) * (size_t)(n_items * k + 1));
    if (!Un || !Ud || !Vn || !Vd) {
        free(Un), free(Ud), free(Vn), free(Vd);
        return -1;
    }
    for (int epoch = 0; epoch < n_epochs; ++epoch) {
        memset(Un, 0, sizeof(float) * (size_t)(n_users * k));
        memset(Ud, 0, sizeof(float) * (size_t)(n_users * k));
        memset(Vn, 0, sizeof(float) * (size_t)(n_items * k));
        memset(Vd, 0, sizeof(float) * (size_t)(n_items * k));
        for (int64_t j = 0; j < nnz; ++j) {                          /* recom_nmf.pyx:227-248 */
            const int64_t u = rid[j], i = cid[j];
            const float r = val[j];
            float r_pred = mu + Bu[u] + Bi[i];
            for (int f = 0; f < k; ++f) r_pred = r_pred + U[u * k + f] * V[i * k + f];
            const float error = r - r_pred;
            if (use_bias) {
                Bu[u] += lr * (error - lambda_bu * Bu[u]);
                Bi[i] += lr * (error - lambda_bi * Bi[i]);
            }
            for (int f = 0; f < k; ++f) {
                Un[u * k + f] += r * V[i * k + f];
                Ud[u * k + f] += r_pred * V[i * k + f];
                Vn[i * k + f] += r * U[u * k + f];
                Vd[i * k + f] += r_pred * U[u * k + f];
            }
        }
        for (int64_t u = 0; u < n_users; ++u)                        /* :251-255 */
            for (int f = 0; f < k; ++f) {
                Ud[u * k + f] += user_counts[u] * lambda_u * U[u * k + f] + eps;
                U[u * k + f] *= Un[u * k + f] / Ud[u * k + f];
            }
        for (int64_t i = 0; i < n_items; ++i)                        /* :258-262 */
            for (int f = 0; f < k; ++f) {
                Vd[i * k + f] += item_counts[i] * lambda_v * V[i * k + f] + eps;
                V[i * k + f] *= Vn[i * k + f] / Vd[i * k + f];
            }
    }
    free(Un), free(Ud), free(Vn), free(Vd);
    return 0;
}
