/* TEST INFRASTRUCTURE: a scalar C restatement of the reference PMF epoch (cornac/models/pmf/cython/pmf.pyx), the
 * oracle the GPU fit is compared with where the compiled reference is not available.
 *
 * The reference extension is built with Python's default flags (no -ffast-math): plain IEEE f64, the dots summed
 * serially in index order.  This file is compiled -O2 -ffp-contract=off so that no multiply-add is fused either.
 * lambda_reg, learning_rate and gamma are C floats used in f64 expressions, as in the reference's signature.
 * The sigmoid calls libm's expf: C++ resolves the reference's exp(float) to the float overload. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define API __attribute__((visibility("default")))

/* pmf.pyx:27-37 */
static float sigmoid(float z)
{
    const float MAX_EXP = 6.0f;
    if (z > MAX_EXP) return 1.0f;
    if (z < -MAX_EXP) return 0.0f;
    return (float)(1.0 / (1.0 + (double)expf(-z)));
}

/* The element loops of one rating (pmf.pyx:86-104 / 148-166) given the weighted error we and the error e.
 * Returns the rating's loss term. */
static double apply_rating(double* Uu, double* Vi, double* cu, double* cv, int k, double e, double we, float lambda_reg,
                           float learning_rate, float gamma)
{
    const double eps = 1e-8;
    double g, norm_u = 0.0, norm_v = 0.0;
    for (int f = 0; f < k; ++f) {                                   /* pmf.pyx:87-90 */
        g = we * Vi[f] - lambda_reg * Uu[f];
        cu[f] = gamma * cu[f] + (1.0 - gamma) * (g * g);
        Uu[f] += learning_rate * (g / (sqrt(cu[f]) + eps));
    }
    for (int f = 0; f < k; ++f) {                                   /* pmf.pyx:93-96: reads the updated U */
        g = we * Uu[f] - lambda_reg * Vi[f];
        cv[f] = gamma * cv[f] + (1.0 - gamma) * (g * g);
        Vi[f] += learning_rate * (g / (sqrt(cv[f]) + eps));
    }
    for (int f = 0; f < k; ++f) {                                   /* pmf.pyx:98-102 */
        norm_u += Uu[f] * Uu[f];
        norm_v += Vi[f] * Vi[f];
    }
    return e * e + lambda_reg * (norm_u + norm_v);                  /* pmf.pyx:104 */
}

/* One epoch of pmf_linear (pmf.pyx:79-104) over the ratings in stored order.  terms (nullable, [nnz]) receives each
 * rating's loss term; the return value is the epoch's loss, summed as the reference sums it. */
API double pmf_linear_epoch(const int32_t* uid, const int32_t* iid, const float* rat, int64_t nnz, int k, double* U,
                            double* V, double* cache_u, double* cache_v, float lambda_reg, float learning_rate,
                            float gamma, double* terms)
{
    double loss = 0.0;
    for (int64_t r = 0; r < nnz; ++r) {
        const int64_t u = uid[r], i = iid[r];
        const double val = rat[r];
        double* Uu = U + u * k;
        double* Vi = V + i * k;
        double s = 0.0;
        for (int f = 0; f < k; ++f) s += Uu[f] * Vi[f];             /* pmf.pyx:81-83 */
        const double e = val - s;
        const double t = apply_rating(Uu, Vi, cache_u + u * k, cache_v + i * k, k, e, e, lambda_reg, learning_rate, gamma);
        if (terms) terms[r] = t;
        loss += t;
    }
    return loss;
}

/* One epoch of pmf_non_linear (pmf.pyx:138-166). */
API double pmf_nonlinear_epoch(const int32_t* uid, const int32_t* iid, const float* rat, int64_t nnz, int k, double* U,
                               double* V, double* cache_u, double* cache_v, float lambda_reg, float learning_rate,
                               float gamma, double* terms)
{
    double loss = 0.0;
    for (int64_t r = 0; r < nnz; ++r) {
        const int64_t u = uid[r], i = iid[r];
        const double val = rat[r];
        double* Uu = U + u * k;
        double* Vi = V + i * k;
        double s = 0.0;
        for (int f = 0; f < k; ++f) s += Uu[f] * Vi[f];             /* pmf.pyx:141-143 */
        const double sg = sigmoid((float)s);                        /* pmf.pyx:144-146 */
        const double e = val - sg;
        const double we = e * sg * (1. - sg);
        const double t = apply_rating(Uu, Vi, cache_u + u * k, cache_v + i * k, k, e, we, lambda_reg, learning_rate, gamma);
        if (terms) terms[r] = t;
        loss += t;
    }
    return loss;
}

/* sigmoid of the n floats whose bit patterns are first, first + 1, ... (the exhaustive comparison of the device
 * sigmoid). */
API void pmf_sigmoid_bits(uint32_t first, int64_t n, float* out)
{
#pragma omp parallel for schedule(static)
    for (int64_t j = 0; j < n; ++j) {
        const uint32_t b = first + (uint32_t)j;
        float z;
        memcpy(&z, &b, sizeof z);
        out[j] = sigmoid(z);
    }
}
