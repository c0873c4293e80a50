/* TEST INFRASTRUCTURE: a scalar C restatement of the graph-edge pass of SoRec (cornac/models/sorec/cython/sorec.pyx:81-109)
 * and MCF (cornac/models/mcf/cython/mcf.pyx:83-111), the oracle the GPU co-factor fit is compared with.
 *
 * An edge update is a pmf_non_linear rating update (same sigmoid, same f64 element steps, same loss term) of two other
 * rows: SoRec's (U[i], Z[j]) with the step lambda_c * learning_rate (two C floats, so an f32 product), MCF's (V[i], Z[j])
 * with learning_rate.  PMF's oracle is included as it stands so that both oracles share one sigmoid and one element step;
 * the rating pass of an epoch is its pmf_nonlinear_epoch.  Same flags: -O2 -ffp-contract=off. */
#include "pmf_oracle.c"

/* One edge pass over the n edges in stored order: A[a[e]] and B[b[e]] with the caches ca / cb, target val[e], and the
 * step `step` (f32, promoted as the reference promotes it).  terms (nullable, [n]) receives each edge's loss term. */
API void cofactor_edge_pass(const int32_t* a, const int32_t* b, const float* val, int64_t n, int k, double* A, double* B,
                            double* ca, double* cb, float lambda_reg, float step, float gamma, double* terms)
{
    for (int64_t e = 0; e < n; ++e) {
        const int64_t i = a[e], j = b[e];
        double* Ai = A + i * k;
        double* Bj = B + j * k;
        double s = 0.0;
        for (int f = 0; f < k; ++f) s += Ai[f] * Bj[f];             /* sorec.pyx:84-86 */
        const double sg = sigmoid((float)s);                        /* sorec.pyx:87-89: sg, err, werr are doubles */
        const double err = (double)val[e] - sg;
        const double werr = err * sg * (1. - sg);
        const double t = apply_rating(Ai, Bj, ca + i * k, cb + j * k, k, err, werr, lambda_reg, step, gamma);
        if (terms) terms[e] = t;
    }
}

/* sorec.pyx:95 `lambda_c * learning_rate * (...)`: the f32 product of two C floats */
API float cofactor_sorec_step(float lambda_c, float learning_rate)
{
    return lambda_c * learning_rate;
}
