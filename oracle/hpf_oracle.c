/* TEST INFRASTRUCTURE: a scalar C restatement of the reference HPF / PF fit (cornac/models/hpf/cpp/cpp_hpf.cpp:139-275),
 * the oracle the GPU fit is compared with where the compiled reference is not available.
 *
 * The reference is built without -ffast-math or -march: no multiply-add is fused and no sum is reordered.  This file is
 * compiled -O2 -ffp-contract=off for the same reason.  The update loops walk the ratings as the reference's do: column
 * by column (items ascending), users ascending inside a column.  The expectations use libm's exp and log and the Cephes
 * digamma (the recurrence to s >= 10, then the asymptotic series), which is the algorithm the reference's Eigen uses.
 *
 * State: Gs, Gr [n, k]; Ls, Lr [d, k]; Kr [n]; Tr [d], row-major f64.  Ratings: CSC (col_ptr [d + 1], row_ind, val). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define API __attribute__((visibility("default")))

static double digamma_pos(double x)
{
    double s = x, w = 0.0, y = 0.0;
    while (s < 10.0) {
        w += 1.0 / s;
        s += 1.0;
    }
    if (s < 1e17) {
        const double z = 1.0 / (s * s);
        double p = 1.0 / 12.0;
        p = p * z + -691.0 / 32760.0;
        p = p * z + 1.0 / 132.0;
        p = p * z + -1.0 / 240.0;
        p = p * z + 1.0 / 252.0;
        p = p * z + -1.0 / 120.0;
        p = p * z + 1.0 / 12.0;
        y = z * p;
    }
    return log(s) - (0.5 / s) - y - w;
}

API double hpf_digamma(double x) { return digamma_pos(x); }

/* E_SpMat_logGamma + exp: an entry whose shape (rate) is not > 0 drops the digamma (log) term; both dropped -> 0. */
API void hpf_expect(const double* shape, const double* rate, int64_t n, double* out)
{
    for (int64_t t = 0; t < n; ++t) {
        const int hs = shape[t] > 0.0, hr = rate[t] > 0.0;
        if (!hs && !hr) {
            out[t] = 0.0;
            continue;
        }
        double e = hs ? digamma_pos(shape[t]) : 0.0;
        if (hr) e = e - log(rate[t]);
        out[t] = exp(e);
    }
}

/* update_kappa_r */
static void kappa(double* Kr, const double* S, const double* R, int64_t n, int k, double a_over_c)
{
    for (int64_t i = 0; i < n; ++i) {
        double sk = 0.0;
        for (int f = 0; f < k; ++f) sk += S[i * k + f] / R[i * k + f];
        Kr[i] = a_over_c + sk;
    }
}

/* update_gamma_r: R[i, f] = shape_s / Kr[i] + sum over the other side's rows of S2 / R2 (R2 <= 0 skipped) */
static void rate(double* R, const double* S2, const double* R2, int64_t n2, const double* Kr, int64_t n, int k,
                 double shape_s)
{
    for (int f = 0; f < k; ++f) {
        double sk = 0.0;
        for (int64_t j = 0; j < n2; ++j)
            if (R2[j * k + f] > 0.0) sk += S2[j * k + f] / R2[j * k + f];
        for (int64_t i = 0; i < n; ++i) R[i * k + f] = shape_s / Kr[i] + sk;
    }
}

/* update_gamma_s (user_side) / update_lambda_s: out = shape0, then the ratings' shares in the reference's walk. */
static void shape_pass(double* out, int64_t n_out, int user_side, const int32_t* col_ptr, const int32_t* row_ind,
                       const double* val, int64_t d, int k, const double* Lt, const double* Lb, double shape0)
{
    const double eps = pow(2, -52);
    for (int64_t t = 0; t < n_out * k; ++t) out[t] = shape0;
    for (int64_t i = 0; i < d; ++i) {
        for (int32_t c = col_ptr[i]; c < col_ptr[i + 1]; ++c) {
            const int64_t u = row_ind[c];
            double dk = eps;
            for (int f = 0; f < k; ++f) dk += Lt[u * k + f] * Lb[i * k + f];
            double* o = out + (user_side ? u : i) * k;
            for (int f = 0; f < k; ++f) o[f] += Lt[u * k + f] * Lb[i * k + f] * val[c] / dk;
        }
    }
}

/* One iteration from given expectations Lt [n, k], Lb [d, k]: G_s, G_r, (HPF) K_r, L_s, L_r, (HPF) T_r. */
API void hpf_update(int hierarchical, int64_t n, int64_t d, int k, const int32_t* col_ptr, const int32_t* row_ind,
                    const double* val, const double* Lt, const double* Lb, double* Gs, double* Gr, double* Ls,
                    double* Lr, double* Kr, double* Tr)
{
    const double a = 0.3, b = 0.3, c = 1.0;
    const double ks = hierarchical ? a + k * a : a;
    const double ts = hierarchical ? b + k * b : b;
    shape_pass(Gs, n, 1, col_ptr, row_ind, val, d, k, Lt, Lb, a);
    rate(Gr, Ls, Lr, d, Kr, n, k, ks);
    if (hierarchical) kappa(Kr, Gs, Gr, n, k, a / c);
    shape_pass(Ls, d, 0, col_ptr, row_ind, val, d, k, Lt, Lb, b);
    rate(Lr, Gs, Gr, n, Tr, d, k, ts);
    if (hierarchical) kappa(Tr, Ls, Lr, d, k, b / c);
}

/* hpf_cpp / pf_cpp: max_iter iterations (HPF sets K_r, T_r from the state first).  Returns 0, or -1 out of memory. */
API int hpf_fit(int hierarchical, int64_t n, int64_t d, int k, const int32_t* col_ptr, const int32_t* row_ind,
                const double* val, double* Gs, double* Gr, double* Ls, double* Lr, double* Kr, double* Tr, int max_iter)
{
    double* Lt = malloc(sizeof(double) * (size_t)(n * k + 1));
    double* Lb = malloc(sizeof(double) * (size_t)(d * k + 1));
    if (!Lt || !Lb) {
        free(Lt);
        free(Lb);
        return -1;
    }
    if (hierarchical) {
        kappa(Kr, Gs, Gr, n, k, 0.3 / 1.0);
        kappa(Tr, Ls, Lr, d, k, 0.3 / 1.0);
    }
    for (int it = 0; it < max_iter; ++it) {
        hpf_expect(Gs, Gr, n * k, Lt);
        hpf_expect(Ls, Lr, d * k, Lb);
        hpf_update(hierarchical, n, d, k, col_ptr, row_ind, val, Lt, Lb, Gs, Gr, Ls, Lr, Kr, Tr);
    }
    free(Lt);
    free(Lb);
    return 0;
}
