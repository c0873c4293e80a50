/* TEST INFRASTRUCTURE: a scalar C restatement of the reference C2PF fits (cornac/models/c2pf/cpp/cpp_c2pf.cpp: c2pf_cpp,
 * tc2pf_cpp, rc2pf_cpp), the oracle the GPU fit is compared with where the compiled reference is not available.
 *
 * The reference is built without -ffast-math or -march: no multiply-add is fused and no sum is reordered.  This file is
 * compiled -O2 -ffp-contract=off for the same reason.  Plain CSC arrays stand in for the reference's Eigen matrices; the
 * loops walk them as the reference's do, and every read of the sparse kappa matrices at the mirrored position (i, row)
 * of a stored (row, i) is a binary search, as SparseMatrix::coeff is.  A mirrored position that is not stored makes the
 * reference insert a zero shape there; this restatement reports it instead (return code -2).
 *
 * variant 0: c2pf_cpp, 1: tc2pf_cpp (L2 is L: pass the same pointers), 2: rc2pf_cpp (no L: Ls, Lr, Lb are NULL).
 * State, row-major f64: Gs, Gr [n, k]; Ls, Lr, L2s, L2r [d, k]; L3s, L3r [nnz(C)] in the CSC order of C; T3r [d].
 * Expectations: Lt [n, k]; Lb, L2b, Lb2 [d, k]; L3b [nnz(C)].  Ratings X and graph pattern C: CSC, rows ascending.
 * util[i] is the reference's util_sum (column sums of C's values), which only c2pf_cpp reads. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define API __attribute__((visibility("default")))

typedef struct {
    int variant;
    int64_t n, d;
    int k;
    const int32_t *xp, *xr;
    const double* xv;
    const int32_t *cp, *cr;
    const double* util;
    double at, bt;
    double *Gs, *Gr, *Ls, *Lr, *L2s, *L2r, *L3s, *L3r, *T3r;
    double *Lt, *Lb, *L2b, *L3b, *Lb2;
} C2pf;

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

/* E_SpMat_logGamma(Mat, Mat) + exp: a term whose argument is not > 0 is dropped; both dropped -> 0 (not stored). */
API void c2pf_expect(const double* shape, const double* rate, int64_t n, double* out)
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

/* E_SpMat_logGamma(SpMat, SpMat) + exp: every stored entry, no filter (shapes must be > 0). */
API void c2pf_expect_sparse(const double* shape, const double* rate, int64_t n, double* out)
{
    for (int64_t t = 0; t < n; ++t) out[t] = exp(digamma_pos(shape[t]) - log(rate[t]));
}

/* position of (row, col) in C, or -1 */
static int64_t find(const C2pf* p, int64_t row, int64_t col)
{
    int64_t lo = p->cp[col], hi = p->cp[col + 1];
    while (lo < hi) {
        const int64_t mid = (lo + hi) / 2;
        if (p->cr[mid] < row)
            lo = mid + 1;
        else
            hi = mid;
    }
    return (lo < p->cp[col + 1] && p->cr[lo] == row) ? lo : -1;
}

API int c2pf_mirrors(int64_t d, const int32_t* cp, const int32_t* cr, int32_t* mir)
{
    C2pf p = {0};
    p.cp = cp;
    p.cr = cr;
    int bad = 0;
    for (int64_t i = 0; i < d; ++i)
        for (int32_t c = cp[i]; c < cp[i + 1]; ++c) {
            mir[c] = (int32_t)find(&p, i, cr[c]);
            if (mir[c] < 0) bad = 1;
        }
    return bad ? -2 : 0;
}

static double item_exp(const C2pf* p, int64_t i, int f)
{
    return p->variant == 2 ? p->Lb2[i * p->k + f] : p->Lb[i * p->k + f] + p->Lb2[i * p->k + f];
}

static double dk_of(const C2pf* p, int64_t u, int64_t i)
{
    double dk = pow(2, -52);
    for (int f = 0; f < p->k; ++f) dk += p->Lt[u * p->k + f] * item_exp(p, i, f);
    return dk;
}

/* the Lb_u row of item i: the users' ordered sum of x * Lt / dk */
static void lbu_row(const C2pf* p, int64_t i, double* lbu)
{
    const int k = p->k;
    for (int f = 0; f < k; ++f) lbu[f] = 0.0;
    for (int32_t c = p->xp[i]; c < p->xp[i + 1]; ++c) {
        const int64_t u = p->xr[c];
        const double dk = dk_of(p, u, i);
        for (int f = 0; f < k; ++f) lbu[f] += p->xv[c] * p->Lt[u * k + f] / dk;
    }
}

/* set_coeffs_to_sparse(L3_s, a_t) + update_gamma_s_context_3_n(_r) */
static int shape_kappa(const C2pf* p, double* lbu)
{
    const int k = p->k;
    for (int64_t e = 0; e < p->cp[p->d]; ++e) p->L3s[e] = p->at;
    for (int64_t i = 0; i < p->d; ++i) {
        lbu_row(p, i, lbu);
        for (int32_t c = p->cp[i]; c < p->cp[i + 1]; ++c) {
            const int64_t r = p->cr[c], m = find(p, i, r);
            if (m < 0) return -2;
            for (int f = 0; f < k; ++f) p->L3s[m] += p->L2b[r * k + f] * p->L3b[m] * lbu[f];
        }
    }
    return 0;
}

/* Sk[f] = sum over users of G_s / G_r (G_r <= 0 skipped) */
static void user_sums(const C2pf* p, double* Sk)
{
    const int k = p->k;
    for (int f = 0; f < k; ++f) {
        Sk[f] = 0.0;
        for (int64_t u = 0; u < p->n; ++u)
            if (p->Gr[u * k + f] > 0.0) Sk[f] += p->Gs[u * k + f] / p->Gr[u * k + f];
    }
}

/* update_gamma_r_context_3_n (c2pf_cpp: k_s = 5, att = a_t) / update_gamma_r_context_3_n_2 (k_s = b_t) */
static void rate_kappa(const C2pf* p, double* Sk)
{
    const int k = p->k;
    user_sums(p, Sk);
    for (int64_t j = 0; j < p->d; ++j) {
        double Sj = 0.0;
        for (int f = 0; f < k; ++f)
            if (p->L2r[j * k + f] > 0.0) Sj += (p->L2s[j * k + f] / p->L2r[j * k + f]) * Sk[f];
        for (int32_t c = p->cp[j]; c < p->cp[j + 1]; ++c) {
            const int64_t r = p->cr[c];
            if (p->variant == 0)
                p->L3r[c] = p->at * (5. + p->at * p->util[r]) / p->T3r[r] + Sj;
            else
                p->L3r[c] = p->bt / p->T3r[r] + Sj;
        }
    }
}

static int context_sums(const C2pf* p)
{
    const int k = p->k;
    for (int64_t i = 0; i < p->d; ++i)
        for (int f = 0; f < k; ++f) {
            double s = 0.0;
            for (int32_t c = p->cp[i]; c < p->cp[i + 1]; ++c) {
                const int64_t r = p->cr[c], m = find(p, i, r);
                if (m < 0) return -2;
                s += p->L2b[r * k + f] * p->L3b[m];
            }
            p->Lb2[i * k + f] = s;
        }
    return 0;
}

/* update_kappa_r_inv_kappa(T3_r, L3_s, L3_r, C, b_t, 1.0, a_t) */
static int kappa_rate(const C2pf* p)
{
    const double b_ = 1.0;
    for (int64_t i = 0; i < p->d; ++i) {
        double Si = 0.0;
        for (int32_t c = p->cp[i]; c < p->cp[i + 1]; ++c) {
            const int64_t m = find(p, i, p->cr[c]);
            if (m < 0) return -2;
            Si += p->L3s[m] / p->L3r[m];
        }
        p->T3r[i] = p->bt / b_ + p->at * Si;
    }
    return 0;
}

/* set_coeffs_to(G_s, 0.3) + update_gamma_s_context(_r) */
static void shape_users(const C2pf* p)
{
    const int k = p->k;
    for (int64_t t = 0; t < p->n * k; ++t) p->Gs[t] = 0.3;
    for (int64_t i = 0; i < p->d; ++i)
        for (int32_t c = p->xp[i]; c < p->xp[i + 1]; ++c) {
            const int64_t u = p->xr[c];
            const double dk = dk_of(p, u, i);
            for (int f = 0; f < k; ++f) p->Gs[u * k + f] += p->Lt[u * k + f] * item_exp(p, i, f) * p->xv[c] / dk;
        }
}

/* update_gamma_r_context_n / update_gamma_r_context_n_r */
static int rate_users(const C2pf* p)
{
    const int k = p->k;
    for (int f = 0; f < k; ++f) {
        double Sk = 0.0;
        for (int64_t i = 0; i < p->d; ++i) {
            if (p->variant != 2) {
                if (!(p->Lr[i * k + f] > 0.0)) continue;
                Sk += p->Ls[i * k + f] / p->Lr[i * k + f];
            }
            for (int32_t c = p->cp[i]; c < p->cp[i + 1]; ++c) {
                const int64_t r = p->cr[c], m = find(p, i, r);
                if (m < 0) return -2;
                Sk += (p->L2s[r * k + f] / p->L2r[r * k + f]) * (p->L3s[m] / p->L3r[m]);
            }
        }
        for (int64_t u = 0; u < p->n; ++u) p->Gr[u * k + f] = 0.3 + Sk;
    }
    return 0;
}

/* set_coeffs_to(L_s, 0.3) + update_lambda_s_context */
static void shape_items(const C2pf* p)
{
    const int k = p->k;
    for (int64_t t = 0; t < p->d * k; ++t) p->Ls[t] = 0.3;
    for (int64_t i = 0; i < p->d; ++i)
        for (int32_t c = p->xp[i]; c < p->xp[i + 1]; ++c) {
            const int64_t u = p->xr[c];
            const double dk = dk_of(p, u, i);
            for (int f = 0; f < k; ++f) p->Ls[i * k + f] += p->Lt[u * k + f] * p->Lb[i * k + f] * p->xv[c] / dk;
        }
}

/* update_gamma_s_context_2_n(_r): adds to L2s (tc2pf: to L_s, after the ratings' shares) */
static int shape_context(const C2pf* p, double* lbu)
{
    const int k = p->k;
    for (int64_t i = 0; i < p->d; ++i) {
        lbu_row(p, i, lbu);
        for (int32_t c = p->cp[i]; c < p->cp[i + 1]; ++c) {
            const int64_t r = p->cr[c], m = find(p, i, r);
            if (m < 0) return -2;
            for (int f = 0; f < k; ++f) p->L2s[r * k + f] += p->L2b[r * k + f] * p->L3b[m] * lbu[f];
        }
    }
    return 0;
}

/* update_gamma_r (tied: first) and update_gamma_r_context_2_n(_tied) */
static void rate_items(const C2pf* p, double* Sk)
{
    const int k = p->k;
    user_sums(p, Sk);
    if (p->variant != 2)
        for (int f = 0; f < k; ++f)
            for (int64_t i = 0; i < p->d; ++i) p->Lr[i * k + f] = 0.3 + Sk[f];
}

static void rate_context(const C2pf* p, const double* Sk)
{
    const int k = p->k;
    for (int f = 0; f < k; ++f)
        for (int64_t j = 0; j < p->d; ++j) {
            double Sj = 0.0;
            for (int32_t c = p->cp[j]; c < p->cp[j + 1]; ++c) Sj += p->L3s[c] / p->L3r[c];
            if (p->variant == 1)
                p->L2r[j * k + f] += Sj * Sk[f];
            else
                p->L2r[j * k + f] = 0.3 + Sj * Sk[f];
        }
}

static int iterate(const C2pf* p, double* lbu, double* Sk)
{
    const int k = p->k;
    const int64_t ne = p->cp[p->d];
    if (shape_kappa(p, lbu)) return -2;
    rate_kappa(p, Sk);
    c2pf_expect_sparse(p->L3s, p->L3r, ne, p->L3b);
    context_sums(p);
    if (p->variant == 0) kappa_rate(p);
    shape_users(p);
    rate_users(p);
    c2pf_expect(p->Gs, p->Gr, p->n * k, p->Lt);
    if (p->variant != 2) shape_items(p);
    if (p->variant == 0) {
        rate_items(p, Sk);
        c2pf_expect(p->Ls, p->Lr, p->d * k, p->Lb);
    }
    if (p->variant != 1)
        for (int64_t t = 0; t < p->d * k; ++t) p->L2s[t] = 0.3;
    shape_context(p, lbu);
    if (p->variant != 0) rate_items(p, Sk);
    rate_context(p, Sk);
    c2pf_expect(p->L2s, p->L2r, p->d * k, p->L2b);
    context_sums(p);
    return 0;
}

#define C2PF_PARAMS                                                                                                    \
    int variant, int64_t n, int64_t d, int k, const int32_t *xp, const int32_t *xr, const double *xv,                  \
        const int32_t *cp, const int32_t *cr, const double *util, double at, double bt, double *Gs, double *Gr,        \
        double *Ls, double *Lr, double *L2s, double *L2r, double *L3s, double *L3r, double *T3r
#define C2PF_INIT(Lt, Lb, L2b, L3b, Lb2)                                                                               \
    {variant, n, d, k, xp, xr, xv, cp, cr, util, at, bt, Gs, Gr, Ls, Lr, L2s, L2r, L3s, L3r, T3r, Lt, Lb, L2b, L3b, Lb2}

/* One iteration from the expectations Lt, Lb, L2b, L3b, Lb2, which are replaced by the ones the iteration computes
 * (tc2pf: L2b is Lb).  Returns 0, -1 out of memory, -2 a stored (r, i) of C without its mirror (i, r). */
API int c2pf_update(C2PF_PARAMS, double* Lt, double* Lb, double* L2b, double* L3b, double* Lb2)
{
    const C2pf p = C2PF_INIT(Lt, Lb, L2b, L3b, Lb2);
    double* tmp = malloc(sizeof(double) * 2 * (size_t)k);
    if (!tmp) return -1;
    const int rc = iterate(&p, tmp, tmp + k);
    free(tmp);
    return rc;
}

/* One call of c2pf_cpp / tc2pf_cpp / rc2pf_cpp with (a_t, b_t) = (at, bt): max_iter iterations on the state. */
API int c2pf_fit(C2PF_PARAMS, int max_iter)
{
    const int64_t ne = cp[d];
    double* buf = malloc(sizeof(double) * (size_t)((n + 3 * d) * k + ne + 2 * k + 1));
    if (!buf) return -1;
    double *Lt = buf, *Lb = Lt + n * k, *L2b = Lb + d * k, *Lb2 = L2b + d * k, *L3b = Lb2 + d * k, *tmp = L3b + ne;
    if (variant == 1) L2b = Lb;
    const C2pf p = C2PF_INIT(Lt, variant == 2 ? NULL : Lb, L2b, L3b, Lb2);
    int rc = 0;
    if (variant == 0) rc = kappa_rate(&p);
    c2pf_expect(Gs, Gr, n * k, Lt);
    if (variant != 2) c2pf_expect(Ls, Lr, d * k, Lb);
    if (variant != 1) c2pf_expect(L2s, L2r, d * k, L2b);
    c2pf_expect_sparse(L3s, L3r, ne, L3b);
    if (!rc) rc = context_sums(&p);
    for (int it = 0; it < max_iter && !rc; ++it) rc = iterate(&p, tmp, tmp + k);
    free(buf);
    return rc;
}
