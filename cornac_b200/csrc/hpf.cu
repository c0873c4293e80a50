// HPF / PF (cornac/models/hpf/cpp/cpp_hpf.cpp:139-275) for sm_90a: the coordinate-ascent variational fit in f64, in the
// reference's update order.
//
// The reference is built without -ffast-math or -march, so it has no FMA and never reorders a sum.  Every product, sum
// and quotient below is an explicitly rounded __d*_rn intrinsic in the reference's order, so given the same expectations
// Lt / Lb an iteration is bit-identical to it.  The expectations themselves use CUDA's exp / log and a restatement of the
// Cephes digamma, so they differ from glibc / Eigen in the last bits; the fit agrees with the reference to rounding.
//
// One iteration (constants a = b = 0.3; HPF: k_s = t_s = 0.3 + 0.3 g, c = 1; PF: k_s = t_s = 0.3, K_r = T_r = 1):
//   1. hpf_expect_kernel: Lt = exp(digamma(G_s) - log(G_r)), Lb likewise; a term whose shape / rate is <= 0 is dropped
//      and an entry with both dropped is 0 (the reference works on sparse matrices that store only positive entries);
//   2. hpf_dk_kernel: dk = 2^-52 + sum_k Lt[u,k] Lb[i,k] for every rating, k ascending;
//   3. hpf_pass_kernel over the CSR rows: G_s[u,k] = a + sum over the row, items ascending, of ((Lt Lb) x) / dk;
//   4. hpf_colsum_kernel: S[k] = sum over items, ascending, of the OLD L_s / L_r (entries with L_r <= 0 skipped);
//      hpf_rate_kernel: G_r[u,k] = k_s / K_r[u] + S[k]; HPF: K_r[u] = a / c + sum_k G_s / G_r;
//   5. hpf_pass_kernel over the CSC columns (users ascending, dk through the CSR -> CSC map): L_s;
//   6. S'[k] over the NEW G_s / G_r, then L_r and (HPF) T_r as in 4.
// A skipped quotient enters the column sums as +0.0: a sum that starts at +0.0 is never -0.0, so adding +0.0 leaves it
// unchanged bit for bit.  The column sums are one sequential chain per factor, as in the reference.
// The kernels of steps 1-3, 5 and the column sums are in hpf_common.cuh, which c2pf.cu shares.
#include "hpf_common.cuh"

namespace b200 {

// Steps 4 and 6, the row updates: a thread per row.  RATE: R[r,f] = shape_s / Kr[r] + colsum[f].  KAPPA: Kr[r] = a/c +
// sum_f S[r,f] / R[r,f] (f ascending, nothing skipped: update_kappa_r).  Q (may be NULL): the quotients the next column
// sum adds, R > 0 ? S / R : +0.0.
template <bool RATE, bool KAPPA>
__global__ void __launch_bounds__(HPF_THREADS) hpf_rate_kernel(int64_t n_rows, int k, const double* __restrict__ S,
                                                               double* __restrict__ R, double* __restrict__ Kr,
                                                               const double* __restrict__ colsum, double shape_s,
                                                               double a_over_c, double* __restrict__ Q)
{
    for (int64_t r = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * HPF_THREADS) {
        const size_t base = (size_t)r * k;
        if constexpr (RATE) {
            const double head = __ddiv_rn(shape_s, Kr[r]);
            for (int f = 0; f < k; ++f) R[base + f] = __dadd_rn(head, __ldg(colsum + f));
        }
        double sum = 0.0;
        for (int f = 0; f < k; ++f) {
            const double rv = R[base + f];
            const double q = __ddiv_rn(__ldg(S + base + f), rv);
            if constexpr (KAPPA) sum = __dadd_rn(sum, q);
            if (Q) Q[base + f] = rv > 0.0 ? q : 0.0;
        }
        if constexpr (KAPPA) Kr[r] = __dadd_rn(a_over_c, sum);
    }
}

struct HpfWork {
    double *dk, *qL, *qG, *S, *S2, *Lt, *Lb;
};

HpfWork hpf_carve(double* w, int64_t n_users, int64_t n_items, int64_t nnz, int k)
{
    HpfWork h;
    h.dk = w;
    h.qL = h.dk + std::max<int64_t>(nnz, 1);
    h.qG = h.qL + n_items * k;
    h.S = h.qG + n_users * k;
    h.S2 = h.S + k;
    h.Lt = h.S2 + k;
    h.Lb = h.Lt + n_users * k;
    return h;
}


template <bool RATE, bool KAPPA>
void hpf_rate(int64_t n_rows, int k, const double* S, double* R, double* Kr, const double* colsum, double shape_s,
              double a_over_c, double* Q, cudaStream_t st)
{
    if (n_rows == 0) return;
    hpf_rate_kernel<RATE, KAPPA><<<hpf_grid(n_rows), HPF_THREADS, 0, st>>>(n_rows, k, S, R, Kr, colsum, shape_s,
                                                                          a_over_c, Q);
    count_launch();
}

struct HpfArgs {
    int hierarchical;
    int64_t n_users, n_items;
    int k;
    SparseArgs<double> r;
    double *Gs, *Gr, *Ls, *Lr, *Kr, *Tr;
};

// Steps 2-6 of one iteration from the expectations Lt, Lb.
void hpf_update(const HpfArgs& a, const double* Lt, const double* Lb, const HpfWork& w, cudaStream_t st)
{
    const int k = a.k;
    const double ks = a.hierarchical ? HPF_A + (double)k * HPF_A : HPF_A;
    const double ts = a.hierarchical ? HPF_B + (double)k * HPF_B : HPF_B;
    const double c = 1.0;
    const unsigned gk = (unsigned)((k + 31) / 32);
    // S from the old L_s / L_r (update_gamma_r before update_lambda_s)
    if (a.n_items * k > 0) {
        hpf_quotient_kernel<<<hpf_grid(a.n_items * k), HPF_THREADS, 0, st>>>(a.Ls, a.Lr, a.n_items * k, w.qL);
        count_launch();
    }
    hpf_colsum_kernel<<<gk, 32, 0, st>>>(w.qL, a.n_items, k, w.S);
    count_launch();
    if (a.r.nnz > 0) {
        hpf_dk_kernel<<<hpf_grid(a.r.nnz), HPF_THREADS, 0, st>>>(a.r.row, a.r.idx, a.r.nnz, k, Lt, Lb, w.dk);
        count_launch();
    }
    if (a.n_users > 0) {
        hpf_pass_kernel<true><<<hpf_grid(a.n_users * k), HPF_THREADS, 0, st>>>(
            a.r.ptr, a.r.idx, a.r.val, nullptr, w.dk, a.n_users, k, Lt, Lb, HPF_A, a.Gs);
        count_launch();
    }
    if (a.hierarchical)
        hpf_rate<true, true>(a.n_users, k, a.Gs, a.Gr, a.Kr, w.S, ks, HPF_A / c, w.qG, st);
    else
        hpf_rate<true, false>(a.n_users, k, a.Gs, a.Gr, a.Kr, w.S, ks, 0.0, w.qG, st);
    hpf_colsum_kernel<<<gk, 32, 0, st>>>(w.qG, a.n_users, k, w.S2);
    count_launch();
    if (a.n_items > 0) {
        hpf_pass_kernel<false><<<hpf_grid(a.n_items * k), HPF_THREADS, 0, st>>>(
            a.r.cptr, a.r.crow, a.r.cval, a.r.cpos, w.dk, a.n_items, k, Lb, Lt, HPF_B, a.Ls);
        count_launch();
    }
    if (a.hierarchical)
        hpf_rate<true, true>(a.n_items, k, a.Ls, a.Lr, a.Tr, w.S2, ts, HPF_B / c, nullptr, st);
    else
        hpf_rate<true, false>(a.n_items, k, a.Ls, a.Lr, a.Tr, w.S2, ts, 0.0, nullptr, st);
}

int hpf_check(const HpfArgs& a, const void* work, const char* what)
{
    if (int rc = sparse_check(a.r, a.n_users, a.n_items, what)) return rc;
    B200_REQUIRE(a.k >= 1, "%s: bad k=%d", what, a.k);
    B200_REQUIRE(work && (a.n_users == 0 || (a.Gs && a.Gr && a.Kr)) && (a.n_items == 0 || (a.Ls && a.Lr && a.Tr)),
                 "%s: null pointer argument", what);
    return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_hpf_workspace_bytes(int64_t n_users, int64_t n_items, int64_t nnz, int k)
{
    if (n_users < 0 || n_items < 0 || nnz < 0 || k < 1) return -1;
    return (int64_t)sizeof(double) * (std::max<int64_t>(nnz, 1) + 2 * (n_users + n_items) * k + 2 * (int64_t)k);
}

extern "C" int b200_hpf_expect(const double* shape, const double* rate, int64_t n, double* out, void* stream)
{
    B200_REQUIRE(n >= 0, "b200_hpf_expect: bad size n=%lld", (long long)n);
    B200_REQUIRE(n == 0 || (shape && rate && out), "b200_hpf_expect: null pointer argument");
    hpf_expect(shape, rate, n, out, (cudaStream_t)stream);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_hpf_update(int hierarchical, int64_t n_users, int64_t n_items, int k, B200_SPARSE(r_, double),
                               const double* Lt, const double* Lb, double* Gs, double* Gr, double* Ls, double* Lr,
                               double* Kr, double* Tr, double* work, void* stream)
{
    const HpfArgs a{hierarchical, n_users, n_items, k, B200_SPARSE_VIEW(r_), Gs, Gr, Ls, Lr, Kr, Tr};
    if (int rc = hpf_check(a, work, "b200_hpf_update")) return rc;
    B200_REQUIRE((n_users == 0 || Lt) && (n_items == 0 || Lb), "b200_hpf_update: null Lt / Lb");
    hpf_update(a, Lt, Lb, hpf_carve(work, n_users, n_items, r_nnz, k), (cudaStream_t)stream);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_hpf_fit(int hierarchical, int64_t n_users, int64_t n_items, int k, B200_SPARSE(r_, double),
                            double* Gs, double* Gr, double* Ls, double* Lr, double* Kr, double* Tr, int max_iter,
                            double* work, void* stream)
{
    const HpfArgs a{hierarchical, n_users, n_items, k, B200_SPARSE_VIEW(r_), Gs, Gr, Ls, Lr, Kr, Tr};
    if (int rc = hpf_check(a, work, "b200_hpf_fit")) return rc;
    B200_REQUIRE(max_iter >= 0, "b200_hpf_fit: bad max_iter=%d", max_iter);
    cudaStream_t st = (cudaStream_t)stream;
    const HpfWork w = hpf_carve(work, n_users, n_items, r_nnz, k);
    // hpf_cpp's update_kappa_r before the loop.  After an iteration K_r and T_r already hold these values, so a fit split
    // into several calls recomputes them bit for bit.
    if (hierarchical) {
        hpf_rate<false, true>(n_users, k, Gs, Gr, Kr, nullptr, 0.0, HPF_A / 1.0, nullptr, st);
        hpf_rate<false, true>(n_items, k, Ls, Lr, Tr, nullptr, 0.0, HPF_B / 1.0, nullptr, st);
    }
    for (int it = 0; it < max_iter; ++it) {
        hpf_expect(Gs, Gr, n_users * k, w.Lt, st);
        hpf_expect(Ls, Lr, n_items * k, w.Lb, st);
        hpf_update(a, w.Lt, w.Lb, w, st);
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
