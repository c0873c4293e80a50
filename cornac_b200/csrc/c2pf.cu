// C2PF (cornac/models/c2pf/cpp/cpp_c2pf.cpp: c2pf_cpp, tc2pf_cpp, rc2pf_cpp) for sm_90a: the coordinate-ascent
// variational fit of Collaborative Context Poisson Factorization in f64, in the reference's update order.
//
// As in hpf.cu, every product, sum and quotient is an explicitly rounded __d*_rn intrinsic in the reference's order and
// association, so given the same expectations an iteration is bit-identical to the reference's arithmetic; exp, log and
// digamma are hpf_common.cuh's.  The context graph C is a d x d CSC pattern (c_ptr, c_row, and c_col: the column of each
// entry) that must be symmetric: c_mir[p] is the position of (i, r) for the entry p = (r, i).  The reference reads kappa
// (L3) at the mirrored position while it walks a column, which is why the mirror map is an input.
//
// One iteration (variant 0 c2pf, 1 tc2pf: L2 is L, 2 rc2pf: no L; E = Lb + Lb2, rc2pf: Lb2):
//   1. dk = 2^-52 + sum_k Lt E per rating; Lb_u[i,k] = sum over item i's users, ascending, of (x Lt) / dk;
//      per edge q = (a, b): L3_s = a_t + sum_k ((L2b[b,k] L3b[q]) Lb_u[a,k]), a chain over k;
//      L3_r = (a_t (5 + a_t util[a])) / T3_r[a] + Sj[b] (c2pf) or b_t / T3_r[a] + Sj[b], Sj[b] = sum_k (L2_s/L2_r)[b,k] S[k],
//      S[k] the ordered sum over users of G_s / G_r; L3b = exp(digamma(L3_s) - log(L3_r)) on every edge;
//   2. Lb2[i,k] = sum over column i, rows ascending, of L2b[r,k] L3b(i,r); (c2pf) T3_r[i] = b_t + a_t sum L3_s/L3_r (i,r);
//   3. G_s as HPF's user pass with E on the item side (new dk); G_r = 0.3 + one chain per factor over all items and,
//      nested inside each item, its context entries: the terms are computed in parallel into scratch in chain order
//      (a skipped term is +0.0) and hpf_colsum_kernel adds them; Lt;
//   4. (not rc2pf) L_s as HPF's item pass (new dk); c2pf: L_r = 0.3 + S'[k], Lb;
//   5. Lb_u again (new dk; tc2pf: step 4's), L2_s[r,k] = 0.3 (tc2pf: L_s[r,k]) + sum over column r, rows i ascending, of
//      (L2b[r,k] L3b(i,r)) Lb_u[i,k]; L2_r = 0.3 + Sj' S' (tc2pf: (0.3 + S') + Sj' S'), Sj'[j] the column sum of
//      L3_s / L3_r; L2b; Lb2.
#include "hpf_common.cuh"

namespace b200 {

constexpr double C2PF_SHAPE = 0.3;              // aa, cc, ee, k_s, t_s of all three variants
constexpr double C2PF_A1 = 5.0;                 // a1_ of c2pf_cpp's L3_r

__global__ void __launch_bounds__(HPF_THREADS) c2pf_add_kernel(const double* __restrict__ a,
                                                               const double* __restrict__ b, int64_t n,
                                                               double* __restrict__ out)
{
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS)
        out[t] = __dadd_rn(a[t], b[t]);
}

// kap = L3_s / L3_r and (L3b != NULL) the sparse expectation: every entry, no filter.  digamma is defined here for
// positive shapes only; anything else gives NaN, never a loop that does not end.
__global__ void __launch_bounds__(HPF_THREADS) c2pf_edge_expect_kernel(const double* __restrict__ S,
                                                                       const double* __restrict__ R, int64_t n,
                                                                       double* __restrict__ kap, double* __restrict__ L3b)
{
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const double s = S[t], r = R[t];
        kap[t] = __ddiv_rn(s, r);
        if (L3b) L3b[t] = s > 0.0 ? exp(__dsub_rn(hpf_digamma(s), log(r))) : __longlong_as_double(0x7ff8000000000000ll);
    }
}

// Lb_u: a thread per (item, factor), the item's users ascending (CSC), dk through the CSR -> CSC map.
__global__ void __launch_bounds__(HPF_THREADS) c2pf_lbu_kernel(const int32_t* __restrict__ ptr,
                                                               const int32_t* __restrict__ uid,
                                                               const double* __restrict__ val,
                                                               const int32_t* __restrict__ pos,
                                                               const double* __restrict__ dk, int64_t d, int k,
                                                               const double* __restrict__ Lt, double* __restrict__ out)
{
    const int64_t n = d * k;
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const int64_t i = t / k;
        const int f = (int)(t - i * k);
        const int32_t lo = __ldg(ptr + i), hi = __ldg(ptr + i + 1);
        double acc = 0.0;
        int32_t c = lo;
        for (; c + HPF_PASS_BATCH <= hi; c += HPF_PASS_BATCH) {
            double o[HPF_PASS_BATCH], x[HPF_PASS_BATCH], q[HPF_PASS_BATCH];
#pragma unroll
            for (int b = 0; b < HPF_PASS_BATCH; ++b) {
                o[b] = __ldg(Lt + (size_t)__ldg(uid + c + b) * k + f);
                x[b] = __ldg(val + c + b);
                q[b] = __ldg(dk + __ldg(pos + c + b));
            }
#pragma unroll
            for (int b = 0; b < HPF_PASS_BATCH; ++b) acc = __dadd_rn(acc, __ddiv_rn(__dmul_rn(x[b], o[b]), q[b]));
        }
        for (; c < hi; ++c)
            acc = __dadd_rn(acc, __ddiv_rn(__dmul_rn(__ldg(val + c), __ldg(Lt + (size_t)__ldg(uid + c) * k + f)),
                                           __ldg(dk + __ldg(pos + c))));
        out[t] = acc;
    }
}

// Sj[j] = sum_k (L2_r > 0) (L2_s / L2_r) S[k]: a thread per item, the chain over k.
__global__ void __launch_bounds__(HPF_THREADS) c2pf_sj_kernel(int64_t d, int k, const double* __restrict__ L2s,
                                                              const double* __restrict__ L2r,
                                                              const double* __restrict__ S, double* __restrict__ Sj)
{
    for (int64_t j = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; j < d; j += (int64_t)gridDim.x * HPF_THREADS) {
        double acc = 0.0;
        for (int f = 0; f < k; ++f) {
            const double r = L2r[j * k + f];
            if (r > 0.0) acc = __dadd_rn(acc, __dmul_rn(__ddiv_rn(L2s[j * k + f], r), __ldg(S + f)));
        }
        Sj[j] = acc;
    }
}

// Step 1 per edge q = (a, b): L3_s (a chain over k), L3_r, kap = L3_s / L3_r and the new L3b (given: taken from there).
template <bool C2PF>
__global__ void __launch_bounds__(HPF_THREADS) c2pf_kappa_kernel(
    int64_t ne, int k, const int32_t* __restrict__ c_row, const int32_t* __restrict__ c_col,
    const double* __restrict__ L2b, const double* __restrict__ Lbu, const double* __restrict__ Sj,
    const double* __restrict__ util, const double* __restrict__ T3r, double at, double bt, double* __restrict__ L3b,
    const double* __restrict__ given, double* __restrict__ L3s, double* __restrict__ L3r, double* __restrict__ kap)
{
    for (int64_t q = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; q < ne; q += (int64_t)gridDim.x * HPF_THREADS) {
        const int32_t a = __ldg(c_row + q), b = __ldg(c_col + q);
        const double* x = L2b + (size_t)b * k;
        const double* y = Lbu + (size_t)a * k;
        const double e = L3b[q];
        double acc = at;
        int f = 0;
        for (; f + HPF_PASS_BATCH <= k; f += HPF_PASS_BATCH) {
            double xv[HPF_PASS_BATCH], yv[HPF_PASS_BATCH];
#pragma unroll
            for (int u = 0; u < HPF_PASS_BATCH; ++u) xv[u] = __ldg(x + f + u), yv[u] = __ldg(y + f + u);
#pragma unroll
            for (int u = 0; u < HPF_PASS_BATCH; ++u) acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(xv[u], e), yv[u]));
        }
        for (; f < k; ++f) acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(__ldg(x + f), e), __ldg(y + f)));
        const double head = C2PF ? __ddiv_rn(__dmul_rn(at, __dadd_rn(C2PF_A1, __dmul_rn(at, __ldg(util + a)))), T3r[a])
                                 : __ddiv_rn(bt, T3r[a]);
        const double r = __dadd_rn(head, __ldg(Sj + b));
        L3s[q] = acc;
        L3r[q] = r;
        kap[q] = __ddiv_rn(acc, r);
        L3b[q] = given ? given[q]
                       : (acc > 0.0 ? exp(__dsub_rn(hpf_digamma(acc), log(r))) : __longlong_as_double(0x7ff8000000000000ll));
    }
}

// Lb2: a thread per (item, factor), the entries of column i with rows ascending, kappa's expectation at the mirror.
__global__ void __launch_bounds__(HPF_THREADS) c2pf_lb2_kernel(int64_t d, int k, const int32_t* __restrict__ c_ptr,
                                                               const int32_t* __restrict__ c_row,
                                                               const int32_t* __restrict__ c_mir,
                                                               const double* __restrict__ L2b,
                                                               const double* __restrict__ L3b, double* __restrict__ Lb2)
{
    const int64_t n = d * k;
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const int64_t i = t / k;
        const int f = (int)(t - i * k);
        double acc = 0.0;
        for (int32_t p = __ldg(c_ptr + i); p < __ldg(c_ptr + i + 1); ++p)
            acc = __dadd_rn(acc, __dmul_rn(__ldg(L2b + (size_t)__ldg(c_row + p) * k + f), __ldg(L3b + __ldg(c_mir + p))));
        Lb2[t] = acc;
    }
}

// The sum of kap over column i, at the mirrors (c_mir != NULL) or in place; KAPPA_RATE: T3_r[i] = b_t + a_t * sum.
template <bool KAPPA_RATE>
__global__ void __launch_bounds__(HPF_THREADS) c2pf_edge_sum_kernel(int64_t d, const int32_t* __restrict__ c_ptr,
                                                                    const int32_t* __restrict__ c_mir,
                                                                    const double* __restrict__ kap, double at, double bt,
                                                                    double* __restrict__ out)
{
    for (int64_t i = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; i < d; i += (int64_t)gridDim.x * HPF_THREADS) {
        double acc = 0.0;
        for (int32_t p = __ldg(c_ptr + i); p < __ldg(c_ptr + i + 1); ++p)
            acc = __dadd_rn(acc, __ldg(kap + (c_mir ? __ldg(c_mir + p) : p)));
        out[i] = KAPPA_RATE ? __dadd_rn(bt, __dmul_rn(at, acc)) : acc;
    }
}

// The terms of G_r's chain in chain order, a thread per (term, factor).  HAS_L: item i's own term L_s / L_r sits at
// row i + c_ptr[i] and its context entries follow it; all of them are +0.0 when L_r[i,k] <= 0.  Otherwise (rc2pf) the
// chain is the edges alone.
template <bool HAS_L>
__global__ void __launch_bounds__(HPF_THREADS) c2pf_gr_terms_kernel(
    int64_t d, int64_t ne, int k, const int32_t* __restrict__ c_ptr, const int32_t* __restrict__ c_row,
    const int32_t* __restrict__ c_col, const int32_t* __restrict__ c_mir, const double* __restrict__ Ls,
    const double* __restrict__ Lr, const double* __restrict__ L2s, const double* __restrict__ L2r,
    const double* __restrict__ kap, double* __restrict__ T)
{
    const int64_t n = (ne + (HAS_L ? d : 0)) * k;
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const int64_t s = t / k;
        const int f = (int)(t - s * k);
        int64_t dst;
        double v;
        if (!HAS_L || s < ne) {
            const int64_t i = __ldg(c_col + s), r = __ldg(c_row + s);
            v = __dmul_rn(__ddiv_rn(L2s[r * k + f], L2r[r * k + f]), __ldg(kap + __ldg(c_mir + s)));
            if (HAS_L && !(Lr[i * k + f] > 0.0)) v = 0.0;
            dst = HAS_L ? i + 1 + s : s;
        } else {
            const int64_t i = s - ne;
            const double lr = Lr[i * k + f];
            v = lr > 0.0 ? __ddiv_rn(Ls[i * k + f], lr) : 0.0;
            dst = i + __ldg(c_ptr + i);
        }
        T[dst * k + f] = v;
    }
}

// The rates: R[r,f] = 0.3 + S[f], or with Sj 0.3 + Sj[r] S[f] (TIED: (0.3 + S[f]) + Sj[r] S[f]).  Q (may be NULL): the
// guarded quotients shape / R the next column sum adds.
__global__ void __launch_bounds__(HPF_THREADS) c2pf_rate_kernel(int64_t n_rows, int k, const double* __restrict__ S,
                                                                const double* __restrict__ Sj, int tied,
                                                                const double* __restrict__ shape, double* __restrict__ R,
                                                                double* __restrict__ Q)
{
    const int64_t n = n_rows * k;
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const int64_t r = t / k;
        const double s = __ldg(S + (t - r * k));
        double v;
        if (!Sj)
            v = __dadd_rn(C2PF_SHAPE, s);
        else if (tied)
            v = __dadd_rn(__dadd_rn(C2PF_SHAPE, s), __dmul_rn(__ldg(Sj + r), s));
        else
            v = __dadd_rn(C2PF_SHAPE, __dmul_rn(__ldg(Sj + r), s));
        R[t] = v;
        if (Q) Q[t] = v > 0.0 ? __ddiv_rn(shape[t], v) : 0.0;
    }
}

// Step 5: a thread per (context item r, factor): out = (init ? init[r,f] : 0.3) + the chain over column r.
__global__ void __launch_bounds__(HPF_THREADS) c2pf_context_kernel(int64_t d, int k, const int32_t* __restrict__ c_ptr,
                                                                   const int32_t* __restrict__ c_row,
                                                                   const double* __restrict__ L2b,
                                                                   const double* __restrict__ L3b,
                                                                   const double* __restrict__ Lbu, const double* init,
                                                                   double* out)
{
    const int64_t n = d * k;
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const int64_t r = t / k;
        const int f = (int)(t - r * k);
        const double e = L2b[t];
        double acc = init ? init[t] : C2PF_SHAPE;
        for (int32_t p = __ldg(c_ptr + r); p < __ldg(c_ptr + r + 1); ++p)
            acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(e, __ldg(L3b + p)), __ldg(Lbu + (size_t)__ldg(c_row + p) * k + f)));
        out[t] = acc;
    }
}

struct C2pfArgs {
    int variant;
    int64_t n, d;
    int k;
    SparseArgs<double> r;
    int64_t ne;
    const int32_t *c_ptr, *c_row, *c_col, *c_mir;
    const double* util;
    double at, bt;
    double *Gs, *Gr, *Ls, *Lr, *L2s, *L2r, *L3s, *L3r, *T3r;
};

struct C2pfExp {
    double *Lt, *Lb, *L2b, *L3b, *Lb2;
};

struct C2pfWork {
    double *dk, *E, *Lbu, *qG, *S, *S2, *Sg, *Sj, *kap, *T;
    C2pfExp own;                                 // b200_c2pf_fit's expectations
};

int64_t c2pf_work_doubles(int64_t n, int64_t d, int64_t nnz, int64_t ne, int k)
{
    return std::max<int64_t>(nnz, 1) + 2 * std::max<int64_t>(ne, 1) + (2 * n + 5 * d) * k + 3 * (int64_t)k + d +
           (d + ne) * k;
}

C2pfWork c2pf_carve(double* w, int64_t n, int64_t d, int64_t nnz, int64_t ne, int k)
{
    C2pfWork h;
    h.dk = w;
    h.E = h.dk + std::max<int64_t>(nnz, 1);
    h.Lbu = h.E + d * k;
    h.qG = h.Lbu + d * k;
    h.S = h.qG + n * k;
    h.S2 = h.S + k;
    h.Sg = h.S2 + k;
    h.Sj = h.Sg + k;
    h.kap = h.Sj + d;
    h.T = h.kap + std::max<int64_t>(ne, 1);
    h.own.Lt = h.T + (d + ne) * k;
    h.own.Lb = h.own.Lt + n * k;
    h.own.L2b = h.own.Lb + d * k;
    h.own.Lb2 = h.own.L2b + d * k;
    h.own.L3b = h.own.Lb2 + d * k;
    return h;
}

#define C2PF_LAUNCH(kernel, count, ...)                                                                                \
    do {                                                                                                               \
        if ((count) > 0) {                                                                                             \
            kernel<<<hpf_grid(count), HPF_THREADS, 0, st>>>(__VA_ARGS__);                                              \
            count_launch();                                                                                            \
        }                                                                                                              \
    } while (0)

void c2pf_colsum(const double* Q, int64_t n_rows, int k, double* out, cudaStream_t st)
{
    hpf_colsum_kernel<<<(unsigned)((k + 31) / 32), 32, 0, st>>>(Q, n_rows, k, out);
    count_launch();
}

// out = the expectation of (shape, rate), or the given one.
void c2pf_expect(const double* shape, const double* rate, int64_t n, double* out, const double* given, cudaStream_t st)
{
    if (given)
        cudaMemcpyAsync(out, given, sizeof(double) * (size_t)n, cudaMemcpyDeviceToDevice, st);
    else
        hpf_expect(shape, rate, n, out, st);
}

// One iteration from the expectations e, which it replaces; g (entries may be NULL): expectations to take instead of
// computing them.
void c2pf_update(C2pfArgs a, const C2pfExp& e, const C2pfExp& g, const C2pfWork& w, cudaStream_t st)
{
    const int k = a.k;
    const int64_t dk_ = a.d * k, nk = a.n * k;
    const bool has_l = a.variant != 2, tied = a.variant == 1;
    double* L2b = tied ? e.Lb : e.L2b;
    if (tied) a.L2s = a.Ls, a.L2r = a.Lr;
    const double* E = has_l ? w.E : e.Lb2;
    auto item_side = [&] {
        if (has_l) C2PF_LAUNCH(c2pf_add_kernel, dk_, e.Lb, e.Lb2, dk_, w.E);
    };
    auto dk_and_lbu = [&](bool lbu) {
        C2PF_LAUNCH(hpf_dk_kernel, a.r.nnz, a.r.row, a.r.idx, a.r.nnz, k, e.Lt, E, w.dk);
        if (lbu) C2PF_LAUNCH(c2pf_lbu_kernel, dk_, a.r.cptr, a.r.crow, a.r.cval, a.r.cpos, w.dk, a.d, k, e.Lt, w.Lbu);
    };
    // 1. kappa
    item_side();
    dk_and_lbu(true);
    C2PF_LAUNCH(hpf_quotient_kernel, nk, a.Gs, a.Gr, nk, w.qG);
    c2pf_colsum(w.qG, a.n, k, w.S, st);
    C2PF_LAUNCH(c2pf_sj_kernel, a.d, a.d, k, a.L2s, a.L2r, w.S, w.Sj);
    if (a.variant == 0)
        C2PF_LAUNCH(c2pf_kappa_kernel<true>, a.ne, a.ne, k, a.c_row, a.c_col, L2b, w.Lbu, w.Sj, a.util, a.T3r, a.at, a.bt,
                    e.L3b, g.L3b, a.L3s, a.L3r, w.kap);
    else
        C2PF_LAUNCH(c2pf_kappa_kernel<false>, a.ne, a.ne, k, a.c_row, a.c_col, L2b, w.Lbu, w.Sj, a.util, a.T3r, a.at, a.bt,
                    e.L3b, g.L3b, a.L3s, a.L3r, w.kap);
    // 2. the context sums and c2pf's T3_r
    C2PF_LAUNCH(c2pf_lb2_kernel, dk_, a.d, k, a.c_ptr, a.c_row, a.c_mir, L2b, e.L3b, e.Lb2);
    item_side();
    if (a.variant == 0) C2PF_LAUNCH(c2pf_edge_sum_kernel<true>, a.d, a.d, a.c_ptr, a.c_mir, w.kap, a.at, a.bt, a.T3r);
    // 3. the users
    dk_and_lbu(false);
    C2PF_LAUNCH(hpf_pass_kernel<true>, nk, a.r.ptr, a.r.idx, a.r.val, nullptr, w.dk, a.n, k, e.Lt, E, C2PF_SHAPE, a.Gs);
    if (has_l)
        C2PF_LAUNCH(c2pf_gr_terms_kernel<true>, (a.ne + a.d) * k, a.d, a.ne, k, a.c_ptr, a.c_row, a.c_col, a.c_mir, a.Ls,
                    a.Lr, a.L2s, a.L2r, w.kap, w.T);
    else
        C2PF_LAUNCH(c2pf_gr_terms_kernel<false>, a.ne * k, a.d, a.ne, k, a.c_ptr, a.c_row, a.c_col, a.c_mir, a.Ls, a.Lr,
                    a.L2s, a.L2r, w.kap, w.T);
    c2pf_colsum(w.T, a.ne + (has_l ? a.d : 0), k, w.Sg, st);
    C2PF_LAUNCH(c2pf_rate_kernel, nk, a.n, k, w.Sg, nullptr, 0, a.Gs, a.Gr, w.qG);
    c2pf_expect(a.Gs, a.Gr, nk, e.Lt, g.Lt, st);
    c2pf_colsum(w.qG, a.n, k, w.S2, st);
    // 4. the items
    if (has_l) {
        dk_and_lbu(tied);
        C2PF_LAUNCH(hpf_pass_kernel<false>, dk_, a.r.cptr, a.r.crow, a.r.cval, a.r.cpos, w.dk, a.d, k, e.Lb, e.Lt,
                    C2PF_SHAPE, a.Ls);
    }
    if (a.variant == 0) {
        C2PF_LAUNCH(c2pf_rate_kernel, dk_, a.d, k, w.S2, nullptr, 0, nullptr, a.Lr, nullptr);
        c2pf_expect(a.Ls, a.Lr, dk_, e.Lb, g.Lb, st);
        item_side();
    }
    // 5. the context items
    if (!tied) dk_and_lbu(true);
    C2PF_LAUNCH(c2pf_context_kernel, dk_, a.d, k, a.c_ptr, a.c_row, L2b, e.L3b, w.Lbu, tied ? a.Ls : nullptr, a.L2s);
    C2PF_LAUNCH(c2pf_edge_sum_kernel<false>, a.d, a.d, a.c_ptr, nullptr, w.kap, 0.0, 0.0, w.Sj);
    C2PF_LAUNCH(c2pf_rate_kernel, dk_, a.d, k, w.S2, w.Sj, (int)tied, nullptr, a.L2r, nullptr);
    c2pf_expect(a.L2s, a.L2r, dk_, L2b, tied ? g.Lb : g.L2b, st);
    C2PF_LAUNCH(c2pf_lb2_kernel, dk_, a.d, k, a.c_ptr, a.c_row, a.c_mir, L2b, e.L3b, e.Lb2);
}

int c2pf_check(const C2pfArgs& a, const void* work, const char* what)
{
    B200_REQUIRE(a.variant >= 0 && a.variant <= 2, "%s: bad variant %d", what, a.variant);
    if (int rc = sparse_check(a.r, a.n, a.d, what)) return rc;
    B200_REQUIRE(a.k >= 1 && a.ne >= 0 && a.ne < (1ll << 31), "%s: bad sizes k=%d n_edges=%lld", what, a.k,
                 (long long)a.ne);
    const bool has_l = a.variant != 2, has_l2 = a.variant != 1;
    B200_REQUIRE(a.c_ptr && work && (a.n == 0 || (a.Gs && a.Gr)) &&
                     (a.d == 0 || ((!has_l || (a.Ls && a.Lr)) && (!has_l2 || (a.L2s && a.L2r)) && a.T3r && a.util)),
                 "%s: null pointer argument", what);
    B200_REQUIRE(a.ne == 0 || (a.c_row && a.c_col && a.c_mir && a.L3s && a.L3r), "%s: null graph arrays", what);
    return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_c2pf_workspace_bytes(int64_t n_users, int64_t n_items, int64_t nnz, int64_t n_edges, int k)
{
    if (n_users < 0 || n_items < 0 || nnz < 0 || n_edges < 0 || k < 1) return -1;
    return (int64_t)sizeof(double) * c2pf_work_doubles(n_users, n_items, nnz, n_edges, k);
}

#define B200_C2PF_ARGS                                                                                                 \
    C2pfArgs a{variant, n_users, n_items, k, B200_SPARSE_VIEW(r_), n_edges, c_ptr, c_row, c_col, c_mir, util, at, bt,  \
               Gs, Gr, Ls, Lr, L2s, L2r, L3s, L3r, T3r}

extern "C" int b200_c2pf_update(B200_C2PF_PARAMS, double* Lt, double* Lb, double* L2b, double* L3b, double* Lb2,
                                const double* given_Lt, const double* given_Lb, const double* given_L2b,
                                const double* given_L3b, double* work, void* stream)
{
    B200_C2PF_ARGS;
    if (int rc = c2pf_check(a, work, "b200_c2pf_update")) return rc;
    B200_REQUIRE((n_users == 0 || Lt) && (n_items == 0 || ((variant == 2 || Lb) && (variant == 1 || L2b) && Lb2)) &&
                     (n_edges == 0 || L3b),
                 "b200_c2pf_update: null expectation");
    const C2pfExp e{Lt, Lb, L2b, L3b, Lb2};
    const C2pfExp g{const_cast<double*>(given_Lt), const_cast<double*>(given_Lb), const_cast<double*>(given_L2b),
                    const_cast<double*>(given_L3b), nullptr};
    c2pf_update(a, e, g, c2pf_carve(work, n_users, n_items, r_nnz, n_edges, k), (cudaStream_t)stream);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_c2pf_fit(B200_C2PF_PARAMS, int n_iter, double* work, void* stream)
{
    B200_C2PF_ARGS;
    if (int rc = c2pf_check(a, work, "b200_c2pf_fit")) return rc;
    B200_REQUIRE(n_iter >= 0, "b200_c2pf_fit: bad n_iter=%d", n_iter);
    cudaStream_t st = (cudaStream_t)stream;
    const C2pfWork w = c2pf_carve(work, n_users, n_items, r_nnz, n_edges, k);
    const C2pfExp& e = w.own;
    const int64_t dk_ = n_items * k;
    // What a call of the reference does before its loop: (c2pf) T3_r from kappa, the expectations, the context sums.
    // They are the values an iteration leaves, so a fit split into several calls recomputes them bit for bit.
    C2PF_LAUNCH(c2pf_edge_expect_kernel, n_edges, L3s, L3r, n_edges, w.kap, e.L3b);
    if (variant == 0) C2PF_LAUNCH(c2pf_edge_sum_kernel<true>, n_items, n_items, c_ptr, c_mir, w.kap, at, bt, T3r);
    hpf_expect(Gs, Gr, n_users * k, e.Lt, st);
    if (variant != 2) hpf_expect(Ls, Lr, dk_, e.Lb, st);
    if (variant != 1) hpf_expect(L2s, L2r, dk_, e.L2b, st);
    C2PF_LAUNCH(c2pf_lb2_kernel, dk_, n_items, k, c_ptr, c_row, c_mir, variant == 1 ? e.Lb : e.L2b, e.L3b, e.Lb2);
    for (int it = 0; it < n_iter; ++it) c2pf_update(a, e, C2pfExp{}, w, st);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
