// The pieces of the HPF / PF fit (hpf.cu) that the C2PF fit (c2pf.cu) shares: the Cephes digamma, the expectation
// exp(digamma(shape) - log(rate)) with the stored-entry rules, the guarded quotients, dk per rating, the ordered per-row
// pass over the ratings and the ordered column sum.  Every operation is an explicitly rounded __d*_rn intrinsic, so each
// kernel is a fixed function of its inputs in whichever file it is compiled.
#pragma once
#include "common.cuh"

#include <algorithm>

namespace b200 {
namespace {

constexpr int HPF_THREADS = 256;
constexpr int HPF_COLSUM_UNROLL = 8;
constexpr int HPF_PASS_BATCH = 8;
constexpr double HPF_DK_EPS = 0x1p-52;          // pow(2, -52), cpp_hpf.cpp:43
constexpr double HPF_A = 0.3;                   // a_ (HPF and PF)
constexpr double HPF_B = 0.3;                   // HPF b_, PF c_: the item-side shape

// psi(x) for x > 0 (the rules of step 1 never pass anything else): the recurrence psi(x) = psi(x + 1) - 1/x up to
// s >= 10, then the asymptotic series log(s) - 1/(2s) - sum_k B_2k / (2k s^2k) with its seven Bernoulli terms in Horner
// form, as the Cephes `psi` routine evaluates it.
__device__ __forceinline__ double hpf_digamma(double x)
{
    double s = x, w = 0.0;
    while (s < 10.0) {
        w = __dadd_rn(w, __ddiv_rn(1.0, s));
        s = __dadd_rn(s, 1.0);
    }
    double y = 0.0;
    if (s < 1e17) {
        const double z = __ddiv_rn(1.0, __dmul_rn(s, s));
        double p = 1.0 / 12.0;                                  // B_14 / 14
        p = __dadd_rn(__dmul_rn(p, z), -691.0 / 32760.0);        // B_12 / 12
        p = __dadd_rn(__dmul_rn(p, z), 1.0 / 132.0);             // B_10 / 10
        p = __dadd_rn(__dmul_rn(p, z), -1.0 / 240.0);            // B_8 / 8
        p = __dadd_rn(__dmul_rn(p, z), 1.0 / 252.0);             // B_6 / 6
        p = __dadd_rn(__dmul_rn(p, z), -1.0 / 120.0);            // B_4 / 4
        p = __dadd_rn(__dmul_rn(p, z), 1.0 / 12.0);              // B_2 / 2
        y = __dmul_rn(z, p);
    }
    return __dsub_rn(__dsub_rn(__dsub_rn(log(s), __ddiv_rn(0.5, s)), y), w);
}

// Step 1: out = exp(digamma(shape) - log(rate)) with the stored-entry rules.
__global__ void __launch_bounds__(HPF_THREADS) hpf_expect_kernel(const double* __restrict__ shape,
                                                                 const double* __restrict__ rate, int64_t n,
                                                                 double* __restrict__ out)
{
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const double s = shape[t], r = rate[t];
        const bool hs = s > 0.0, hr = r > 0.0;
        double v = 0.0;
        if (hs || hr) {
            double e = hs ? hpf_digamma(s) : 0.0;
            if (hr) e = __dsub_rn(e, log(r));
            v = exp(e);
        }
        out[t] = v;
    }
}

// Q = R > 0 ? S / R : +0.0, the quotients the column sums add.
__global__ void __launch_bounds__(HPF_THREADS) hpf_quotient_kernel(const double* __restrict__ S,
                                                                   const double* __restrict__ R, int64_t n,
                                                                   double* __restrict__ Q)
{
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const double r = R[t];
        Q[t] = r > 0.0 ? __ddiv_rn(S[t], r) : 0.0;
    }
}

// Step 2: a thread per rating (CSR order).
__global__ void __launch_bounds__(HPF_THREADS) hpf_dk_kernel(const int32_t* __restrict__ row,
                                                             const int32_t* __restrict__ col, int64_t nnz, int k,
                                                             const double* __restrict__ Lt,
                                                             const double* __restrict__ Lb, double* __restrict__ dk)
{
    for (int64_t j = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; j < nnz; j += (int64_t)gridDim.x * HPF_THREADS) {
        const double* a = Lt + (size_t)__ldg(row + j) * k;
        const double* b = Lb + (size_t)__ldg(col + j) * k;
        double d = HPF_DK_EPS;
        for (int f = 0; f < k; ++f) d = __dadd_rn(d, __dmul_rn(__ldg(a + f), __ldg(b + f)));
        dk[j] = d;
    }
}

// Steps 3 and 5: a thread per (row, factor) of the side being updated.  Row r's entries are [ptr[r], ptr[r+1]); entry c
// pairs r with row oid[c] of the other side, has rating val[c] and its dk at dk[pos ? pos[c] : c].  USER_SIDE: the
// product is own[r,f] * other[o,f] (Lt * Lb); otherwise other[o,f] * own[r,f] (again Lt * Lb).
template <bool USER_SIDE>
__global__ void __launch_bounds__(HPF_THREADS) hpf_pass_kernel(const int32_t* __restrict__ ptr,
                                                               const int32_t* __restrict__ oid,
                                                               const double* __restrict__ val,
                                                               const int32_t* __restrict__ pos,
                                                               const double* __restrict__ dk, int64_t n_rows, int k,
                                                               const double* __restrict__ own,
                                                               const double* __restrict__ other, double shape0,
                                                               double* __restrict__ out)
{
    const int64_t n = n_rows * k;
    for (int64_t t = (int64_t)blockIdx.x * HPF_THREADS + threadIdx.x; t < n; t += (int64_t)gridDim.x * HPF_THREADS) {
        const int64_t r = t / k;
        const int f = (int)(t - r * k);
        const double e = __ldg(own + t);
        const int32_t lo = __ldg(ptr + r), hi = __ldg(ptr + r + 1);
        auto term = [&](double o, double x, double d) {
            const double p = USER_SIDE ? __dmul_rn(e, o) : __dmul_rn(o, e);
            return __ddiv_rn(__dmul_rn(p, x), d);
        };
        double acc = shape0;
        int32_t c = lo;
        // the gathers of HPF_PASS_BATCH entries are issued together (the division's slow path is a call the compiler
        // does not schedule loads across), then the terms are added in entry order
        for (; c + HPF_PASS_BATCH <= hi; c += HPF_PASS_BATCH) {
            double o[HPF_PASS_BATCH], x[HPF_PASS_BATCH], d[HPF_PASS_BATCH];
#pragma unroll
            for (int q = 0; q < HPF_PASS_BATCH; ++q) {
                o[q] = __ldg(other + (size_t)__ldg(oid + c + q) * k + f);
                x[q] = __ldg(val + c + q);
                d[q] = __ldg(dk + (pos ? __ldg(pos + c + q) : c + q));
            }
#pragma unroll
            for (int q = 0; q < HPF_PASS_BATCH; ++q) acc = __dadd_rn(acc, term(o[q], x[q], d[q]));
        }
        for (; c < hi; ++c)
            acc = __dadd_rn(acc, term(__ldg(other + (size_t)__ldg(oid + c) * k + f), __ldg(val + c),
                                      __ldg(dk + (pos ? __ldg(pos + c) : c))));
        out[t] = acc;
    }
}

// Steps 4 and 6, the column sums: a thread per factor, one sequential chain over the rows.  The loads run ahead of the
// chain in groups of HPF_COLSUM_UNROLL rows; the adds stay in row order.
__global__ void __launch_bounds__(32) hpf_colsum_kernel(const double* __restrict__ Q, int64_t n_rows, int k,
                                                        double* __restrict__ out)
{
    const int f = blockIdx.x * 32 + threadIdx.x;
    if (f >= k) return;
    double acc = 0.0;
    int64_t r = 0;
    for (; r + HPF_COLSUM_UNROLL <= n_rows; r += HPF_COLSUM_UNROLL) {
        double q[HPF_COLSUM_UNROLL];
#pragma unroll
        for (int u = 0; u < HPF_COLSUM_UNROLL; ++u) q[u] = __ldg(Q + (size_t)(r + u) * k + f);
#pragma unroll
        for (int u = 0; u < HPF_COLSUM_UNROLL; ++u) acc = __dadd_rn(acc, q[u]);
    }
    for (; r < n_rows; ++r) acc = __dadd_rn(acc, __ldg(Q + (size_t)r * k + f));
    out[f] = acc;
}

unsigned hpf_grid(int64_t n)
{
    const int64_t cap = (int64_t)sm_count() * 16;
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>(cap, (n + HPF_THREADS - 1) / HPF_THREADS));
}

void hpf_expect(const double* shape, const double* rate, int64_t n, double* out, cudaStream_t st)
{
    if (n == 0) return;
    hpf_expect_kernel<<<hpf_grid(n), HPF_THREADS, 0, st>>>(shape, rate, n, out);
    count_launch();
}

}  // namespace
}  // namespace b200
