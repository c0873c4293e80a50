// Shared helpers for the sm_90a kernels of the BPR / MF / score+rank hot path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200cornac.h"

namespace b200 {

// ---------------------------------------------------------------------------
// error plumbing: every C-ABI entry returns 0 or a non-zero status; the text
// is kept per thread and returned by b200_last_error().
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define B200_CUDA(call)                                                        \
    do {                                                                       \
        cudaError_t _e = (call);                                               \
        if (_e != cudaSuccess) return ::b200::cuda_fail(_e, #call, __FILE__, __LINE__); \
    } while (0)

#define B200_REQUIRE(cond, ...)                                                \
    do {                                                                       \
        if (!(cond)) {                                                         \
            ::b200::set_error(__VA_ARGS__);                                    \
            return B200_ERR_INVALID;                                           \
        }                                                                      \
    } while (0)

int sm_count();   // cached multiProcessorCount of the current device
void count_launch(int n = 1);   // one tick per kernel this library launches (b200_kernel_launches)

// ---------------------------------------------------------------------------
// Philox4x32-10 counter-based RNG (Salmon et al., SC'11).  Stateless: the
// (u,i,j) triplet of sample s in epoch e is a pure function of (seed, e, s),
// so any grid shape / shard layout draws the same stream.
struct Philox4 {
    uint32_t x, y, z, w;
};

__host__ __device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b)
{
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

__host__ __device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                          uint32_t k0, uint32_t k1)
{
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = mulhi32(M0, c0), lo0 = M0 * c0;
        uint32_t hi1 = mulhi32(M1, c2), lo1 = M1 * c2;
        uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    return Philox4{c0, c1, c2, c3};
}

// unbiased-enough range reduction: floor(r64 * n / 2^64), bias <= n / 2^64
__host__ __device__ __forceinline__ uint64_t range64(uint32_t lo, uint32_t hi, uint64_t n)
{
    uint64_t r = ((uint64_t)hi << 32) | lo;
#ifdef __CUDA_ARCH__
    return __umul64hi(r, n);
#else
    return (uint64_t)(((unsigned __int128)r * n) >> 64);
#endif
}

// ---------------------------------------------------------------------------
// The sample law of the throughput-mode BPR epoch, shared by the kernels and by b200_bpr_draw_host.
// Unblocked (wn = bn = 1): sample s draws i_index uniformly from [0, nnz) and j uniformly from [0, n_neg) -- the
// reference's law (recom_bpr.pyx:237-239).
// Cache-blocked (B200_BPR_BLOCKED): the SAME marginal law -- every interaction is drawn once per epoch in expectation,
// every negative is uniform over all items and independent of the interaction -- but the epoch's nnz samples are
// visited in an order that keeps the rows they touch in the L2: the interaction list (CSR order = grouped by user) is
// cut into `wn` windows and the items into `bn` blocks; the epoch is cut into wn * bn runs of s_sub = ceil(nnz / (wn bn))
// consecutive sample indices; run (w, b) draws its interactions from window w and its negatives from item block
// (b + epoch) % bn.  Every window meets every item block once per epoch, so each user still sees negatives from the whole
// catalogue every epoch; what changes is only the order in which the triplets of an epoch are applied, which Hogwild
// does not define anyway (stratified SGD: Gemulla et al., KDD 2011).
struct SampleLaw {
    int64_t nnz, n_neg;
    int64_t s_sub;          // samples per (window, block) run
    uint32_t wn, bn;        // windows of the interaction list / blocks of the items (1, 1 = unblocked)
    uint32_t epoch_mod_bn;
    int64_t w_base, b_base; // floor(nnz / wn), floor(n_neg / bn): window w = [w w_base + min(w, w_rem), ...) of w_base (+1) entries
    uint32_t w_rem, b_rem;
};

__host__ __device__ __forceinline__ SampleLaw make_law(int64_t nnz, int64_t n_neg, uint32_t wn, uint32_t bn, uint64_t epoch)
{
    SampleLaw L;
    L.nnz = nnz; L.n_neg = n_neg;
    L.wn = wn < 1 ? 1 : wn; L.bn = bn < 1 ? 1 : bn;
    if ((int64_t)L.wn > nnz) L.wn = nnz > 0 ? (uint32_t)nnz : 1;
    if ((int64_t)L.bn > n_neg) L.bn = n_neg > 0 ? (uint32_t)n_neg : 1;
    const int64_t runs = (int64_t)L.wn * L.bn;
    L.s_sub = (nnz + runs - 1) / runs;
    if (L.s_sub < 1) L.s_sub = 1;
    L.epoch_mod_bn = (uint32_t)(epoch % L.bn);
    L.w_base = nnz / L.wn; L.w_rem = (uint32_t)(nnz % L.wn);
    L.b_base = n_neg / L.bn; L.b_rem = (uint32_t)(n_neg % L.bn);
    return L;
}

// ranges [lo, lo + len) the sample with epoch-local index s draws its interaction index and its negative from
__host__ __device__ __forceinline__ void law_ranges(const SampleLaw& L, uint64_t s, int64_t& i_lo, int64_t& i_len,
                                                    int64_t& j_lo, int64_t& j_len)
{
    if (L.wn == 1 && L.bn == 1) { i_lo = 0; i_len = L.nnz; j_lo = 0; j_len = L.n_neg; return; }
    const uint32_t runs = L.wn * L.bn;
    const uint32_t run = (uint32_t)((s / (uint64_t)L.s_sub) % runs);           // the one 64-bit division of the law
    const uint32_t w = run / L.bn;
    uint32_t b = run - w * L.bn + L.epoch_mod_bn;
    if (b >= L.bn) b -= L.bn;
    i_lo = (int64_t)w * L.w_base + (w < L.w_rem ? w : L.w_rem);
    i_len = L.w_base + (w < L.w_rem ? 1 : 0);
    j_lo = (int64_t)b * L.b_base + (b < L.b_rem ? b : L.b_rem);
    j_len = L.b_base + (b < L.b_rem ? 1 : 0);
}

// ---------------------------------------------------------------------------
// sub-warp (G-lane group) sum; G is a power of two <= 32, groups are aligned.  The shuffle
// mask names only the group's own lanes, so groups of one warp may diverge (different trip
// counts, skipped samples) without dead-locking each other.
template <int G>
__device__ __forceinline__ unsigned group_mask()
{
    if constexpr (G >= 32) {
        return 0xffffffffu;
    } else {
        const unsigned lane = threadIdx.x & 31u;
        return ((1u << G) - 1u) << (lane & ~(unsigned)(G - 1));
    }
}
template <int G>
__device__ __forceinline__ float group_sum(float v)
{
    const unsigned m = group_mask<G>();
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(m, v, o);
    return v;
}

// has_non_zero: lower_bound over the sorted CSR row [lo, hi)
__device__ __forceinline__ bool row_contains(const int32_t* __restrict__ indices, int64_t lo, int64_t hi, int32_t col)
{
    const int64_t end = hi;
    while (lo < hi) {
        int64_t mid = lo + ((hi - lo) >> 1);
        int32_t v = __ldg(indices + mid);
        if (v < col) lo = mid + 1; else hi = mid;
    }
    return lo < end && __ldg(indices + lo) == col;
}

// order-preserving float -> uint32 key (larger float => larger key; -0.0 maps to +0.0)
__host__ __device__ __forceinline__ uint32_t float_key(float f)
{
#ifdef __CUDA_ARCH__
    uint32_t b = __float_as_uint(f);
#else
    union { float f; uint32_t u; } cv; cv.f = f; uint32_t b = cv.u;
#endif
    if (b == 0x80000000u) b = 0u;   // -0.0 ties with +0.0, as in a float compare
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

}  // namespace b200
