// Exact scores and exact top-k for sm_90a (the reproducible reference path of the rank
// side; the tensor-core fused kernel in rank_fused.cu is checked against these).
//
// Replaces fast_dot (reference: cornac/utils/fast_dot.pyx:40-43) as used by BPR.score
// (cornac/models/bpr/recom_bpr.pyx:290-293) / MF.score (cornac/models/mf/recom_mf.py:272-278)
// and the argpartition/argsort of Recommender.rank (cornac/models/recommender.py:521-528).
//
// score_batch_kernel: out[q,i] = (item_base[i] + user_off[q]) + f32( sum_f f64(U[q,f]) * f64(V[i,f]) ),
//   f ascending.  Every f32 x f32 product is exact in f64, so the only rounding is the f64
//   accumulation (fixed order) and the final f64 -> f32 conversion: bit-reproducible.
// topk_rows_kernel: per row, exclusion-aware 4 x 8-bit radix select of the k-th largest
//   key, ordered collection (ties by ascending id), bitonic sort of the k survivors by
//   (score desc, id asc).
#include "common.cuh"

namespace b200 {

constexpr int SC_THREADS = 128;
constexpr int SC_ITEMS = 256;     // items per block (2 per thread)
constexpr int SC_KC = 32;         // factor chunk
constexpr int SC_Q = 8;           // queries per block pass

__global__ void __launch_bounds__(SC_THREADS) score_batch_kernel(
    const float* __restrict__ U, const int64_t* __restrict__ user_idx, int64_t n_q,
    const float* __restrict__ V, int64_t n_items, int k,
    const float* __restrict__ item_base, const float* __restrict__ user_off, float* __restrict__ out,
    float user_off_all = 0.f)
{
    __shared__ float Vs[SC_ITEMS][SC_KC + 1];
    __shared__ double Us[SC_Q][SC_KC];
    __shared__ int64_t urow[SC_Q];
    const int tid = threadIdx.x;
    const int64_t item0 = (int64_t)blockIdx.x * SC_ITEMS;
    const int64_t n_qt = (n_q + SC_Q - 1) / SC_Q;

    for (int64_t qt = blockIdx.y; qt < n_qt; qt += gridDim.y) {
        const int64_t q0 = qt * SC_Q;
        __syncthreads();
        if (tid < SC_Q) {
            const int64_t q = q0 + tid;
            urow[tid] = (q < n_q) ? (user_idx ? user_idx[q] : q) : -1;
        }
        double acc0[SC_Q], acc1[SC_Q];
#pragma unroll
        for (int q = 0; q < SC_Q; ++q) { acc0[q] = 0.0; acc1[q] = 0.0; }

        for (int f0 = 0; f0 < k; f0 += SC_KC) {
            __syncthreads();
            // V chunk: SC_ITEMS x SC_KC, each warp reads 32 consecutive floats of one row
            for (int idx = tid; idx < SC_ITEMS * SC_KC; idx += SC_THREADS) {
                const int it = idx / SC_KC, f = idx % SC_KC;
                const int64_t gi = item0 + it;
                float v = 0.f;
                if (gi < n_items && f0 + f < k) v = __ldg(V + (size_t)gi * k + f0 + f);
                Vs[it][f] = v;
            }
            for (int idx = tid; idx < SC_Q * SC_KC; idx += SC_THREADS) {
                const int q = idx / SC_KC, f = idx % SC_KC;
                float u = 0.f;
                if (urow[q] >= 0 && f0 + f < k) u = __ldg(U + (size_t)urow[q] * k + f0 + f);
                Us[q][f] = (double)u;
            }
            __syncthreads();
#pragma unroll 4
            for (int f = 0; f < SC_KC; ++f) {
                const double v0 = (double)Vs[tid][f], v1 = (double)Vs[tid + SC_THREADS][f];
#pragma unroll
                for (int q = 0; q < SC_Q; ++q) {
                    const double uq = Us[q][f];
                    acc0[q] = fma(uq, v0, acc0[q]);
                    acc1[q] = fma(uq, v1, acc1[q]);
                }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t gi = item0 + tid + h * SC_THREADS;
            if (gi < n_items) {
                const float base = item_base ? __ldg(item_base + gi) : 0.f;
#pragma unroll
                for (int q = 0; q < SC_Q; ++q) {
                    const int64_t gq = q0 + q;
                    if (gq < n_q) {
                        const float uo = user_off ? __ldg(user_off + gq) : user_off_all;
                        const double a = h ? acc1[q] : acc0[q];
                        out[(size_t)gq * n_items + gi] = __fadd_rn(__fadd_rn(base, uo), __double2float_rn(a));
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
constexpr int TK_THREADS = 512;
constexpr int TK_WARPS = TK_THREADS / 32;
constexpr int TK_MAX = 4096;     // largest supported top-k

// Walk one warp's contiguous span of a row in 32-item steps; fn(item_id, key, score, valid) is
// called by every lane each step (valid = in range and not excluded).  The exclusion list
// is sorted, so a warp-uniform cursor makes the membership test O(1) amortised.
template <typename F>
__device__ __forceinline__ void scan_span(const float* __restrict__ row, int64_t n, int64_t span_lo, int64_t span_hi,
                                          const int32_t* __restrict__ excl, int64_t n_excl, F fn)
{
    const int lane = threadIdx.x & 31;
    int64_t c = 0;
    if (n_excl > 0) {   // lower_bound(excl, span_lo)
        int64_t lo = 0, hi = n_excl;
        while (lo < hi) {
            int64_t mid = (lo + hi) >> 1;
            if ((int64_t)__ldg(excl + mid) < span_lo) lo = mid + 1; else hi = mid;
        }
        c = lo;
    }
    for (int64_t base = span_lo; base < span_hi; base += 32) {
        unsigned exmask = 0u;
        while (c < n_excl) {
            const int64_t e = (int64_t)__ldg(excl + c);
            if (e >= base + 32) break;
            if (e >= base) exmask |= 1u << (unsigned)(e - base);
            ++c;
        }
        const int64_t i = base + lane;
        const bool valid = (i < n) && (i < span_hi) && !((exmask >> lane) & 1u);
        const float s = (i < n) ? __ldg(row + i) : 0.f;
        fn(i, float_key(s), s, valid);
    }
}

__global__ void __launch_bounds__(TK_THREADS) topk_rows_kernel(
    const float* __restrict__ scores, int64_t n_q, int64_t n_items,
    const int64_t* __restrict__ excl_indptr, const int32_t* __restrict__ excl_indices,
    int topk, int sort_n, int32_t* __restrict__ out_ids, float* __restrict__ out_scores)
{
    extern __shared__ unsigned long long sort_buf[];   // sort_n entries
    __shared__ unsigned int hist[256];
    __shared__ unsigned int sel_prefix, sel_remaining;
    __shared__ unsigned int w_gt[TK_WARPS], w_eq[TK_WARPS];
    __shared__ unsigned int n_cand_total;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t span = ((n_items + TK_WARPS - 1) / TK_WARPS + 31) / 32 * 32;
    const int64_t span_lo = min((int64_t)warp * span, n_items), span_hi = min(span_lo + span, n_items);

    for (int64_t q = blockIdx.x; q < n_q; q += gridDim.x) {
        const float* row = scores + (size_t)q * n_items;
        const int32_t* excl = nullptr;
        int64_t n_excl = 0;
        if (excl_indptr) {
            const int64_t a = excl_indptr[q], b = excl_indptr[q + 1];
            excl = excl_indices + a;
            n_excl = b - a;
        }
        // ---- number of candidates (row length minus in-range exclusions; duplicates not expected)
        __syncthreads();
        if (tid == 0) n_cand_total = 0;
        __syncthreads();
        {
            unsigned cnt = 0;
            scan_span(row, n_items, span_lo, span_hi, excl, n_excl,
                      [&](int64_t, uint32_t, float, bool valid) { cnt += valid; });
            cnt = __reduce_add_sync(0xffffffffu, cnt);
            if (lane == 0) atomicAdd(&n_cand_total, cnt);
        }
        __syncthreads();
        const unsigned kk = min((unsigned)topk, n_cand_total);

        // ---- radix select of the kk-th largest key, 8 bits per pass from the top
        if (tid == 0) { sel_prefix = 0; sel_remaining = kk; }
        for (int pass = 3; pass >= 0 && kk > 0; --pass) {
            __syncthreads();
            if (tid < 256) hist[tid] = 0;
            __syncthreads();
            const unsigned prefix = sel_prefix;
            const int shift = pass * 8;
            scan_span(row, n_items, span_lo, span_hi, excl, n_excl,
                      [&](int64_t, uint32_t key, float, bool valid) {
                          const bool m = valid && (pass == 3 || (key >> (shift + 8)) == prefix);
                          const unsigned digit = (key >> shift) & 0xffu;
                          // warp-aggregated histogram update
                          const unsigned act = __ballot_sync(0xffffffffu, m);
                          if (m) {
                              const unsigned peers = __match_any_sync(act, digit);
                              if ((int)(__ffs(peers) - 1) == lane) atomicAdd(&hist[digit], (unsigned)__popc(peers));
                          }
                      });
            __syncthreads();
            if (tid == 0) {
                unsigned rem = sel_remaining, cum = 0;
                int d = 255;
                for (; d > 0; --d) {
                    if (cum + hist[d] >= rem) break;
                    cum += hist[d];
                }
                sel_remaining = rem - cum;
                sel_prefix = (prefix << 8) | (unsigned)d;
            }
        }
        __syncthreads();
        const unsigned T = sel_prefix;              // key of the kk-th largest candidate
        const unsigned need_eq = sel_remaining;     // how many == T entries to take (smallest ids)
        const unsigned n_gt = kk - need_eq;

        // ---- per-warp counts, then ordered collection into the sort buffer
        {
            unsigned cg = 0, ce = 0;
            if (kk > 0)
                scan_span(row, n_items, span_lo, span_hi, excl, n_excl,
                          [&](int64_t, uint32_t key, float, bool valid) {
                              cg += (valid && key > T);
                              ce += (valid && key == T);
                          });
            cg = __reduce_add_sync(0xffffffffu, cg);
            ce = __reduce_add_sync(0xffffffffu, ce);
            if (lane == 0) { w_gt[warp] = cg; w_eq[warp] = ce; }
        }
        for (int x = tid; x < sort_n; x += TK_THREADS) sort_buf[x] = 0ull;   // below every real entry
        __syncthreads();
        if (kk > 0) {
            unsigned off_gt = 0, off_eq = 0;
            for (int w = 0; w < warp; ++w) { off_gt += w_gt[w]; off_eq += w_eq[w]; }
            scan_span(row, n_items, span_lo, span_hi, excl, n_excl,
                      [&](int64_t i, uint32_t key, float, bool valid) {
                          const bool gt = valid && key > T, eq = valid && key == T;
                          const unsigned mg = __ballot_sync(0xffffffffu, gt), me = __ballot_sync(0xffffffffu, eq);
                          const unsigned below = (1u << lane) - 1u;
                          // entry = key in the high word, (~id) in the low word: descending 64-bit order
                          // is (score desc, id asc)
                          const unsigned long long ent = ((unsigned long long)key << 32) | (unsigned)(0xffffffffu - (unsigned)i);
                          if (gt) sort_buf[off_gt + __popc(mg & below)] = ent;
                          if (eq) {
                              const unsigned rk = off_eq + __popc(me & below);
                              if (rk < need_eq) sort_buf[n_gt + rk] = ent;
                          }
                          off_gt += __popc(mg);
                          off_eq += __popc(me);
                      });
        }
        __syncthreads();
        // ---- bitonic sort, descending
        for (int size = 2; size <= sort_n; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int x = tid; x < sort_n / 2; x += TK_THREADS) {
                    const int lo = 2 * x - (x & (stride - 1));
                    const int hi = lo + stride;
                    const bool desc = ((lo & size) == 0);
                    const unsigned long long a = sort_buf[lo], b = sort_buf[hi];
                    if ((a < b) == desc) { sort_buf[lo] = b; sort_buf[hi] = a; }
                }
                __syncthreads();
            }
        }
        for (int x = tid; x < topk; x += TK_THREADS) {
            int32_t id = -1;
            float sc = -INFINITY;
            if ((unsigned)x < kk) {
                const unsigned long long ent = sort_buf[x];
                id = (int32_t)(0xffffffffu - (unsigned)(ent & 0xffffffffull));
                sc = __ldg(row + id);
            }
            out_ids[(size_t)q * topk + x] = id;
            out_scores[(size_t)q * topk + x] = sc;
        }
    }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_score_batch(const float* U, const int64_t* user_idx, int64_t n_q,
                                const float* V, int64_t n_items, int k,
                                const float* item_base, const float* user_off,
                                float* out, void* stream)
{
    B200_REQUIRE(U && V && out, "b200_score_batch: null pointer argument");
    B200_REQUIRE(n_q >= 0 && n_items >= 0 && k >= 1, "b200_score_batch: bad sizes n_q=%lld n_items=%lld k=%d",
                 (long long)n_q, (long long)n_items, k);
    if (n_q == 0 || n_items == 0) return B200_OK;
    const int64_t n_it = (n_items + SC_ITEMS - 1) / SC_ITEMS;
    const int64_t n_qt = (n_q + SC_Q - 1) / SC_Q;
    dim3 grid((unsigned)n_it, (unsigned)(n_qt < 65535 ? n_qt : 65535));
    score_batch_kernel<<<grid, SC_THREADS, 0, (cudaStream_t)stream>>>(U, user_idx, n_q, V, n_items, k, item_base, user_off, out); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

// The single-user form of SURVEY 8(b): out = (item_base + user_off) + fast_dot(U[user_idx], V)  -- what one call of
// BPR.score / MF.score computes (recom_bpr.pyx:290-293, mf/recom_mf.py:272-278: user_off = mu + Bu[u]).
extern "C" int b200_score(const float* U, int64_t user_idx, const float* V, int64_t n_items, int k,
                          const float* item_base, float user_off, float* out, void* stream)
{
    B200_REQUIRE(U && V && out, "b200_score: null pointer argument");
    B200_REQUIRE(user_idx >= 0 && n_items >= 0 && k >= 1, "b200_score: bad arguments user_idx=%lld n_items=%lld k=%d",
                 (long long)user_idx, (long long)n_items, k);
    if (n_items == 0) return B200_OK;
    const int64_t n_it = (n_items + SC_ITEMS - 1) / SC_ITEMS;
    dim3 grid((unsigned)n_it, 1u);
    score_batch_kernel<<<grid, SC_THREADS, 0, (cudaStream_t)stream>>>(U + (size_t)user_idx * k, nullptr, 1, V, n_items, k, item_base, nullptr,
                                                                     out, user_off); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_topk_rows(const float* scores, int64_t n_q, int64_t n_items,
                              const int64_t* excl_indptr, const int32_t* excl_indices,
                              int topk, int32_t* out_ids, float* out_scores, void* stream)
{
    B200_REQUIRE(scores && out_ids && out_scores, "b200_topk_rows: null pointer argument");
    B200_REQUIRE(topk >= 1 && topk <= TK_MAX, "b200_topk_rows: topk=%d out of range [1, %d]", topk, TK_MAX);
    B200_REQUIRE(n_q >= 0 && n_items >= 1 && n_items < (1ll << 31), "b200_topk_rows: bad sizes");
    B200_REQUIRE((excl_indptr == nullptr) == (excl_indices == nullptr) || excl_indptr,
                 "b200_topk_rows: excl_indices given without excl_indptr");
    if (n_q == 0) return B200_OK;
    int sort_n = 2;
    while (sort_n < topk) sort_n <<= 1;
    const size_t smem = (size_t)sort_n * sizeof(unsigned long long);
    int64_t grid = (int64_t)sm_count() * 2;
    if (n_q < grid) grid = n_q;
    topk_rows_kernel<<<(unsigned)grid, TK_THREADS, smem, (cudaStream_t)stream>>>(
        scores, n_q, n_items, excl_indptr, excl_indptr ? excl_indices : nullptr, topk, sort_n, out_ids, out_scores); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
