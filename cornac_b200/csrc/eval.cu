// Top-k ranking metrics of a batch of ranked lists, on the device.
//
// Reference: the body of the per-user loop of `ranking_eval`
// (cornac/eval_methods/base_method.py:169-220) calls `metric.compute(gt_pos, pd_rank)` for every metric;
// for the @k metrics (cornac/metrics/ranking.py:67-123 NDCG, :126-178 NCRR, :240-275 MeasureAtK and its
// subclasses HitRatio / Precision / Recall / FMeasure) only `np.isin(pd_rank[:k], gt_pos)` matters.
// Here: one warp per ranked list; the hit bitmap of the list against the user's sorted test positives is
// built once in shared memory (coalesced id loads, binary search per lane), then every metric reduces a
// prefix of the bitmap.  HBM traffic = the ids (4 B each) + the positives the searches touch; integer work
// except for the final f64 ratios.
#include "common.cuh"

namespace {

constexpr int EV_THREADS = 256;
constexpr int EV_WARPS = EV_THREADS / 32;
constexpr int EV_MAX_TOPK = 4096;
constexpr int EV_MAX_METRICS = 32;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(EV_THREADS)
topk_metrics_kernel(const int32_t* __restrict__ ids, long long n_q, int topk, long long ids_stride,
                    const long long* __restrict__ user_idx, const long long* __restrict__ pos_indptr,
                    const int32_t* __restrict__ pos_indices, const int32_t* __restrict__ kinds,
                    const int32_t* __restrict__ ks, int n_metrics, double* __restrict__ out) {
    extern __shared__ double disc[];                       // [topk] 1/log2(r+2), then per-warp bitmaps
    uint32_t* bitmap = reinterpret_cast<uint32_t*>(disc + topk) + (threadIdx.x >> 5) * ((topk + 31) / 32);
    __shared__ int s_kind[EV_MAX_METRICS], s_k[EV_MAX_METRICS];
    for (int r = threadIdx.x; r < topk; r += EV_THREADS) disc[r] = 1.0 / log2((double)(r + 2));
    if (threadIdx.x < n_metrics) {
        s_kind[threadIdx.x] = kinds[threadIdx.x];
        int k = ks[threadIdx.x];
        s_k[threadIdx.x] = k < topk ? k : topk;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int words = (topk + 31) / 32;
    for (long long q = (long long)blockIdx.x * EV_WARPS + (threadIdx.x >> 5); q < n_q;
         q += (long long)gridDim.x * EV_WARPS) {
        const long long u = user_idx ? user_idx[q] : q;
        const long long lo = pos_indptr[u];
        const int npos = (int)(pos_indptr[u + 1] - lo);
        const int32_t* pos = pos_indices + lo;
        for (int w = 0; w < words; ++w) {
            int r = w * 32 + lane;
            int id = r < topk ? ids[q * ids_stride + r] : -1;
            bool hit = false;
            if (id >= 0) {
                int a = 0, b = npos;                       // lower bound in the sorted positives
                while (a < b) {
                    int m = (a + b) >> 1;
                    if (pos[m] < id) a = m + 1; else b = m;
                }
                hit = a < npos && pos[a] == id;
            }
            uint32_t bits = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) bitmap[w] = bits;
        }
        __syncwarp();
        for (int m = 0; m < n_metrics; ++m) {
            const int kind = s_kind[m], k = s_k[m];
            const int k_nominal = ks[m];                   // tp_fp uses the requested k (ranking.py:272)
            int tp = 0;
            double dcg = 0.0, crr = 0.0;
            for (int r = lane; r < k; r += 32) {
                if ((bitmap[r >> 5] >> (r & 31)) & 1u) {
                    ++tp;
                    dcg += disc[r];
                    crr += 1.0 / (double)(r + 1);
                }
            }
            tp = __reduce_add_sync(0xffffffffu, tp);
            double val = 0.0;
            if (kind == B200_METRIC_NDCG || kind == B200_METRIC_NCRR) {
                const bool nd = kind == B200_METRIC_NDCG;
                double num = warp_sum(nd ? dcg : crr);
                int ideal = npos < k ? npos : k;
                double den = 0.0;
                for (int r = lane; r < ideal; r += 32) den += nd ? disc[r] : 1.0 / (double)(r + 1);
                den = warp_sum(den);
                val = num / den;                           // npos >= 1 is the caller's contract (base_method.py:180)
            } else {
                double prec = (double)tp / (double)k_nominal;
                double rec = (double)tp / (double)npos;
                if (kind == B200_METRIC_PRECISION) val = prec;
                else if (kind == B200_METRIC_RECALL) val = rec;
                else if (kind == B200_METRIC_HIT) val = tp > 0 ? 1.0 : 0.0;
                else val = (prec + rec) > 0.0 ? 2.0 * prec * rec / (prec + rec) : 0.0;   // ranking.py FMeasure
            }
            if (lane == 0) out[(long long)m * n_q + q] = val;
        }
        __syncwarp();
    }
}

}  // namespace

extern "C" int b200_topk_metrics(const int32_t* ids, int64_t n_q, int topk, int64_t ids_stride,
                                 const int64_t* user_idx, const int64_t* pos_indptr, const int32_t* pos_indices,
                                 const int32_t* metric_kind, const int32_t* metric_k, int n_metrics,
                                 double* out, void* stream) {
    B200_REQUIRE(ids && pos_indptr && pos_indices && metric_kind && metric_k && out, "null pointer");
    B200_REQUIRE(topk >= 1 && topk <= EV_MAX_TOPK, "topk out of range [1, 4096]");
    B200_REQUIRE(n_metrics >= 1 && n_metrics <= EV_MAX_METRICS, "n_metrics out of range [1, 32]");
    B200_REQUIRE(ids_stride >= topk, "ids_stride < topk");
    if (n_q == 0) return 0;
    const int sms = ::b200::sm_count();
    size_t smem = (size_t)topk * sizeof(double) + (size_t)EV_WARPS * ((topk + 31) / 32) * sizeof(uint32_t);
    long long blocks = (n_q + EV_WARPS - 1) / EV_WARPS;
    long long cap = (long long)sms * 8;
    if (blocks > cap) blocks = cap;
    topk_metrics_kernel<<<(unsigned)blocks, EV_THREADS, smem, (cudaStream_t)stream>>>(
        ids, (long long)n_q, topk, (long long)ids_stride, (const long long*)user_idx,
        (const long long*)pos_indptr, pos_indices, metric_kind, metric_k, n_metrics, out); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
// Full-vector ranking metrics (AUC, MAP, MRR): cornac/metrics/ranking.py:473-485 (AUC = sum_p #{n : s_p > s_n} /
// (|P| |N|)), :522-525 (AP = mean_p L_p / rank_p with rankdata(-scores, "max")) and :213-222 (MRR = 1 / position of the
// first positive of the ranked list).  All three only need, per test positive p of a user, HOW MANY CANDIDATES SCORE
// BELOW IT -- not the sorted list: one block per user sorts the user's (few) positive scores in shared memory, then
// streams the score row once; every candidate does one binary search among the positives and bumps one counter; prefix
// sums of the counters are the "less than" counts.  Excluded items (the user's seen items) are blanked to NaN first, so
// they compare false everywhere.  Integer output; the ratios are formed by the caller in f64 like the reference.
namespace {

constexpr int FC_THREADS = 256;
constexpr int FC_TILE = 1024;                 // positives per pass (shared memory)

__global__ void __launch_bounds__(FC_THREADS)
blank_excluded_kernel(float* __restrict__ scores, long long n_q, long long n_items, const long long* __restrict__ excl_indptr,
                      const int32_t* __restrict__ excl_indices)
{
    for (long long q = blockIdx.x; q < n_q; q += gridDim.x) {
        const long long lo = excl_indptr[q], hi = excl_indptr[q + 1];
        for (long long e = lo + threadIdx.x; e < hi; e += FC_THREADS) {
            const int32_t i = excl_indices[e];
            if (i >= 0 && i < n_items) scores[q * n_items + i] = __int_as_float(0x7fc00000);
        }
    }
}

__global__ void __launch_bounds__(FC_THREADS)
rank_counts_kernel(const float* __restrict__ scores, long long n_q, long long n_items, const long long* __restrict__ user_idx,
                   const long long* __restrict__ pos_indptr, const int32_t* __restrict__ pos_indices,
                   long long* __restrict__ less_out, float* __restrict__ pos_score_out, long long* __restrict__ n_cand_out,
                   long long* __restrict__ before_first_out)
{
    __shared__ float sp[FC_TILE];             // positive scores of the current pass, ascending
    __shared__ int sidx[FC_TILE];             // their positions in the user's positives row
    __shared__ unsigned int hist[FC_TILE + 1];
    __shared__ unsigned long long red[FC_THREADS / 32][3];
    __shared__ float best_s;
    __shared__ int best_id;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (long long q = blockIdx.x; q < n_q; q += gridDim.x) {
        const float* row = scores + q * n_items;
        const long long u = user_idx ? user_idx[q] : q;
        const long long plo = pos_indptr[u];
        const int npos = (int)(pos_indptr[u + 1] - plo);
        const int32_t* pos = pos_indices + plo;
        // the positive that leads the ranked list: largest score, smallest id among equals (total order of rank())
        if (tid == 0) {
            float bs = -INFINITY; int bi = 0x7fffffff;
            for (int t = 0; t < npos; ++t) {
                const float s = row[pos[t]];
                if (s > bs || (s == bs && pos[t] < bi) || (t == 0)) { bs = s; bi = pos[t]; }
            }
            best_s = bs; best_id = bi;
        }
        __syncthreads();
        const float bsc = best_s;
        const int bid = best_id;
        for (int p0 = 0; p0 < (npos > 0 ? npos : 1); p0 += FC_TILE) {
            const int np = min(FC_TILE, npos - p0);
            // load + bitonic sort of this pass's positives, ascending by (float_key(score), position): a total order, also
            // for +inf and NaN scores.  Padding = (the NaN of the largest key, INT_MAX) sorts after every positive, so the
            // first np entries are exactly the pass's positives
            for (int t = tid; t < FC_TILE; t += FC_THREADS) {
                sp[t] = t < np ? row[pos[p0 + t]] : __int_as_float(0x7fffffff);
                sidx[t] = t < np ? p0 + t : 0x7fffffff;
            }
            for (int t = tid; t <= FC_TILE; t += FC_THREADS) hist[t] = 0;
            __syncthreads();
            int n2 = 2;
            while (n2 < np) n2 <<= 1;
            for (int size = 2; size <= n2; size <<= 1) {
                for (int stride = size >> 1; stride > 0; stride >>= 1) {
                    for (int x = tid; x < n2 / 2; x += FC_THREADS) {
                        const int lo = 2 * x - (x & (stride - 1));
                        const int hi = lo + stride;
                        const bool asc = ((lo & size) == 0);
                        const float a = sp[lo], b = sp[hi];
                        const int ia = sidx[lo], ib = sidx[hi];
                        const unsigned long long ka = ((unsigned long long)::b200::float_key(a) << 32) | (unsigned)ia;
                        const unsigned long long kb = ((unsigned long long)::b200::float_key(b) << 32) | (unsigned)ib;
                        if ((ka > kb) == asc) {
                            sp[lo] = b; sp[hi] = a;
                            sidx[lo] = ib; sidx[hi] = ia;
                        }
                    }
                    __syncthreads();
                }
            }
            // stream the candidates: hist[j] += 1 with j = first position whose positive scores ABOVE the candidate
            unsigned long long below_all = 0, ncand = 0, before = 0;
            for (long long c = tid; c < n_items; c += FC_THREADS) {
                const float s = row[c];
                if (s != s) continue;                               // excluded (NaN)
                ++ncand;
                before += (s > bsc) || (s == bsc && c < (long long)bid);
                int a = 0, b = np;                                  // upper bound: first t with sp[t] > s
                while (a < b) {
                    const int m = (a + b) >> 1;
                    if (sp[m] > s) b = m; else a = m + 1;
                }
                if (a == 0) ++below_all; else atomicAdd(&hist[a], 1u);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                below_all += __shfl_xor_sync(0xffffffffu, below_all, o);
                ncand += __shfl_xor_sync(0xffffffffu, ncand, o);
                before += __shfl_xor_sync(0xffffffffu, before, o);
            }
            if (lane == 0) { red[warp][0] = below_all; red[warp][1] = ncand; red[warp][2] = before; }
            __syncthreads();
            if (tid == 0) {
                unsigned long long t0 = 0, t1 = 0, t2 = 0;
                for (int w = 0; w < FC_THREADS / 32; ++w) { t0 += red[w][0]; t1 += red[w][1]; t2 += red[w][2]; }
                // serial prefix over the pass's positives (<= 1024): candidates scoring below sp[t]
                unsigned long long acc = t0;
                for (int t = 0; t < np; ++t) {
                    acc += hist[t];                                  // hist[0] stays 0 (counted in below_all)
                    less_out[plo + sidx[t]] = (long long)acc;
                    pos_score_out[plo + sidx[t]] = sp[t];
                }
                if (p0 == 0) { n_cand_out[q] = (long long)t1; before_first_out[q] = (long long)t2; }
            }
            __syncthreads();
        }
    }
}

}  // namespace

extern "C" int b200_rank_counts(float* scores, int64_t n_q, int64_t n_items,
                                const int64_t* excl_indptr, const int32_t* excl_indices,
                                const int64_t* user_idx, const int64_t* pos_indptr, const int32_t* pos_indices,
                                int64_t* less, float* pos_score, int64_t* n_cand, int64_t* before_first, void* stream) {
    B200_REQUIRE(scores && pos_indptr && pos_indices && less && pos_score && n_cand && before_first, "b200_rank_counts: null pointer");
    B200_REQUIRE(n_q >= 0 && n_items >= 1, "b200_rank_counts: bad sizes");
    if (n_q == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const long long cap = (long long)::b200::sm_count() * 8;
    const unsigned grid = (unsigned)(n_q < cap ? n_q : cap);
    if (excl_indptr) {
        B200_REQUIRE(excl_indices != nullptr, "b200_rank_counts: excl_indices missing");
        blank_excluded_kernel<<<grid, FC_THREADS, 0, st>>>(scores, (long long)n_q, (long long)n_items,
                                                           (const long long*)excl_indptr, excl_indices); ::b200::count_launch();
    }
    rank_counts_kernel<<<grid, FC_THREADS, 0, st>>>(scores, (long long)n_q, (long long)n_items, (const long long*)user_idx,
                                                    (const long long*)pos_indptr, pos_indices, (long long*)less, pos_score,
                                                    (long long*)n_cand, (long long*)before_first); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return 0;
}
