// K7: neighbourhood models (UserKNN / ItemKNN).  Dense f64 similarity of the rows of a weight matrix, its compaction
// into CSR, and the top-k neighbour score rows.
//
// Similarity (restates compute_similarity, cornac/models/knn/similarity.pyx:51-105): for row r and every stored (c, w_rc)
// of r in stored order, for every stored (x, w_xc) of column c in ascending x:
//     S[r,x] += w_xc * w_rc;   if (w_rc != 0 && w_xc != 0) { D1[r,x] += w_rc^2; D2[r,x] += w_xc^2; }
// then S[r,x] /= sqrt(D1 * D2) where S[r,x] != 0 -- the compiled reference (-O3 -ffast-math, no FMA) evaluates
// sqrt(D1) * sqrt(D2) as sqrt(D1 * D2), see DESIGN.md section 1.  Each S[r,x] is therefore an ordered sum over the
// columns r and x share; the kernel keeps that order (one barrier between consecutive columns, no atomics) and rounds
// every product and sum separately, so the result is bit-identical to the compiled reference.  The terms of S[x,r] are
// those of S[r,x] in the same order, so only x >= r is computed and the lower triangle is mirrored.
//
// Scores (restate compute_score / compute_score_single, similarity.pyx:109-201 with SparseNeighbors / TopK,
// similarity.h:15-89): the candidates (weight, value) of one (user, item) are visited in descending neighbour index;
// the first k are kept, later ones only when weight > the smallest kept weight, replacing the smallest kept
// (weight, value) pair.  score = mean[u] + sum(w v) / (sum |w| + 1e-8).
#include "common.cuh"

namespace b200 {
namespace knn {

constexpr int SIM_THREADS = 256;
constexpr int SIM_WS_CTAS = 264;              // CTAs of the similarity pass when its accumulators live in the workspace
constexpr int SCORE_WS_CTAS = 264;            // same for the score pass
constexpr int SCORE_WS_THREADS = 128;
constexpr size_t SMEM_LIMIT = 220 * 1024;
constexpr size_t STAGE_LIMIT = 96 * 1024;     // UserKNN: largest similarity row staged in shared memory

__device__ __forceinline__ double amplify_map(double s, double alpha)
{
    return s > 0.0 ? pow(s, alpha) : -pow(-s, alpha);
}

// one CTA per row r (persistent, rows in `order`); acc = S, D1, D2 for x in [r, n), in shared memory or the workspace
__global__ void __launch_bounds__(SIM_THREADS) knn_sim_kernel(
    int n, const int32_t* __restrict__ rp, const int32_t* __restrict__ ri, const double* __restrict__ rd,
    const int32_t* __restrict__ cp, const int32_t* __restrict__ ci, const double* __restrict__ cd,
    const int32_t* __restrict__ order, double alpha, double* ws, double* __restrict__ out)
{
    extern __shared__ double smem[];
    double* S = ws ? ws + (size_t)blockIdx.x * 3 * n : smem;
    double* D1 = S + n;
    double* D2 = D1 + n;
    const int tid = threadIdx.x;
    for (int t = blockIdx.x; t < n; t += gridDim.x) {
        const int r = __ldg(order + t);
        const int m = n - r;
        for (int x = tid; x < m; x += SIM_THREADS) S[x] = D1[x] = D2[x] = 0.0;
        __syncthreads();
        const int pe = __ldg(rp + r + 1);
        for (int p = __ldg(rp + r); p < pe; ++p) {
            const int c = __ldg(ri + p);
            const double w = __ldg(rd + p);
            const double ww = __dmul_rn(w, w);
            int lo = __ldg(cp + c), hi = __ldg(cp + c + 1);
            const int e = hi;
            while (lo < hi) {                                   // first entry of column c with x >= r
                const int mid = (lo + hi) >> 1;
                if (__ldg(ci + mid) < r) lo = mid + 1; else hi = mid;
            }
            for (int j = lo + tid; j < e; j += SIM_THREADS) {   // distinct x within one column: no conflicts
                const int x = __ldg(ci + j) - r;
                const double v = __ldg(cd + j);
                S[x] = __dadd_rn(S[x], __dmul_rn(v, w));
                if (w != 0.0 && v != 0.0) {
                    D1[x] = __dadd_rn(D1[x], ww);
                    D2[x] = __dadd_rn(D2[x], __dmul_rn(v, v));
                }
            }
            __syncthreads();                                    // column c's terms land before column c+1's
        }
        double* row = out + (size_t)r * n + r;
        for (int x = tid; x < m; x += SIM_THREADS) {
            double s = S[x];
            if (s != 0.0) {
                s = __ddiv_rn(s, __dsqrt_rn(__dmul_rn(D1[x], D2[x])));
                if (alpha != 1.0) s = amplify_map(s, alpha);
            }
            row[x] = s;
        }
        __syncthreads();
    }
}

// out[x][r] = out[r][x] for x > r, 32x32 tiles at or below the diagonal
__global__ void knn_mirror_kernel(int n, double* out)
{
    __shared__ double tile[32][33];
    const int R = blockIdx.y, C = blockIdx.x;
    if (R < C) return;
    const int tx = threadIdx.x;
    for (int ty = threadIdx.y; ty < 32; ty += blockDim.y) {
        const int row = C * 32 + ty, col = R * 32 + tx;
        if (row < n && col < n) tile[ty][tx] = out[(size_t)row * n + col];
    }
    __syncthreads();
    for (int ty = threadIdx.y; ty < 32; ty += blockDim.y) {
        const int row = R * 32 + ty, col = C * 32 + tx;
        if (row < n && col < n && row > col) out[(size_t)row * n + col] = tile[tx][ty];
    }
}

__global__ void knn_row_nnz_kernel(int n, const double* __restrict__ S, int32_t* __restrict__ counts)
{
    for (int r = blockIdx.x; r < n; r += gridDim.x) {
        const double* row = S + (size_t)r * n;
        int total = 0;
        for (int x0 = 0; x0 < n; x0 += blockDim.x) {
            const int x = x0 + threadIdx.x;
            total += __syncthreads_count(x < n && row[x] != 0.0);
        }
        if (threadIdx.x == 0) counts[r] = total;
    }
}

// ordered compaction of row r into [indptr[r], indptr[r+1]); blockDim.x == 256
__global__ void __launch_bounds__(256) knn_compact_kernel(int n, const double* __restrict__ S, const int32_t* __restrict__ indptr,
                                                          int32_t* __restrict__ indices, double* __restrict__ data)
{
    __shared__ int warp_tot[8];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int r = blockIdx.x; r < n; r += gridDim.x) {
        const double* row = S + (size_t)r * n;
        int base = indptr[r];
        for (int x0 = 0; x0 < n; x0 += 256) {
            const int x = x0 + threadIdx.x;
            const double s = x < n ? row[x] : 0.0;
            const unsigned b = __ballot_sync(0xffffffffu, s != 0.0);
            if (lane == 0) warp_tot[wid] = __popc(b);
            __syncthreads();
            int off = base + __popc(b & ((1u << lane) - 1u)), tot = 0;
            for (int w = 0; w < 8; ++w) {
                const int c = warp_tot[w];
                if (w < wid) off += c;
                tot += c;
            }
            if (s != 0.0) {
                indices[off] = x;
                data[off] = s;
            }
            base += tot;
            __syncthreads();
        }
    }
}

// ---- neighbour selection: one thread per (user, item) stream; its kept pairs at kw[s * stride], kv[s * stride] ----
struct Kept {
    double* w;
    double* v;
    int stride, k, cnt, pos;   // pos: slot of the smallest kept pair (valid once cnt == k)
    double mw, mv;

    __device__ __forceinline__ void find_min()
    {
        pos = 0;
        mw = w[0];
        mv = v[0];
        for (int s = 1; s < k; ++s) {
            const double a = w[(size_t)s * stride], b = v[(size_t)s * stride];
            if (a < mw || (a == mw && b < mv)) { pos = s; mw = a; mv = b; }
        }
    }
    __device__ __forceinline__ void offer(double a, double b)
    {
        if (cnt < k) {
            w[(size_t)cnt * stride] = a;
            v[(size_t)cnt * stride] = b;
            if (++cnt == k) find_min();
        } else if (a > mw) {
            w[(size_t)pos * stride] = a;
            v[(size_t)pos * stride] = b;
            find_min();
        }
    }
    __device__ __forceinline__ void sum(double& num, double& den) const
    {
        for (int s = 0; s < cnt; ++s) {
            const double a = w[(size_t)s * stride];
            num = __dadd_rn(num, __dmul_rn(a, v[(size_t)s * stride]));
            den = __dadd_rn(den, fabs(a));
        }
    }
};

__device__ __forceinline__ double finish(double mean, double num, double den)
{
    return __dadd_rn(mean, __ddiv_rn(num, __dadd_rn(den, 1e-8)));
}

// ItemKNN: candidates of (u, i) are the items j rated by u (ui[u,j] != 0) with S[j,i] != 0, in descending j.
// Every thread walks the same rating row, so S[j, i0 .. i0+T) is read coalesced (S is symmetric).
__global__ void knn_score_items_kernel(const int64_t* __restrict__ users, int64_t n_q, int n_items,
                                       const int32_t* __restrict__ ui_ptr, const int32_t* __restrict__ ui_idx,
                                       const double* __restrict__ ui_val, const double* __restrict__ S,
                                       const double* __restrict__ mean, int k, double* ws, double* __restrict__ out)
{
    extern __shared__ double smem[];
    const int T = blockDim.x;
    double* kw = ws ? ws + (size_t)blockIdx.x * 2 * k * T : smem;
    Kept kept;
    kept.w = kw + threadIdx.x;
    kept.v = kw + (size_t)k * T + threadIdx.x;
    kept.stride = T;
    kept.k = k;
    for (int64_t q = blockIdx.x; q < n_q; q += gridDim.x) {
        const int64_t u = users[q];
        const int b = ui_ptr[u], e = ui_ptr[u + 1];
        const bool all = e - b <= k;                              // every candidate is kept: sum as we go
        const double mu = mean[u];
        for (int i = threadIdx.x; i < n_items; i += T) {
            double num = 0.0, den = 0.0;
            kept.cnt = 0;
            for (int p = e - 1; p >= b; --p) {
                const double val = __ldg(ui_val + p);
                if (val == 0.0) continue;
                const double wt = __ldg(S + (size_t)__ldg(ui_idx + p) * n_items + i);
                if (wt == 0.0) continue;
                if (all) {
                    num = __dadd_rn(num, __dmul_rn(wt, val));
                    den = __dadd_rn(den, fabs(wt));
                } else {
                    kept.offer(wt, val);
                }
            }
            if (!all) kept.sum(num, den);
            out[q * n_items + i] = finish(mu, num, den);
        }
    }
}

// UserKNN: candidates of (u, i) are the users v who rated i (row i of the item-user matrix) with S[u,v] != 0, in
// descending v.  Row u of S is staged in shared memory when `stage` is set.
__global__ void knn_score_users_kernel(const int64_t* __restrict__ users, int64_t n_q, int n_users, int n_items,
                                       const int32_t* __restrict__ iu_ptr, const int32_t* __restrict__ iu_idx,
                                       const double* __restrict__ iu_val, const double* __restrict__ S,
                                       const double* __restrict__ mean, int k, int stage, double* ws,
                                       double* __restrict__ out)
{
    extern __shared__ double smem[];
    const int T = blockDim.x;
    double* srow_s = smem;
    double* kw = ws ? ws + (size_t)blockIdx.x * 2 * k * T : smem + (stage ? n_users : 0);
    Kept kept;
    kept.w = kw + threadIdx.x;
    kept.v = kw + (size_t)k * T + threadIdx.x;
    kept.stride = T;
    kept.k = k;
    for (int64_t q = blockIdx.x; q < n_q; q += gridDim.x) {
        const int64_t u = users[q];
        const double* srow = S + (size_t)u * n_users;
        if (stage) {
            __syncthreads();
            for (int x = threadIdx.x; x < n_users; x += T) srow_s[x] = __ldg(srow + x);
            __syncthreads();
            srow = srow_s;
        }
        const double mu = mean[u];
        for (int i = threadIdx.x; i < n_items; i += T) {
            const int b = __ldg(iu_ptr + i), e = __ldg(iu_ptr + i + 1);
            const bool all = e - b <= k;
            double num = 0.0, den = 0.0;
            kept.cnt = 0;
            for (int p = e - 1; p >= b; --p) {
                const double wt = srow[__ldg(iu_idx + p)];
                if (wt == 0.0) continue;
                const double val = __ldg(iu_val + p);
                if (all) {
                    num = __dadd_rn(num, __dmul_rn(wt, val));
                    den = __dadd_rn(den, fabs(wt));
                } else {
                    kept.offer(wt, val);
                }
            }
            if (!all) kept.sum(num, den);
            out[q * n_items + i] = finish(mu, num, den);
        }
    }
}

// ---- launch plans (shared by the workspace queries and the launches) ----
static bool sim_in_smem(int64_t n) { return (size_t)n * 3 * sizeof(double) <= SMEM_LIMIT; }

struct ScorePlan {
    int threads;       // block size
    bool stage;        // UserKNN row of S in shared memory
    bool kept_smem;    // kept pairs in shared memory (else the workspace)
    size_t smem;
    int64_t ws_bytes;
};

static ScorePlan score_plan(int64_t n_q, int64_t n_stage, int k)
{
    ScorePlan p;
    p.stage = n_stage > 0 && (size_t)n_stage * sizeof(double) <= STAGE_LIMIT;
    const size_t stage_b = p.stage ? (size_t)n_stage * sizeof(double) : 0;
    for (int t = 256; t >= 64; t >>= 1) {
        const size_t kb = (size_t)2 * k * t * sizeof(double);
        if (stage_b + kb <= SMEM_LIMIT) {
            p.threads = t; p.kept_smem = true; p.smem = stage_b + kb; p.ws_bytes = 0;
            return p;
        }
    }
    p.threads = SCORE_WS_THREADS;
    p.kept_smem = false;
    p.smem = stage_b;
    const int64_t ctas = n_q < SCORE_WS_CTAS ? n_q : SCORE_WS_CTAS;
    p.ws_bytes = ctas * 2 * (int64_t)k * SCORE_WS_THREADS * (int64_t)sizeof(double);
    return p;
}

}  // namespace knn
}  // namespace b200

using namespace b200;

extern "C" int64_t b200_knn_similarity_workspace_bytes(int64_t n)
{
    if (n <= 0 || knn::sim_in_smem(n)) return 0;
    const int64_t ctas = n < knn::SIM_WS_CTAS ? n : knn::SIM_WS_CTAS;
    return ctas * 3 * n * (int64_t)sizeof(double);
}

extern "C" int b200_knn_similarity(int64_t n, const int32_t* row_indptr, const int32_t* row_indices, const double* row_data,
                                   int64_t n_cols, const int32_t* col_indptr, const int32_t* col_indices, const double* col_data,
                                   const int32_t* order, double amplify, void* workspace, double* out, void* stream)
{
    B200_REQUIRE(n >= 1 && n < (1LL << 31) && n_cols >= 1 && n_cols < (1LL << 31), "b200_knn_similarity: bad sizes n=%lld n_cols=%lld",
                 (long long)n, (long long)n_cols);
    B200_REQUIRE(row_indptr && row_indices && row_data && col_indptr && col_indices && col_data && order && out,
                 "b200_knn_similarity: null pointer argument");
    const bool smem = knn::sim_in_smem(n);
    B200_REQUIRE(smem || workspace, "b200_knn_similarity: n=%lld needs a workspace of %lld bytes", (long long)n,
                 (long long)b200_knn_similarity_workspace_bytes(n));
    cudaStream_t st = (cudaStream_t)stream;
    const size_t sm_bytes = smem ? (size_t)n * 3 * sizeof(double) : 0;
    int grid;
    if (smem) {
        B200_CUDA(cudaFuncSetAttribute(knn::knn_sim_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_bytes));
        int per_sm = 0;
        B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, knn::knn_sim_kernel, knn::SIM_THREADS, sm_bytes));
        const int64_t cap = (int64_t)sm_count() * (per_sm > 0 ? per_sm : 1);
        grid = (int)(n < cap ? n : cap);
    } else {
        grid = (int)(n < knn::SIM_WS_CTAS ? n : knn::SIM_WS_CTAS);
    }
    knn::knn_sim_kernel<<<grid, knn::SIM_THREADS, sm_bytes, st>>>((int)n, row_indptr, row_indices, row_data, col_indptr,
                                                                  col_indices, col_data, order, amplify,
                                                                  smem ? nullptr : (double*)workspace, out); ::b200::count_launch();
    const unsigned tiles = (unsigned)((n + 31) / 32);
    knn::knn_mirror_kernel<<<dim3(tiles, tiles), dim3(32, 8), 0, st>>>((int)n, out); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_knn_row_nnz(int64_t n, const double* sim, int32_t* counts, void* stream)
{
    B200_REQUIRE(n >= 1 && n < (1LL << 31) && sim && counts, "b200_knn_row_nnz: bad argument");
    const int64_t cap = (int64_t)sm_count() * 8;
    knn::knn_row_nnz_kernel<<<(unsigned)(n < cap ? n : cap), 256, 0, (cudaStream_t)stream>>>((int)n, sim, counts); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_knn_compact(int64_t n, const double* sim, const int32_t* indptr, int32_t* indices, double* data, void* stream)
{
    B200_REQUIRE(n >= 1 && n < (1LL << 31) && sim && indptr && indices && data, "b200_knn_compact: bad argument");
    const int64_t cap = (int64_t)sm_count() * 8;
    knn::knn_compact_kernel<<<(unsigned)(n < cap ? n : cap), 256, 0, (cudaStream_t)stream>>>((int)n, sim, indptr, indices, data);
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int64_t b200_knn_score_workspace_bytes(int64_t n_q, int64_t n_stage, int k)
{
    if (n_q <= 0 || k < 1) return 0;
    return knn::score_plan(n_q, n_stage, k).ws_bytes;
}

static int knn_score_launch(bool user_mode, const int64_t* users, int64_t n_q, int64_t n_users, int64_t n_items,
                            const int32_t* indptr, const int32_t* indices, const double* data, const double* sim,
                            const double* mean, int k, void* workspace, double* out, void* stream, const char* what)
{
    B200_REQUIRE(n_q >= 0 && n_users >= 1 && n_users < (1LL << 31) && n_items >= 1 && n_items < (1LL << 31) && k >= 1,
                 "%s: bad sizes n_q=%lld n_users=%lld n_items=%lld k=%d", what, (long long)n_q, (long long)n_users,
                 (long long)n_items, k);
    B200_REQUIRE(users && indptr && indices && data && sim && mean && out, "%s: null pointer argument", what);
    if (n_q == 0) return B200_OK;
    const knn::ScorePlan p = knn::score_plan(n_q, user_mode ? n_users : 0, k);
    B200_REQUIRE(p.kept_smem || workspace, "%s: k=%d needs a workspace of %lld bytes", what, k, (long long)p.ws_bytes);
    double* ws = p.kept_smem ? nullptr : (double*)workspace;
    const int64_t grid = p.kept_smem ? n_q : (n_q < knn::SCORE_WS_CTAS ? n_q : knn::SCORE_WS_CTAS);
    const unsigned g = (unsigned)(grid < (1LL << 31) - 1 ? grid : (1LL << 31) - 1);
    cudaStream_t st = (cudaStream_t)stream;
    if (user_mode) {
        B200_CUDA(cudaFuncSetAttribute(knn::knn_score_users_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
        knn::knn_score_users_kernel<<<g, p.threads, p.smem, st>>>(users, n_q, (int)n_users, (int)n_items, indptr, indices, data,
                                                                 sim, mean, k, p.stage ? 1 : 0, ws, out);
    } else {
        B200_CUDA(cudaFuncSetAttribute(knn::knn_score_items_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
        knn::knn_score_items_kernel<<<g, p.threads, p.smem, st>>>(users, n_q, (int)n_items, indptr, indices, data, sim, mean, k,
                                                                 ws, out);
    }
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_knn_score_items(const int64_t* users, int64_t n_q, int64_t n_items, const int32_t* ui_indptr,
                                    const int32_t* ui_indices, const double* ui_data, const double* sim, const double* mean,
                                    int k, void* workspace, double* out, void* stream)
{
    return knn_score_launch(false, users, n_q, 1, n_items, ui_indptr, ui_indices, ui_data, sim, mean, k, workspace, out, stream,
                            "b200_knn_score_items");
}

extern "C" int b200_knn_score_users(const int64_t* users, int64_t n_q, int64_t n_users, int64_t n_items,
                                    const int32_t* iu_indptr, const int32_t* iu_indices, const double* iu_data,
                                    const double* sim, const double* mean, int k, void* workspace, double* out, void* stream)
{
    return knn_score_launch(true, users, n_q, n_users, n_items, iu_indptr, iu_indices, iu_data, sim, mean, k, workspace, out,
                            stream, "b200_knn_score_users");
}
