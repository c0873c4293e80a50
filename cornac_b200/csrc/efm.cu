// EFM (cornac/models/efm/recom_efm.pyx:268-353, 471-528) for sm_90a: the multiplicative-update fit over the ratings A,
// the user aspect attentions X and the item aspect qualities Y, and the per-user query vectors of its aspect-weighted
// rank.
//
// The reference's extension is built without extra compile flags (setup.py:205-210): no OpenMP, so its prange loops run
// serially, and plain IEEE f32 with no FMA.  One iteration of the reference is
//   1. for each entry of A, X, Y in CSR order: a prediction p from the factors the iteration started with, and the
//      accumulators  num += (lam * s) * other,  den += (lam * p) * other  of both rows it joins (lam = 1 for A);
//   2. x *= sqrt(num / (den + (((float)count * lam_reg) * x + eps))) element-wise (f32 sqrt: the module is C++).
// The predictions are BLAS sdot calls, whose order is unspecified; here a dot is DEFINED as the f64 sum in index order of
// the exact f32 products, rounded once to f32 (as b200_score_batch), and the A prediction is f32(U) + f32(H) in f32.
// Each accumulator element is an ordered f32 chain:
//   U1[u]: A row u, then X row u       H1[u]: A row u
//   U2[i]: A column i (users ascending), then Y row i       H2[i]: A column i
//   V[a]:  X column a (users ascending), then Y column a (items ascending)
// so an iteration runs as
//   * efm_pred_kernel: every prediction of A, X and Y, a thread per entry;
//   * efm_pass_kernel: a warp per (row, 32-factor chunk) walks the row's chains in order (lane per factor) and writes
//     the updated chunk to the second buffer of its factor matrix.  Work items are the aspects (longest chains first),
//     then the items (longest first), then the users, so the long aspect chains start first and the other rows fill
//     the machine around them.  Every pass reads only the iteration's starting factors, so one launch serves all three.
// No atomics touch the factors, so every sum has the reference's order.  -ftz=false and -prec-div/-prec-sqrt=true stay.
#include "common.cuh"

#include <algorithm>

namespace b200 {

constexpr int EFM_WARPS = 4;              // pass kernel: warps per CTA
constexpr int EFM_PRED_THREADS = 256;
constexpr int EFM_QUERY_THREADS = 128;
constexpr float EFM_EPS = 1e-9f;

__device__ __forceinline__ void efm_loss_add(double* loss, double x)
{
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (loss && (threadIdx.x & 31) == 0 && x != 0.0) atomicAdd(loss, x);
}

// The defined sdot: f64 sum in index order of exact f32 products (an f64 FMA of an exact product is that sum), one
// rounding to f32.
__device__ __forceinline__ float efm_dot(const float* __restrict__ a, const float* __restrict__ b, int n)
{
    double acc = 0.0;
    for (int f = 0; f < n; ++f) acc = __fma_rn((double)__ldg(a + f), (double)__ldg(b + f), acc);
    return __double2float_rn(acc);
}

// One segment of a chain: entries [ptr[r], ptr[r+1]) of a CSR (or of a CSC through pos, the stored index of each CSC
// entry), each naming the `other` factor row oid[c] (row length ld), with value val[c] and prediction pred[pos[c]]
// (pos == nullptr: pred[c]); lam scales both terms.
struct EfmSeg {
    const int32_t* ptr;
    const int32_t* oid;
    const float* val;
    const int32_t* pos;
    const float* pred;
    const float* other;
    int ld;
    float lam;
};

// Accumulate one segment of row r into num / den for factor f (lanes with f >= ld add nothing).
__device__ __forceinline__ void efm_chain(const EfmSeg& s, int64_t r, int f, float& num, float& den)
{
    const int lane = threadIdx.x & 31;
    const int32_t lo = __ldg(s.ptr + r), hi = __ldg(s.ptr + r + 1);
    for (int32_t c0 = lo; c0 < hi; c0 += 32) {
        const int n = min(32, hi - c0);
        int32_t o_l = 0;
        float r_l = 0.0f, p_l = 0.0f;
        if (lane < n) {
            const int32_t c = c0 + lane;
            o_l = __ldg(s.oid + c);
            r_l = __fmul_rn(s.lam, __ldg(s.val + c));                        // lambda * score
            p_l = __fmul_rn(s.lam, __ldg(s.pred + (s.pos ? __ldg(s.pos + c) : c)));   // lambda * prediction
        }
#pragma unroll 4
        for (int t = 0; t < n; ++t) {
            const int32_t o = __shfl_sync(0xffffffffu, o_l, t);
            const float rr = __shfl_sync(0xffffffffu, r_l, t);
            const float pp = __shfl_sync(0xffffffffu, p_l, t);
            if (f < s.ld) {
                const float y = __ldg(s.other + (size_t)o * s.ld + f);
                num = __fadd_rn(num, __fmul_rn(rr, y));
                den = __fadd_rn(den, __fmul_rn(pp, y));
            }
        }
    }
}

struct EfmPass {
    SparseArgs<float> a, x, y;                   // A (users x items), X (users x aspects), Y (items x aspects)
    const int32_t *item_order, *aspect_order;
    const float *pA, *pX, *pY;
    int64_t n_users, n_items, n_aspects;
    int E, L;
    float lx, ly, lu, lh, lv;
};

// The update of one 32-factor chunk of row r of X_in (row length ld) from the chains of seg1 then seg2.
__device__ __forceinline__ void efm_update(const EfmSeg& s1, const EfmSeg* s2, int64_t r, int f0, int ld, int cnt,
                                           float lam, const float* X_in, float* X_out, double& lsum, bool want_loss)
{
    const int f = f0 + (threadIdx.x & 31);
    float num = 0.0f, den = 0.0f;
    efm_chain(s1, r, f, num, den);
    if (s2) efm_chain(*s2, r, f, num, den);
    if (f < ld) {
        const float x = X_in[(size_t)r * ld + f];
        const float d = __fadd_rn(den, __fadd_rn(__fmul_rn(__fmul_rn(__int2float_rn(cnt), lam), x), EFM_EPS));
        X_out[(size_t)r * ld + f] = __fmul_rn(x, __fsqrt_rn(__fdiv_rn(num, d)));
        if (want_loss) lsum += (double)__fmul_rn(__fmul_rn(lam, x), x);
    }
}

// Every prediction of the iteration: pA[e] = f32(U1[u].U2[i]) + f32(H1[u].H2[i]), pX[e] = f32(U1[u].V[a]),
// pY[e] = f32(U2[i].V[a]).  loss (optional) += (p - s)^2 of every entry.
__global__ void __launch_bounds__(EFM_PRED_THREADS) efm_pred_kernel(
    const int32_t* __restrict__ a_row, const int32_t* __restrict__ a_idx, const float* __restrict__ a_val, int64_t nA,
    const int32_t* __restrict__ x_row, const int32_t* __restrict__ x_idx, const float* __restrict__ x_val, int64_t nX,
    const int32_t* __restrict__ y_row, const int32_t* __restrict__ y_idx, const float* __restrict__ y_val, int64_t nY,
    const float* __restrict__ U1, const float* __restrict__ U2, const float* __restrict__ V, const float* __restrict__ H1,
    const float* __restrict__ H2, int E, int L, float* __restrict__ pA, float* __restrict__ pX, float* __restrict__ pY,
    double* loss)
{
    double lsum = 0.0;
    const int64_t total = nA + nX + nY;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        float p, s;
        if (e < nA) {
            const int64_t u = __ldg(a_row + e), i = __ldg(a_idx + e);
            p = __fadd_rn(efm_dot(U1 + u * E, U2 + i * E, E), efm_dot(H1 + u * L, H2 + i * L, L));
            s = __ldg(a_val + e);
            pA[e] = p;
        } else if (e < nA + nX) {
            const int64_t c = e - nA;
            p = efm_dot(U1 + (int64_t)__ldg(x_row + c) * E, V + (int64_t)__ldg(x_idx + c) * E, E);
            s = __ldg(x_val + c);
            pX[c] = p;
        } else {
            const int64_t c = e - nA - nX;
            p = efm_dot(U2 + (int64_t)__ldg(y_row + c) * E, V + (int64_t)__ldg(y_idx + c) * E, E);
            s = __ldg(y_val + c);
            pY[c] = p;
        }
        if (loss) {
            const float d = __fsub_rn(p, s);
            lsum += (double)d * (double)d;
        }
    }
    if (loss) {
        for (int o = 16; o; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if ((threadIdx.x & 31) == 0 && lsum != 0.0) atomicAdd(loss, lsum);
    }
}

// All three update passes of one iteration.  Work item w (a warp each, grid-stride): the first n_aspects * cE are
// (aspect_order[w / cE], chunk w % cE); then n_items * (cE + cL) items in item_order, then n_users * (cE + cL) users;
// chunks [0, cE) of an item or user are its explicit factors, [cE, cE + cL) its latent ones.
__global__ void __launch_bounds__(EFM_WARPS * 32, 4) efm_pass_kernel(
    EfmPass P, const float* __restrict__ U1, const float* __restrict__ U2, const float* __restrict__ V,
    const float* __restrict__ H1, const float* __restrict__ H2, float* __restrict__ U1o, float* __restrict__ U2o,
    float* __restrict__ Vo, float* __restrict__ H1o, float* __restrict__ H2o, double* loss)
{
    const int cE = (P.E + 31) >> 5, cL = (P.L + 31) >> 5, cR = cE + cL;
    const int64_t nw_a = P.n_aspects * cE, nw_i = P.n_items * cR, nw_u = P.n_users * cR;
    const int64_t n_work = nw_a + nw_i + nw_u;
    const int64_t n_warps = (int64_t)gridDim.x * EFM_WARPS;
    double lsum = 0.0;
    const bool want_loss = loss != nullptr;
    for (int64_t w = (int64_t)blockIdx.x * EFM_WARPS + (threadIdx.x >> 5); w < n_work; w += n_warps) {
        if (w < nw_a) {                                          // V[a]: X column a, then Y column a
            const int64_t a = __ldg(P.aspect_order + w / cE);
            const int q = (int)(w % cE);
            const EfmSeg sx{P.x.cptr, P.x.crow, P.x.cval, P.x.cpos, P.pX, U1, P.E, P.lx};
            const EfmSeg sy{P.y.cptr, P.y.crow, P.y.cval, P.y.cpos, P.pY, U2, P.E, P.ly};
            const int cnt = (__ldg(P.x.cptr + a + 1) - __ldg(P.x.cptr + a)) + (__ldg(P.y.cptr + a + 1) - __ldg(P.y.cptr + a));
            efm_update(sx, &sy, a, q * 32, P.E, cnt, P.lv, V, Vo, lsum, want_loss);
        } else if (w < nw_a + nw_i) {                            // U2[i]: A column i, then Y row i; H2[i]: A column i
            const int64_t v = w - nw_a;
            const int64_t i = __ldg(P.item_order + v / cR);
            const int q = (int)(v % cR);
            const int cA = __ldg(P.a.cptr + i + 1) - __ldg(P.a.cptr + i);
            if (q < cE) {
                const EfmSeg sa{P.a.cptr, P.a.crow, P.a.cval, P.a.cpos, P.pA, U1, P.E, 1.0f};
                const EfmSeg sy{P.y.ptr, P.y.idx, P.y.val, nullptr, P.pY, V, P.E, P.ly};
                const int cnt = cA + (__ldg(P.y.ptr + i + 1) - __ldg(P.y.ptr + i));
                efm_update(sa, &sy, i, q * 32, P.E, cnt, P.lu, U2, U2o, lsum, want_loss);
            } else {
                const EfmSeg sa{P.a.cptr, P.a.crow, P.a.cval, P.a.cpos, P.pA, H1, P.L, 1.0f};
                efm_update(sa, nullptr, i, (q - cE) * 32, P.L, cA, P.lh, H2, H2o, lsum, want_loss);
            }
        } else {                                                 // U1[u]: A row u, then X row u; H1[u]: A row u
            const int64_t v = w - nw_a - nw_i;
            const int64_t u = v / cR;
            const int q = (int)(v % cR);
            const int cA = __ldg(P.a.ptr + u + 1) - __ldg(P.a.ptr + u);
            if (q < cE) {
                const EfmSeg sa{P.a.ptr, P.a.idx, P.a.val, nullptr, P.pA, U2, P.E, 1.0f};
                const EfmSeg sx{P.x.ptr, P.x.idx, P.x.val, nullptr, P.pX, V, P.E, P.lx};
                const int cnt = cA + (__ldg(P.x.ptr + u + 1) - __ldg(P.x.ptr + u));
                efm_update(sa, &sx, u, q * 32, P.E, cnt, P.lu, U1, U1o, lsum, want_loss);
            } else {
                const EfmSeg sa{P.a.ptr, P.a.idx, P.a.val, nullptr, P.pA, H2, P.L, 1.0f};
                efm_update(sa, nullptr, u, (q - cE) * 32, P.L, cA, P.lh, H1, H1o, lsum, want_loss);
            }
        }
    }
    efm_loss_add(loss, lsum);
}

// The query vector of each listed user (b200_efm_queries): a CTA per user.
//   X_[a] = f32(U1[u].V[a]) for every aspect (the defined dot), kept in shared memory;
//   the top m = min(N, n_aspects) aspects a_0..a_{m-1} in the order (X_ desc, aspect id asc), by m block-wide argmax;
//   Q[q, f]     = f32(c * sum_t X_[a_t] * V[a_t, f] + beta * U1[u, f])   (f < E; the sum in f64 over t ascending)
//   Q[q, E + f] = f32(beta * H1[u, f])                                     (f < L)
// with c = alpha / (N * rating_scale) and beta = 1 - alpha given in f64, every f64 operation rounded separately.
__global__ void __launch_bounds__(EFM_QUERY_THREADS) efm_query_kernel(
    const int64_t* __restrict__ users, int64_t n_q, const float* __restrict__ U1, const float* __restrict__ H1,
    const float* __restrict__ V, int64_t n_aspects, int E, int L, int m, double c, double beta, float* __restrict__ Q)
{
    extern __shared__ float efm_qsmem[];
    float* xs = efm_qsmem;                                   // X_ of the user
    int32_t* top = reinterpret_cast<int32_t*>(efm_qsmem + n_aspects);   // the chosen aspects, in order
    uint8_t* taken = reinterpret_cast<uint8_t*>(top + m);
    __shared__ float r_val[EFM_QUERY_THREADS / 32];
    __shared__ int32_t r_id[EFM_QUERY_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int64_t q = blockIdx.x; q < n_q; q += gridDim.x) {
        const int64_t u = __ldg(users + q);
        const float* U1r = U1 + u * E;
        for (int64_t a = tid; a < n_aspects; a += EFM_QUERY_THREADS) {
            xs[a] = efm_dot(U1r, V + a * E, E);
            taken[a] = 0;
        }
        __syncthreads();
        for (int t = 0; t < m; ++t) {
            // the best untaken aspect: larger X_, then the smaller id
            float bv = 0.0f;
            int32_t bi = -1;
            for (int64_t a = tid; a < n_aspects; a += EFM_QUERY_THREADS)
                if (!taken[a] && (bi < 0 || xs[a] > bv)) bv = xs[a], bi = (int32_t)a;
            for (int o = 16; o; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
                const int32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (oi >= 0 && (bi < 0 || ov > bv || (ov == bv && oi < bi))) bv = ov, bi = oi;
            }
            if (lane == 0) r_val[wid] = bv, r_id[wid] = bi;
            __syncthreads();
            if (tid == 0) {
                float v0 = r_val[0];
                int32_t i0 = r_id[0];
                for (int k = 1; k < EFM_QUERY_THREADS / 32; ++k) {
                    const float ov = r_val[k];
                    const int32_t oi = r_id[k];
                    if (oi >= 0 && (i0 < 0 || ov > v0 || (ov == v0 && oi < i0))) v0 = ov, i0 = oi;
                }
                top[t] = i0;
                taken[i0] = 1;
            }
            __syncthreads();
        }
        for (int f = tid; f < E + L; f += EFM_QUERY_THREADS) {
            double out;
            if (f < E) {
                double s = 0.0;
                for (int t = 0; t < m; ++t) {
                    const int32_t a = top[t];
                    s = __dadd_rn(s, __dmul_rn((double)xs[a], (double)__ldg(V + (int64_t)a * E + f)));
                }
                out = __dadd_rn(__dmul_rn(c, s), __dmul_rn(beta, (double)__ldg(U1r + f)));
            } else {
                out = __dmul_rn(beta, (double)__ldg(H1 + u * L + (f - E)));
            }
            Q[q * (E + L) + f] = __double2float_rn(out);
        }
        __syncthreads();
    }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_efm_fit(B200_EFM_DATA, int E, int L, float* U1, float* U2, float* V, float* H1, float* H2,
                            float* work, float* pred, int n_iter, float lambda_x, float lambda_y, float lambda_u,
                            float lambda_h, float lambda_v, double* loss, void* stream)
{
    const EfmPass P{B200_SPARSE_VIEW(a_), B200_SPARSE_VIEW(x_), B200_SPARSE_VIEW(y_), item_order, aspect_order,
                    pred, pred + a_nnz, pred + a_nnz + x_nnz, n_users, n_items, n_aspects, E, L, lambda_x, lambda_y,
                    lambda_u, lambda_h, lambda_v};
    if (int rc = sparse_check(P.a, n_users, n_items, "b200_efm_fit")) return rc;
    if (int rc = sparse_check(P.x, n_users, n_aspects, "b200_efm_fit")) return rc;
    if (int rc = sparse_check(P.y, n_items, n_aspects, "b200_efm_fit")) return rc;
    B200_REQUIRE(E >= 1 && L >= 1 && n_iter >= 0, "b200_efm_fit: bad sizes E=%d L=%d n_iter=%d", E, L, n_iter);
    B200_REQUIRE(item_order && aspect_order && U1 && U2 && V && H1 && H2 && work && pred,
                 "b200_efm_fit: null pointer argument");
    if (n_iter == 0) return B200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t sz[5] = {(size_t)n_users * E, (size_t)n_items * E, (size_t)n_aspects * E, (size_t)n_users * L,
                          (size_t)n_items * L};
    float* cur[5] = {U1, U2, V, H1, H2};
    float* nxt[5];
    for (int m = 0; m < 5; ++m) {                           // the second buffer of each factor matrix
        nxt[m] = work;
        work += sz[m];
    }
    const int64_t n_pred = a_nnz + x_nnz + y_nnz;
    const unsigned cap = (unsigned)sm_count() * 16;
    const unsigned grid_p = (unsigned)std::max<int64_t>(1, std::min<int64_t>(cap, (n_pred + EFM_PRED_THREADS - 1) / EFM_PRED_THREADS));
    const int64_t cR = (E + 31) / 32 + (L + 31) / 32;
    const int64_t n_work = n_aspects * ((E + 31) / 32) + (n_items + n_users) * cR;
    const unsigned grid_w = (unsigned)std::max<int64_t>(1, std::min<int64_t>(cap, (n_work + EFM_WARPS - 1) / EFM_WARPS));
    for (int it = 0; it < n_iter; ++it) {
        double* le = loss ? loss + it : nullptr;
        if (n_pred > 0) {
            efm_pred_kernel<<<grid_p, EFM_PRED_THREADS, 0, st>>>(a_row, a_idx, a_val, a_nnz, x_row, x_idx, x_val, x_nnz,
                                                                 y_row, y_idx, y_val, y_nnz, cur[0], cur[1], cur[2],
                                                                 cur[3], cur[4], E, L, pred, pred + a_nnz,
                                                                 pred + a_nnz + x_nnz, le);
            ::b200::count_launch();
        }
        if (n_work > 0) {
            efm_pass_kernel<<<grid_w, EFM_WARPS * 32, 0, st>>>(P, cur[0], cur[1], cur[2], cur[3], cur[4], nxt[0], nxt[1],
                                                               nxt[2], nxt[3], nxt[4], le);
            ::b200::count_launch();
        }
        B200_CUDA(cudaGetLastError());
        for (int m = 0; m < 5; ++m) std::swap(cur[m], nxt[m]);
    }
    float* orig[5] = {U1, U2, V, H1, H2};
    for (int m = 0; m < 5; ++m)
        if (cur[m] != orig[m] && sz[m])
            B200_CUDA(cudaMemcpyAsync(orig[m], cur[m], sizeof(float) * sz[m], cudaMemcpyDeviceToDevice, st));
    return B200_OK;
}

extern "C" int b200_efm_queries(const int64_t* users, int64_t n_q, const float* U1, const float* H1, const float* V,
                                int64_t n_aspects, int E, int L, int num_most_cared, double alpha, double rating_scale,
                                float* Q, void* stream)
{
    B200_REQUIRE(E >= 1 && L >= 1 && n_q >= 0 && n_aspects >= 0 && num_most_cared >= 0,
                 "b200_efm_queries: bad sizes E=%d L=%d n_q=%lld n_aspects=%lld N=%d", E, L, (long long)n_q,
                 (long long)n_aspects, num_most_cared);
    B200_REQUIRE(n_q == 0 || (users && U1 && H1 && Q && (n_aspects == 0 || V)), "b200_efm_queries: null pointer argument");
    if (n_q == 0) return B200_OK;
    const int m = (int)std::min<int64_t>(num_most_cared, n_aspects);
    const size_t smem = (size_t)n_aspects * (sizeof(float) + 1) + (size_t)m * sizeof(int32_t) + 16;
    int dev = 0, optin = 0;
    B200_CUDA(cudaGetDevice(&dev));
    B200_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    B200_REQUIRE(smem <= (size_t)optin, "b200_efm_queries: %lld aspects do not fit one CTA's shared memory",
                 (long long)n_aspects);
    if (smem > 48 * 1024)
        B200_CUDA(cudaFuncSetAttribute(efm_query_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const double c = alpha / ((double)num_most_cared * rating_scale);
    const double beta = 1.0 - alpha;
    const unsigned grid = (unsigned)std::min<int64_t>(n_q, (int64_t)sm_count() * 16);
    efm_query_kernel<<<grid, EFM_QUERY_THREADS, smem, (cudaStream_t)stream>>>(users, n_q, U1, H1, V, n_aspects, E, L, m, c,
                                                                             beta, Q);
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
