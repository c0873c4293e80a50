// NMF (cornac/models/nmf/recom_nmf.pyx:182-267) for sm_90a: the multiplicative-update fit, bit-identical to the
// compiled reference.
//
// The reference's extension is built without extra compile flags (setup.py:155-160): no OpenMP, so its prange loops run
// serially, and plain IEEE f32 with no FMA.  Every operation below is an explicitly rounded __f*_rn intrinsic in the
// reference's order; nvcc's defaults -ftz=false and -prec-div=true stay (the updates can produce subnormals).
//
// One epoch of the reference is
//   1. for each rating j = (u, i, r) in stored (CSR) order: rp = ((mu + Bu[u]) + Bi[i]) + U[u,0]*V[i,0] + ... (serial);
//      with use_bias, Bu[u] and Bi[i] take an SGD step; the four accumulators Un/Ud[u] and Vn/Vd[i] gain r*V[i],
//      rp*V[i], r*U[u], rp*U[u];
//   2. U[u,f] *= Un / (Ud + ((count_u * lambda_u) * U[u,f] + eps));
//   3. V[i,f] *= Vn / (Vd + ((count_i * lambda_v) * V[i,f] + eps)).
// U and V do not change during 1, so rp of a rating depends on earlier ratings only through the biases.  Un/Ud of a user
// are an ordered sum over its CSR row and Vn/Vd of an item an ordered sum over its ratings in stored order (a stable
// CSC transpose), so the fit runs as:
//   * nmf_level_kernel (use_bias only): rp and the bias steps over b200_pmf_schedule's level schedule, one CTA, a barrier
//     between levels; the biases live in shared memory when they fit;
//   * nmf_user_kernel: a warp per user walks its row in order (lane per factor), computing rp first when the biases are
//     not trained, and writes the updated row to a second buffer (the item sums still need the old U);
//   * nmf_item_kernel: a warp per item walks its CSC column in order and updates V in place.
// No atomics touch the factors, so every sum has the reference's order.
#include "common.cuh"

#include <algorithm>

namespace b200 {

constexpr int NMF_WARPS = 4;               // user / item kernels: warps per CTA (short CTAs spread long columns over SMs)
constexpr int NMF_LEVEL_THREADS = 512;     // level kernel: one CTA
constexpr float NMF_EPS = 1e-9f;

__device__ __forceinline__ void nmf_loss_add(double* loss, double x)
{
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (loss && (threadIdx.x & 31) == 0 && x != 0.0) atomicAdd(loss, x);
}

// The ordered sums of one row (a user's CSR row or an item's CSC column) and the multiplicative update of its factors.
// Entry c of the row: `other` row oid[c], rating val[c], prediction rp[pos[c]] (pos == nullptr: rp[c]).
// X_out[f] = X[f] * (num / (den + ((cnt * lam) * X[f] + eps))).  Lane q*32 + lane handles factor f0 + q*32 + lane.
template <int FPL>
__device__ __forceinline__ void nmf_row_update(int32_t lo, int32_t hi, const int32_t* __restrict__ oid,
                                               const float* __restrict__ val, const int32_t* __restrict__ pos,
                                               const float* rp, const float* __restrict__ other, int k, const float* X,
                                               float* X_out, float lam, double& lsum, bool err_loss, bool reg_loss)
{
    const int lane = threadIdx.x & 31;
    const float cl = __fmul_rn(__int2float_rn(hi - lo), lam);
    for (int f0 = 0; f0 < k; f0 += 32 * FPL) {
        float num[FPL], den[FPL];
#pragma unroll
        for (int q = 0; q < FPL; ++q) num[q] = den[q] = 0.0f;
        for (int32_t c0 = lo; c0 < hi; c0 += 32) {
            const int n = min(32, hi - c0);
            int32_t o_l = 0;
            float r_l = 0.0f, p_l = 0.0f;
            if (lane < n) {
                const int32_t c = c0 + lane;
                o_l = __ldg(oid + c);
                r_l = __ldg(val + c);
                p_l = rp[pos ? __ldg(pos + c) : c];
                if (err_loss && f0 == 0) {
                    const float e = __fsub_rn(r_l, p_l);
                    lsum += (double)e * (double)e;
                }
            }
#pragma unroll 4
            for (int t = 0; t < n; ++t) {
                const int32_t o = __shfl_sync(0xffffffffu, o_l, t);
                const float r = __shfl_sync(0xffffffffu, r_l, t);
                const float p = __shfl_sync(0xffffffffu, p_l, t);
                const float* Orow = other + (size_t)o * k;
#pragma unroll
                for (int q = 0; q < FPL; ++q) {
                    const int f = f0 + q * 32 + lane;
                    if (f < k) {
                        const float y = __ldg(Orow + f);
                        num[q] = __fadd_rn(num[q], __fmul_rn(r, y));
                        den[q] = __fadd_rn(den[q], __fmul_rn(p, y));
                    }
                }
            }
        }
#pragma unroll
        for (int q = 0; q < FPL; ++q) {
            const int f = f0 + q * 32 + lane;
            if (f < k) {
                const float x = X[f];
                const float d = __fadd_rn(den[q], __fadd_rn(__fmul_rn(cl, x), NMF_EPS));
                X_out[f] = __fmul_rn(x, __fdiv_rn(num[q], d));
                if (reg_loss) lsum += (double)__fmul_rn(__fmul_rn(lam, x), x);
            }
        }
    }
}

// Phase 2 (and phase 1 when the biases are not trained): a warp per user.  U_out must not alias U.
template <bool COMPUTE_RP, int FPL>
__global__ void __launch_bounds__(NMF_WARPS * 32, 8) nmf_user_kernel(
    const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ rating,
    int64_t n_users, int k, const float* __restrict__ U, const float* __restrict__ V, const float* __restrict__ Bu,
    const float* __restrict__ Bi, float mu, float lambda_u, float* rp, float* __restrict__ U_out, double* loss)
{
    const int lane = threadIdx.x & 31;
    const int64_t n_warps = (int64_t)gridDim.x * NMF_WARPS;
    double lsum = 0.0;
    for (int64_t u = (int64_t)blockIdx.x * NMF_WARPS + (threadIdx.x >> 5); u < n_users; u += n_warps) {
        const int32_t lo = __ldg(indptr + u), hi = __ldg(indptr + u + 1);
        const float* Ur = U + (size_t)u * k;
        if constexpr (COMPUTE_RP) {           // recom_nmf.pyx:232-234, a lane per rating
            const float base = __fadd_rn(mu, __ldg(Bu + u));
            for (int32_t j = lo + lane; j < hi; j += 32) {
                const int32_t i = __ldg(indices + j);
                const float* Vr = V + (size_t)i * k;
                float x = __fadd_rn(base, __ldg(Bi + i));
                for (int f = 0; f < k; ++f) x = __fadd_rn(x, __fmul_rn(__ldg(Ur + f), __ldg(Vr + f)));
                rp[j] = x;
            }
            __syncwarp();
        }
        nmf_row_update<FPL>(lo, hi, indices, rating, nullptr, rp, V, k, Ur, U_out + (size_t)u * k, lambda_u, lsum,
                            loss != nullptr, loss != nullptr);
    }
    nmf_loss_add(loss, lsum);
}

// Phase 3: a warp per item, items in decreasing degree (item_order) so that the long columns start first.
template <int FPL>
__global__ void __launch_bounds__(NMF_WARPS * 32, 8) nmf_item_kernel(
    const int32_t* __restrict__ csc_ptr, const int32_t* __restrict__ csc_row, const float* __restrict__ csc_val,
    const int32_t* __restrict__ csc_pos, const int32_t* __restrict__ item_order, int64_t n_items, int k,
    const float* __restrict__ U, float* V, const float* __restrict__ rp, float lambda_v, double* loss)
{
    const int64_t n_warps = (int64_t)gridDim.x * NMF_WARPS;
    double lsum = 0.0;
    for (int64_t w = (int64_t)blockIdx.x * NMF_WARPS + (threadIdx.x >> 5); w < n_items; w += n_warps) {
        const int32_t i = __ldg(item_order + w);
        float* Vr = V + (size_t)i * k;
        nmf_row_update<FPL>(__ldg(csc_ptr + i), __ldg(csc_ptr + i + 1), csc_row, csc_val, csc_pos, rp, U, k, Vr, Vr,
                            lambda_v, lsum, false, loss != nullptr);
    }
    nmf_loss_add(loss, lsum);
}

// Phase 1 with use_bias: the ratings level by level (b200_pmf_schedule); ratings of one level touch disjoint users and
// items.  s_uid / s_iid / s_rat / s_pos are the ratings in schedule order (s_pos = stored index, where rp goes).
// Thread t handles slot level_ptr[l] + t (+ multiples of the CTA width).  Everything that does not depend on the
// biases -- the slot's ids and rating, and for k <= KP the two factor rows -- is loaded one level ahead, so that only
// the bias loads, the k-long add chain and the bias steps sit between two barriers.  KP == 0: the rows are read after
// the barrier.  SMEM: Bu and Bi are staged in dynamic shared memory.
template <bool SMEM, int KP>
__global__ void __launch_bounds__(NMF_LEVEL_THREADS, 1) nmf_level_kernel(
    const int32_t* __restrict__ s_uid, const int32_t* __restrict__ s_iid, const float* __restrict__ s_rat,
    const int32_t* __restrict__ s_pos, const int32_t* __restrict__ level_ptr, int32_t n_levels, int64_t n_users,
    int64_t n_items, int k, const float* __restrict__ U, const float* __restrict__ V, float* Bu_g, float* Bi_g, float mu,
    float lr, float lambda_bu, float lambda_bi, float* __restrict__ rp)
{
    extern __shared__ float nmf_smem[];
    const int tid = threadIdx.x;
    float* Bu = Bu_g;
    float* Bi = Bi_g;
    if constexpr (SMEM) {
        Bu = nmf_smem;
        Bi = nmf_smem + n_users;
        for (int64_t x = tid; x < n_users; x += NMF_LEVEL_THREADS) Bu[x] = Bu_g[x];
        for (int64_t x = tid; x < n_items; x += NMF_LEVEL_THREADS) Bi[x] = Bi_g[x];
        __syncthreads();
    }
    constexpr int KR = KP > 0 ? KP : 1;
    // the thread's first slot of the next level: ids, rating, stored index, factor rows
    int32_t nu = 0, ni = 0, np = -1;
    float nr = 0.0f;
    float pu[KR], pv[KR];
    auto fetch = [&](int32_t s) {
        nu = __ldg(s_uid + s), ni = __ldg(s_iid + s), nr = __ldg(s_rat + s), np = __ldg(s_pos + s);
        if constexpr (KP > 0) {
            const float* Ur = U + (size_t)nu * k;
            const float* Vr = V + (size_t)ni * k;
#pragma unroll
            for (int f = 0; f < KP; ++f)
                if (f < k) pu[f] = __ldg(Ur + f), pv[f] = __ldg(Vr + f);
        }
    };
    auto apply = [&](int32_t u, int32_t i, float r, int32_t j, bool prefetched) {
        // recom_nmf.pyx:232-242
        float x = __fadd_rn(__fadd_rn(mu, Bu[u]), Bi[i]);
        const float* Ur = U + (size_t)u * k;
        const float* Vr = V + (size_t)i * k;
        if (KP > 0 && prefetched) {
#pragma unroll
            for (int f = 0; f < KR; ++f)
                if (f < k) x = __fadd_rn(x, __fmul_rn(pu[f], pv[f]));
        } else {
            for (int f = 0; f < k; ++f) x = __fadd_rn(x, __fmul_rn(__ldg(Ur + f), __ldg(Vr + f)));
        }
        const float e = __fsub_rn(r, x);
        const float bu = Bu[u], bi = Bi[i];
        Bu[u] = __fadd_rn(bu, __fmul_rn(lr, __fsub_rn(e, __fmul_rn(lambda_bu, bu))));
        Bi[i] = __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(e, __fmul_rn(lambda_bi, bi))));
        rp[j] = x;
    };
    int32_t lo = n_levels > 0 ? __ldg(level_ptr) : 0, hi = n_levels > 0 ? __ldg(level_ptr + 1) : 0;
    if (lo + tid < hi) fetch(lo + tid);
    for (int32_t l = 0; l < n_levels; ++l) {
        const int32_t hi2 = l + 2 <= n_levels ? __ldg(level_ptr + l + 2) : hi;
        if (lo + tid < hi) {
            const int32_t u = nu, i = ni, j = np;
            const float r = nr;
            apply(u, i, r, j, KP > 0);
            if (hi + tid < hi2) fetch(hi + tid);       // next level's slot: loads in flight across the barrier
            for (int32_t s = lo + tid + NMF_LEVEL_THREADS; s < hi; s += NMF_LEVEL_THREADS)
                apply(__ldg(s_uid + s), __ldg(s_iid + s), __ldg(s_rat + s), __ldg(s_pos + s), false);
        } else if (hi + tid < hi2) {
            fetch(hi + tid);
        }
        __syncthreads();
        lo = hi, hi = hi2;
    }
    if constexpr (SMEM) {
        for (int64_t x = tid; x < n_users; x += NMF_LEVEL_THREADS) Bu_g[x] = Bu[x];
        for (int64_t x = tid; x < n_items; x += NMF_LEVEL_THREADS) Bi_g[x] = Bi[x];
    }
}

template <int FPL>
void launch_user(bool compute_rp, unsigned grid, cudaStream_t st, const int32_t* indptr, const int32_t* indices,
                 const float* rating, int64_t n_users, int k, const float* U, const float* V, const float* Bu,
                 const float* Bi, float mu, float lambda_u, float* rp, float* U_out, double* loss)
{
    if (compute_rp)
        nmf_user_kernel<true, FPL><<<grid, NMF_WARPS * 32, 0, st>>>(indptr, indices, rating, n_users, k, U, V, Bu, Bi, mu,
                                                                    lambda_u, rp, U_out, loss);
    else
        nmf_user_kernel<false, FPL><<<grid, NMF_WARPS * 32, 0, st>>>(indptr, indices, rating, n_users, k, U, V, Bu, Bi,
                                                                     mu, lambda_u, rp, U_out, loss);
}

template <bool SMEM>
void launch_level(int k, size_t smem, cudaStream_t st, const int32_t* s_uid, const int32_t* s_iid, const float* s_rat,
                  const int32_t* s_pos, const int32_t* level_ptr, int32_t n_levels, int64_t n_users, int64_t n_items,
                  const float* U, const float* V, float* Bu, float* Bi, float mu, float lr, float lbu, float lbi, float* rp)
{
#define B200_NMF_LEVEL(KP)                                                                                           \
    nmf_level_kernel<SMEM, KP><<<1, NMF_LEVEL_THREADS, smem, st>>>(s_uid, s_iid, s_rat, s_pos, level_ptr, n_levels,   \
                                                                   n_users, n_items, k, U, V, Bu, Bi, mu, lr, lbu, lbi, rp)
    if (k <= 16) B200_NMF_LEVEL(16);
    else if (k <= 32) B200_NMF_LEVEL(32);
    else B200_NMF_LEVEL(0);
#undef B200_NMF_LEVEL
}

}  // namespace b200

using namespace b200;

extern "C" int b200_nmf_fit(int64_t n_users, int64_t n_items, B200_SPARSE(r_, float), const int32_t* item_order,
                            const int32_t* s_uid, const int32_t* s_iid, const float* s_rat, const int32_t* s_pos,
                            const int32_t* level_ptr, int32_t n_levels, int k, float* U, float* V, float* Bu, float* Bi,
                            float* rp, float* U_work, int n_epochs, float mu, float learning_rate, float lambda_u,
                            float lambda_v, float lambda_bu, float lambda_bi, int use_bias, double* loss, void* stream)
{
    const SparseArgs<float> r = B200_SPARSE_VIEW(r_);
    if (int rc = sparse_check(r, n_users, n_items, "b200_nmf_fit")) return rc;
    const int64_t nnz = r.nnz;
    B200_REQUIRE(k >= 1 && n_epochs >= 0 && n_levels >= 0, "b200_nmf_fit: bad sizes k=%d n_epochs=%d n_levels=%d", k,
                 n_epochs, n_levels);
    B200_REQUIRE(item_order && U && V && Bu && Bi && U_work && U_work != U && (nnz == 0 || rp),
                 "b200_nmf_fit: null or aliased pointer argument");
    B200_REQUIRE(!use_bias || nnz == 0 || (s_uid && s_iid && s_rat && s_pos && level_ptr && n_levels > 0),
                 "b200_nmf_fit: use_bias needs the level schedule");
    if (n_epochs == 0 || n_users == 0 || n_items == 0) return B200_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned cap = (unsigned)sm_count() * 16;
    const unsigned grid_u = (unsigned)std::min<int64_t>(cap, (n_users + NMF_WARPS - 1) / NMF_WARPS);
    const unsigned grid_i = (unsigned)std::min<int64_t>(cap, (n_items + NMF_WARPS - 1) / NMF_WARPS);
    const bool bias_pass = use_bias && nnz > 0;
    size_t smem = 0;
    bool in_smem = false;
    if (bias_pass) {
        int dev = 0, optin = 0;
        B200_CUDA(cudaGetDevice(&dev));
        B200_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        smem = (size_t)(n_users + n_items) * sizeof(float);
        in_smem = smem <= (size_t)optin;
        if (in_smem) {
            B200_CUDA(cudaFuncSetAttribute(nmf_level_kernel<true, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            B200_CUDA(cudaFuncSetAttribute(nmf_level_kernel<true, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            B200_CUDA(cudaFuncSetAttribute(nmf_level_kernel<true, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        } else {
            smem = 0;
        }
    }
    float* cur = U;
    float* nxt = U_work;
    for (int e = 0; e < n_epochs; ++e) {
        double* le = loss ? loss + e : nullptr;
        if (bias_pass) {
            if (in_smem)
                launch_level<true>(k, smem, st, s_uid, s_iid, s_rat, s_pos, level_ptr, n_levels, n_users, n_items, cur, V, Bu,
                                   Bi, mu, learning_rate, lambda_bu, lambda_bi, rp);
            else
                launch_level<false>(k, 0, st, s_uid, s_iid, s_rat, s_pos, level_ptr, n_levels, n_users, n_items, cur, V, Bu,
                                    Bi, mu, learning_rate, lambda_bu, lambda_bi, rp);
            ::b200::count_launch();
        }
        if (k <= 32)
            launch_user<1>(!bias_pass, grid_u, st, r.ptr, r.idx, r.val, n_users, k, cur, V, Bu, Bi, mu, lambda_u, rp, nxt, le);
        else if (k <= 64)
            launch_user<2>(!bias_pass, grid_u, st, r.ptr, r.idx, r.val, n_users, k, cur, V, Bu, Bi, mu, lambda_u, rp, nxt, le);
        else
            launch_user<4>(!bias_pass, grid_u, st, r.ptr, r.idx, r.val, n_users, k, cur, V, Bu, Bi, mu, lambda_u, rp, nxt, le);
        if (k <= 32)
            nmf_item_kernel<1><<<grid_i, NMF_WARPS * 32, 0, st>>>(r.cptr, r.crow, r.cval, r.cpos, item_order, n_items, k,
                                                                  cur, V, rp, lambda_v, le);
        else if (k <= 64)
            nmf_item_kernel<2><<<grid_i, NMF_WARPS * 32, 0, st>>>(r.cptr, r.crow, r.cval, r.cpos, item_order, n_items, k,
                                                                  cur, V, rp, lambda_v, le);
        else
            nmf_item_kernel<4><<<grid_i, NMF_WARPS * 32, 0, st>>>(r.cptr, r.crow, r.cval, r.cpos, item_order, n_items, k,
                                                                  cur, V, rp, lambda_v, le);
        ::b200::count_launch(2);
        B200_CUDA(cudaGetLastError());
        std::swap(cur, nxt);
    }
    if (cur != U) B200_CUDA(cudaMemcpyAsync(U, cur, sizeof(float) * (size_t)n_users * k, cudaMemcpyDeviceToDevice, st));
    return B200_OK;
}
