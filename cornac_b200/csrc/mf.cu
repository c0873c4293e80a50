// Biased matrix-factorisation SGD epochs for sm_90a.
//
// Replaces one epoch of backend_cpu.fit_sgd (reference: cornac/models/mf/backend_cpu.pyx:58-83):
//   * mf_hogwild_kernel : every G-lane group owns one rating at a time (grid-stride over the
//     stored rating list), gathers U[u] / V[i] with 128-bit L2-only loads, warp-shuffle dot,
//     scatter-update (plain stores or red.global.add), per-epoch sum(err^2) reduced per block.
//   * mf_replay_kernel  : one warp, ratings applied strictly in stored order (the seeded
//     single-thread reference, mf/recom_mf.py:124-125), loss accumulated in the same order.
#include <stdlib.h>

#include "sgd_common.cuh"

namespace b200 {

template <typename IdT>
struct MfParams {
    const IdT* __restrict__ rid;
    const IdT* __restrict__ cid;
    const float* __restrict__ val;
    int64_t n;
    float* U;
    float* V;
    float* Bu;
    float* Bi;
    int k;
    float lr, reg, mu;
    int use_bias;
    float* loss;
    int64_t max_groups;      // cap on concurrently running ratings (Hogwild staleness bound)
};

template <typename IdT, int G, int NPL, bool VEC, bool ATOMIC, int S>
__global__ void __launch_bounds__(256) mf_hogwild_kernel(const MfParams<IdT> p)
{
    using Frag = RowFrag<NPL, VEC>;
    constexpr int E = NPL * Frag::W;
    const int lg = threadIdx.x & (G - 1);
    const int n_units = VEC ? p.k / 4 : p.k;
    const int64_t groups_per_block = blockDim.x / G;
    const int64_t n_groups = (int64_t)gridDim.x * groups_per_block;
    const int64_t gid = (int64_t)blockIdx.x * groups_per_block + threadIdx.x / G;
    const size_t k = (size_t)p.k;
    float loss = 0.f;

    // group g takes ratings g, g + n_groups, ... : consecutive groups read consecutive ratings
    for (int64_t j0 = gid; j0 < p.n; j0 += n_groups * S) {
        int64_t u[S], it[S];
        float r[S], bu[S], bi[S];
        bool live[S];
        Frag fu[S], fi[S];
#pragma unroll
        for (int t = 0; t < S; ++t) {
            const int64_t j = j0 + (int64_t)t * n_groups;
            live[t] = j < p.n;
            const int64_t jj = live[t] ? j : j0;
            u[t] = (int64_t)__ldg(p.rid + jj);
            it[t] = (int64_t)__ldg(p.cid + jj);
            r[t] = __ldg(p.val + jj);
        }
#pragma unroll
        for (int t = 0; t < S; ++t) {
            row_load<G, NPL, VEC>(fu[t], p.U + (size_t)u[t] * k, lg, n_units);
            row_load<G, NPL, VEC>(fi[t], p.V + (size_t)it[t] * k, lg, n_units);
            bu[t] = __ldcg(p.Bu + u[t]);
            bi[t] = __ldcg(p.Bi + it[t]);
        }
#pragma unroll
        for (int t = 0; t < S; ++t) {
            float part = 0.f;
#pragma unroll
            for (int e = 0; e < E; ++e) part = fmaf(fu[t].v[e], fi[t].v[e], part);
            const float r_pred = (p.mu + bu[t] + bi[t]) + group_sum<G>(part);   // backend_cpu.pyx:67-69
            if (!live[t]) continue;
            const float err = r[t] - r_pred;                                    // :71
            if (lg == 0) loss += err * err;                                     // :72
            const float lr = p.lr, reg = p.reg;
            float* pu = p.U + (size_t)u[t] * k;
            float* pi = p.V + (size_t)it[t] * k;
            if (ATOMIC) {
                Frag du, di;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const float uf = fu[t].v[e], vf = fi[t].v[e];
                    du.v[e] = lr * (err * vf - reg * uf);
                    di.v[e] = lr * (err * uf - reg * vf);
                }
                row_red_add<G, NPL, VEC>(du, pu, lg, n_units);
                row_red_add<G, NPL, VEC>(di, pi, lg, n_units);
                if (p.use_bias && lg == 0) {
                    red_add_f32(p.Bu + u[t], lr * (err - reg * bu[t]));
                    red_add_f32(p.Bi + it[t], lr * (err - reg * bi[t]));
                }
            } else {
#pragma unroll
                for (int e = 0; e < E; ++e) {                                   // :75-78
                    const float uf = fu[t].v[e], vf = fi[t].v[e];
                    fu[t].v[e] = uf + lr * (err * vf - reg * uf);
                    fi[t].v[e] = vf + lr * (err * uf - reg * vf);
                }
                row_store<G, NPL, VEC>(fu[t], pu, lg, n_units);
                row_store<G, NPL, VEC>(fi[t], pi, lg, n_units);
                if (p.use_bias && lg == 0) {                                    // :81-83
                    __stcg(p.Bu + u[t], bu[t] + lr * (err - reg * bu[t]));
                    __stcg(p.Bi + it[t], bi[t] + lr * (err - reg * bi[t]));
                }
            }
        }
    }

    __shared__ float sh_loss[8];
    loss = group_sum<32>(loss);                 // all lanes are converged again here
    if ((threadIdx.x & 31) == 0) sh_loss[threadIdx.x >> 5] = loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tot = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += sh_loss[w];
        atomicAdd(p.loss, tot);
    }
}

template <typename IdT>
__global__ void __launch_bounds__(32) mf_replay_kernel(const MfParams<IdT> p)
{
    const int lane = threadIdx.x;
    const size_t k = (size_t)p.k;
    float loss = 0.f;
    for (int64_t base = 0; base < p.n; base += 32) {
        const int64_t s = base + lane;
        int64_t mu_ = 0, mi_ = 0;
        float mr = 0.f;
        if (s < p.n) { mu_ = (int64_t)p.rid[s]; mi_ = (int64_t)p.cid[s]; mr = p.val[s]; }
        const int n_here = (int)min((int64_t)32, p.n - base);
        for (int t = 0; t < n_here; ++t) {
            const int64_t u = __shfl_sync(0xffffffffu, mu_, t);
            const int64_t i = __shfl_sync(0xffffffffu, mi_, t);
            const float r = __shfl_sync(0xffffffffu, mr, t);
            float* pu = p.U + (size_t)u * k;
            float* pi = p.V + (size_t)i * k;
            const float bu = __ldcg(p.Bu + u), bi = __ldcg(p.Bi + i);
            float part = 0.f;
            for (int f = lane; f < p.k; f += 32) part = __fadd_rn(part, __fmul_rn(__ldcg(pu + f), __ldcg(pi + f)));
            const float r_pred = __fadd_rn(__fadd_rn(__fadd_rn(p.mu, bu), bi), group_sum<32>(part));
            const float err = __fsub_rn(r, r_pred);
            loss = __fadd_rn(loss, __fmul_rn(err, err));
            const float lr = p.lr, reg = p.reg;
            for (int f = lane; f < p.k; f += 32) {
                const float uf = __ldcg(pu + f), vf = __ldcg(pi + f);
                __stcg(pu + f, __fadd_rn(uf, __fmul_rn(lr, __fsub_rn(__fmul_rn(err, vf), __fmul_rn(reg, uf)))));
                __stcg(pi + f, __fadd_rn(vf, __fmul_rn(lr, __fsub_rn(__fmul_rn(err, uf), __fmul_rn(reg, vf)))));
            }
            if (p.use_bias && lane == 0) {
                __stcg(p.Bu + u, __fadd_rn(bu, __fmul_rn(lr, __fsub_rn(err, __fmul_rn(reg, bu)))));
                __stcg(p.Bi + i, __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(err, __fmul_rn(reg, bi)))));
            }
            __syncwarp();
        }
    }
    if (lane == 0) *p.loss = loss;
}

// Ordered mode, windowed (same idea as bpr_replay_window_kernel): 32 consecutive ratings are resolved at a
// time, one per warp, and applied as soon as no EARLIER pending rating of the window has the same user or
// the same item.  Ratings that share neither commute exactly; the per-epoch loss is summed in rating order
// afterwards from the per-rating squared errors so that it matches the reference's f32 accumulator.
template <typename IdT>
__global__ void __launch_bounds__(1024) mf_replay_window_kernel(const MfParams<IdT> p)
{
    __shared__ long long s_u[32], s_i[32];
    __shared__ int s_pending[32];
    __shared__ float s_err2[32];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t k = (size_t)p.k;
    float loss = 0.f;                               // meaningful in thread 0 only
    for (int64_t base = 0; base < p.n; base += 32) {
        const int64_t s = base + w;
        long long mu = -1, mi = -1;
        float mr = 0.f;
        bool todo = false;
        if (s < p.n) { mu = (long long)p.rid[s]; mi = (long long)p.cid[s]; mr = p.val[s]; todo = true; }
        __syncthreads();
        if (lane == 0) { s_u[w] = mu; s_i[w] = mi; s_pending[w] = todo ? 1 : 0; s_err2[w] = 0.f; }
        for (;;) {
            if (!__syncthreads_or(todo)) break;
            bool run = false;
            if (todo) {
                bool conflict = false;
                if (lane < w && s_pending[lane]) conflict = (s_u[lane] == mu) | (s_i[lane] == mi);
                run = !__any_sync(0xffffffffu, conflict);
            }
            __syncthreads();
            if (run) {
                float* pu = p.U + (size_t)mu * k;
                float* pi = p.V + (size_t)mi * k;
                const float bu = __ldcg(p.Bu + mu), bi = __ldcg(p.Bi + mi);
                float part = 0.f;
                for (int f = lane; f < p.k; f += 32) part = __fadd_rn(part, __fmul_rn(__ldcg(pu + f), __ldcg(pi + f)));
                const float r_pred = __fadd_rn(__fadd_rn(__fadd_rn(p.mu, bu), bi), group_sum<32>(part));
                const float err = __fsub_rn(mr, r_pred);
                const float lr = p.lr, reg = p.reg;
                for (int f = lane; f < p.k; f += 32) {
                    const float uf = __ldcg(pu + f), vf = __ldcg(pi + f);
                    __stcg(pu + f, __fadd_rn(uf, __fmul_rn(lr, __fsub_rn(__fmul_rn(err, vf), __fmul_rn(reg, uf)))));
                    __stcg(pi + f, __fadd_rn(vf, __fmul_rn(lr, __fsub_rn(__fmul_rn(err, uf), __fmul_rn(reg, vf)))));
                }
                if (lane == 0) {
                    if (p.use_bias) {
                        __stcg(p.Bu + mu, __fadd_rn(bu, __fmul_rn(lr, __fsub_rn(err, __fmul_rn(reg, bu)))));
                        __stcg(p.Bi + mi, __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(err, __fmul_rn(reg, bi)))));
                    }
                    s_err2[w] = __fmul_rn(err, err);
                    s_pending[w] = 0;
                }
                todo = false;
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {                     // loss += err^2 in rating order (backend_cpu.pyx:72)
            const int n_here = (int)min((int64_t)32, p.n - base);
            for (int t = 0; t < n_here; ++t) loss = __fadd_rn(loss, s_err2[t]);
        }
    }
    if (threadIdx.x == 0) *p.loss = loss;
}

template <typename IdT, int G, int NPL, bool VEC, bool ATOMIC>
static int launch_mf(const MfParams<IdT>& p, cudaStream_t st)
{
    constexpr int E = NPL * (VEC ? 4 : 1);
    constexpr int S = (E <= 4) ? 2 : 1;
    auto kern = mf_hogwild_kernel<IdT, G, NPL, VEC, ATOMIC, S>;
    const int threads = 256;
    int occ = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, 0));
    if (occ < 1) occ = 1;
    const int64_t groups_per_block = threads / G;
    int64_t want = (p.n + groups_per_block * S - 1) / (groups_per_block * S);
    int64_t grid = (int64_t)sm_count() * occ;
    if (want < grid) grid = want;
    const int64_t cap = (p.max_groups + groups_per_block * S - 1) / (groups_per_block * S);
    if (cap < grid) grid = cap;
    if (grid < 1) grid = 1;
    kern<<<(unsigned)grid, threads, 0, st>>>(p); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

template <typename IdT>
static int mf_epoch_impl(const IdT* rid, const IdT* cid, const float* val, int64_t n,
                         int64_t n_users, int64_t n_items, float* U, float* V, float* Bu, float* Bi, int k,
                         float lr, float reg, float mu, int use_bias, int ordered,
                         unsigned flags, float* loss, cudaStream_t st)
{
    MfParams<IdT> p;
    p.rid = rid; p.cid = cid; p.val = val; p.n = n;
    p.U = U; p.V = V; p.Bu = Bu; p.Bi = Bi; p.k = k;
    p.lr = lr; p.reg = reg; p.mu = mu; p.use_bias = use_bias; p.loss = loss;
    {
        const int64_t rows = n_users < n_items ? n_users : n_items;
        p.max_groups = rows / 4 < 16 ? 16 : rows / 4;
        if (flags & B200_SGD_UNBOUNDED) p.max_groups = INT64_MAX / 1024;
    }
    B200_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), st));
    if (n == 0) return B200_OK;
    if (ordered) {
        const char* serial = getenv("B200_REPLAY_SERIAL");
        ::b200::count_launch();
        if (serial && serial[0] == '1') mf_replay_kernel<IdT><<<1, 32, 0, st>>>(p);
        else mf_replay_window_kernel<IdT><<<1, 1024, 0, st>>>(p);
        B200_CUDA(cudaGetLastError());
        return B200_OK;
    }
    const RowLayout L = pick_layout(k);
    B200_REQUIRE(L.npl <= 8, "b200_mf_epoch: k=%d not supported (scalar rows are limited to k <= 256)", k);
    if (L.vec) {
        B200_REQUIRE((((uintptr_t)U | (uintptr_t)V) & 15) == 0, "b200_mf_epoch: U/V must be 16-byte aligned");
    }
    const bool atomic = flags & B200_SGD_ATOMIC;
#define CALL(G_, NPL_, VEC_)                                                              \
    do {                                                                                  \
        int rc = atomic ? launch_mf<IdT, G_, NPL_, VEC_, true>(p, st)                     \
                        : launch_mf<IdT, G_, NPL_, VEC_, false>(p, st);                   \
        if (rc) return rc;                                                                \
    } while (0)
    B200_DISPATCH_LAYOUT(L, CALL);
#undef CALL
    return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_mf_epoch(const void* rid, const void* cid, const float* val, int64_t n, int ids_are_i32,
                             int64_t n_users, int64_t n_items, float* U, float* V, float* Bu, float* Bi, int k,
                             float lr, float reg, float mu, int use_bias, int ordered,
                             unsigned flags, float* loss, void* stream)
{
    B200_REQUIRE(Bu && Bi && loss && (k == 0 || (U && V)), "b200_mf_epoch: null pointer argument");
    B200_REQUIRE(n >= 0 && (n == 0 || (rid && cid && val)), "b200_mf_epoch: bad rating arrays");
    B200_REQUIRE(k >= 0 && k <= 1024, "b200_mf_epoch: k=%d out of range [0, 1024]", k);
    B200_REQUIRE(n_users >= 1 && n_items >= 1, "b200_mf_epoch: bad n_users/n_items");
    cudaStream_t st = (cudaStream_t)stream;
    if (ids_are_i32)
        return mf_epoch_impl<int32_t>((const int32_t*)rid, (const int32_t*)cid, val, n, n_users, n_items, U, V, Bu, Bi, k, lr, reg, mu,
                                      use_bias, ordered, flags, loss, st);
    return mf_epoch_impl<int64_t>((const int64_t*)rid, (const int64_t*)cid, val, n, n_users, n_items, U, V, Bu, Bi, k, lr, reg, mu,
                                  use_bias, ordered, flags, loss, st);
}
