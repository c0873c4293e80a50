// PMF (cornac/models/pmf/cython/pmf.pyx:55-173) for sm_90a: the level schedule of the ratings (host) and the fit,
// all epochs in one launch of one CTA that walks the levels with a barrier between consecutive levels.  SoRec and MCF
// (sorec.pyx / mcf.pyx) are the same epoch over a mixed stream of graph edges and ratings: b200_cofactor_schedule /
// b200_cofactor_fit below, on the same level rule, sigmoid and RMSProp step.
//
// The reference's extension is built without extra compile flags (setup.py:161-165): plain IEEE f64, no FMA, dots summed
// serially in index order.  Every operation below is therefore an explicitly rounded __d*_rn intrinsic, in the
// reference's order.  lambda_reg, learning_rate and gamma arrive as C floats and are used in f64 expressions; the
// ratings are f32 promoted to f64.
//
// Thread mapping: one thread per rating.  A rating's dot is a serial chain of k products and sums whatever the mapping,
// and the element-wise RMSProp steps of one rating are independent across f, so a single thread keeps them in flight
// together; the ratings of one level run side by side.  A level wider than the CTA is a loop.
#include "common.cuh"
#include "expf.cuh"

#include <algorithm>
#include <vector>

namespace b200 {

constexpr int PMF_THREADS = 256;

// pmf.pyx:27-37
__device__ __forceinline__ float pmf_sigmoid(float z)
{
    if (z > 6.0f) return 1.0f;
    if (z < -6.0f) return 0.0f;
    return __double2float_rn(__ddiv_rn(1.0, __dadd_rn(1.0, (double)pmf_expf(-z))));
}

// One RMSProp element step (pmf.pyx:88-90 / 94-96): g = we*other - lam*x; c = gam*c + (1-gam)*g*g;
// x += lr * (g / (sqrt(c) + eps)).  Returns the new x.
__device__ __forceinline__ double rmsprop(double x, double other, double we, double& c, double lam, double gam, double omg,
                                          double lr)
{
    const double g = __dsub_rn(__dmul_rn(we, other), __dmul_rn(lam, x));
    c = __dadd_rn(__dmul_rn(gam, c), __dmul_rn(omg, __dmul_rn(g, g)));
    return __dadd_rn(x, __dmul_rn(lr, __ddiv_rn(g, __dadd_rn(__dsqrt_rn(c), 1e-8))));
}

template <bool NON_LINEAR>
__global__ void __launch_bounds__(PMF_THREADS) pmf_fit_kernel(
    const int32_t* __restrict__ uid, const int32_t* __restrict__ iid, const float* __restrict__ rat,
    const int32_t* __restrict__ level_ptr, int32_t n_levels, int64_t nnz, int k,
    double* U, double* V, double* cache_u, double* cache_v,
    int n_epochs, float lambda_reg, float learning_rate, float gamma,
    double* __restrict__ loss, const int32_t* __restrict__ order)
{
    const double lam = (double)lambda_reg, lr = (double)learning_rate, gam = (double)gamma;
    const double omg = __dsub_rn(1.0, gam);
    for (int epoch = 0; epoch < n_epochs; ++epoch) {
        for (int32_t l = 0; l < n_levels; ++l) {
            const int32_t lo = __ldg(level_ptr + l), hi = __ldg(level_ptr + l + 1);
            for (int32_t s = lo + (int32_t)threadIdx.x; s < hi; s += PMF_THREADS) {
                const int32_t u = __ldg(uid + s), i = __ldg(iid + s);
                const double val = (double)__ldg(rat + s);
                // rows written by other threads of this CTA in earlier levels: plain (coherent) loads, ordered by the barrier
                double* Ur = U + (size_t)u * k;
                double* Vr = V + (size_t)i * k;
                double* cu = cache_u + (size_t)u * k;
                double* cv = cache_v + (size_t)i * k;
                double dot = 0.0;
                for (int f = 0; f < k; ++f) dot = __dadd_rn(dot, __dmul_rn(Ur[f], Vr[f]));
                double e, we;
                if constexpr (NON_LINEAR) {                    // pmf.pyx:144-146
                    const double sg = (double)pmf_sigmoid(__double2float_rn(dot));
                    e = __dsub_rn(val, sg);
                    we = __dmul_rn(__dmul_rn(e, sg), __dsub_rn(1.0, sg));
                } else {                                       // pmf.pyx:84
                    e = __dsub_rn(val, dot);
                    we = e;
                }
                // The user loop reads V before the item loop changes it and element f of the item loop reads only the
                // new U[f]: one fused pass over f applies both loops in the reference's order.
                double nu = 0.0, nv = 0.0;
                for (int f = 0; f < k; ++f) {
                    double c_u = cu[f], c_v = cv[f];
                    const double v0 = Vr[f];
                    const double u1 = rmsprop(Ur[f], v0, we, c_u, lam, gam, omg, lr);
                    const double v1 = rmsprop(v0, u1, we, c_v, lam, gam, omg, lr);
                    Ur[f] = u1; Vr[f] = v1; cu[f] = c_u; cv[f] = c_v;
                    nu = __dadd_rn(nu, __dmul_rn(u1, u1));
                    nv = __dadd_rn(nv, __dmul_rn(v1, v1));
                }
                if (loss)                                      // pmf.pyx:98-104
                    loss[(size_t)epoch * nnz + __ldg(order + s)] = __dadd_rn(__dmul_rn(e, e), __dmul_rn(lam, __dadd_rn(nu, nv)));
            }
            __syncthreads();
        }
    }
}

// The co-factor fit of SoRec (cornac/models/sorec/cython/sorec.pyx:40-147) and MCF (cornac/models/mcf/cython/mcf.pyx:43-148):
// per epoch the non-linear PMF update over the graph edges, then over the ratings.  Slot s updates rows a[s] of A and b[s]
// of B with one of two bindings (is_edge[s]: the edge pass's, else the rating pass's); a cache belongs to its matrix, so
// a row shared by both passes (SoRec's U, MCF's V) steps one cache.  The two rows of one update are always different
// matrices, so the fused loop over f is pmf_fit_kernel's.  A kernel of its own rather than a second binding in
// pmf_fit_kernel: PMF's slot stays three loads and no select.
struct CofactorBinding {
    double* A;
    double* B;
    double* cache_a;
    double* cache_b;
    double step;                     // the factor of g / (sqrt(c) + eps): (double) of the reference's f32 step
};

__global__ void __launch_bounds__(PMF_THREADS) cofactor_fit_kernel(
    const int32_t* __restrict__ a_id, const int32_t* __restrict__ b_id, const float* __restrict__ val,
    const uint8_t* __restrict__ is_edge, const int32_t* __restrict__ level_ptr, int32_t n_levels, int64_t n_total, int k,
    CofactorBinding edge, CofactorBinding rating, int n_epochs, float lambda_reg, float gamma,
    double* __restrict__ loss, const int32_t* __restrict__ order)
{
    const double lam = (double)lambda_reg, gam = (double)gamma;
    const double omg = __dsub_rn(1.0, gam);
    for (int epoch = 0; epoch < n_epochs; ++epoch) {
        for (int32_t l = 0; l < n_levels; ++l) {
            const int32_t lo = __ldg(level_ptr + l), hi = __ldg(level_ptr + l + 1);
            for (int32_t s = lo + (int32_t)threadIdx.x; s < hi; s += PMF_THREADS) {
                const bool ed = __ldg(is_edge + s) != 0;      // field-wise selects: no copy of a parameter struct
                const size_t oa = (size_t)__ldg(a_id + s) * k, ob = (size_t)__ldg(b_id + s) * k;
                const double v = (double)__ldg(val + s), step = ed ? edge.step : rating.step;
                double* Ar = (ed ? edge.A : rating.A) + oa;
                double* Br = (ed ? edge.B : rating.B) + ob;
                double* ca = (ed ? edge.cache_a : rating.cache_a) + oa;
                double* cb = (ed ? edge.cache_b : rating.cache_b) + ob;
                double dot = 0.0;
                for (int f = 0; f < k; ++f) dot = __dadd_rn(dot, __dmul_rn(Ar[f], Br[f]));
                const double sg = (double)pmf_sigmoid(__double2float_rn(dot));      // sorec.pyx:87-89
                const double e = __dsub_rn(v, sg);
                const double we = __dmul_rn(__dmul_rn(e, sg), __dsub_rn(1.0, sg));
                double na = 0.0, nb = 0.0;
                for (int f = 0; f < k; ++f) {
                    double c_a = ca[f], c_b = cb[f];
                    const double b0 = Br[f];
                    const double a1 = rmsprop(Ar[f], b0, we, c_a, lam, gam, omg, step);
                    const double b1 = rmsprop(b0, a1, we, c_b, lam, gam, omg, step);
                    Ar[f] = a1; Br[f] = b1; ca[f] = c_a; cb[f] = c_b;
                    na = __dadd_rn(na, __dmul_rn(a1, a1));
                    nb = __dadd_rn(nb, __dmul_rn(b1, b1));
                }
                if (loss)                                      // sorec.pyx:103-109 / 134-140 (x + y == y + x exactly)
                    loss[(size_t)epoch * n_total + __ldg(order + s)] = __dadd_rn(__dmul_rn(e, e), __dmul_rn(lam, __dadd_rn(na, nb)));
            }
            __syncthreads();
        }
    }
}

__global__ void pmf_sigmoid_kernel(const float* __restrict__ z, int64_t n, float* __restrict__ out)
{
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x)
        out[j] = pmf_sigmoid(__ldg(z + j));
}

// The level schedule of n updates that each touch two rows of one id space of n_rows rows (rows(r, a, b) gives update r's
// rows, already range-checked): level(r) = 1 + max(level of the previous update of row a, of row b).  Writes order (the
// update of each slot, level-major, stored order inside a level), level_ptr[0 .. depth] and returns depth.
template <class Rows>
int32_t level_schedule(int64_t n, int64_t n_rows, Rows rows, int32_t* order, int32_t* level_ptr)
{
    std::vector<int32_t> last((size_t)n_rows, 0), level((size_t)n);
    int32_t depth = 0;
    for (int64_t r = 0; r < n; ++r) {
        int64_t a, b;
        rows(r, a, b);
        const int32_t lv = std::max(last[a], last[b]) + 1;
        last[a] = last[b] = level[r] = lv;
        depth = std::max(depth, lv);
    }
    // counting sort by level, stable: level_ptr[l] = first slot of level l (levels numbered from 0 here)
    std::fill(level_ptr, level_ptr + depth + 1, 0);
    for (int64_t r = 0; r < n; ++r) ++level_ptr[level[r]];
    for (int32_t l = 0; l < depth; ++l) level_ptr[l + 1] += level_ptr[l];
    std::vector<int32_t> next(level_ptr, level_ptr + depth);
    for (int64_t r = 0; r < n; ++r) order[next[level[r] - 1]++] = (int32_t)r;
    return depth;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_pmf_schedule(const int32_t* uid, const int32_t* iid, int64_t nnz, int64_t n_users, int64_t n_items,
                                 int32_t* order, int32_t* level_ptr, int32_t* n_levels)
{
    B200_REQUIRE(n_levels && level_ptr && (nnz == 0 || (uid && iid && order)), "b200_pmf_schedule: null pointer argument");
    B200_REQUIRE(nnz >= 0 && nnz < (1ll << 31) && n_users >= 0 && n_items >= 0, "b200_pmf_schedule: bad sizes nnz=%lld",
                 (long long)nnz);
    for (int64_t r = 0; r < nnz; ++r) {
        const int32_t u = uid[r], i = iid[r];
        B200_REQUIRE(u >= 0 && u < n_users && i >= 0 && i < n_items,
                     "b200_pmf_schedule: rating %lld has (user %d, item %d) outside [0, %lld) x [0, %lld)", (long long)r, u, i,
                     (long long)n_users, (long long)n_items);
    }
    // rows: users [0, n_users), then items
    *n_levels = level_schedule(nnz, n_users + n_items, [&](int64_t r, int64_t& a, int64_t& b) {
        a = uid[r];
        b = n_users + iid[r];
    }, order, level_ptr);
    return B200_OK;
}

extern "C" int b200_cofactor_schedule(int variant, const int32_t* net_a, const int32_t* net_b, int64_t n_edges,
                                      const int32_t* uid, const int32_t* iid, int64_t n_ratings, int64_t n_users,
                                      int64_t n_items, int32_t* order, int32_t* level_ptr, int32_t* n_levels)
{
    B200_REQUIRE(variant == B200_COFACTOR_SOREC || variant == B200_COFACTOR_MCF, "b200_cofactor_schedule: unknown variant %d",
                 variant);
    B200_REQUIRE(n_levels && level_ptr && (n_edges == 0 || (net_a && net_b)) && (n_ratings == 0 || (uid && iid)) &&
                 (n_edges + n_ratings == 0 || order), "b200_cofactor_schedule: null pointer argument");
    B200_REQUIRE(n_edges >= 0 && n_ratings >= 0 && n_edges + n_ratings < (1ll << 31) && n_users >= 0 && n_items >= 0,
                 "b200_cofactor_schedule: bad sizes n_edges=%lld n_ratings=%lld", (long long)n_edges, (long long)n_ratings);
    // SoRec's edges join users (U row, Z row), MCF's join items (V row, Z row); Z has as many rows as the graph has nodes
    const bool sorec = variant == B200_COFACTOR_SOREC;
    const int64_t n_nodes = sorec ? n_users : n_items;
    for (int64_t e = 0; e < n_edges; ++e)
        B200_REQUIRE(net_a[e] >= 0 && net_a[e] < n_nodes && net_b[e] >= 0 && net_b[e] < n_nodes,
                     "b200_cofactor_schedule: edge %lld has (%d, %d) outside [0, %lld) x [0, %lld)", (long long)e, net_a[e],
                     net_b[e], (long long)n_nodes, (long long)n_nodes);
    for (int64_t r = 0; r < n_ratings; ++r)
        B200_REQUIRE(uid[r] >= 0 && uid[r] < n_users && iid[r] >= 0 && iid[r] < n_items,
                     "b200_cofactor_schedule: rating %lld has (user %d, item %d) outside [0, %lld) x [0, %lld)", (long long)r,
                     uid[r], iid[r], (long long)n_users, (long long)n_items);
    // rows: U [0, n_users), V [n_users, n_users + n_items), Z after them; edges are updates [0, n_edges), ratings follow
    const int64_t v0 = n_users, z0 = n_users + n_items, a0 = sorec ? 0 : v0;
    *n_levels = level_schedule(n_edges + n_ratings, z0 + n_nodes, [&](int64_t s, int64_t& a, int64_t& b) {
        if (s < n_edges) {
            a = a0 + net_a[s];
            b = z0 + net_b[s];
        } else {
            a = uid[s - n_edges];
            b = v0 + iid[s - n_edges];
        }
    }, order, level_ptr);
    return B200_OK;
}

extern "C" int b200_pmf_fit(int variant, const int32_t* uid, const int32_t* iid, const float* rat, const int32_t* level_ptr,
                            int32_t n_levels, int64_t nnz, int k, double* U, double* V, double* cache_u, double* cache_v,
                            int n_epochs, float lambda_reg, float learning_rate, float gamma, double* loss,
                            const int32_t* order, void* stream)
{
    B200_REQUIRE(variant == B200_PMF_LINEAR || variant == B200_PMF_NON_LINEAR, "b200_pmf_fit: unknown variant %d", variant);
    B200_REQUIRE(k >= 1 && n_epochs >= 0 && n_levels >= 0 && nnz >= 0 && nnz < (1ll << 31),
                 "b200_pmf_fit: bad sizes k=%d n_epochs=%d n_levels=%d nnz=%lld", k, n_epochs, n_levels, (long long)nnz);
    B200_REQUIRE(U && V && cache_u && cache_v && level_ptr, "b200_pmf_fit: null pointer argument");
    B200_REQUIRE(nnz == 0 || (uid && iid && rat), "b200_pmf_fit: null rating arrays");
    B200_REQUIRE(!loss || order, "b200_pmf_fit: loss needs order");
    if (n_epochs == 0 || nnz == 0) return B200_OK;
    if (variant == B200_PMF_NON_LINEAR)
        pmf_fit_kernel<true><<<1, PMF_THREADS, 0, (cudaStream_t)stream>>>(uid, iid, rat, level_ptr, n_levels, nnz, k, U, V, cache_u,
                                                                        cache_v, n_epochs, lambda_reg, learning_rate, gamma, loss, order);
    else
        pmf_fit_kernel<false><<<1, PMF_THREADS, 0, (cudaStream_t)stream>>>(uid, iid, rat, level_ptr, n_levels, nnz, k, U, V, cache_u,
                                                                         cache_v, n_epochs, lambda_reg, learning_rate, gamma, loss, order);
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_cofactor_fit(int variant, const int32_t* a_id, const int32_t* b_id, const float* val,
                                 const uint8_t* is_edge, const int32_t* level_ptr, int32_t n_levels, int64_t n_edges,
                                 int64_t n_ratings, int k, double* U, double* V, double* Z, double* cache_u, double* cache_v,
                                 double* cache_z, int n_epochs, float lambda_c, float lambda_reg, float learning_rate,
                                 float gamma, double* loss, const int32_t* order, void* stream)
{
    B200_REQUIRE(variant == B200_COFACTOR_SOREC || variant == B200_COFACTOR_MCF, "b200_cofactor_fit: unknown variant %d",
                 variant);
    const int64_t n_total = n_edges + n_ratings;
    B200_REQUIRE(k >= 1 && n_epochs >= 0 && n_levels >= 0 && n_edges >= 0 && n_ratings >= 0 && n_total < (1ll << 31),
                 "b200_cofactor_fit: bad sizes k=%d n_epochs=%d n_levels=%d n_edges=%lld n_ratings=%lld", k, n_epochs,
                 n_levels, (long long)n_edges, (long long)n_ratings);
    B200_REQUIRE(U && V && Z && cache_u && cache_v && cache_z && level_ptr, "b200_cofactor_fit: null pointer argument");
    B200_REQUIRE(n_total == 0 || (a_id && b_id && val && is_edge), "b200_cofactor_fit: null slot arrays");
    B200_REQUIRE(!loss || order, "b200_cofactor_fit: loss needs order");
    if (n_epochs == 0 || n_total == 0) return B200_OK;
    // sorec.pyx:95 `lambda_c * learning_rate * (...)`: two C floats, so the step is their f32 product
    const float edge_step = variant == B200_COFACTOR_SOREC ? lambda_c * learning_rate : learning_rate;
    const CofactorBinding edge = variant == B200_COFACTOR_SOREC
                                     ? CofactorBinding{U, Z, cache_u, cache_z, (double)edge_step}
                                     : CofactorBinding{V, Z, cache_v, cache_z, (double)edge_step};
    const CofactorBinding rating{U, V, cache_u, cache_v, (double)learning_rate};
    cofactor_fit_kernel<<<1, PMF_THREADS, 0, (cudaStream_t)stream>>>(a_id, b_id, val, is_edge, level_ptr, n_levels, n_total,
                                                                    k, edge, rating, n_epochs, lambda_reg, gamma, loss, order);
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_pmf_sigmoid(const float* z, int64_t n, float* out, void* stream)
{
    B200_REQUIRE(n >= 0 && (n == 0 || (z && out)), "b200_pmf_sigmoid: bad arguments");
    if (n == 0) return B200_OK;
    int64_t grid = (n + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    pmf_sigmoid_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(z, n, out);
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
