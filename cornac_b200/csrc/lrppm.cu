// LRPPM (cornac/models/lrppm/recom_lrppm.pyx:356-560) for sm_90a: the fit, bit-identical to the reference's compiled
// float loop given the same sample draws and stopping where it converges, and the aspect-mixed rank rows.
//
// One iteration of the reference reads the parameters it started with everywhere and writes them only in its final
// dense step, so it splits into independent chains:
//   phase 1  a thread per sample: the predictions, the skip test and the sample's coefficients (del_sqerror of a rating
//            sample; del_ranking and del_rating of a ranking sample), and a mark on every row it touches.
//   phase 2  a warp per touched row, a lane per factor: the row's `del` as one ordered f32 chain over the samples that
//            touch it (rating samples first, then per ranking sample its ranking term and then its rating term).  The
//            warp finds the samples 32 at a time with a ballot and adds them in sample order.
//   phase 3  the dense step over every element, fused with numpy's isclose against the value the iteration started
//            with; an element that is not close sets the iteration's "changed" flag.
// After the last barrier every block reads the flag and stops after the first iteration that changed nothing, as the
// reference's `np.all(np.isclose(...))` test does.  A call of n iterations is one cooperative launch.
//
// The arithmetic is the one gcc -O3 -ffast-math made of the float specialisation of `_fit` (x86-64, SSE2, no FMA):
//   * the rating dot U[u] . I[i] is a serial f32 sum in k order;
//   * get_score is vectorised over pairs of k: lane k % 2 sums (UA[a, k] + I[i, k]) * U[u, k] + IA[a, k] * I[i, k],
//     the two lanes are added, and an odd k leaves a scalar tail (score_k below); k <= 3 runs the scalar code alone;
//   * exp(pred) is glibc's expf, z = f32(1.0 / (1.0 + (double)expf(pred)));
//   * the clamp `if x < 0: x = 0` is maxss(x, 0): NaN and -0.0 become +0.0;
//   * the test `del != 0` is comiss: a NaN del takes the `del == 0` branch.  For U, I and IA that branch only clamps;
//     for UA it still subtracts lr * del (so a NaN del gives 0).
#include "common.cuh"
#include "expf.cuh"

#include <cooperative_groups.h>

#include <algorithm>

namespace cg = cooperative_groups;

namespace b200 {

constexpr int LR_THREADS = 256;
enum { L_U = 0, L_I, L_UA, L_IA, L_N };

struct LrppmArgs {
    int64_t rows[L_N];
    int k;
    const int32_t *r_u, *r_i;
    const float* r_val;
    int64_t n_r;
    const int32_t *x_u, *x_i, *x_a;
    const float* x_l;
    int64_t n_x;
    const int32_t* akeys;        // sorted distinct get_key3(u, i, a) of the review triples (C int, wrapped)
    int64_t n_akeys;
    const int32_t* rkeys;        // sorted distinct get_key(u, i) of the ratings, and the f32 value the dict keeps
    const float* rvals;
    int64_t n_rkeys;
    int n_s, n_rank, n_iter;
    const int32_t* draws;        // [n_iter][n_s + 2 n_rank]: pos, pos_uia, neg_uia
    float* P[L_N];
    float* D[L_N];
    float* coef;                 // [n_s + 2 n_rank]: del_sqerror per rating sample, (del_ranking, del_rating) per ranking
    int32_t* ids;                // [2 n_s + 5 n_rank]: (u, i) per rating sample, (u, i, a, a_j, live) per ranking sample
    uint8_t* touched;            // per row of U, I, UA, IA
    int64_t row_off[L_N];
    float lr, reg, ld;
    unsigned int* changed;       // [2]: per iteration parity
    unsigned long long* counts;  // += correct, skipped, iterations run; [3] = 1 when the fit converged
    double* losses;              // += loss, ranking_loss, r_loss (f64) or NULL
    int philox;
    uint32_t key0, key1;
    uint64_t iter0;
    unsigned long long* phase_ns;
};

// get_key of recom_mter.pyx in C int: (i + j) (i + j + 1) // 2 + j with two's-complement wrap
__host__ __device__ __forceinline__ int32_t lr_key(int32_t i, int32_t j)
{
    const uint32_t s = (uint32_t)i + (uint32_t)j;
    const int32_t p = (int32_t)(s * (s + 1u));
    return (int32_t)((uint32_t)(p >> 1) + (uint32_t)j);
}

__device__ __forceinline__ int64_t sorted_find(const int32_t* keys, int64_t n, int32_t key)
{
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo) / 2;
        if (keys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return (lo < n && keys[lo] == key) ? lo : -1;
}

__device__ __forceinline__ int64_t lr_draw(const LrppmArgs& a, const int32_t* dr, int it, int64_t j, int64_t n)
{
    if (!a.philox) return dr[j];
    const uint64_t itg = a.iter0 + (uint64_t)it;
    const Philox4 r = philox4x32_10((uint32_t)j, (uint32_t)itg, (uint32_t)(itg >> 32), 0x4c525050u, a.key0, a.key1);
    return (int64_t)range64(r.x, r.y, (uint64_t)n);
}

__device__ __forceinline__ float dot_serial(const float* x, const float* y, int k)
{
    float s = 0.f;
    for (int f = 0; f < k; ++f) s = __fadd_rn(s, __fmul_rn(x[f], y[f]));
    return s;
}

// get_score as compiled: see the file comment
__device__ float score_k(const float* U, const float* I, const float* UA, const float* IA, int k)
{
    auto t = [&](int f) { return __fmul_rn(__fadd_rn(UA[f], I[f]), U[f]); };
    auto w = [&](int f) { return __fmul_rn(IA[f], I[f]); };
    float s = 0.f;
    int f = 0;
    if (k > 3) {
        float l0 = 0.f, l1 = 0.f;
        for (; f + 1 < k; f += 2) {
            l0 = __fadd_rn(l0, __fadd_rn(t(f), w(f)));
            l1 = __fadd_rn(l1, __fadd_rn(t(f + 1), w(f + 1)));
        }
        s = __fadd_rn(l1, l0);
        if (f < k) s = __fadd_rn(__fadd_rn(s, w(f)), t(f));
        return s;
    }
    if (k > 0) s = __fadd_rn(__fadd_rn(s, w(0)), t(0));
    if (k > 1) s = __fadd_rn(__fadd_rn(s, t(1)), w(1));
    if (k > 2) s = __fadd_rn(s, __fadd_rn(t(2), w(2)));
    return s;
}

__device__ __forceinline__ void mark(const LrppmArgs& a, int m, int32_t row)
{
    a.touched[a.row_off[m] + row] = 1;
}

// phase 1
__device__ void lr_predict(const LrppmArgs& a, const int32_t* dr, int it)
{
    const int k = a.k;
    const float *U = a.P[L_U], *I = a.P[L_I], *UA = a.P[L_UA], *IA = a.P[L_IA];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < a.n_s + a.n_rank; w += stride) {
        if (w < a.n_s) {
            const int64_t idx = lr_draw(a, dr, it, w, a.n_r);
            const int32_t u = a.r_u[idx], i = a.r_i[idx];
            const float score = a.r_val[idx];
            const float rp = dot_serial(U + (int64_t)u * k, I + (int64_t)i * k, k);
            const float d = __fsub_rn(rp, score);
            a.coef[w] = __fadd_rn(d, d);
            a.ids[2 * w] = u;
            a.ids[2 * w + 1] = i;
            mark(a, L_U, u);
            mark(a, L_I, i);
            if (a.losses) atomicAdd(a.losses, (double)__fmul_rn(d, d));
        } else {
            const int64_t t = w - a.n_s;
            const int64_t idx = lr_draw(a, dr, it, a.n_s + t, a.n_x);
            const int32_t aj = (int32_t)lr_draw(a, dr, it, a.n_s + a.n_rank + t, a.rows[L_UA]);
            const int32_t u = a.x_u[idx], i = a.x_i[idx], as = a.x_a[idx];
            int32_t* id = a.ids + 2ll * a.n_s + 5 * t;
            id[0] = u; id[1] = i; id[2] = as; id[3] = aj;
            if (sorted_find(a.akeys, a.n_akeys, lr_key(lr_key(u, i), aj)) >= 0) {
                id[4] = 0;
                atomicAdd(a.counts + 1, 1ull);
                continue;
            }
            id[4] = 1;
            const float *Uu = U + (int64_t)u * k, *Ii = I + (int64_t)i * k;
            const float sa = score_k(Uu, Ii, UA + (int64_t)as * k, IA + (int64_t)as * k, k);
            const float sj = score_k(Uu, Ii, UA + (int64_t)aj * k, IA + (int64_t)aj * k, k);
            const float pred = __fsub_rn(sa, sj);
            const float z = __double2float_rn(__ddiv_rn(1.0, __dadd_rn(1.0, (double)glibc_expf(pred))));
            if (z < 0.5f) atomicAdd(a.counts + 0, 1ull);
            const float rp = dot_serial(Uu, Ii, k);
            const int64_t kp = sorted_find(a.rkeys, a.n_rkeys, lr_key(u, i));
            const float score = kp >= 0 ? a.rvals[kp] : 0.f;       // operator[] of an absent key reads 0
            const float l = a.x_l[idx];
            const float diff = __fsub_rn(score, rp);
            a.coef[a.n_s + 2 * t] = __fmul_rn(a.ld, z);
            a.coef[a.n_s + 2 * t + 1] = __fmul_rn(__fmul_rn(2.f, l), diff);    // f32(2.0 * l * diff): one rounding
            mark(a, L_U, u);
            mark(a, L_I, i);
            mark(a, L_UA, as);
            mark(a, L_UA, aj);
            mark(a, L_IA, as);
            mark(a, L_IA, aj);
            if (a.losses) {
                atomicAdd(a.losses + 1, (double)a.ld * log(1.0 / (1.0 + (double)glibc_expf(-pred))));
                atomicAdd(a.losses + 2, (double)__fmul_rn(__fmul_rn(l, diff), diff));
            }
        }
    }
}

// phase 2: the del row of (matrix m, row) in the reference's order; a lane per factor
__device__ void lr_row_chain(const LrppmArgs& a, int m, int32_t row, int lane)
{
    const int k = a.k;
    const float *U = a.P[L_U], *I = a.P[L_I], *UA = a.P[L_UA], *IA = a.P[L_IA];
    for (int f0 = 0; f0 < k; f0 += 32) {
        const int f = f0 + lane;
        const bool on = f < k;
        float acc = 0.f;
        if (m <= L_I) {
            for (int64_t b = 0; b < a.n_s; b += 32) {
                const int64_t t = b + lane;
                const bool hit = t < a.n_s && a.ids[2 * t + m] == row;
                unsigned mask = __ballot_sync(0xffffffffu, hit);
                while (mask) {
                    const int64_t s = b + __ffs(mask) - 1;
                    mask &= mask - 1;
                    if (on) {
                        const float c = a.coef[s];
                        const int32_t o = a.ids[2 * s + 1 - m];
                        acc = __fadd_rn(acc, __fmul_rn(c, (m == L_U ? I : U)[(int64_t)o * k + f]));
                    }
                }
            }
        }
        const int32_t* ids = a.ids + 2ll * a.n_s;
        for (int64_t b = 0; b < a.n_rank; b += 32) {
            const int64_t t = b + lane;
            bool hit = false;
            if (t < a.n_rank && ids[5 * t + 4]) {
                const int32_t* id = ids + 5 * t;
                hit = m <= L_I ? id[m] == row : (id[2] == row || id[3] == row);
            }
            unsigned mask = __ballot_sync(0xffffffffu, hit);
            while (mask) {
                const int64_t s = b + __ffs(mask) - 1;
                mask &= mask - 1;
                if (!on) continue;
                const int32_t* id = ids + 5 * s;
                const int64_t u = id[0], i = id[1], as = id[2], aj = id[3];
                const float dr = a.coef[a.n_s + 2 * s], dt = a.coef[a.n_s + 2 * s + 1];
                if (m == L_U) {
                    acc = __fsub_rn(acc, __fmul_rn(dr, __fsub_rn(UA[as * k + f], UA[aj * k + f])));
                    acc = __fadd_rn(acc, __fmul_rn(dt, I[i * k + f]));
                } else if (m == L_I) {
                    acc = __fsub_rn(acc, __fmul_rn(dr, __fsub_rn(IA[as * k + f], IA[aj * k + f])));
                    acc = __fadd_rn(acc, __fmul_rn(dt, U[u * k + f]));
                } else {
                    const float v = __fmul_rn(dr, (m == L_UA ? U[u * k + f] : I[i * k + f]));
                    acc = as == row ? __fsub_rn(acc, v) : __fadd_rn(acc, v);
                }
            }
        }
        if (on) a.D[m][(int64_t)row * k + f] = acc;
    }
}

__device__ void lr_gradients(const LrppmArgs& a)
{
    const int64_t n_rows = a.row_off[L_IA] + a.rows[L_IA];
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5); r < n_rows; r += warps) {
        if (!a.touched[r]) continue;
        int m = L_IA;
        while (r < a.row_off[m]) --m;
        lr_row_chain(a, m, (int32_t)(r - a.row_off[m]), lane);
        __syncwarp();
        if (lane == 0) a.touched[r] = 0;
    }
}

// numpy 2 isclose(x, y) of f32 arrays: |x - y| <= f32(1e-8) + f32(1e-5) |y| with y finite, or x == y
__device__ __forceinline__ bool lr_isclose(float x, float y)
{
    const float tol = __fadd_rn(1e-8f, __fmul_rn(1e-5f, fabsf(y)));
    return (fabsf(__fsub_rn(x, y)) <= tol && isfinite(y)) || x == y;
}

// phase 3
__device__ void lr_step(const LrppmArgs& a, unsigned int* changed)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    bool diff = false;
    for (int m = 0; m < L_N; ++m) {
        float *x = a.P[m], *del = a.D[m];
        for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < a.rows[m] * a.k; e += stride) {
            const float xv = x[e];
            float d = del[e];
            float nx;
            if (d != 0.f && !isnan(d)) {
                d = __fadd_rn(d, __fmul_rn(a.reg, xv));
                del[e] = 0.f;
                nx = __fsub_rn(xv, __fmul_rn(a.lr, d));
            } else if (m == L_UA) {
                del[e] = 0.f;
                nx = __fsub_rn(xv, __fmul_rn(a.lr, d));
            } else {
                del[e] = 0.f;
                nx = xv;
            }
            nx = nx > 0.f ? nx : 0.f;                   // maxss(nx, 0): NaN and -0.0 give +0.0
            x[e] = nx;
            diff |= !lr_isclose(nx, xv);
        }
    }
    if (__syncthreads_or(diff) && threadIdx.x == 0) atomicAdd(changed, 1u);
}

__device__ __forceinline__ uint64_t lr_ns()
{
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__global__ void __launch_bounds__(LR_THREADS) lrppm_fit_kernel(LrppmArgs a)
{
    cg::grid_group grid = cg::this_grid();
    const int64_t per_iter = a.n_s + 2ll * a.n_rank;
    const bool timer = a.phase_ns && blockIdx.x == 0 && threadIdx.x == 0;
    uint64_t t0 = timer ? lr_ns() : 0;
    auto tick = [&](int p) {
        if (timer) {
            const uint64_t t1 = lr_ns();
            a.phase_ns[p] += t1 - t0;
            t0 = t1;
        }
    };
    int it = 0;
    bool converged = false;
    while (it < a.n_iter) {
        lr_predict(a, a.draws + (a.philox ? 0 : per_iter * it), it);
        grid.sync();
        tick(0);
        // every block read the flag of the other parity after the last iteration's final barrier
        if (blockIdx.x == 0 && threadIdx.x == 0) a.changed[(it + 1) & 1] = 0;
        lr_gradients(a);
        grid.sync();
        tick(1);
        lr_step(a, a.changed + (it & 1));
        grid.sync();
        tick(2);
        ++it;
        if (*(volatile unsigned int*)(a.changed + ((it - 1) & 1)) == 0) {
            converged = true;
            break;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.counts[2] += (unsigned long long)it;
        if (converged) a.counts[3] = 1;
    }
}

// The rank rows (recom_lrppm.pyx:519-530) of user u over items [0, n_items), in f64:
//   s[i, a] = f32(f32(f32(UA[a] . U[u]) + f32(I[i] . IA[a])) + f32(I[i] . U[u]))   (each dot an f64 index-order sum)
//   out[i] = alpha * (sum over the n_top largest s[i, :] of s * q[i, a]) / n_top * rating_scale
//            + f32(f32(1 - alpha) * f32(I[i] . U[u]))   (numpy's f32 product of the reference)
// q is the item x aspect quality CSR (f64; an absent entry is 0).  A block per (tile of LR_ITEMS items, user) stages
// UA . U[u] in shared memory; a warp per item holds s[i, lane + 32 j] in registers and the item's q row in a dense
// shared strip.  With n_top < n_aspects the n_top-th largest value is found exactly by bisection over the 32 bits of an
// order-preserving key; values above it are taken, and at a tie the smaller aspect ids (numpy's argsort there is not
// stable, so this is a choice).
constexpr int LR_RANK_THREADS = 256, LR_ITEMS = 64;

__device__ __forceinline__ uint32_t f32_key(float v)
{
    const uint32_t b = __float_as_uint(v);
    return (b >> 31) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ float dot_f64(const float* x, const float* y, int k)
{
    double s = 0.0;
    for (int f = 0; f < k; ++f) s = __dadd_rn(s, __dmul_rn((double)x[f], (double)y[f]));
    return __double2float_rn(s);
}

template <int J>
__global__ void __launch_bounds__(LR_RANK_THREADS) lrppm_rank_kernel(
    const float* __restrict__ U, const float* __restrict__ I, const float* __restrict__ UA, const float* __restrict__ IA,
    const int32_t* __restrict__ q_ptr, const int32_t* __restrict__ q_idx, const double* __restrict__ q_val,
    const int64_t* __restrict__ users, int64_t n_items, int k, int n_aspects, int n_top, double alpha_scale,
    double beta, double* __restrict__ out)
{
    extern __shared__ double lr_sh[];
    double* qd = lr_sh;                                      // [warps][n_aspects]
    float* uau = (float*)(lr_sh + (LR_RANK_THREADS / 32) * n_aspects);
    const int64_t u = users[blockIdx.y];
    const float* Uu = U + u * k;
    for (int e = threadIdx.x; e < n_aspects; e += blockDim.x) uau[e] = dot_f64(UA + (int64_t)e * k, Uu, k);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* q = qd + warp * n_aspects;
    for (int e = lane; e < n_aspects; e += 32) q[e] = 0.0;
    __syncthreads();
    const int64_t i1 = min(n_items, (int64_t)(blockIdx.x + 1) * LR_ITEMS);
    for (int64_t i = (int64_t)blockIdx.x * LR_ITEMS + warp; i < i1; i += LR_RANK_THREADS / 32) {
        const float* Ii = I + i * k;
        for (int p = q_ptr[i] + lane; p < q_ptr[i + 1]; p += 32) q[q_idx[p]] = q_val[p];
        __syncwarp();
        const float du = dot_f64(Ii, Uu, k);
        float s[J];
        uint32_t key[J];
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int as = lane + 32 * j;
            s[j] = 0.f;
            key[j] = 0u;                                     // below every aspect's key
            if (as < n_aspects) {
                s[j] = __fadd_rn(__fadd_rn(uau[as], dot_f64(Ii, IA + (int64_t)as * k, k)), du);
                key[j] = f32_key(s[j]);
            }
        }
        uint32_t kth = 0;                                    // 0: every aspect is taken
        if (n_top < n_aspects)
            for (int bit = 31; bit >= 0; --bit) {
                const uint32_t cand = kth | (1u << bit);
                int c = 0;
#pragma unroll
                for (int j = 0; j < J; ++j) c += key[j] >= cand;
                if (__reduce_add_sync(0xffffffffu, c) >= n_top) kth = cand;
            }
        int above = 0;
#pragma unroll
        for (int j = 0; j < J; ++j) above += key[j] > kth;
        int need = n_top - __reduce_add_sync(0xffffffffu, above);  // ties at the n_top-th place still to take
        double acc = 0.0;
#pragma unroll
        for (int j = 0; j < J; ++j) {
            const int as = lane + 32 * j;
            const bool tie = n_top < n_aspects && key[j] == kth && as < n_aspects;
            const unsigned tm = __ballot_sync(0xffffffffu, tie);
            const bool take = key[j] > kth || (n_top >= n_aspects && as < n_aspects) ||
                              (tie && __popc(tm & ((1u << lane) - 1u)) < need);
            need -= __popc(tm);
            if (take) acc = __dadd_rn(acc, __dmul_rn((double)s[j], q[as < n_aspects ? as : 0]));
        }
        for (int off = 16; off > 0; off >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, off));
        if (lane == 0)
            out[(int64_t)blockIdx.y * n_items + i] =
                __dadd_rn(__dmul_rn(alpha_scale, __ddiv_rn(acc, (double)n_top)), (double)__fmul_rn((float)beta, du));
        __syncwarp();
        for (int p = q_ptr[i] + lane; p < q_ptr[i + 1]; p += 32) q[q_idx[p]] = 0.0;
        __syncwarp();
    }
}

}  // namespace b200

using namespace b200;

// The workspace: del (f32 per parameter) and the touched marks lead and must be zero between calls; then the changed
// flags and the per-iteration sample buffers.
struct LrppmLayout {
    int64_t del, touched, changed, coef, ids, total;
};

static LrppmLayout lrppm_layout(int64_t n_users, int64_t n_items, int64_t n_aspects, int k, int n_s, int n_rank)
{
    auto up = [](int64_t b) { return (b + 255) / 256 * 256; };
    const int64_t rows = n_users + n_items + 2 * n_aspects;
    LrppmLayout l{};
    l.del = 0;
    l.touched = up(4 * rows * k);
    l.changed = l.touched + up(rows);
    l.coef = l.changed + 256;
    l.ids = l.coef + up(4 * ((int64_t)n_s + 2ll * n_rank));
    l.total = l.ids + up(4 * (2ll * n_s + 5ll * n_rank));
    return l;
}

extern "C" int64_t b200_lrppm_workspace_bytes(int64_t n_users, int64_t n_items, int64_t n_aspects, int k, int n_samples,
                                              int n_ranking_samples)
{
    return lrppm_layout(n_users, n_items, n_aspects, k, n_samples, n_ranking_samples).total;
}

extern "C" int b200_lrppm_fit(int64_t n_users, int64_t n_items, int64_t n_aspects, int k, const int32_t* r_u,
                              const int32_t* r_i, const float* r_val, int64_t n_r, const int32_t* x_u,
                              const int32_t* x_i, const int32_t* x_a, const float* x_l, int64_t n_x,
                              const int32_t* akeys, int64_t n_akeys, const int32_t* rkeys, const float* rvals,
                              int64_t n_rkeys, int n_samples, int n_ranking_samples, int n_iter, const int32_t* draws,
                              float* const* params, void* work, float lr, float reg, float ld, int flags, uint64_t seed,
                              uint64_t iter0, unsigned long long* counts, double* losses, unsigned long long* phase_ns,
                              void* stream)
{
    B200_REQUIRE(n_users > 0 && n_items > 0 && n_aspects > 0 && k > 0 && n_r > 0 && n_x > 0 && n_akeys > 0 &&
                     n_rkeys > 0 && n_samples >= 0 && n_ranking_samples >= 0 && n_iter >= 0,
                 "b200_lrppm_fit: bad sizes (users %lld items %lld aspects %lld factors %d ratings %lld triples %lld "
                 "keys %lld/%lld samples %d/%d iterations %d)",
                 (long long)n_users, (long long)n_items, (long long)n_aspects, k, (long long)n_r, (long long)n_x,
                 (long long)n_akeys, (long long)n_rkeys, n_samples, n_ranking_samples, n_iter);
    B200_REQUIRE(n_users < (1ll << 31) && n_items < (1ll << 31) && n_aspects < (1ll << 31) && n_r < (1ll << 31) &&
                     n_x < (1ll << 31) && 2ll * n_samples + 5ll * n_ranking_samples < (1ll << 31),
                 "b200_lrppm_fit: sizes beyond int32 ids");
    B200_REQUIRE(r_u && r_i && r_val && x_u && x_i && x_a && x_l && akeys && rkeys && rvals && params && work &&
                     counts,
                 "b200_lrppm_fit: null pointer argument");
    B200_REQUIRE((flags & ~B200_LRPPM_PHILOX) == 0, "b200_lrppm_fit: unknown flags %d", flags);
    if (n_iter == 0) return B200_OK;
    B200_REQUIRE(draws || (flags & B200_LRPPM_PHILOX), "b200_lrppm_fit: null draws");
    LrppmArgs a{};
    a.rows[L_U] = n_users; a.rows[L_I] = n_items; a.rows[L_UA] = n_aspects; a.rows[L_IA] = n_aspects;
    a.k = k;
    a.r_u = r_u; a.r_i = r_i; a.r_val = r_val; a.n_r = n_r;
    a.x_u = x_u; a.x_i = x_i; a.x_a = x_a; a.x_l = x_l; a.n_x = n_x;
    a.akeys = akeys; a.n_akeys = n_akeys; a.rkeys = rkeys; a.rvals = rvals; a.n_rkeys = n_rkeys;
    a.n_s = n_samples; a.n_rank = n_ranking_samples; a.n_iter = n_iter; a.draws = draws;
    const LrppmLayout l = lrppm_layout(n_users, n_items, n_aspects, k, n_samples, n_ranking_samples);
    char* w = (char*)work;
    float* del = (float*)(w + l.del);
    int64_t off = 0;
    for (int m = 0; m < L_N; ++m) {
        a.P[m] = params[m];
        B200_REQUIRE(a.P[m], "b200_lrppm_fit: null parameter %d", m);
        a.D[m] = del;
        del += a.rows[m] * k;
        a.row_off[m] = off;
        off += a.rows[m];
    }
    a.touched = (uint8_t*)(w + l.touched);
    a.changed = (unsigned int*)(w + l.changed);
    a.coef = (float*)(w + l.coef);
    a.ids = (int32_t*)(w + l.ids);
    a.lr = lr; a.reg = reg; a.ld = ld;
    a.counts = counts; a.losses = losses; a.phase_ns = phase_ns;
    a.philox = (flags & B200_LRPPM_PHILOX) != 0;
    a.key0 = (uint32_t)seed;
    a.key1 = (uint32_t)(seed >> 32);
    a.iter0 = iter0;
    B200_CUDA(cudaMemsetAsync(a.changed, 0, 2 * sizeof(unsigned int), (cudaStream_t)stream));
    int per_sm = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lrppm_fit_kernel, LR_THREADS, 0));
    B200_REQUIRE(per_sm > 0, "b200_lrppm_fit: the fit kernel does not fit on an SM");
    const int blocks = sm_count() * per_sm;
    void* kargs[] = {&a};
    count_launch();
    B200_CUDA(cudaLaunchCooperativeKernel((const void*)lrppm_fit_kernel, dim3(blocks), dim3(LR_THREADS), kargs, 0,
                                          (cudaStream_t)stream));
    return B200_OK;
}

extern "C" int b200_lrppm_rank_rows(const float* U, const float* I, const float* UA, const float* IA,
                                    const int32_t* q_indptr, const int32_t* q_indices, const double* q_data,
                                    const int64_t* users, int64_t n_q, int64_t n_items, int k, int64_t n_aspects,
                                    int n_top, double alpha, double rating_scale, double* out, void* stream)
{
    B200_REQUIRE(n_q >= 0 && n_items >= 0 && k > 0 && n_aspects > 0 && n_aspects <= 1024 && n_top > 0 &&
                     n_top <= n_aspects,
                 "b200_lrppm_rank_rows: bad sizes n_q=%lld n_items=%lld k=%d aspects=%lld top=%d", (long long)n_q,
                 (long long)n_items, k, (long long)n_aspects, n_top);
    B200_REQUIRE(U && I && UA && IA && q_indptr && q_indices && q_data && users && out,
                 "b200_lrppm_rank_rows: null pointer argument");
    if (n_q == 0 || n_items == 0) return B200_OK;
    const size_t smem = 8 * (size_t)(LR_RANK_THREADS / 32) * n_aspects + 4 * (size_t)n_aspects;
    const int na = (int)n_aspects;
    auto launch = [&](auto kernel) -> int {
        B200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const int64_t tiles = (n_items + LR_ITEMS - 1) / LR_ITEMS;
        for (int64_t q0 = 0; q0 < n_q; q0 += 65535) {
            const int64_t nq = std::min<int64_t>(65535, n_q - q0);
            count_launch();
            kernel<<<dim3((unsigned)tiles, (unsigned)nq), LR_RANK_THREADS, smem, (cudaStream_t)stream>>>(
                U, I, UA, IA, q_indptr, q_indices, q_data, users + q0, n_items, k, na, n_top, alpha * rating_scale,
                1.0 - alpha, out + q0 * n_items);
            B200_CUDA(cudaGetLastError());
        }
        return B200_OK;
    };
    if (na <= 32) return launch(lrppm_rank_kernel<1>);
    if (na <= 64) return launch(lrppm_rank_kernel<2>);
    if (na <= 128) return launch(lrppm_rank_kernel<4>);
    if (na <= 256) return launch(lrppm_rank_kernel<8>);
    if (na <= 512) return launch(lrppm_rank_kernel<16>);
    return launch(lrppm_rank_kernel<32>);
}
