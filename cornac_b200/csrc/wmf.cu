// Weighted matrix factorisation (Hu / Koren / Volinsky, Pan et al.) training step for sm_90a.
//
// Replaces one `sess.run([model.opt, model.loss])` of the reference's TensorFlow-1 graph
//     cornac/models/wmf/wmf.py:34-55          (loss, gradients, clip to [-5, 5], AdamOptimizer)
//     cornac/models/wmf/recom_wmf.py:186-199  (dense rating / confidence slabs of one item mini-batch)
// for a mini-batch of `b` item ids:
//     V_b  = V[ids];   pred = U V_b^T;   W = C_b * (R_b - pred),  C_b = a where R_b != 0, else b_conf
//     loss = sum(C_b (R_b - pred)^2) + lambda_u |U|^2 / 2 + lambda_v |V_b|^2 / 2
//     gU   = -2 W V_b + lambda_u U            (dense:   every user row moves in every step)
//     gV_b = -2 W^T U + lambda_v V_b          (sparse:  IndexedSlices over ids)
//     both clipped elementwise to [-5, 5]; Adam with the TF-1 semantics: the sparse update decays the moments of the
//     WHOLE item matrix and moves every row (non-lazy), the beta powers advance once per step (host side).
//
// Kernel A (wmf_users_kernel): one CTA per tile of TU users.  V_b and the tile's U rows live in shared memory; the dense
// R_b tile is scattered from the CSC columns of the batch items (binary search of the tile's user range per column), so
// the rating matrix is never densified in HBM.  The CTA forms W in place, then its share of gV_b (from the OLD user
// rows; red.global.add into a b x k scratch), then gU for its rows, clips, and applies the dense Adam step.
// Kernel B (wmf_items_kernel): elementwise over all of V: decay, scatter-add of the clipped batch gradient, move.
// f32 throughout like the graph; plain FFMA (the step is latency/bandwidth bound at Cornac's sizes, and faithful f32
// keeps it comparable with a CPU restatement of the graph).
#include "common.cuh"

namespace b200 {

namespace wmf {

constexpr int THREADS = 256;

struct UsersParams {
    const int32_t* __restrict__ indptr;    // CSC: [n_items + 1]
    const int32_t* __restrict__ rows;      // user index of every stored rating, sorted within a column
    const float* __restrict__ vals;
    const int32_t* __restrict__ ids;       // [b] item ids of the mini-batch
    int b, k, tu;
    int64_t n_users;
    float* U;
    float* mU;
    float* vU;
    const float* V;
    float* gV;                             // [b, k] zeroed by the caller; receives -2 W^T U
    float a_conf, b_conf, lambda_u;
    float lr_t, beta1, beta2, eps;
    double* loss;                          // += sum(C E^2) + lambda_u |U_tile|^2 / 2
};

__device__ __forceinline__ float clip5(float g) { return fminf(fmaxf(g, -5.f), 5.f); }

__global__ void __launch_bounds__(THREADS) wmf_users_kernel(const UsersParams p)
{
    extern __shared__ __align__(16) float sm[];
    const int k = p.k, b = p.b, tu = p.tu;
    const int kp = k + 1;                       // padded row stride: conflict-free column walks
    const int bp = b + 1;
    float* Vs = sm;                             // [b][kp]
    float* Us = Vs + (size_t)b * kp;            // [tu][kp]
    float* Ws = Us + (size_t)tu * kp;           // [tu][bp]   R_b tile -> W tile
    __shared__ double red[THREADS / 32];
    const int tid = threadIdx.x;
    double loss_acc = 0.0;

    for (int i = tid; i < b * k; i += THREADS) {
        const int j = i / k, f = i - j * k;
        Vs[j * kp + f] = __ldg(p.V + (size_t)p.ids[j] * k + f);
    }
    for (int64_t u0 = (int64_t)blockIdx.x * tu; u0 < p.n_users; u0 += (int64_t)gridDim.x * tu) {
        const int nu = (int)min((int64_t)tu, p.n_users - u0);
        __syncthreads();
        for (int i = tid; i < tu * k; i += THREADS) {
            const int u = i / k, f = i - u * k;
            Us[u * kp + f] = u < nu ? p.U[(size_t)(u0 + u) * k + f] : 0.f;
        }
        for (int i = tid; i < tu * bp; i += THREADS) Ws[i] = 0.f;
        __syncthreads();
        // dense ratings of the tile: column j of the batch restricted to users [u0, u0 + nu)
        for (int j = tid >> 3; j < b; j += THREADS >> 3) {       // 8 lanes per column
            const int32_t item = p.ids[j];
            int lo = __ldg(p.indptr + item), hi = __ldg(p.indptr + item + 1);
            const int end = hi;
            while (lo < hi) {                                     // first entry with user >= u0
                const int mid = (lo + hi) >> 1;
                if ((int64_t)__ldg(p.rows + mid) < u0) lo = mid + 1; else hi = mid;
            }
            for (int e = lo + (tid & 7); e < end; e += 8) {
                const int64_t u = __ldg(p.rows + e);
                if (u >= u0 + nu) break;
                Ws[(int)(u - u0) * bp + j] = __ldg(p.vals + e);
            }
        }
        __syncthreads();
        // W = C * (R - U V_b^T), loss += C * E^2        (recom_wmf.py:187-189: C = a where R != 0)
        for (int i = tid; i < tu * b; i += THREADS) {
            const int u = i / b, j = i - u * b;
            float w = 0.f;
            if (u < nu) {
                float pred = 0.f;
                const float* ur = Us + u * kp;
                const float* vr = Vs + j * kp;
                for (int f = 0; f < k; ++f) pred = fmaf(ur[f], vr[f], pred);
                const float r = Ws[u * bp + j];
                const float c = (r != 0.f) ? p.a_conf : p.b_conf;
                const float e = r - pred;
                w = c * e;
                loss_acc += (double)(w * e);
            }
            Ws[u * bp + j] = w;
        }
        __syncthreads();
        // this tile's share of gV_b = -2 W^T U  (OLD user rows)
        for (int i = tid; i < b * k; i += THREADS) {
            const int j = i / k, f = i - j * k;
            float s = 0.f;
            for (int u = 0; u < nu; ++u) s = fmaf(Ws[u * bp + j], Us[u * kp + f], s);
            atomicAdd(p.gV + (size_t)j * k + f, -2.f * s);
        }
        // gU = -2 W V_b + lambda_u U, clip, dense Adam (tf.train.AdamOptimizer._apply_dense)
        for (int i = tid; i < nu * k; i += THREADS) {
            const int u = i / k, f = i - u * k;
            float s = 0.f;
            const float* wr = Ws + u * bp;
            for (int j = 0; j < b; ++j) s = fmaf(wr[j], Vs[j * kp + f], s);
            const float uo = Us[u * kp + f];
            loss_acc += 0.5 * (double)p.lambda_u * (double)(uo * uo);
            const float g = clip5(fmaf(-2.f, s, p.lambda_u * uo));
            const size_t at = (size_t)(u0 + u) * k + f;
            const float m = p.beta1 * p.mU[at] + (1.f - p.beta1) * g;
            const float v = p.beta2 * p.vU[at] + (1.f - p.beta2) * g * g;
            p.mU[at] = m;
            p.vU[at] = v;
            p.U[at] = uo - p.lr_t * m / (sqrtf(v) + p.eps);
        }
    }
    // block reduction of the loss share
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, o);
    if ((tid & 31) == 0) red[tid >> 5] = loss_acc;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < THREADS / 32; ++w) t += red[w];
        atomicAdd(p.loss, t);
    }
}

// slot_of[ids[j]] = j (set) / -1 (clear)
__global__ void wmf_slots_kernel(const int32_t* __restrict__ ids, int b, int32_t* __restrict__ slot_of, int set)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < b) slot_of[ids[j]] = set ? j : -1;
}

// tf.train.AdamOptimizer._apply_sparse_shared on V: m *= beta1, v *= beta2 for EVERY row, the clipped batch gradient is
// scatter-added into the batch rows, then every row moves by lr_t * m / (sqrt(v) + eps).
__global__ void wmf_items_kernel(float* __restrict__ V, float* __restrict__ mV, float* __restrict__ vV,
                                 const float* __restrict__ gV, const int32_t* __restrict__ slot_of, int64_t n_items, int k,
                                 float lambda_v, float lr_t, float beta1, float beta2, float eps, double* loss)
{
    const int64_t total = n_items * k;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    double reg = 0.0;
    for (int64_t at = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; at < total; at += stride) {
        const int64_t i = at / k;
        const int f = (int)(at - i * k);
        const int slot = __ldg(slot_of + i);
        const float x = V[at];
        float m = beta1 * mV[at], v = beta2 * vV[at];
        if (slot >= 0) {
            const float g = clip5(gV[(size_t)slot * k + f] + lambda_v * x);
            m += (1.f - beta1) * g;
            v += (1.f - beta2) * g * g;
            reg += 0.5 * (double)lambda_v * (double)(x * x);
        }
        mV[at] = m;
        vV[at] = v;
        V[at] = x - lr_t * m / (sqrtf(v) + eps);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) reg += __shfl_xor_sync(0xffffffffu, reg, o);
    if ((threadIdx.x & 31) == 0 && reg != 0.0) atomicAdd(loss, reg);
}

static size_t users_smem(int b, int k, int tu) { return ((size_t)(b + tu) * (k + 1) + (size_t)tu * (b + 1)) * sizeof(float); }

}  // namespace wmf
}  // namespace b200

using namespace b200;

extern "C" int b200_wmf_step(const int32_t* csc_indptr, const int32_t* csc_rows, const float* csc_vals,
                             const int32_t* ids, int b, int64_t n_users, int64_t n_items, int k,
                             float* U, float* V, float* mU, float* vU, float* mV, float* vV,
                             float a_conf, float b_conf, float lambda_u, float lambda_v,
                             float lr_t, float beta1, float beta2, float epsilon,
                             int32_t* slot_of, float* gV_scratch, double* loss, void* stream)
{
    B200_REQUIRE(csc_indptr && csc_rows && csc_vals && ids && U && V && mU && vU && mV && vV && slot_of && gV_scratch && loss,
                 "b200_wmf_step: null pointer argument");
    B200_REQUIRE(b >= 1 && k >= 1 && n_users >= 1 && n_items >= 1, "b200_wmf_step: bad sizes b=%d k=%d n_users=%lld n_items=%lld",
                 b, k, (long long)n_users, (long long)n_items);
    cudaStream_t st = (cudaStream_t)stream;
    int tu = 64;
    const size_t limit = 220 * 1024;
    while (tu > 4 && wmf::users_smem(b, k, tu) > limit) tu >>= 1;
    B200_REQUIRE(wmf::users_smem(b, k, tu) <= limit, "b200_wmf_step: batch_size=%d x k=%d does not fit the shared memory of one SM", b, k);
    B200_CUDA(cudaMemsetAsync(gV_scratch, 0, (size_t)b * k * sizeof(float), st));
    B200_CUDA(cudaMemsetAsync(loss, 0, sizeof(double), st));
    wmf::wmf_slots_kernel<<<(b + 127) / 128, 128, 0, st>>>(ids, b, slot_of, 1); ::b200::count_launch();
    wmf::UsersParams p;
    p.indptr = csc_indptr; p.rows = csc_rows; p.vals = csc_vals; p.ids = ids; p.b = b; p.k = k; p.tu = tu; p.n_users = n_users;
    p.U = U; p.mU = mU; p.vU = vU; p.V = V; p.gV = gV_scratch;
    p.a_conf = a_conf; p.b_conf = b_conf; p.lambda_u = lambda_u;
    p.lr_t = lr_t; p.beta1 = beta1; p.beta2 = beta2; p.eps = epsilon; p.loss = loss;
    const size_t smem = wmf::users_smem(b, k, tu);
    B200_CUDA(cudaFuncSetAttribute(wmf::wmf_users_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int64_t tiles = (n_users + tu - 1) / tu;
    const int64_t cap = (int64_t)sm_count();
    const unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
    wmf::wmf_users_kernel<<<grid, wmf::THREADS, smem, st>>>(p); ::b200::count_launch();
    const int64_t total = n_items * (int64_t)k;
    int64_t ib = (total + 255) / 256;
    if (ib > (int64_t)sm_count() * 16) ib = (int64_t)sm_count() * 16;
    wmf::wmf_items_kernel<<<(unsigned)ib, 256, 0, st>>>(V, mV, vV, gV_scratch, slot_of, n_items, k, lambda_v, lr_t, beta1, beta2,
                                                        epsilon, loss); ::b200::count_launch();
    wmf::wmf_slots_kernel<<<(b + 127) / 128, 128, 0, st>>>(ids, b, slot_of, 0); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
