// K10: EASE (Steck 2019).  The inverse P = G^-1 of the symmetric positive definite Gram matrix G = X^T X + lambda I, the
// weights B = P / -diag(P) and the score rows X[u, :] . B.  G itself is b200_ease_gram (the raw mode of knn.cu's ordered
// row-pair sums).
//
// Inverse (Cholesky route, about n^3 flop, in place in one row-major n x n f64 buffer, lower triangle in):
//   potrf  G = L L^T, right-looking over NB-wide block columns: the diagonal block is factored by one CTA, which also
//          writes inv(L_kk); the panel below it becomes A_panel . inv(L_kk)^T and the trailing lower triangle
//          loses panel . panel^T.
//   trtri  Z = L^-T (upper triangular), stored in the upper triangle; Z_jj = inv(L_jj)^T, and block column j above the
//          diagonal is Z[0:j, j] = -(Z[0:j, 0:j] . L[j, 0:j]^T) . inv(L_jj)^T.
//   lauum  P = Z Z^T, lower triangle only (P[i, j] = sum over k >= i of Z[i, k] Z[j, k]), written over L.
// All three are products C = beta C + alpha A B^T of row-major operands, done by one FP64 tensor-core tile kernel
// (mma.sync m16n8k16 f64, cp.async double-buffered shared-memory tiles).  Sums are in a fixed order (no split-K, no
// atomics), so two runs give the same bits; the upper triangle is a mirror of the lower, so P is exactly symmetric.
#include "common.cuh"

namespace b200 {
namespace ease {

constexpr int NB = 64;                  // block size of the factorisation = tile edge of the product kernel
constexpr int KC = 32;                  // k extent of one staged tile
constexpr int LDS = KC + 4;             // padded shared row: the f64 fragment loads of a half-warp hit distinct banks
constexpr int GEMM_THREADS = 128;       // 4 warps, 32 x 32 outputs each
constexpr size_t GEMM_SMEM = 2 * 2 * NB * LDS * sizeof(double);

enum : unsigned {
    C_LOWER = 1,        // only tiles with tile row >= tile col (C square); diagonal tiles write row >= col only
    A_UPPER = 2,        // A[r, k] is taken as 0 for k < r (upper triangular operand, whatever is stored below)
    B_UPPER = 4,        // same for B[r, k]
    K_FROM_ROW = 8,     // the k loop of a tile starts at its first row (A is upper triangular)
    DIAG_ALT = 16,      // C_LOWER: diagonal tiles go to alt + tile * NB * NB (ld NB) instead of C
};

struct Gemm {
    int M, N, K;
    const double* A; int64_t lda;
    const double* B; int64_t ldb;
    double* C; int64_t ldc;
    double alpha;
    int beta;           // 0: C = alpha A B^T, 1: C += alpha A B^T
    unsigned flags;
    double* alt;
};

__device__ __forceinline__ void cp_async8(double* dst, const double* src, bool valid)
{
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(d), "l"(src), "r"(valid ? 8 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::); }

__device__ __forceinline__ void dmma(double (&d)[4], const double (&a)[8], const double (&b)[4])
{
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
        "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
        : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
          "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// rows [r0, r0 + NB) x k [k0, k0 + KC) of a row-major operand into S[NB][LDS]; outside [0, rows) x [0, kend): zeros
__device__ __forceinline__ void stage(double* S, const double* X, int64_t ld, int r0, int rows, int k0, int kend)
{
    for (int e = threadIdx.x; e < NB * KC; e += GEMM_THREADS) {
        const int r = e / KC, k = e % KC;
        const bool ok = r0 + r < rows && k0 + k < kend;
        cp_async8(S + r * LDS + k, ok ? X + (int64_t)(r0 + r) * ld + k0 + k : X, ok);
    }
}

// One CTA per NB x NB tile of C.  Warp w owns rows 32 (w >> 1) .. +32 and columns 32 (w & 1) .. +32: 2 x 4 mma tiles.
// Fragments of m16n8k16 f64 (g = lane >> 2, t = lane & 3): a[i] = A[g + 8 (i & 1)][t + 4 (i >> 1)],
// b[i] = B[k = t + 4 i][n = g], c[i] = C[g + 8 (i >> 1)][2 t + (i & 1)].
__global__ void __launch_bounds__(GEMM_THREADS, 3) ease_gemm_kernel(Gemm p)
{
    extern __shared__ double smem[];
    double* As = smem;                   // [2][NB][LDS]
    double* Bs = smem + 2 * NB * LDS;    // [2][NB][LDS]
    int tm, tn;
    if (p.flags & C_LOWER) {             // triangular tile numbering: t = tm (tm + 1) / 2 + tn, tn <= tm
        const int64_t t = blockIdx.x;
        tm = (int)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
        while ((int64_t)tm * (tm + 1) / 2 > t) --tm;
        while ((int64_t)(tm + 1) * (tm + 2) / 2 <= t) ++tm;
        tn = (int)(t - (int64_t)tm * (tm + 1) / 2);
    } else {
        tm = blockIdx.x;
        tn = blockIdx.y;
    }
    const int m0 = tm * NB, n0 = tn * NB;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t4 = lane & 3;
    const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
    double acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[i][j][c] = 0.0;

    const int kbeg = (p.flags & K_FROM_ROW) ? (m0 < p.K ? m0 : p.K) : 0;
    const int nchunks = (p.K - kbeg + KC - 1) / KC;
    if (nchunks > 0) {
        stage(As, p.A, p.lda, m0, p.M, kbeg, p.K);
        stage(Bs, p.B, p.ldb, n0, p.N, kbeg, p.K);
        cp_async_commit();
    }
    for (int c = 0; c < nchunks; ++c) {
        const int buf = c & 1;
        const int k0 = kbeg + c * KC;
        cp_async_wait_all();
        __syncthreads();                                  // chunk c landed; every warp is done with chunk c - 1
        if (c + 1 < nchunks) {
            stage(As + (buf ^ 1) * NB * LDS, p.A, p.lda, m0, p.M, k0 + KC, p.K);
            stage(Bs + (buf ^ 1) * NB * LDS, p.B, p.ldb, n0, p.N, k0 + KC, p.K);
            cp_async_commit();
        }
        const double* Ab = As + buf * NB * LDS;
        const double* Bb = Bs + buf * NB * LDS;
#pragma unroll
        for (int kk = 0; kk < KC; kk += 16) {
            double a[2][8], b[4][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const int r = wm + i * 16 + g + 8 * (e & 1), k = kk + t4 + 4 * (e >> 1);
                    double v = Ab[r * LDS + k];
                    if ((p.flags & A_UPPER) && k0 + k < m0 + r) v = 0.0;
                    a[i][e] = v;
                }
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = wn + j * 8 + g, k = kk + t4 + 4 * e;
                    double v = Bb[r * LDS + k];
                    if ((p.flags & B_UPPER) && k0 + k < n0 + r) v = 0.0;
                    b[j][e] = v;
                }
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) dmma(acc[i][j], a[i], b[j]);
        }
    }

    const bool diag = (p.flags & C_LOWER) && tm == tn;
    double* C = p.C;
    int64_t ldc = p.ldc;
    int cr0 = m0, cc0 = n0;
    if (diag && (p.flags & DIAG_ALT)) {
        C = p.alt + (int64_t)tm * NB * NB;
        ldc = NB;
        cr0 = cc0 = 0;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = wm + i * 16 + g + 8 * (e >> 1), col = wn + j * 8 + 2 * t4 + (e & 1);
                if (m0 + r >= p.M || n0 + col >= p.N || (diag && col > r)) continue;
                double* dst = C + (int64_t)(cr0 + r) * ldc + cc0 + col;
                const double v = p.alpha * acc[i][j][e];
                *dst = p.beta ? __dadd_rn(*dst, v) : v;
            }
}

// Cholesky of the diagonal block at (kb, kb) (bs = min(NB, n - kb) rows; padded with the identity) in shared memory,
// written back over its lower triangle, and inv(L_kk) (lower, zeros above) to dinv.  A pivot that is not a positive
// finite number sets *info = kb + j + 1 unless an earlier column already failed.
__global__ void __launch_bounds__(256) ease_potrf_diag_kernel(int64_t n, double* A, int64_t kb, double* __restrict__ dinv,
                                                              int* info)
{
    __shared__ double a[NB][NB + 1];    // L in the lower triangle; inv(L)[i][c] (i >= c) then goes to a[c][i]
    __shared__ double ldiag[NB];
    const int tid = threadIdx.x;
    const int bs = (int)(n - kb < NB ? n - kb : NB);
    for (int e = tid; e < NB * NB; e += blockDim.x) {
        const int i = e / NB, j = e % NB;
        a[i][j] = (i < bs && j < bs) ? A[(kb + i) * n + kb + j] : (i == j ? 1.0 : 0.0);
    }
    __syncthreads();
    for (int j = 0; j < NB; ++j) {
        if (tid == 0) {
            const double d = a[j][j];
            if (!(d > 0.0) || !isfinite(d)) {
                atomicCAS(info, 0, (int)(kb + j + 1));
                a[j][j] = 1.0;                            // keeps the rest finite; the result is discarded
            } else {
                a[j][j] = __dsqrt_rn(d);
            }
        }
        __syncthreads();
        for (int i = j + 1 + tid; i < NB; i += blockDim.x) a[i][j] = __ddiv_rn(a[i][j], a[j][j]);
        __syncthreads();
        for (int e = tid; e < NB * NB; e += blockDim.x) {
            const int i = e / NB, k = e % NB;
            if (k > j && i >= k) a[i][k] = __dsub_rn(a[i][k], __dmul_rn(a[i][j], a[k][j]));
        }
        __syncthreads();
    }
    for (int e = tid; e < NB * NB; e += blockDim.x) {
        const int i = e / NB, j = e % NB;
        if (i < bs && j <= i) A[(kb + i) * n + kb + j] = a[i][j];
    }
    if (tid < NB) ldiag[tid] = a[tid][tid];
    __syncthreads();
    if (tid < NB) {                                       // column c of inv(L) by forward substitution
        const int c = tid;
        for (int i = c; i < NB; ++i) {
            double s = i == c ? 1.0 : 0.0;
            for (int k = c; k < i; ++k) s = __dsub_rn(s, __dmul_rn(a[i][k], a[c][k]));
            a[c][i] = __ddiv_rn(s, ldiag[i]);
        }
    }
    __syncthreads();
    for (int e = tid; e < NB * NB; e += blockDim.x) {
        const int i = e / NB, c = e % NB;
        dinv[e] = i >= c ? a[c][i] : 0.0;
    }
}

// Z_jj = inv(L_jj)^T into the upper triangle (diagonal included) of every diagonal block
__global__ void ease_zdiag_kernel(int64_t n, double* A, const double* __restrict__ dinv)
{
    const int64_t kb = (int64_t)blockIdx.x * NB;
    const int bs = (int)(n - kb < NB ? n - kb : NB);
    const double* D = dinv + (int64_t)blockIdx.x * NB * NB;
    for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
        const int r = e / NB, c = e % NB;
        if (r < bs && c < bs && c >= r) A[(kb + r) * n + kb + c] = D[c * NB + r];
    }
}

// P's lower triangle is in A outside the diagonal blocks and in alt (ld NB) for them: write the full symmetric P
__global__ void ease_finish_kernel(int64_t n, double* A, const double* __restrict__ alt)
{
    __shared__ double tile[32][33];
    const int R = blockIdx.y, Cb = blockIdx.x;            // 32 x 32 tiles at or above the diagonal: R <= Cb
    if (R > Cb) return;
    const int tx = threadIdx.x;
    for (int ty = threadIdx.y; ty < 32; ty += blockDim.y) {   // tile[ty][tx] = P[Cb*32 + ty][R*32 + tx] (lower)
        const int64_t row = (int64_t)Cb * 32 + ty, col = (int64_t)R * 32 + tx;
        if (row < n && col < n && row >= col) {
            tile[ty][tx] = row / NB == col / NB ? alt[(row / NB) * NB * NB + (row % NB) * NB + col % NB] : A[row * n + col];
        }
    }
    __syncthreads();
    for (int ty = threadIdx.y; ty < 32; ty += blockDim.y) {
        const int64_t row = (int64_t)R * 32 + ty, col = (int64_t)Cb * 32 + tx;   // upper element P[row][col], row <= col
        if (row < n && col < n && row <= col) {
            const double v = tile[tx][ty];
            A[row * n + col] = v;
            if (row / NB == col / NB) A[col * n + row] = v;                 // the lower part of a diagonal block
        }
    }
}

__global__ void ease_diag_kernel(int64_t n, const double* __restrict__ P, double* __restrict__ d)
{
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) d[j] = P[j * n + j];
}

// B = P / -diag(P) column-wise, B[j, j] = 0, negatives to 0 under posB: numpy's expression, element by element
__global__ void ease_weights_kernel(int64_t n, double* P, const double* __restrict__ d, int posB)
{
    const int64_t total = n * n;
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = e / n, j = e - i * n;
        double b = __ddiv_rn(P[e], -__ldg(d + j));
        if (i == j) b = 0.0;
        if (posB && b < 0.0) b = 0.0;
        P[e] = b;
    }
}

constexpr int SCORE_COLS = 128;         // columns of B per CTA: the strip every user of a grid row reads
constexpr int SCORE_USERS = 8;          // users per CTA

// out[q, j] = sum over the stored (i, x) of row users[q] of x * B[i, j], in stored order, from +0.0, no FMA
__global__ void __launch_bounds__(SCORE_COLS) ease_score_kernel(const int64_t* __restrict__ users, int64_t n_q, int64_t n,
                                                                const int32_t* __restrict__ indptr,
                                                                const int32_t* __restrict__ indices,
                                                                const double* __restrict__ data, const double* __restrict__ B,
                                                                double* __restrict__ out)
{
    const int64_t j = (int64_t)blockIdx.y * SCORE_COLS + threadIdx.x;
    if (j >= n) return;
    const int64_t q_end = ((int64_t)blockIdx.x + 1) * SCORE_USERS < n_q ? ((int64_t)blockIdx.x + 1) * SCORE_USERS : n_q;
    for (int64_t q = (int64_t)blockIdx.x * SCORE_USERS; q < q_end; ++q) {
        const int64_t u = __ldg(users + q);
        double acc = 0.0;
        const int pe = __ldg(indptr + u + 1);
        for (int p = __ldg(indptr + u); p < pe; ++p)
            acc = __dadd_rn(acc, __dmul_rn(__ldg(data + p), __ldg(B + (int64_t)__ldg(indices + p) * n + j)));
        out[q * n + j] = acc;
    }
}

static int gemm(const Gemm& p, cudaStream_t st)
{
    if (p.M <= 0 || p.N <= 0) return B200_OK;
    dim3 grid;
    if (p.flags & C_LOWER) {
        const int64_t tm = (p.M + NB - 1) / NB;
        grid = dim3((unsigned)(tm * (tm + 1) / 2));
    } else {
        grid = dim3((unsigned)((p.M + NB - 1) / NB), (unsigned)((p.N + NB - 1) / NB));
    }
    ease_gemm_kernel<<<grid, GEMM_THREADS, GEMM_SMEM, st>>>(p);
    ::b200::count_launch();
    return B200_OK;
}

}  // namespace ease
}  // namespace b200

using namespace b200;

extern "C" int64_t b200_spd_inverse_workspace_bytes(int64_t n)
{
    if (n <= 0) return 0;
    const int64_t nb = (n + ease::NB - 1) / ease::NB;
    // inv(L_kk) blocks (later P's diagonal blocks) + the trtri product T [n, NB] + info
    return (nb * ease::NB * ease::NB + n * ease::NB) * (int64_t)sizeof(double) + 256;
}

extern "C" int b200_spd_inverse(int64_t n, double* A, void* workspace, int* info, int phases, void* stream)
{
    using namespace ease;
    B200_REQUIRE(n >= 1 && n < (1LL << 31) - NB, "b200_spd_inverse: bad size n=%lld", (long long)n);
    B200_REQUIRE(A && workspace && info, "b200_spd_inverse: null pointer argument");
    B200_REQUIRE(phases >= 1 && phases <= 7, "b200_spd_inverse: bad phase mask %d", phases);
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA(cudaFuncSetAttribute(ease_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GEMM_SMEM));
    const int64_t nb = (n + NB - 1) / NB;
    double* dinv = (double*)workspace;
    double* T = dinv + nb * NB * NB;
    if (phases & B200_SPD_POTRF) {
        B200_CUDA(cudaMemsetAsync(info, 0, sizeof(int), st));
        for (int64_t k = 0; k < nb; ++k) {
            const int64_t kb = k * NB, rest = n - kb - NB;
            ease_potrf_diag_kernel<<<1, 256, 0, st>>>(n, A, kb, dinv + k * NB * NB, info); ::b200::count_launch();
            if (rest <= 0) break;
            double* panel = A + (kb + NB) * n + kb;
            // panel = panel . inv(L_kk)^T: one tile column, so each CTA reads its rows whole before it overwrites them
            gemm(Gemm{(int)rest, NB, NB, panel, n, dinv + k * NB * NB, NB, panel, n, 1.0, 0, 0, nullptr}, st);
            gemm(Gemm{(int)rest, (int)rest, NB, panel, n, panel, n, panel + NB, n, -1.0, 1, C_LOWER, nullptr}, st);
        }
    }
    if (phases & B200_SPD_TRTRI) {
        ease_zdiag_kernel<<<(unsigned)nb, 256, 0, st>>>(n, A, dinv); ::b200::count_launch();
        for (int64_t j = 1; j < nb; ++j) {
            const int64_t jb = j * NB;
            const int bs = (int)(n - jb < NB ? n - jb : NB);
            // T = Z[0:jb, 0:jb] . L[jb:jb+bs, 0:jb]^T, then Z[0:jb, jb:jb+bs] = -T . inv(L_jj)^T
            gemm(Gemm{(int)jb, bs, (int)jb, A, n, A + jb * n, n, T, NB, 1.0, 0, A_UPPER | K_FROM_ROW, nullptr}, st);
            gemm(Gemm{(int)jb, bs, bs, T, NB, dinv + j * NB * NB, NB, A + jb, n, -1.0, 0, 0, nullptr}, st);
        }
    }
    if (phases & B200_SPD_LAUUM) {
        // P = Z Z^T, lower; the diagonal tiles (where Z_ii still lives) go to the free inv(L) blocks
        gemm(Gemm{(int)n, (int)n, (int)n, A, n, A, n, A, n, 1.0, 0, C_LOWER | A_UPPER | B_UPPER | K_FROM_ROW | DIAG_ALT, dinv},
             st);
        const unsigned t32 = (unsigned)((n + 31) / 32);
        ease_finish_kernel<<<dim3(t32, t32), dim3(32, 8), 0, st>>>(n, A, dinv); ::b200::count_launch();
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_ease_weights(int64_t n, double* P, double* diag_workspace, int posB, void* stream)
{
    B200_REQUIRE(n >= 1 && P && diag_workspace, "b200_ease_weights: bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t cap = (int64_t)sm_count() * 16;
    const int64_t g1 = (n + 255) / 256;
    ease::ease_diag_kernel<<<(unsigned)(g1 < cap ? g1 : cap), 256, 0, st>>>(n, P, diag_workspace); ::b200::count_launch();
    const int64_t g2 = (n * n + 255) / 256;
    ease::ease_weights_kernel<<<(unsigned)(g2 < cap ? g2 : cap), 256, 0, st>>>(n, P, diag_workspace, posB ? 1 : 0);
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_ease_score(const int64_t* users, int64_t n_q, int64_t n_items, const int32_t* indptr, const int32_t* indices,
                               const double* data, const double* B, double* out, void* stream)
{
    B200_REQUIRE(n_q >= 0 && n_items >= 1 && (n_items + ease::SCORE_COLS - 1) / ease::SCORE_COLS < 65536,
                 "b200_ease_score: bad sizes n_q=%lld n_items=%lld", (long long)n_q, (long long)n_items);
    B200_REQUIRE(users && indptr && indices && data && B && out, "b200_ease_score: null pointer argument");
    if (n_q == 0) return B200_OK;
    // grid x (user batches) runs fastest, so the CTAs in flight share one column strip of B in the L2
    const dim3 grid((unsigned)((n_q + ease::SCORE_USERS - 1) / ease::SCORE_USERS),
                    (unsigned)((n_items + ease::SCORE_COLS - 1) / ease::SCORE_COLS));
    ease::ease_score_kernel<<<grid, ease::SCORE_COLS, 0, (cudaStream_t)stream>>>(users, n_q, n_items, indptr, indices, data, B, out);
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}
