// Tensor-core fused score + top-k for sm_90a (wgmma / TMA bulk copies / mbarrier).
//
// Replaces, for a batch of users, the reference's per-user pipeline
//     fast_dot(U[u], V, bias)            cornac/utils/fast_dot.pyx:40-43
//     argpartition / argsort top-k       cornac/models/recommender.py:521-528
// driven once per test user by ranking_eval (cornac/eval_methods/base_method.py:177-220).
//
// Plan of one call (users are processed in chunks so the candidate lists stay small):
//   1. pack   V (and the chunk's U rows) to fp16 in the GMMA "K-major, no swizzle" core-matrix
//             layout, tile by tile, so that one tile is ONE contiguous cp.async.bulk.  Both
//             sides are first multiplied by a power of two (exact) that brings their largest element
//             to [2^13, 2^14), so the fp16 range is never left and the rounding error is the 2^-11
//             relative one (8x smaller than bf16's: 8x tighter candidate filter); an extra K slice
//             carries the item base (two fp16 per item against a constant on the user side), so the
//             MMA adds it; per-row norms give the rigorous error bound eps(u) ~ 2^-10 |u| max|v|
//             (+ subnormal, accumulation and base terms, see `row_eps`) of the fp16 pass;
//   2. rank_tc_kernel  persistent, one CTA per SM, warp-specialised:
//               warp 0   TMA producer: U tile once per 128 users, V stages (128 items, half of a
//                        packed 256-item tile) through a ring of smem stages released by the consumers
//               warps 4-11  two consumer warpgroups, each owning 64 user rows: wgmma (M=64, N=128,
//                        K=16 per instruction, fp16 x fp16 -> f32 in registers), then the accumulator is
//                        passed through shared memory so that every thread owns one (user row, 64-column
//                        strip); it keeps every score above the row's running threshold in the thread's
//                        candidate list; the threshold is raised (never above the approximate k-th best
//                        minus 2*eps) by lock-step scans of the lists
//   3. rank_tc_finish_kernel  per row: exact re-score of the candidates (the f64-accumulated
//             arithmetic of score_batch_kernel), total order (score desc, id asc), top-k.
// The tensor pass only NOMINATES: every item whose exact score can reach the top-k is provably
// in the list, so ids and scores are identical to the exact path (score.cu).  Rows whose list
// overflows (degenerate score distributions) are redone by the exact path.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "common.cuh"

namespace b200 {

namespace tc {

constexpr int TM = 128;            // users per tile (two warpgroups of M = 64)
constexpr int TN = 256;            // items per packed V tile (the padding unit of the item side)
constexpr int SN = 128;            // items per pipeline stage (wgmma N): half of a packed tile, itself a contiguous tile image
constexpr int ST = 2;              // column strips of a stage: 64 columns per epilogue thread
constexpr int STRIP_N = SN / ST;
constexpr int EPI_WARPS = 4 * ST;  // 8 consumer warps = 2 warpgroups
constexpr int THREADS = 128 + 32 * EPI_WARPS;     // warps 0-3: TMA producer (warp 0) + idle, warps 4-11: consumers
constexpr int LDT = SN + 8;        // row stride (floats) of the accumulator hand-off: conflict-free fragment stores
constexpr int MAX_ST = 4;          // per-row slots of row_cnt / row_flag / row_tau (the finish reads `strips` of them)
constexpr int KX = 16;             // extra K slice carrying the item base: U gets (cA, cA, 1, 0...), V gets (hi, lo, pad ? -inf : 0, 0...)
constexpr int CAP = 1024;          // candidate-list capacity of one (row, strip) list
constexpr int NB = 32;             // score bins of a threshold raise (one pass over the list, counters in shared memory)
constexpr int MAX_TOPK = 256;
constexpr int MAX_KP = 128 + KX;
constexpr int CHUNK_TILES = 132 * 4;   // user tiles per chunk (4 waves of the H100's 132 SMs)

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    const uint32_t addr = smem_u32(bar);
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!ok);
}
// same, for the single-thread TMA producer: back off between polls so the spinning lane does not steal issue slots
// from the consumer warps that share its scheduler
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity)
{
    const uint32_t addr = smem_u32(bar);
    uint32_t ok;
    for (;;) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(addr), "r"(parity)
            : "memory");
        if (ok) break;
        __nanosleep(40);
    }
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// named barrier of `n` threads
__device__ __forceinline__ void named_sync(int id, int n)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}

// GMMA shared-memory descriptor, K-major, no swizzle ("interleaved" core matrices):
// a core matrix is 8 rows x 16 bytes stored as 128 contiguous bytes; LBO = byte distance between
// the two K-halves (16-byte chunks) of one K=16 instruction, SBO = byte distance between 8-row
// groups ("((8,n),2):((1,SBO),LBO)" in 16-byte units).
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;                        // base_offset = 0, layout_type (bits 62-63) = no swizzle
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, fp16 operands from shared memory (both K-major), f32 accumulators in
// registers: thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8), columns 8 j + 2 (t % 4) (+ 1)
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

// shared memory of rank_tc_kernel besides the U tile and the V ring: the accumulator hand-off of the two warpgroups,
// the barriers, the per-row threshold / exchange slots and the score-bin counters of a raise
constexpr int SMEM_FIXED = 2 * 64 * LDT * 4 + 16 * 8 + ST * TM * 8 + ST * TM * 4 * 4 + ST * NB * TM * 2 + 1024;
constexpr int SMEM_MAX = 227 * 1024;   // opt-in shared memory per block on sm_90

// V-stage ring depth that fits next to the U tile and the fixed part (2..4)
__host__ __device__ __forceinline__ int num_stages(int kp)
{
    const int budget = SMEM_MAX - SMEM_FIXED - TM * kp * 2;
    int ns = budget / (SN * kp * 2);
    return ns > 4 ? 4 : (ns < 2 ? 2 : ns);
}

// byte offset of element (row r, column c) inside a packed tile of `kp` fp16 columns
__host__ __device__ __forceinline__ size_t packed_offset(int r, int c, int kp)
{
    return ((size_t)(r >> 3) * (kp >> 3) + (c >> 3)) * 128 + (size_t)(r & 7) * 16 + (size_t)(c & 7) * 2;
}

// ---------------------------------------------------------------- scales, norms, pack kernels
// Scalars of one call, device resident (workspace `scal`, 16 x 32 bit):
//   [0] max |v| (L2 norm, bits)   [1] max |base| (bits)   [2] max |V element| (bits)   [4] sV   [5] sB  (floats)
// The tensor pass computes, for user row r,  S_r * (u.v + base)  with  S_r = sU_r * sV  from  u * sU_r,  v * sV,
// base * sB (hi + lo)  and the user-side constant  cA_r = S_r / sB.  All scales are powers of two (exact); every
// user row has its own (thresholds are per row, so rows of very different magnitude each keep full fp16 precision).
constexpr int SC_VNORM = 0, SC_BMAX = 1, SC_VABS = 2, SC_SV = 4, SC_SB = 5;

// power of two s with m * s in [2^13, 2^14) (1 for m == 0); exponent clamped so that products of two scales stay
// finite (operands beyond 2^+-46 are not brought into range: eps grows and such rows end up on the exact path)
__device__ __forceinline__ float pow2_scale(float m)
{
    if (!(m > 0.f)) return 1.f;
    int e;
    frexpf(m, &e);                              // m = fr * 2^e, fr in [0.5, 1)
    int x = 14 - e;
    x = x > 60 ? 60 : (x < -60 ? -60 : x);
    return ldexpf(1.f, x);
}

__global__ void scale_items_kernel(unsigned int* scal)
{
    float* f = reinterpret_cast<float*>(scal);
    f[SC_SV] = pow2_scale(__uint_as_float(scal[SC_VABS]));
    f[SC_SB] = pow2_scale(__uint_as_float(scal[SC_BMAX]));
}

// scales of one user row from its largest |element|
struct UserScale { float sU, cA, S; };
__device__ __forceinline__ UserScale user_scale(const unsigned int* scal, float row_absmax)
{
    const float* f = reinterpret_cast<const float*>(scal);
    const float sV = f[SC_SV], sB = f[SC_SB];
    UserScale r;
    r.sU = pow2_scale(row_absmax);
    r.cA = 0.f;
    if (__uint_as_float(scal[SC_BMAX]) > 0.f) {
        r.cA = r.sU * sV / sB;                  // powers of two: exact
        if (r.cA > 32768.f) { r.sU *= 32768.f / r.cA; r.cA = 32768.f; }      // keep cA an fp16 power of two
        if (r.cA < 5.9604645e-8f) r.cA = 0.f;   // below 2^-24: the base is left out and charged to eps
    }
    r.S = r.sU * sV;
    return r;
}

// |approx / S - exact| <= row_eps for every item, `un` = |u| (x 1.0001):
//   fp16 rounding of both operands (2^-11 each; 2^-25 absolute in the subnormal range, in scaled units)
//   + f32 accumulation inside the tensor core + the base carried as two fp16 (2^-22 relative)
__device__ __forceinline__ float row_eps(const unsigned int* scal, const UserScale& us, float un, int k)
{
    const float* f = reinterpret_cast<const float*>(scal);
    const float vmax = __uint_as_float(scal[SC_VNORM]), bmax = __uint_as_float(scal[SC_BMAX]);
    float eps = 0.00098f * un * vmax + 2.99e-8f * sqrtf((float)k) * (vmax / us.sU + un / f[SC_SV])
                + 2e-6f * (un * vmax + bmax) + 4.8e-7f * bmax + 6e-8f * us.cA / us.S;
    if (us.cA == 0.f) eps += bmax * 1.0001f;
    return eps;
}

// one thread per (row, 16-byte chunk): 8 consecutive factors -> 8 fp16.  The last KX columns are the
// base slice: user rows carry (cA, cA, 1, 0, ...), item rows carry (hi, lo, 0, ...) with hi + lo = base * sB split
// into two fp16, so the MMA itself adds S * base and the epilogue has no bias add.  Padding item rows carry
// -inf in the third slot (against the users' 1): they are never nominated.
template <int TR, bool ITEMS>
__global__ void pack_kernel(const float* __restrict__ src, const int64_t* __restrict__ row_idx, int64_t n_rows,
                            int64_t n_rows_padded, int k, int kp, const float* __restrict__ base,
                            const unsigned int* __restrict__ scal, const float* __restrict__ row_absmax,
                            uint8_t* __restrict__ dst)
{
    const float* sf = reinterpret_cast<const float*>(scal);
    const int chunks = kp >> 3;
    const int k16 = kp - KX;                    // first column of the base slice
    const int64_t total = n_rows_padded * chunks;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
        const int64_t row = t / chunks;
        const int kc = (int)(t % chunks);
        float s = sf[SC_SV], sb = sf[SC_SB];
        if (!ITEMS) {
            const UserScale us = user_scale(scal, row < n_rows ? row_absmax[row] : 0.f);
            s = us.sU; sb = us.cA;
        }
        __half v[8];
#pragma unroll
        for (int x = 0; x < 8; ++x) v[x] = __float2half_rn(0.f);
        if (kc * 8 == k16) {                    // base slice, first chunk (the second one stays zero)
            if (ITEMS) {
                if (row < n_rows) {
                    const float b = (base ? __ldg(base + row) : 0.f) * sb;
                    const __half hi = __float2half_rn(b);
                    v[0] = hi;
                    v[1] = __float2half_rn(b - __half2float(hi));
                } else {
                    v[2] = __float2half_rn(-INFINITY);
                }
            } else if (row < n_rows) {
                v[0] = __float2half_rn(sb);
                v[1] = __float2half_rn(sb);
                v[2] = __float2half_rn(1.f);
            }
        } else if (kc * 8 < k16 && row < n_rows) {
            const int64_t srow = row_idx ? row_idx[row] : row;
            const float* p = src + (size_t)srow * k + kc * 8;
#pragma unroll
            for (int x = 0; x < 8; ++x)
                if (kc * 8 + x < k) v[x] = __float2half_rn(__ldg(p + x) * s);
        }
        const int64_t tile = row / TR;
        const int r = (int)(row % TR);
        uint8_t* out = dst + (size_t)tile * TR * kp * 2 + packed_offset(r, kc * 8, kp);
        *reinterpret_cast<uint4*>(out) = *reinterpret_cast<const uint4*>(v);
    }
}

// warp per row, four rows in flight per warp: L2 norm (f32 rows) -> norm_out; the maxima over all rows of the norm,
// of |element| and of |base| are max-reduced into scal[] (as uint bits, values >= 0)
__global__ void norm_kernel(const float* __restrict__ src, const int64_t* __restrict__ row_idx, int64_t n_rows, int k,
                            float* __restrict__ norm_out, float* __restrict__ rowabs_out,
                            unsigned int* __restrict__ max_out, unsigned int* __restrict__ absmax_out,
                            const float* __restrict__ base, unsigned int* __restrict__ base_absmax_out)
{
    const int lane = threadIdx.x & 31;
    const int64_t wstride = (int64_t)gridDim.x * (blockDim.x >> 5) * 4;
    float m_norm = 0.f, m_abs = 0.f, m_base = 0.f;
    const bool vec4 = (k % 4 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
    for (int64_t row0 = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 4; row0 < n_rows; row0 += wstride) {
        float s[4] = {0.f, 0.f, 0.f, 0.f}, a[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int64_t row = row0 + r;
            if (row < n_rows) {
                const int64_t srow = row_idx ? row_idx[row] : row;
                const float* p = src + (size_t)srow * k;
                if (vec4) {                     // one 16-byte load per lane covers a 128-wide row
                    for (int f = lane * 4; f < k; f += 128) {
                        const float4 x = __ldg(reinterpret_cast<const float4*>(p + f));
                        s[r] = fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, fmaf(x.w, x.w, s[r]))));
                        a[r] = fmaxf(fmaxf(a[r], fmaxf(fabsf(x.x), fabsf(x.y))), fmaxf(fabsf(x.z), fabsf(x.w)));
                    }
                } else {
                    for (int f = lane; f < k; f += 32) {
                        const float x = __ldg(p + f);
                        s[r] = fmaf(x, x, s[r]);
                        a[r] = fmaxf(a[r], fabsf(x));
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int64_t row = row0 + r;
            const float nrm = sqrtf(group_sum<32>(s[r])) * 1.0001f;
            float ra = a[r];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ra = fmaxf(ra, __shfl_xor_sync(0xffffffffu, ra, o));
            m_abs = fmaxf(m_abs, ra);
            if (row < n_rows && lane == 0) {
                if (norm_out) norm_out[row] = nrm;
                if (rowabs_out) rowabs_out[row] = ra;
                m_norm = fmaxf(m_norm, nrm);
                if (base) m_base = fmaxf(m_base, fabsf(__ldg(base + row)));
            }
        }
    }
    // one shared maximum each: reduce per warp and look before the atomic, or a million rows serialise on one address
    if (lane == 0) {
        if (max_out && __float_as_uint(m_norm) > *reinterpret_cast<volatile unsigned int*>(max_out))
            atomicMax(max_out, __float_as_uint(m_norm));
        if (absmax_out && __float_as_uint(m_abs) > *reinterpret_cast<volatile unsigned int*>(absmax_out))
            atomicMax(absmax_out, __float_as_uint(m_abs));
        if (base_absmax_out && __float_as_uint(m_base) > *reinterpret_cast<volatile unsigned int*>(base_absmax_out))
            atomicMax(base_absmax_out, __float_as_uint(m_base));
    }
}

// ---------------------------------------------------------------- main kernel
struct RankTcParams {
    const uint8_t* __restrict__ Upack;     // [n_ut][TM x kp fp16 tile image]
    const uint8_t* __restrict__ Vpack;     // [n_it][TN x kp fp16 tile image]
    const float* __restrict__ unorm;       // [n_ut * TM] |u| per chunk row
    const float* __restrict__ uabs;        // [n_ut * TM] max |element| per chunk row (-> the row's scales)
    const unsigned int* __restrict__ scal; // [0] = max |v| bits, [1] = max |base| bits
    const int64_t* __restrict__ excl_indptr;   // already offset to the chunk's first row (may be null)
    const int32_t* __restrict__ excl_indices;
    int64_t n_rows;                        // valid rows in this chunk
    int n_ut, n_it, kp, topk;
    unsigned long long* __restrict__ lists;    // [n_ut * 4 ST warps][cap][32 lanes] interleaved lists: (score bits << 32) | item id
    int* __restrict__ row_cnt;             // [n_ut * TM][MAX_ST strips]
    int* __restrict__ row_flag;            // [n_ut * TM][MAX_ST] 1 = list overflow -> exact path
    float* __restrict__ row_tau;           // [n_ut * TM][MAX_ST] final filter tau - 2 eps of the strip (scaled units): the finish drops entries below the row's largest
    float* __restrict__ dump;              // debug: dense approximate scores [n_ut*TM][n_it*TN] or null
    int debug;                             // B200_RANK_DEBUG: timing only: 8 = screening only (no candidate is listed);
                                           // 4 = raise schedule with ratio 1.41 instead of 2 (results stay exact)
};

// Per-thread epilogue state: one thread owns one (user row, column strip) and its candidate list of up to `cap` 8-byte
// entries (score bits << 32 | item id) in global memory, interleaved with the lists of the other 31 lanes of its warp
// (entry e at list[e * 32]) and appended to with one store and a pointer bump.  Items reach a list in increasing id order and every in-place compaction keeps that order; the user's
// exclusion list (sorted too) is merged against the NEW tail of the list whenever the threshold is raised, and once
// more in the finish kernel -- the hot loop never branches on it.  Entries that fall below a later threshold are NOT
// removed eagerly: the finish kernel drops everything below the row's final filter, and a list is compacted in place
// only when more than half of it is dead.
struct RowState {
    unsigned long long* list;      // entries [cap]
    unsigned long long* wp;        // append position (hot loop); cnt is derived from it between stages
    const int32_t* ex;
    int n_ex;
    int ex_c;                      // exclusion cursor: entries [0, ex_c) have been loaded into the window
    int32_t ex_w0, ex_w1, ex_w2, ex_w3;   // next excluded ids (sorted), 0x7fffffff = none
    int cnt;                       // entries in the list
    int checked;                   // entries [0, checked) are already exclusion-filtered
    float tau, tau_f;              // tau_f = tau - 2 eps is the filter applied to every score
    float hi;                      // largest score seen at the last raise (bin range)
};

__device__ __forceinline__ float ent_score(unsigned long long e) { return __uint_as_float((unsigned)(e >> 32)); }

// sequential scan of a list with 16 independent loads in flight.  The 32 lists of a warp are INTERLEAVED in memory
// (entry e of lane l at list[e * 32 + l]), so the lock-step scans of a raise are fully coalesced: one 256-byte request
// per warp and entry (thread-private contiguous lists cost 32 sectors per request -- measured 3x slower raises).
template <int B, typename F>
__device__ __forceinline__ void scan_list(const unsigned long long* list, int L, F f)
{
    // Every batch -- the last, partial one too -- is ONE round trip of B predicated independent loads: a list lives in L2
    // (~1 us away under load) and a raise is nothing but such trips in sequence.  (An element-by-element tail loop cost one
    // trip per entry: 60 us per raise on short lists, 13 % of the epilogue warps' time, profiles/r02_rank_tc.md.)
    for (int e = 0; e < L; e += B) {
        unsigned long long v[B];
#pragma unroll
        for (int i = 0; i < B; ++i) v[i] = (e + i < L) ? list[(size_t)(e + i) * 32] : 0ull;
#pragma unroll
        for (int i = 0; i < B; ++i)
            if (e + i < L) f(v[i]);
    }
}

// named barrier of the ST epilogue warps that own the column strips of the same 32 user rows
template <int ST>
__device__ __forceinline__ void pair_sync(int bar_id)
{
    __syncwarp();
    asm volatile("bar.sync %0, %1;" :: "r"(bar_id), "n"(32 * ST) : "memory");
}

// lower edge of bin j of the range [a, a + NB * step): ONE expression, used both to bin a score and to turn the chosen
// bin back into a threshold, so that "score in bin >= j" and "score >= bin_edge(j)" are the same predicate bit for bit
__device__ __forceinline__ float bin_edge(float a, float step, int j) { return fmaf((float)j, step, a); }

// Raise the threshold of a row: tau = (approximately) the K-th largest listed score, never above it.  All 32 lanes run
// this together, each on its own list.  Steps: (1) merge the new tail of the list against the user's exclusion list and
// drop excluded items (in place); (2) ONE pass over the scores: NB-bin histogram of [lo, hi] in this thread's private
// shared-memory counters; the largest bin edge t with #(score >= t) >= K becomes tau; (3) only if more than half of the
// list is now below the filter tau - 2 eps: order-preserving compaction.
// JOINT (the scheduled raises, which all column strips of a row reach at the same stage): the ST threads of a row read
// each other's counters, so the K-th best is taken over the UNION of the row's lists -- together they keep ~K
// candidates instead of ~K each.  The control flow between the pair barriers is the same for every thread (rows that
// cannot be raised count nothing).  Solo (a list hit TRIGGER between two scheduled raises): the list's own K-th best,
// a valid lower bound; always compacts.
// `share` points at this row's exchange slots: slot s (strip s) at share[s * TM * 4]; `hist` at this row's counters:
// bin j of strip s at hist[(s * NB + j) * TM]; `tau_row` likewise at tau_row[s * TM].
template <bool JOINT, int ST>
__device__ __forceinline__ void raise_threshold(RowState& st, int K, float eps2, uint32_t tile, int strip, int cap,
                                                unsigned long long* tau_row, int* share, unsigned short* hist, int bar_id,
                                                bool dbg_nocompact = false)
{
    constexpr int SCAN_B = ST == 2 ? 32 : 16;      // loads in flight per scan batch (the chunk registers are dead during a raise)
    unsigned long long* my_tau = tau_row + strip * TM;
    int* pair_mine = share + strip * (TM * 4);
    unsigned short* hist_mine = hist + (size_t)strip * NB * TM;
    unsigned long long* __restrict__ list = st.list;
    // The other column strips of this row publish their own lower bound of the row's k-th best score; any such bound
    // (even an old one) is valid for the whole row, so take the largest.  The tag rejects a value the sibling warp left
    // behind from the previous user tile.
#pragma unroll
    for (int o = 0; o < ST; ++o) {
        if (o == strip) continue;
        const unsigned long long v = *reinterpret_cast<const volatile unsigned long long*>(tau_row + o * TM);
        const float other = __uint_as_float((unsigned)(v & 0xffffffffull));
        if ((uint32_t)(v >> 32) == tile && other > st.tau) { st.tau = other; st.tau_f = other - eps2; }
    }
    // ---- (1) exclusion merge over entries [checked, cnt).  The list tail is sorted by id and every id in it is larger
    //      than anything merged before, so one cursor walks the exclusion list once per sweep; it is read four entries
    //      per round trip (independent loads) into a register window.  Entries are moved only after the first hit.
    if (st.n_ex > 0 && st.checked < st.cnt) {
        int w = st.checked;
        for (int e0 = st.checked; e0 < st.cnt; e0 += 16) {      // 16 independent id loads per round trip;
            unsigned long long v[16];                             // a batch is read before it is written (w <= e0)
            const int nb = st.cnt - e0 < 16 ? st.cnt - e0 : 16;
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] = i < nb ? list[(size_t)(e0 + i) * 32] : 0ull;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                if (i < nb) {
                    const int32_t id = (int32_t)(v[i] & 0xffffffffull);
                    while (st.ex_w0 < id) {                       // advance the window past ids below `id`
                        st.ex_w0 = st.ex_w1; st.ex_w1 = st.ex_w2; st.ex_w2 = st.ex_w3; st.ex_w3 = 0x7fffffff;
                        if (st.ex_w0 == 0x7fffffff && st.ex_c < st.n_ex) {      // window empty: refill
                            const int c = st.ex_c;
                            st.ex_w0 = __ldg(st.ex + c);
                            st.ex_w1 = c + 1 < st.n_ex ? __ldg(st.ex + c + 1) : 0x7fffffff;
                            st.ex_w2 = c + 2 < st.n_ex ? __ldg(st.ex + c + 2) : 0x7fffffff;
                            st.ex_w3 = c + 3 < st.n_ex ? __ldg(st.ex + c + 3) : 0x7fffffff;
                            st.ex_c = c + 4;
                        }
                    }
                    if (st.ex_w0 != id) {
                        if (w != e0 + i) list[(size_t)w * 32] = v[i];
                        ++w;
                    }
                }
            }
        }
        st.cnt = w;
    }
    st.checked = st.cnt;
    const int L = st.cnt;
    // ---- (2) score range; the NB-bin histogram of [a, b]
    float lo = st.tau_f, hi = st.hi;
    if (L == 0) { lo = INFINITY; hi = -INFINITY; }
    else if (!(hi > -INFINITY) || !(lo > -1.0e37f)) {  // this list's score range is not known yet
        lo = INFINITY; hi = -INFINITY;
        scan_list<SCAN_B>(list, L, [&](unsigned long long ent) {
            const float sc = ent_score(ent);
            lo = fminf(lo, sc);
            hi = fmaxf(hi, sc);
        });
    }
    float a = lo, b = hi;                       // #(score >= a) >= K whenever the row can be raised at all
    bool act = L >= K;
#pragma unroll
    for (int j = 0; j < NB; ++j) hist_mine[j * TM] = 0;
    if (JOINT) {
        pair_mine[0] = L; pair_mine[1] = __float_as_int(lo); pair_mine[2] = __float_as_int(hi);
        pair_sync<ST>(bar_id);
        int Ltot = 0;
#pragma unroll
        for (int o = 0; o < ST; ++o) {          // every thread of the row reads the same ST slots in the same order
            const int* t = share + o * (TM * 4);
            Ltot += t[0];
            a = o == 0 ? __int_as_float(t[1]) : fminf(a, __int_as_float(t[1]));
            b = o == 0 ? __int_as_float(t[2]) : fmaxf(b, __int_as_float(t[2]));
        }
        act = Ltot >= K;                        // the same decision in all threads of the row
    } else if (!act) {
        return;
    }
    const float step = (b - a) * (1.f / NB);
    const bool ok = act && (step > 0.f) && isfinite(step) && isfinite(a);
    if (!JOINT && !ok) return;
    float new_hi = -INFINITY;
    if (ok) {
        const float inv = 1.f / step;
        scan_list<SCAN_B>(list, L, [&](unsigned long long ent) {
            const float sc = ent_score(ent);
            new_hi = fmaxf(new_hi, sc);
            if (sc >= a) {
                int j = (int)((sc - a) * inv);                  // within +-1 of the bin; made exact against bin_edge()
                j = j > NB - 1 ? NB - 1 : j;
                if (sc < bin_edge(a, step, j)) --j;
                else if (j < NB - 1 && sc >= bin_edge(a, step, j + 1)) ++j;
                if (j >= 0) hist_mine[j * TM] += 1;
            }
        });
    }
    if (JOINT) pair_sync<ST>(bar_id);           // all counters of the row are complete
    int chosen = -1, acc = 0;
    if (ok) {
#pragma unroll 4
        for (int j = NB - 1; j >= 0; --j) {
            int t = 0;
            if (JOINT) {
#pragma unroll
                for (int o = 0; o < ST; ++o) t += hist[(size_t)(o * NB + j) * TM];
            } else {
                t = hist_mine[j * TM];
            }
            acc += t;
            if (acc >= K && chosen < 0) chosen = j;
        }
    }
    if (JOINT) pair_sync<ST>(bar_id);           // everybody has read the row's slots and counters: they may be reused
    if (L > 0) st.hi = fmaxf(hi, new_hi);       // scores above the old range only make the top bin fuller
    const bool raised = ok && chosen >= 0;
    bool want = false;
    if (raised) {
        const float t_new = bin_edge(a, step, chosen);
        if (t_new > st.tau) st.tau = t_new;
        st.tau_f = st.tau - eps2;
        *reinterpret_cast<volatile unsigned long long*>(my_tau) = ((unsigned long long)tile << 32) | __float_as_uint(st.tau);
        // upper bound on this list's entries >= tau_f: its counters from the filter's bin on
        int alive = 0;
        int jf = (int)((st.tau_f - a) * (1.f / step)) - 1;
        jf = jf < 0 ? 0 : (jf > NB - 1 ? NB - 1 : jf);
#pragma unroll 4
        for (int j = NB - 1; j >= 0; --j) alive += (j >= jf) ? (int)hist_mine[j * TM] : 0;
        want = true;                            // lists stay short: the finish reads them with a 256-byte stride
        (void)alive;
    }
    // ---- (3) compaction (order-preserving), when at least half of the list is dead weight (always after a solo raise).
    //      Joint raises decide per warp (the lanes run in lock step anyway); no lane has left the function before this
    //      vote.  A solo raise decides per lane: lanes that could not raise returned above.
    bool go = want;
    if (JOINT) go = __any_sync(0xffffffffu, want);
    if (dbg_nocompact && L < cap / 2) go = false;      // timing experiment (debug bit 16): compact only lists that are half full
    if (go) {
        int w = 0;          // writes trail the reads (w <= e); each batch of 16 is read before it is written
        scan_list<SCAN_B>(list, L, [&](unsigned long long ent) {
            if (ent_score(ent) >= st.tau_f) { list[(size_t)w * 32] = ent; ++w; }
        });
        st.cnt = w;
        st.checked = w;
    }
}

__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// append the scores of one group of four that pass the filter to the calling lane's list
__device__ __noinline__ unsigned long long* append4(unsigned long long* wp, float tau_f, float s0, float s1, float s2,
                                                    float s3, int32_t id)
{
    if (s0 > tau_f) { *wp = ((unsigned long long)__float_as_uint(s0) << 32) | (uint32_t)id; wp += 32; }
    if (s1 > tau_f) { *wp = ((unsigned long long)__float_as_uint(s1) << 32) | (uint32_t)(id + 1); wp += 32; }
    if (s2 > tau_f) { *wp = ((unsigned long long)__float_as_uint(s2) << 32) | (uint32_t)(id + 2); wp += 32; }
    if (s3 > tau_f) { *wp = ((unsigned long long)__float_as_uint(s3) << 32) | (uint32_t)(id + 3); wp += 32; }
    return wp;
}

// one 32-column chunk of the accumulator (the item base is already in it: extra K slice of the MMA):
// append every score above tau_f.  Scores are screened four at a time -- max of the four against the
// row's filter, one warp vote -- and only when some lane of the warp has a hit (a few percent of the
// groups once the thresholds have risen) does the warp run the predicated appends for that group.
// ~1.25 instructions per score on the common path.
template <bool DUMP>
__device__ __forceinline__ void epilogue_chunk(uint32_t (&r)[32], RowState& st, int32_t id0,
                                               float* __restrict__ dump_row, bool valid, float invS)
{
    if (DUMP) {
        if (valid) {
#pragma unroll
            for (int x = 0; x < 32; ++x) dump_row[id0 + x] = __uint_as_float(r[x]) * invS;
        }
    } else {
    // phase 1: maxima of the eight groups of four and of the whole
    // chunk; ONE vote decides whether any of the warp's 32 x 32 scores passes the filter at all
    float m[8];
#pragma unroll
    for (int j4 = 0; j4 < 8; ++j4)
        m[j4] = fmaxf(fmax3(__uint_as_float(r[j4 * 4 + 0]), __uint_as_float(r[j4 * 4 + 1]), __uint_as_float(r[j4 * 4 + 2])),
                      __uint_as_float(r[j4 * 4 + 3]));
    const float mall = fmax3(fmax3(m[0], m[1], m[2]), fmax3(m[3], m[4], m[5]), fmaxf(m[6], m[7]));
    if (!__any_sync(0xffffffffu, mall > st.tau_f)) return;
    // the eight group votes back to back (no branch between them, so their latencies overlap)
    bool hit[8];
#pragma unroll
    for (int j4 = 0; j4 < 8; ++j4) hit[j4] = __any_sync(0xffffffffu, m[j4] > st.tau_f);          // warp-uniform
    // phase 2: predicated appends for the groups some lane of the warp has a hit in (out of line: thirty-two
    // inlined copies of the append sequence made the hot loop overflow the instruction cache)
#pragma unroll
    for (int j4 = 0; j4 < 8; ++j4) {
        if (hit[j4])
            st.wp = append4(st.wp, st.tau_f, __uint_as_float(r[j4 * 4 + 0]), __uint_as_float(r[j4 * 4 + 1]),
                            __uint_as_float(r[j4 * 4 + 2]), __uint_as_float(r[j4 * 4 + 3]), id0 + j4 * 4);
    }
    }
}

// One CTA per SM works on 128-user tiles; per tile it streams the packed item side in stages of SN = 128 items.
// Barrier protocol:
//   full[s], u_full      armed by the TMA producer (expect_tx), completed by the bulk copies
//   empty[s], u_empty    EPI_WARPS arrivals: every consumer warp, once its wgmma reading the stage (the U tile) retired
// Each consumer warpgroup computes its 64 rows x SN columns with wgmma into registers, passes them through its own
// shared-memory block (row stride LDT) and reads back one (row, 64-column strip) per thread: warp w of warpgroup g owns
// rows 64 g + 32 (w & 1) + lane, strip w >> 1 -- the 32-row quarter q = 2 g + (w & 1) of the tile, as in the list layout
// the finish kernels read.
// DBG: the timing-experiment switches (B200_RANK_DEBUG) are compiled into a separate instantiation; the production kernel
// carries none of their branches.
template <bool DUMP, bool DBG = false>
__global__ void __launch_bounds__(THREADS, 1) rank_tc_kernel(const RankTcParams p)
{
    const int dbg = DBG ? p.debug : 0;
    constexpr int CAP_T = CAP;
    constexpr int TRIGGER = CAP_T / 2;
    extern __shared__ __align__(1024) uint8_t smem[];
    const int kp = p.kp;
    const uint32_t u_bytes = TM * kp * 2, s_bytes = SN * kp * 2;
    const int NS = num_stages(kp);
    const int n_st = p.n_it * (TN / SN);          // stages per user tile
    uint8_t* sU = smem;
    uint8_t* sV = sU + u_bytes;
    float* sT = reinterpret_cast<float*>(sV + (size_t)NS * s_bytes);          // [2 warpgroups][64 rows][LDT]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sT + 2 * 64 * LDT);
    uint64_t* full = bars;            // [NS]  V stage landed                TMA -> consumers
    uint64_t* empty = bars + 4;       // [NS]  wgmma reading the stage retired  consumers -> TMA
    uint64_t* u_full = bars + 8;      // U tile landed
    uint64_t* u_empty = bars + 9;     // all wgmma of the user tile retired
    // [ST strips][TM rows] last published row threshold, tagged with the tile it belongs to: (tile << 32) | f32 bits
    unsigned long long* tau_share = reinterpret_cast<unsigned long long*>(bars + 16);
    // [ST strips][TM rows][4] list length and score range exchanged by the ST threads of a row
    int* pair_share = reinterpret_cast<int*>(tau_share + ST * TM);
    // [ST strips][NB bins][TM rows] per-thread score-bin counters of a threshold raise
    unsigned short* hist_share = reinterpret_cast<unsigned short*>(pair_share + ST * TM * 4);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < NS; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, EPI_WARPS); }
        mbar_init(u_full, 1);
        mbar_init(u_empty, EPI_WARPS);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            uint32_t it_global = 0, tile_no = 0;
            for (int ut = blockIdx.x; ut < p.n_ut; ut += gridDim.x, ++tile_no) {
                if (tile_no > 0) mbar_wait_backoff(u_empty, (tile_no - 1) & 1);
                mbar_expect_tx(u_full, u_bytes);
                bulk_g2s(sU, p.Upack + (size_t)ut * u_bytes, u_bytes, u_full);
                for (int it = 0; it < n_st; ++it, ++it_global) {
                    const int s = it_global % NS;
                    const uint32_t round = it_global / NS;
                    if (round > 0) mbar_wait_backoff(empty + s, (round - 1) & 1);
                    mbar_expect_tx(full + s, s_bytes);
                    bulk_g2s(sV + (size_t)s * s_bytes, p.Vpack + (size_t)it * s_bytes, s_bytes, full + s);
                }
            }
        }
    } else if (warp >= 4) {
        // ===================== consumers: wgmma, then one (user row, column strip) per thread =====================
        const int g = (warp - 4) >> 2;                   // warpgroup: rows [64 g, 64 g + 64) of the tile
        const int w = warp & 3;                          // warp of the warpgroup
        const int q = 2 * g + (w & 1);                   // 32-row quarter of the tile
        const int half = w >> 1;                         // column strip: columns [half * STRIP_N, (half + 1) * STRIP_N)
        float* tg = sT + (size_t)g * 64 * LDT;
        const uint32_t lbo = 128, sbo = (uint32_t)(kp >> 3) * 128;
        const uint32_t a_base = smem_u32(sU) + (uint32_t)g * 8 * sbo;      // the warpgroup's 64 rows = 8 core-matrix rows
        uint32_t it_global = 0, tile_no = 0;
        for (int ut = blockIdx.x; ut < p.n_ut; ut += gridDim.x, ++tile_no) {
            const int64_t row = (int64_t)ut * TM + q * 32 + lane;
            const bool valid = row < p.n_rows;
            const float un = valid ? p.unorm[row] : 0.f;
            // scores, thresholds and eps live in the scaled units of the accumulator (x S, a power of two)
            const UserScale us = user_scale(p.scal, valid ? p.uabs[row] : 0.f);
            const float eps = us.S * row_eps(p.scal, us, un, p.kp - KX);
            const float invS = 1.f / us.S;
            const float eps2 = 2.f * eps;
            RowState st;
            st.list = p.lists + ((size_t)(ut * EPI_WARPS + half * 4 + q) * CAP_T) * 32 + lane;
            st.ex = nullptr; st.n_ex = 0; st.ex_c = 0;
            st.ex_w0 = st.ex_w1 = st.ex_w2 = st.ex_w3 = 0x7fffffff;
            if (valid && p.excl_indptr) {
                const int64_t a = p.excl_indptr[row], b = p.excl_indptr[row + 1];
                st.ex = p.excl_indices + a;
                st.n_ex = (int)(b - a);
                if (st.n_ex > 0) {                         // first window (ids are < 0x7fffffff by construction)
                    st.ex_w0 = __ldg(st.ex);
                    st.ex_w1 = 1 < st.n_ex ? __ldg(st.ex + 1) : 0x7fffffff;
                    st.ex_w2 = 2 < st.n_ex ? __ldg(st.ex + 2) : 0x7fffffff;
                    st.ex_w3 = 3 < st.n_ex ? __ldg(st.ex + 3) : 0x7fffffff;
                    st.ex_c = 4;
                }
            }
            st.cnt = 0; st.checked = 0;
            st.tau = -INFINITY; st.hi = -INFINITY;
            tau_share[half * TM + q * 32 + lane] = ((unsigned long long)(uint32_t)ut << 32) | 0xff800000u;   // -inf
            st.tau_f = valid ? -1.0e38f : INFINITY;       // padding items score -inf: never above the filter
            if (dbg & 8) st.tau_f = INFINITY;         // timing experiment: screening only (nothing is ever listed)
            if ((dbg & 32) && valid) {                // timing experiment: start from the PREVIOUS call's final filters (perfect thresholds)
                float t = -INFINITY;
#pragma unroll
                for (int x = 0; x < ST; ++x) t = fmaxf(t, p.row_tau[row * MAX_ST + x]);
                st.tau_f = t; st.tau = t + eps2;
            }
            int flag = 0;
            float* dump_row = DUMP ? p.dump + (size_t)(valid ? row : 0) * ((size_t)p.n_it * TN) : nullptr;
            int next_sched = 2;
            mbar_wait(u_full, tile_no & 1);
            for (int it = 0; it < n_st; ++it, ++it_global) {
                const int s = it_global % NS;
                mbar_wait(full + s, (it_global / NS) & 1);
                const uint32_t b_base = smem_u32(sV + (size_t)s * s_bytes);
                float acc[64];                              // set here so that it is dead during the screening
#pragma unroll
                for (int x = 0; x < 64; ++x) acc[x] = 0.f;
                __syncwarp();
                wgmma_fence();
                for (int ks = 0; ks < (kp >> 4); ++ks)
                    wgmma_m64n128k16(acc, gmma_desc(a_base + ks * 256, lbo, sbo), gmma_desc(b_base + ks * 256, lbo, sbo),
                                     ks > 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait_all();
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(empty + s);                 // the stage may be refilled
                    if (it == n_st - 1) mbar_arrive(u_empty);
                }
                // accumulator fragments -> the warpgroup's block -> one 64-column row strip per thread
                named_sync(5 + g, 128);                     // every thread has read the previous stage's block
                {
                    const int fr = 16 * w + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
                    for (int j = 0; j < SN / 8; ++j) {
                        *reinterpret_cast<float2*>(tg + (size_t)fr * LDT + 8 * j + fc) = make_float2(acc[4 * j], acc[4 * j + 1]);
                        *reinterpret_cast<float2*>(tg + (size_t)(fr + 8) * LDT + 8 * j + fc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
                    }
                }
                named_sync(5 + g, 128);
                uint32_t r0[32], r1[32];
                {
                    const float4* src = reinterpret_cast<const float4*>(tg + (size_t)((w & 1) * 32 + lane) * LDT + half * STRIP_N);
#pragma unroll
                    for (int x = 0; x < 8; ++x) {
                        const float4 v0 = src[x], v1 = src[8 + x];
                        r0[4 * x] = __float_as_uint(v0.x); r0[4 * x + 1] = __float_as_uint(v0.y);
                        r0[4 * x + 2] = __float_as_uint(v0.z); r0[4 * x + 3] = __float_as_uint(v0.w);
                        r1[4 * x] = __float_as_uint(v1.x); r1[4 * x + 1] = __float_as_uint(v1.y);
                        r1[4 * x + 2] = __float_as_uint(v1.z); r1[4 * x + 3] = __float_as_uint(v1.w);
                    }
                }
                const int32_t item0 = it * SN + half * STRIP_N;
                st.wp = st.list + (size_t)st.cnt * 32;
                epilogue_chunk<DUMP>(r0, st, item0, dump_row, valid, invS);
                epilogue_chunk<DUMP>(r1, st, item0 + 32, dump_row, valid, invS);
                st.cnt = (int)((st.wp - st.list) >> 5);
                if (!DUMP) {
                    // Raise schedule: after stages 2, 4, 8, 16, ... for EVERY warp at once (doing it in all warps at the
                    // same stage costs one stall instead of eight), plus whenever a list reaches TRIGGER.  Between two
                    // scheduled raises a list gains ~K ln 2 entries, so the lists stay short.  A list grows by at most
                    // STRIP_N entries per stage: keep cnt <= CAP - STRIP_N.
                    const int done = it + 1;
                    // ... and once more after the LAST stage: the lists then hold ~K ln(n_st / last raise) entries above a
                    // stale threshold, every one of which the finish kernel would re-score exactly (a 512-byte gather from V
                    // per candidate: the finish is HBM-bound on those gathers)
                    const bool scheduled = (done == next_sched && !(dbg & 64)) || done == n_st;      // bit 64: timing experiment, final raise only
                    if (scheduled) {               // geometric schedule, ratio 2 (or ~1.41 with debug bit 4)
                        const int grown = (dbg & 4) ? (done * 181) >> 7 : done * 2;
                        next_sched = grown > done ? grown : done + 1;
                    }
                    int* share = pair_share + ((q * 32 + lane) << 2);
                    unsigned short* hist = hist_share + q * 32 + lane;
                    unsigned long long* tau_row = tau_share + q * 32 + lane;
                    if (scheduled)
                        raise_threshold<true, ST>(st, p.topk, eps2, (uint32_t)ut, half, CAP_T, tau_row, share, hist, 1 + q, (dbg & 16) != 0);
                    else if (__any_sync(0xffffffffu, st.cnt >= TRIGGER))
                        raise_threshold<false, ST>(st, p.topk, eps2, (uint32_t)ut, half, CAP_T, tau_row, share, hist, 1 + q);
                    if (st.cnt > CAP_T - STRIP_N) { flag = 1; st.cnt = 0; st.checked = 0; st.tau_f = INFINITY; }
                }
            }
            if (valid && !DUMP) {
                p.row_cnt[row * MAX_ST + half] = st.cnt;
                p.row_flag[row * MAX_ST + half] = flag;
                p.row_tau[row * MAX_ST + half] = st.tau_f;
            }
        }
    }
}

// ---------------------------------------------------------------- finish kernel
struct FinishParams {
    const float* __restrict__ U;
    const int64_t* __restrict__ user_idx;      // offset to the chunk (may be null: rows q0..)
    int64_t q0;                                // first query of the chunk
    const float* __restrict__ V;
    const float* __restrict__ item_base;
    const float* __restrict__ user_off;        // indexed by global query
    int64_t n_rows;
    int k, topk;
    const unsigned long long* __restrict__ lists;   // thread-private lists of (score bits << 32 | id) entries (see RankTcParams)
    const int* __restrict__ row_cnt;
    const int* __restrict__ row_flag;
    const float* __restrict__ row_tau;         // final filter of each (row, strip), scaled units
    const int64_t* __restrict__ excl_indptr;   // offset to the chunk (may be null)
    const int32_t* __restrict__ excl_indices;
    int32_t* __restrict__ out_ids;             // offset to the chunk
    float* __restrict__ out_scores;
    int* __restrict__ overflow_rows;           // [0] = count, [1..] = global query indices
    int* __restrict__ big_rows;                // [0] = count, [1..] = chunk rows whose lists exceed the warp kernel's capacity
    const int* __restrict__ row_list;          // block kernel: null = every row, else [0] = count, [1..] = chunk rows
    int strips, cap;                           // column strips per row (2 or 4) and the capacity of one strip list
};

// list block of (user tile ut, row r of the tile, strip s)
__device__ __forceinline__ const unsigned long long* finish_list(const FinishParams& p, int64_t ut, int r, int s)
{
    return p.lists + ((size_t)(ut * (4 * p.strips) + s * 4 + (r >> 5)) * p.cap) * 32 + (r & 31);      // entry e at [e * 32]
}

// STAGED: the candidates' item rows are gathered warp-cooperatively (one coalesced 16-byte cp.async per lane
// and row, 32 rows in flight per warp) into shared memory, then every lane runs the serial f64 chain of ITS
// candidate out of shared memory (row stride = k*4 + 16 bytes: conflict-free 16-byte reads).  A thread
// gathering its own row from global memory touches 32 different lines per load instruction and thrashes L1.
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src_gmem)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(smem_u32(dst_smem)), "l"(src_gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }

template <bool STAGED>
__global__ void __launch_bounds__(128) rank_tc_finish_kernel(const FinishParams p)
{
    extern __shared__ __align__(16) unsigned char fin_stage[];      // STAGED: [128 rows][k*4 + 16 bytes]
    __shared__ unsigned long long sort_buf[2 * CAP];
    __shared__ double su[MAX_KP];                   // the user's factors, widened once per row
    __shared__ int cand_n;                          // survivors of the row's lists
    const int tid = threadIdx.x;
    const bool vec4 = (p.k % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.V) & 15) == 0);
    const int stride = p.k * 4 + 16;
    const int64_t n_iter = p.row_list ? (int64_t)p.row_list[0] : p.n_rows;
    for (int64_t it = blockIdx.x; it < n_iter; it += gridDim.x) {
        const int64_t row = p.row_list ? (int64_t)p.row_list[1 + it] : it;
        __syncthreads();
        int Ls[MAX_ST] = {0, 0, 0, 0};
        int any_flag = 0;
        float tau_f = -INFINITY;                    // the row's final filter: the largest of its strips' (each is valid)
#pragma unroll
        for (int x = 0; x < MAX_ST; ++x) {
            if (x < p.strips) {
                Ls[x] = p.row_cnt[row * MAX_ST + x];
                any_flag |= p.row_flag[row * MAX_ST + x];
                tau_f = fmaxf(tau_f, p.row_tau[row * MAX_ST + x]);
            }
        }
        if (any_flag) {
            if (tid == 0) {
                const int slot = atomicAdd(p.overflow_rows, 1);
                p.overflow_rows[1 + slot] = (int)(p.q0 + row);
            }
            continue;
        }
        const int64_t ut = row / TM;
        const int r = (int)(row % TM);
        const int64_t gq = p.q0 + row;
        const int64_t urow = p.user_idx ? p.user_idx[row] : gq;
        const float* u = p.U + (size_t)urow * p.k;
        const float uo = p.user_off ? __ldg(p.user_off + gq) : 0.f;
        const int32_t* ex = nullptr;
        int n_ex = 0;
        if (p.excl_indptr) {
            const int64_t a = p.excl_indptr[row], b = p.excl_indptr[row + 1];
            ex = p.excl_indices + a;
            n_ex = (int)(b - a);
        }
        // survivors of the row's lists (approximate score >= the final filter) -> sort_buf[0, L) (ids, any order)
        if (tid == 0) cand_n = 0;
        for (int f = tid; f < p.k; f += 128) su[f] = (double)__ldg(u + f);
        __syncthreads();
        for (int x = 0; x < p.strips; ++x) {
            const unsigned long long* list = finish_list(p, ut, r, x);
            for (int e = tid; e < Ls[x]; e += 128) {
                const unsigned long long ent = list[(size_t)e * 32];
                if (ent_score(ent) >= tau_f) {
                    const int pos = atomicAdd(&cand_n, 1);
                    sort_buf[pos] = ent & 0xffffffffull;
                }
            }
        }
        __syncthreads();
        const int L = cand_n;                       // <= strips * cap = 2 * CAP
        int sort_n = 32;                            // power of two >= L (padding keys are 0 = below every entry)
        while (sort_n < L) sort_n <<= 1;
        for (int e = tid; e < sort_n; e += 128) {
            unsigned long long key = 0ull;
            int32_t id = -1;
            if (e < L) {
                id = (int32_t)(uint32_t)sort_buf[e];
                if (n_ex) {                         // entries appended after the last merge are still unfiltered
                    int lo = 0, hi = n_ex;
                    while (lo < hi) {
                        const int mid = (lo + hi) >> 1;
                        if (__ldg(ex + mid) < id) lo = mid + 1; else hi = mid;
                    }
                    if (lo < n_ex && __ldg(ex + lo) == id) id = -1;
                }
            }
            double acc = 0.0;                      // f ascending, one f64 fma per factor: == score_batch_kernel
            if (STAGED) {
                // sort_n is a multiple of 32 and e advances by 128: whole warps stay together in this loop
                const int lane = tid & 31;
                unsigned char* wstage = fin_stage + (size_t)(tid & ~31) * stride;
                if (__any_sync(0xffffffffu, id >= 0)) {
#pragma unroll 8
                    for (int c = 0; c < 32; ++c) {
                        const int32_t idc = __shfl_sync(0xffffffffu, id, c);
                        if (idc >= 0 && lane * 4 < p.k)
                            cp_async16(wstage + (size_t)c * stride + lane * 16, p.V + (size_t)idc * p.k + lane * 4);
                    }
                    cp_async_wait_all();
                    __syncwarp();
                    if (id >= 0) {
                        const float4* rowp = reinterpret_cast<const float4*>(wstage + (size_t)lane * stride);
                        for (int f = 0; f < p.k; f += 4) {
                            const float4 x = rowp[f >> 2];
                            acc = fma(su[f], (double)x.x, acc);
                            acc = fma(su[f + 1], (double)x.y, acc);
                            acc = fma(su[f + 2], (double)x.z, acc);
                            acc = fma(su[f + 3], (double)x.w, acc);
                        }
                    }
                    __syncwarp();                   // the stage is rewritten by the next batch
                }
            } else if (id >= 0) {
                const float* v = p.V + (size_t)id * p.k;
                if (vec4) {
                    // the row gather is latency bound: keep 8 independent 16-byte loads in flight
                    for (int f = 0; f < p.k; f += 32) {
                        float4 x[8];
#pragma unroll
                        for (int i = 0; i < 8; ++i)
                            x[i] = (f + 4 * i < p.k) ? __ldg(reinterpret_cast<const float4*>(v + f + 4 * i))
                                                     : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            if (f + 4 * i < p.k) {
                                acc = fma(su[f + 4 * i], (double)x[i].x, acc);
                                acc = fma(su[f + 4 * i + 1], (double)x[i].y, acc);
                                acc = fma(su[f + 4 * i + 2], (double)x[i].z, acc);
                                acc = fma(su[f + 4 * i + 3], (double)x[i].w, acc);
                            }
                        }
                    }
                } else {
                    for (int f = 0; f < p.k; ++f) acc = fma(su[f], (double)__ldg(v + f), acc);
                }
            }
            if (id >= 0) {
                const float base = p.item_base ? __ldg(p.item_base + id) : 0.f;
                const float sc = __fadd_rn(__fadd_rn(base, uo), __double2float_rn(acc));      // == score_batch_kernel
                key = ((unsigned long long)float_key(sc) << 32) | (unsigned)(0xffffffffu - (unsigned)id);
            }
            sort_buf[e] = key;
        }
        __syncthreads();
        for (int size = 2; size <= sort_n; size <<= 1) {
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                for (int x = tid; x < sort_n / 2; x += 128) {
                    const int lo = 2 * x - (x & (stride - 1));
                    const int hi = lo + stride;
                    const bool desc = ((lo & size) == 0);
                    const unsigned long long a = sort_buf[lo], b = sort_buf[hi];
                    if ((a < b) == desc) { sort_buf[lo] = b; sort_buf[hi] = a; }
                }
                __syncthreads();
            }
        }
        for (int x = tid; x < p.topk; x += 128) {
            int32_t id = -1;
            float sc = -INFINITY;
            const unsigned long long ent = x < sort_n ? sort_buf[x] : 0ull;
            if (ent != 0ull) {                              // excluded / padding keys are 0 and sort last
                id = (int32_t)(0xffffffffu - (unsigned)(ent & 0xffffffffull));
                const unsigned kb = (unsigned)(ent >> 32);           // invert float_key
                const unsigned bits = (kb & 0x80000000u) ? (kb & 0x7fffffffu) : ~kb;
                sc = __uint_as_float(bits);
            }
            p.out_ids[(size_t)row * p.topk + x] = id;
            p.out_scores[(size_t)row * p.topk + x] = sc;
        }
    }
}

// One WARP per row (the common case: a few hundred candidates): no block barriers anywhere, ten rows in flight per
// SM instead of two, so the dependent chain list -> exclusion search -> row gather -> f64 dot -> sort of one row
// hides behind the other rows'.  Rows with more than FW_KEYS candidates go to the block kernel (big_rows).
constexpr int FW_KEYS = 512;
__host__ __device__ inline size_t finish_warp_smem(int k) { return (size_t)FW_KEYS * 8 + (size_t)MAX_KP * 8 + (size_t)32 * (k * 4 + 16); }

__global__ void __launch_bounds__(32) rank_tc_finish_warp_kernel(const FinishParams p)
{
    extern __shared__ __align__(16) unsigned char fw_smem[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(fw_smem);               // [FW_KEYS]
    double* su = reinterpret_cast<double*>(fw_smem + (size_t)FW_KEYS * 8);                   // [MAX_KP]
    unsigned char* stage = fw_smem + (size_t)FW_KEYS * 8 + (size_t)MAX_KP * 8;               // [32][k*4 + 16]
    const int lane = threadIdx.x;
    const int stride = p.k * 4 + 16;
    for (int64_t row = blockIdx.x; row < p.n_rows; row += gridDim.x) {
        __syncwarp();
        int Ls[MAX_ST] = {0, 0, 0, 0};
        int any_flag = 0;
        float tau_f = -INFINITY;                    // the row's final filter: the largest of its strips' (each is valid)
#pragma unroll
        for (int x = 0; x < MAX_ST; ++x) {
            if (x < p.strips) {
                Ls[x] = p.row_cnt[row * MAX_ST + x];
                any_flag |= p.row_flag[row * MAX_ST + x];
                tau_f = fmaxf(tau_f, p.row_tau[row * MAX_ST + x]);
            }
        }
        if (any_flag) {
            if (lane == 0) {
                const int slot = atomicAdd(p.overflow_rows, 1);
                p.overflow_rows[1 + slot] = (int)(p.q0 + row);
            }
            continue;
        }
        const int64_t ut = row / TM;
        const int r = (int)(row % TM);
        // survivors of the row's lists (approximate score >= the final filter): ids -> keys[0, L), coalesced reads of the
        // thread-private list blocks, order-preserving warp compaction
        int L = 0;
        for (int x = 0; x < p.strips; ++x) {
            const unsigned long long* list = finish_list(p, ut, r, x);
            for (int e0 = 0; e0 < Ls[x]; e0 += 32) {
                const int e = e0 + lane;
                const unsigned long long ent = e < Ls[x] ? list[(size_t)e * 32] : 0ull;
                const bool keep = e < Ls[x] && ent_score(ent) >= tau_f;
                const unsigned m = __ballot_sync(0xffffffffu, keep);
                const int pos = L + __popc(m & ((1u << lane) - 1u));
                if (keep && pos < FW_KEYS) keys[pos] = ent & 0xffffffffull;
                L += __popc(m);
            }
        }
        if (L > FW_KEYS) {
            if (lane == 0) {
                const int slot = atomicAdd(p.big_rows, 1);
                p.big_rows[1 + slot] = (int)row;
            }
            continue;
        }
        __syncwarp();
        const int64_t gq = p.q0 + row;
        const int64_t urow = p.user_idx ? p.user_idx[row] : gq;
        const float* u = p.U + (size_t)urow * p.k;
        const float uo = p.user_off ? __ldg(p.user_off + gq) : 0.f;
        const int32_t* ex = nullptr;
        int n_ex = 0;
        if (p.excl_indptr) {
            const int64_t a = p.excl_indptr[row], b = p.excl_indptr[row + 1];
            ex = p.excl_indices + a;
            n_ex = (int)(b - a);
        }
        int sort_n = 32;                            // power of two >= L (padding keys are 0 = below every entry)
        while (sort_n < L) sort_n <<= 1;
        for (int f = lane; f < p.k; f += 32) su[f] = (double)__ldg(u + f);
        __syncwarp();
        // resolve every candidate first (list entry -> id, membership in the sorted exclusion list by a
        // branch-free lower bound): four independent chains per lane are in flight per pass
        int pow2 = 1;
        while (pow2 < n_ex) pow2 <<= 1;
        for (int e0 = lane; e0 < sort_n; e0 += 128) {
            int32_t cid[4];
            int lo[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int e = e0 + 32 * j;
                cid[j] = -1;
                lo[j] = 0;
                if (e < L) cid[j] = (int32_t)(uint32_t)keys[e];
            }
            if (n_ex) {                             // entries appended after the last merge are still unfiltered
                for (int half = pow2; half > 0; half >>= 1) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int mid = lo[j] + half;
                        if (mid <= n_ex && __ldg(ex + mid - 1) < cid[j]) lo[j] = mid;
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (cid[j] >= 0 && lo[j] < n_ex && __ldg(ex + lo[j]) == cid[j]) cid[j] = -1;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (e0 + 32 * j < sort_n) keys[e0 + 32 * j] = (unsigned long long)(uint32_t)cid[j];
        }
        __syncwarp();
        for (int e = lane; e < sort_n; e += 32) {
            unsigned long long key = 0ull;
            const int32_t id = (int32_t)(uint32_t)keys[e];
            if (__any_sync(0xffffffffu, id >= 0)) {
#pragma unroll 8
                for (int c = 0; c < 32; ++c) {
                    const int32_t idc = __shfl_sync(0xffffffffu, id, c);
                    if (idc >= 0 && lane * 4 < p.k)
                        cp_async16(stage + (size_t)c * stride + lane * 16, p.V + (size_t)idc * p.k + lane * 4);
                }
                cp_async_wait_all();
                __syncwarp();
                if (id >= 0) {
                    const float4* rowp = reinterpret_cast<const float4*>(stage + (size_t)lane * stride);
                    double acc = 0.0;              // f ascending, one f64 fma per factor: == score_batch_kernel
                    for (int f = 0; f < p.k; f += 4) {
                        const float4 x = rowp[f >> 2];
                        acc = fma(su[f], (double)x.x, acc);
                        acc = fma(su[f + 1], (double)x.y, acc);
                        acc = fma(su[f + 2], (double)x.z, acc);
                        acc = fma(su[f + 3], (double)x.w, acc);
                    }
                    const float base = p.item_base ? __ldg(p.item_base + id) : 0.f;
                    const float sc = __fadd_rn(__fadd_rn(base, uo), __double2float_rn(acc));      // == score_batch_kernel
                    key = ((unsigned long long)float_key(sc) << 32) | (unsigned)(0xffffffffu - (unsigned)id);
                }
                __syncwarp();                       // the stage is rewritten by the next batch
            }
            keys[e] = key;
        }
        __syncwarp();
        for (int size = 2; size <= sort_n; size <<= 1) {
            for (int st = size >> 1; st > 0; st >>= 1) {
                for (int x = lane; x < sort_n / 2; x += 32) {
                    const int lo = 2 * x - (x & (st - 1));
                    const int hi = lo + st;
                    const bool desc = ((lo & size) == 0);
                    const unsigned long long a = keys[lo], b = keys[hi];
                    if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
                }
                __syncwarp();
            }
        }
        for (int x = lane; x < p.topk; x += 32) {
            int32_t id = -1;
            float sc = -INFINITY;
            const unsigned long long ent = x < sort_n ? keys[x] : 0ull;
            if (ent != 0ull) {                              // excluded / padding keys are 0 and sort last
                id = (int32_t)(0xffffffffu - (unsigned)(ent & 0xffffffffull));
                const unsigned kb = (unsigned)(ent >> 32);           // invert float_key
                const unsigned bits = (kb & 0x80000000u) ? (kb & 0x7fffffffu) : ~kb;
                sc = __uint_as_float(bits);
            }
            p.out_ids[(size_t)row * p.topk + x] = id;
            p.out_scores[(size_t)row * p.topk + x] = sc;
        }
    }
}

// ---------------------------------------------------------------- workspace layout
struct Layout {
    int kp;
    int64_t n_it, chunk_rows, chunk_ut;
    size_t off_vpack, off_scal, off_upack, off_unorm, off_uabs, off_lists, off_cnt, off_flag, off_tau, off_over, off_big, off_slab, total;
};

static Layout make_layout(int64_t n_q, int64_t n_items, int k)
{
    Layout L;
    L.kp = (k + 15) / 16 * 16 + KX;
    L.n_it = (n_items + TN - 1) / TN;
    int64_t n_ut = (n_q + TM - 1) / TM;
    L.chunk_ut = n_ut < CHUNK_TILES ? n_ut : CHUNK_TILES;
    L.chunk_rows = L.chunk_ut * TM;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t at = o; o += (bytes + 1023) / 1024 * 1024; return at; };
    L.off_vpack = take((size_t)L.n_it * TN * L.kp * 2);
    L.off_scal = take(64);
    L.off_upack = take((size_t)L.chunk_ut * TM * L.kp * 2);
    L.off_unorm = take((size_t)L.chunk_rows * 4);
    L.off_uabs = take((size_t)L.chunk_rows * 4);
    L.off_lists = take((size_t)L.chunk_ut * EPI_WARPS * CAP * 32 * 8);  // = EPI_WARPS x 32 lanes x CAP x (score + id)
    L.off_cnt = take((size_t)L.chunk_rows * MAX_ST * 4);
    L.off_flag = take((size_t)L.chunk_rows * MAX_ST * 4);
    L.off_tau = take((size_t)L.chunk_rows * MAX_ST * 4);
    L.off_over = take((size_t)(L.chunk_rows + 1) * 4);
    L.off_big = take((size_t)(L.chunk_rows + 1) * 4);
    L.off_slab = take((size_t)n_items * 4);          // one exact score row for overflowed users
    L.total = o;
    return L;
}

static size_t smem_bytes_for(int kp)
{
    return (size_t)TM * kp * 2 + (size_t)num_stages(kp) * SN * kp * 2 + SMEM_FIXED;
}

template <bool DUMP, bool DBG = false>
static int launch_rank_tc_t(const RankTcParams& p, cudaStream_t st)
{
    auto kern = rank_tc_kernel<DUMP, DBG>;
    const size_t smem = smem_bytes_for(p.kp);
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = p.n_ut < sm_count() ? p.n_ut : sm_count();
    ::b200::count_launch();
    kern<<<grid, THREADS, smem, st>>>(p);
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

template <bool DUMP>
static int launch_rank_tc(const RankTcParams& p, cudaStream_t st)
{
    if (!DUMP && p.debug != 0) return launch_rank_tc_t<false, true>(p, st);     // timing experiments: the instantiation that carries the switches
    return launch_rank_tc_t<DUMP>(p, st);
}

}  // namespace tc

using namespace tc;

int rank_tc_supported(int64_t n_q, int64_t n_items, int k, int topk)
{
    if (const char* e = getenv("B200_RANK_TC")) {
        if (e[0] == '0') return 0;
    }
    if (k < 8 || (k + 15) / 16 * 16 + KX > MAX_KP) return 0;
    if (topk < 1 || topk > MAX_TOPK) return 0;
    if (n_items < 4 * TN || n_items >= (1ll << 31) - TN) return 0;     // tiny catalogues: the exact path is fine
    if (n_q < 1) return 0;
    return 1;
}

int64_t rank_tc_workspace_bytes(int64_t n_q, int64_t n_items, int k, int topk)
{
    (void)topk;
    return (int64_t)make_layout(n_q, n_items, k).total;
}

// The packed item side (fp16 tile images of V with the base slice + the scalars of the scaling): laid out exactly like the
// head of the workspace (off_vpack = 0, then off_scal), so b200_rank_pack_items can build it once into a caller-owned
// buffer and every later call on the same (V, item_base) skips the norm + pack kernels (b200_rank_topk_packed).
int64_t rank_tc_items_bytes(int64_t n_items, int k)
{
    const Layout L = make_layout(1, n_items, k);
    return (int64_t)(L.off_scal + 1024);
}

static int pack_items(const float* V, int64_t n_items, int k, const float* item_base, const Layout& L, uint8_t* ws,
                      cudaStream_t st)
{
    const int64_t n_pad = L.n_it * TN;
    B200_CUDA(cudaMemsetAsync(ws + L.off_scal, 0, 64, st));
    const int grid = sm_count() * 8;
    unsigned int* scal = reinterpret_cast<unsigned int*>(ws + L.off_scal);
    norm_kernel<<<grid, 256, 0, st>>>(V, nullptr, n_items, k, nullptr, nullptr, scal + SC_VNORM, scal + SC_VABS, item_base, scal + SC_BMAX); ::b200::count_launch();
    scale_items_kernel<<<1, 1, 0, st>>>(scal); ::b200::count_launch();
    pack_kernel<TN, true><<<grid, 256, 0, st>>>(V, nullptr, n_items, n_pad, k, L.kp, item_base, scal, nullptr, ws + L.off_vpack); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

// per chunk of users: norms + element maximum, the chunk's scales, fp16 tile images
static int pack_users(const float* Usrc, const int64_t* uidx, int64_t rows, int64_t n_ut, int k, const Layout& L, uint8_t* ws,
                      const uint8_t* items, cudaStream_t st)
{
    const int grid = sm_count() * 8;
    const unsigned int* scal = reinterpret_cast<const unsigned int*>(items + L.off_scal);
    float* uabs = reinterpret_cast<float*>(ws + L.off_uabs);
    norm_kernel<<<grid, 256, 0, st>>>(Usrc, uidx, rows, k, reinterpret_cast<float*>(ws + L.off_unorm), uabs, nullptr, nullptr,
                                      nullptr, nullptr); ::b200::count_launch();
    pack_kernel<TM, false><<<grid, 256, 0, st>>>(Usrc, uidx, rows, n_ut * TM, k, L.kp, nullptr, scal, uabs, ws + L.off_upack); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

int rank_tc_pack_items(const float* V, int64_t n_items, int k, const float* item_base, void* packed, int64_t packed_bytes,
                       cudaStream_t st)
{
    const Layout L = make_layout(1, n_items, k);
    B200_REQUIRE(packed && packed_bytes >= rank_tc_items_bytes(n_items, k), "b200_rank_pack_items: buffer too small (%lld < %lld bytes)",
                 (long long)packed_bytes, (long long)rank_tc_items_bytes(n_items, k));
    B200_REQUIRE((((uintptr_t)packed) & 127) == 0, "b200_rank_pack_items: buffer must be 128-byte aligned");
    return pack_items(V, n_items, k, item_base, L, static_cast<uint8_t*>(packed), st);
}

int rank_tc(const float* U, const int64_t* user_idx, int64_t n_q, const float* V, int64_t n_items, int k,
            const float* item_base, const float* user_off, const int64_t* excl_indptr, const int32_t* excl_indices,
            int topk, int32_t* out_ids, float* out_scores, void* workspace, int64_t workspace_bytes, const void* packed_items,
            cudaStream_t st)
{
    const Layout L = make_layout(n_q, n_items, k);
    B200_REQUIRE((int64_t)L.total <= workspace_bytes, "rank_tc: workspace too small");
    B200_REQUIRE((((uintptr_t)workspace) & 127) == 0, "rank_tc: workspace must be 128-byte aligned");
    B200_REQUIRE((((uintptr_t)packed_items) & 127) == 0, "rank_tc: packed items must be 128-byte aligned");
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    // the packed item side: the caller's (built once by b200_rank_pack_items) or this call's own, in the workspace
    const uint8_t* items = packed_items ? static_cast<const uint8_t*>(packed_items) : ws;
    int rc = packed_items ? B200_OK : pack_items(V, n_items, k, item_base, L, ws, st);
    if (rc) return rc;
    for (int64_t q0 = 0; q0 < n_q; q0 += L.chunk_rows) {
        const int64_t rows = (n_q - q0 < L.chunk_rows) ? n_q - q0 : L.chunk_rows;
        const int64_t n_ut = (rows + TM - 1) / TM;
        const int64_t* uidx = user_idx ? user_idx + q0 : nullptr;
        const float* Usrc = user_idx ? U : U + (size_t)q0 * k;
        rc = pack_users(Usrc, uidx, rows, n_ut, k, L, ws, items, st);
        if (rc) return rc;
        B200_CUDA(cudaMemsetAsync(ws + L.off_over, 0, 4, st));
        RankTcParams p;
        p.Upack = ws + L.off_upack; p.Vpack = items + L.off_vpack;
        p.unorm = reinterpret_cast<const float*>(ws + L.off_unorm);
        p.uabs = reinterpret_cast<const float*>(ws + L.off_uabs);
        p.scal = reinterpret_cast<const unsigned int*>(items + L.off_scal);
        p.excl_indptr = excl_indptr ? excl_indptr + q0 : nullptr;
        p.excl_indices = excl_indices;
        p.n_rows = rows; p.n_ut = (int)n_ut; p.n_it = (int)L.n_it; p.kp = L.kp; p.topk = topk;
        p.lists = reinterpret_cast<unsigned long long*>(ws + L.off_lists);
        p.row_cnt = reinterpret_cast<int*>(ws + L.off_cnt);
        p.row_flag = reinterpret_cast<int*>(ws + L.off_flag);
        p.row_tau = reinterpret_cast<float*>(ws + L.off_tau);
        p.dump = nullptr;
        { const char* d = getenv("B200_RANK_DEBUG"); p.debug = d ? atoi(d) : 0; }
        rc = launch_rank_tc<false>(p, st);
        if (rc) return rc;
        FinishParams f;
        f.U = U; f.user_idx = uidx; f.q0 = q0; f.V = V; f.item_base = item_base; f.user_off = user_off;
        f.n_rows = rows; f.k = k; f.topk = topk;
        f.lists = p.lists; f.row_cnt = p.row_cnt; f.row_flag = p.row_flag; f.row_tau = p.row_tau;
        f.excl_indptr = p.excl_indptr; f.excl_indices = p.excl_indices;
        f.out_ids = out_ids + (size_t)q0 * topk; f.out_scores = out_scores + (size_t)q0 * topk;
        f.overflow_rows = reinterpret_cast<int*>(ws + L.off_over);
        f.strips = ST; f.cap = CAP;
        f.big_rows = reinterpret_cast<int*>(ws + L.off_big);
        f.row_list = nullptr;
        const bool staged = (k % 4 == 0) && k <= 128 && ((reinterpret_cast<uintptr_t>(V) & 15) == 0);
        const char* fmode = getenv("B200_RANK_FINISH");        // dev knob: "block" = block-per-row kernel for every row
        if (staged && !(fmode && fmode[0] == 'b')) {
            // warp per row; the few rows with more than FW_KEYS candidates are redone by the block kernel
            B200_CUDA(cudaMemsetAsync(f.big_rows, 0, 4, st));
            const size_t wsmem = finish_warp_smem(k);
            B200_CUDA(cudaFuncSetAttribute(rank_tc_finish_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem));
            int occ = 1;
            B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rank_tc_finish_warp_kernel, 32, wsmem));
            if (occ < 1) occ = 1;
            const int64_t cap = (int64_t)sm_count() * occ;
            rank_tc_finish_warp_kernel<<<(int)(rows < cap ? rows : cap), 32, wsmem, st>>>(f); ::b200::count_launch();
            B200_CUDA(cudaGetLastError());
            f.row_list = f.big_rows;
            const size_t fsmem = (size_t)128 * (k * 4 + 16);
            B200_CUDA(cudaFuncSetAttribute(rank_tc_finish_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
            rank_tc_finish_kernel<true><<<sm_count(), 128, fsmem, st>>>(f); ::b200::count_launch();
        } else if (staged) {
            const size_t fsmem = (size_t)128 * (k * 4 + 16);
            B200_CUDA(cudaFuncSetAttribute(rank_tc_finish_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
            int occ = 1;
            B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rank_tc_finish_kernel<true>, 128, fsmem));
            if (occ < 1) occ = 1;
            const int64_t cap = (int64_t)sm_count() * occ;
            rank_tc_finish_kernel<true><<<(int)(rows < cap ? rows : cap), 128, fsmem, st>>>(f); ::b200::count_launch();
        } else {
            // latency-bound gathers: as many rows in flight per SM as the thread limit allows (16 x 128 threads)
            const int fgrid = (int)(rows < (int64_t)sm_count() * 16 ? rows : (int64_t)sm_count() * 16);
            rank_tc_finish_kernel<false><<<fgrid, 128, 0, st>>>(f); ::b200::count_launch();
        }
        B200_CUDA(cudaGetLastError());
        // rows whose candidate list overflowed: exact path, one row at a time (rare; needs the count on the host)
        int n_over = 0;
        B200_CUDA(cudaMemcpyAsync(&n_over, ws + L.off_over, 4, cudaMemcpyDeviceToHost, st));
        B200_CUDA(cudaStreamSynchronize(st));
        // Many overflowed rows = a degenerate score distribution (a diverged model: inf / NaN factors; thousands of exact ties):
        // row-by-row repair would cost a host round trip per user.  Redo the whole chunk on the exact path instead, in slabs
        // of score rows cut from the (now idle) candidate-list area -- same ids and scores, bounded time.
        const int64_t list_bytes = (int64_t)L.chunk_ut * EPI_WARPS * CAP * 32 * 8;
        const int64_t slab_rows = list_bytes / (n_items * (int64_t)sizeof(float));
        if (n_over > 256 && slab_rows >= 8) {
            float* slab = reinterpret_cast<float*>(ws + L.off_lists);
            for (int64_t r0 = 0; r0 < rows; r0 += slab_rows) {
                const int64_t nq = rows - r0 < slab_rows ? rows - r0 : slab_rows;
                const int64_t g0 = q0 + r0;
                const float* Uq = user_idx ? U : U + (size_t)g0 * k;
                rc = b200_score_batch(Uq, user_idx ? user_idx + g0 : nullptr, nq, V, n_items, k, item_base,
                                      user_off ? user_off + g0 : nullptr, slab, st);
                if (!rc) rc = b200_topk_rows(slab, nq, n_items, excl_indptr ? excl_indptr + g0 : nullptr, excl_indices, topk,
                                             out_ids + (size_t)g0 * topk, out_scores + (size_t)g0 * topk, st);
                if (rc) return rc;
            }
            B200_CUDA(cudaStreamSynchronize(st));
        } else if (n_over > 0) {
            int* rows_h = new int[n_over];
            cudaError_t e = cudaMemcpy(rows_h, ws + L.off_over + 4, (size_t)n_over * 4, cudaMemcpyDeviceToHost);
            if (e != cudaSuccess) { delete[] rows_h; return cuda_fail(e, "cudaMemcpy overflow rows", __FILE__, __LINE__); }
            float* slab = reinterpret_cast<float*>(ws + L.off_slab);
            for (int x = 0; x < n_over; ++x) {
                const int64_t gq = rows_h[x];
                const float* Uq = user_idx ? U : U + (size_t)gq * k;
                rc = b200_score_batch(Uq, user_idx ? user_idx + gq : nullptr, 1, V, n_items, k, item_base,
                                      user_off ? user_off + gq : nullptr, slab, st);
                if (!rc) rc = b200_topk_rows(slab, 1, n_items, excl_indptr ? excl_indptr + gq : nullptr, excl_indices, topk,
                                             out_ids + (size_t)gq * topk, out_scores + (size_t)gq * topk, st);
                if (rc) { delete[] rows_h; return rc; }
            }
            delete[] rows_h;
            B200_CUDA(cudaStreamSynchronize(st));
        }
    }
    return B200_OK;
}

}  // namespace b200

using namespace b200;
using namespace b200::tc;

// Debug / validation entry: dense APPROXIMATE scores of the tensor-core pass (scaled fp16 operands, f32
// accumulation, + item base, unscaled again), out[n_q_pad128, n_items_pad256] row-major.  Not part of the rank path.
extern "C" int b200_rank_tc_debug_scores(const float* U, int64_t n_q, const float* V, int64_t n_items, int k,
                                         const float* item_base, float* out, int64_t out_elems,
                                         void* workspace, int64_t workspace_bytes, void* stream)
{
    B200_REQUIRE(U && V && out && workspace, "b200_rank_tc_debug_scores: null pointer argument");
    B200_REQUIRE(k >= 8 && (k + 15) / 16 * 16 + KX <= MAX_KP, "b200_rank_tc_debug_scores: k=%d unsupported", k);
    const Layout L = make_layout(n_q, n_items, k);
    B200_REQUIRE(n_q <= L.chunk_rows, "b200_rank_tc_debug_scores: n_q too large for one chunk");
    B200_REQUIRE((int64_t)L.total <= workspace_bytes, "b200_rank_tc_debug_scores: workspace too small (%lld needed)", (long long)L.total);
    const int64_t n_ut = (n_q + TM - 1) / TM;
    B200_REQUIRE(out_elems >= n_ut * TM * L.n_it * TN, "b200_rank_tc_debug_scores: out too small");
    cudaStream_t st = (cudaStream_t)stream;
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    int rc = pack_items(V, n_items, k, item_base, L, ws, st);
    if (rc) return rc;
    rc = pack_users(U, nullptr, n_q, n_ut, k, L, ws, ws, st);
    if (rc) return rc;
    RankTcParams p;
    p.Upack = ws + L.off_upack; p.Vpack = ws + L.off_vpack;
    p.unorm = reinterpret_cast<const float*>(ws + L.off_unorm);
    p.uabs = reinterpret_cast<const float*>(ws + L.off_uabs);
    p.scal = reinterpret_cast<const unsigned int*>(ws + L.off_scal);
    p.excl_indptr = nullptr; p.excl_indices = nullptr;
    p.n_rows = n_q; p.n_ut = (int)n_ut; p.n_it = (int)L.n_it; p.kp = L.kp; p.topk = 1;
    p.lists = reinterpret_cast<unsigned long long*>(ws + L.off_lists);
    p.row_cnt = reinterpret_cast<int*>(ws + L.off_cnt);
    p.row_flag = reinterpret_cast<int*>(ws + L.off_flag);
    p.row_tau = reinterpret_cast<float*>(ws + L.off_tau);
    p.dump = out;
    p.debug = 0;
    return launch_rank_tc<true>(p, st);
}
