// BPR SGD epochs for sm_90a.
//
// Replaces BPR._fit_sgd (reference: cornac/models/bpr/recom_bpr.pyx:208-269) with
//   * bpr_hogwild_kernel : throughput mode.  Persistent grid; every G-lane group draws its
//     own (u, i+, j-) triplets from the CSR matrix with a counter-based RNG, gathers the
//     three factor rows with 128-bit L2-only loads, reduces the pairwise dot with warp
//     shuffles and scatters the update back (plain 128-bit stores = the reference's
//     lock-free Hogwild, or red.global.add.v4.f32 when B200_SGD_ATOMIC is set).
//   * bpr_replay_kernel  : parity mode.  One warp applies an explicit sample stream with
//     the same result as the sequential seeded reference (num_threads = 1,
//     recom_bpr.pyx:132-133): sample metadata (u, i, j, skip test) is resolved 32 samples
//     at a time in parallel (read-only data), the updates are applied strictly in order.
//
// HBM-bound integer/gather work: no tensor cores here by design (DESIGN.md, K1).
#include <stdlib.h>

#include "sgd_common.cuh"

namespace b200 {

// Interaction store of the throughput kernel (built once per fit by b200_bpr_prepare):
//   pairs  int2[nnz]   (u, i) of every interaction: ONE 8-byte gather yields the user and the
//                      positive item of a sampled interaction (instead of coo_row[] + indices[]);
//   table  u64[slots]  open-addressing set of the keys (u << 32 | i), 4-slot (32-byte) buckets at
//                      load <= 0.5: has_non_zero(u, j) is ONE 32-byte gather that can be issued
//                      together with the factor rows, instead of a ~log2(deg)-deep dependent
//                      binary search.  Costs 8 + ~21 bytes of HBM per interaction -- 3.6 GB for
//                      125 M interactions on an 80 GB part, and it removes ~7 serialized memory round trips per sample.
constexpr unsigned long long TABLE_EMPTY = ~0ull;

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x)
{
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
    x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
    x ^= x >> 33;
    return x;
}

struct BprParams {
    const int2* __restrict__ pairs;
    const unsigned long long* __restrict__ table;   // 4 slots (32 B) per bucket
    uint64_t bucket_mask;
    int64_t nnz;
    int64_t n_neg;
    int64_t n_samples;
    int64_t max_groups;          // cap on concurrently running samples (Hogwild staleness bound)
    int exact_exp;               // B200_SGD_EXACT_EXP
    int debug_skip;              // profiling only (B200_BPR_DEBUG_SKIP): bit0 U, bit1 V+, bit2 V- scatter off
    int hinge;                   // MMMF (recom_mmmf.pyx:129-154): skip correctly ranked pairs, z = 1 otherwise
    int neg_weighted;            // WBPR: negatives drawn from the interaction list (popularity-weighted)
    SampleLaw law;               // unblocked or cache-blocked sample order (common.cuh)
    float* U;
    float* V;
    float* B;
    int k;
    float lr, reg;
    int use_bias;
    uint32_t seed_lo, seed_hi;
    uint32_t epoch_lo, epoch_hi;
    uint64_t sample_base;
    unsigned long long* stats;   // {correct, skipped}
};

// z = 1 / (1 + exp(score))   (recom_bpr.pyx:252); `exact` is warp-uniform
__device__ __forceinline__ float bpr_z(float score, int exact)
{
    if (exact) return (float)(1.0 / (1.0 + exp((double)score)));
    return __frcp_rn(1.f + __expf(score));
}

// resident blocks per SM the register allocator is asked to make room for: the kernel is
// latency-bound on dependent gathers, so samples in flight per SM (= groups x S) is the lever
template <int NPL, bool VEC, int S>
constexpr int hogwild_min_blocks()
{
    constexpr int E = NPL * (VEC ? 4 : 1);
    return (E * S <= 4) ? 5 : (E * S <= 8) ? 4 : (E * S <= 16) ? 2 : 1;
}

template <int G, int NPL, bool VEC, bool ATOMIC, int S, int MINB>
__global__ void __launch_bounds__(256, MINB) bpr_hogwild_kernel(const BprParams p)
{
    using Frag = RowFrag<NPL, VEC>;
    constexpr int E = NPL * Frag::W;
    const int lg = threadIdx.x & (G - 1);
    const int n_units = VEC ? p.k / 4 : p.k;
    const int64_t groups_per_block = blockDim.x / G;
    const int64_t n_groups = (int64_t)gridDim.x * groups_per_block;
    const int64_t gid = (int64_t)blockIdx.x * groups_per_block + threadIdx.x / G;
    const size_t k = (size_t)p.k;

    unsigned int n_correct = 0, n_skipped = 0;

    for (int64_t s0 = gid * S; s0 < p.n_samples; s0 += n_groups * S) {
        int32_t u[S], it[S], jt[S];
        bool live[S];
        Frag fu[S], fi[S], fj[S];
        float bi[S], bj[S];
        // ---- phase A: draw the triplets (every lane of the group computes the same values);
        //      the negative row does not depend on the interaction gather, so it goes out first
        int2 pr[S];
#pragma unroll
        for (int t = 0; t < S; ++t) {
            const uint64_t s = p.sample_base + (uint64_t)(s0 + t);
            live[t] = (s0 + t) < p.n_samples;
            Philox4 r = philox4x32_10((uint32_t)s, (uint32_t)(s >> 32), p.epoch_lo, p.epoch_hi, p.seed_lo, p.seed_hi);
            int64_t i_lo, i_len, j_lo, j_len;
            law_ranges(p.law, s, i_lo, i_len, j_lo, j_len);
            const int64_t ii = i_lo + (int64_t)range64(r.x, r.y, (uint64_t)i_len);
            jt[t] = p.neg_weighted ? __ldg(p.pairs + range64(r.z, r.w, (uint64_t)p.nnz)).y
                                   : (int32_t)(j_lo + (int64_t)range64(r.z, r.w, (uint64_t)j_len));
            pr[t] = __ldg(p.pairs + ii);
            row_load<G, NPL, VEC>(fj[t], p.V + (size_t)jt[t] * k, lg, n_units);
            bj[t] = __ldcg(p.B + jt[t]);
        }
        // ---- phase B: user row, positive row and the membership bucket, all in flight together.
        //      The 32-byte bucket is read by the first four lanes of the group, 8 bytes each.
        unsigned long long slot[S];
        uint64_t bkt[S];
#pragma unroll
        for (int t = 0; t < S; ++t) {
            u[t] = pr[t].x;
            it[t] = pr[t].y;
            const uint64_t key = ((uint64_t)(uint32_t)u[t] << 32) | (uint32_t)jt[t];
            bkt[t] = mix64(key) & p.bucket_mask;
            slot[t] = (lg < 4) ? __ldg(p.table + 4 * bkt[t] + lg) : 0ull;
            row_load<G, NPL, VEC>(fu[t], p.U + (size_t)u[t] * k, lg, n_units);
            row_load<G, NPL, VEC>(fi[t], p.V + (size_t)it[t] * k, lg, n_units);
            bi[t] = __ldcg(p.B + it[t]);
        }
        // ---- phase C: has_non_zero(u, j)  (recom_bpr.pyx:241-243) = key (u, j) in the table
        const unsigned gmask = group_mask<G>();
#pragma unroll
        for (int t = 0; t < S; ++t) {
            const uint64_t key = ((uint64_t)(uint32_t)u[t] << 32) | (uint32_t)jt[t];
            unsigned hit = __ballot_sync(gmask, lg < 4 && slot[t] == key) & gmask;
            unsigned full = __ballot_sync(gmask, lg == 3 && slot[t] != TABLE_EMPTY) & gmask;
            uint64_t bb = bkt[t];
            while (!hit && full) {            // rare: the bucket overflowed into the next one
                bb = (bb + 1) & p.bucket_mask;
                const unsigned long long sl = (lg < 4) ? __ldg(p.table + 4 * bb + lg) : 0ull;
                hit = __ballot_sync(gmask, lg < 4 && sl == key) & gmask;
                full = __ballot_sync(gmask, lg == 3 && sl != TABLE_EMPTY) & gmask;
            }
            if (live[t] && hit) {
                live[t] = false;
                ++n_skipped;
            }
        }
        // ---- phase D: score, z, update (recom_bpr.pyx:249-267)
#pragma unroll
        for (int t = 0; t < S; ++t) {
            float part = 0.f;
#pragma unroll
            for (int e = 0; e < E; ++e) part = fmaf(fu[t].v[e], fi[t].v[e] - fj[t].v[e], part);
            const float score = (bi[t] - bj[t]) + group_sum<G>(part);
            if (!live[t]) continue;     // group-uniform
            float z;
            if (p.hinge) {
                if (score > 0.f) { ++n_correct; continue; }
                z = 1.f;
            } else {
                z = bpr_z(score, p.exact_exp);
                n_correct += (z < .5f);
            }
            const float lr = p.lr, reg = p.reg;
            float* pu = p.U + (size_t)u[t] * k;
            float* pi = p.V + (size_t)it[t] * k;
            float* pj = p.V + (size_t)jt[t] * k;
            if (ATOMIC) {
                Frag du, di, dj;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const float uf = fu[t].v[e], vi = fi[t].v[e], vj = fj[t].v[e];
                    du.v[e] = lr * (z * (vi - vj) - reg * uf);
                    di.v[e] = lr * (z * uf - reg * vi);
                    dj.v[e] = lr * (-z * uf - reg * vj);
                }
                row_red_add<G, NPL, VEC>(du, pu, lg, n_units);
                row_red_add<G, NPL, VEC>(di, pi, lg, n_units);
                row_red_add<G, NPL, VEC>(dj, pj, lg, n_units);
                if (p.use_bias && lg == 0) {
                    red_add_f32(p.B + it[t], lr * (z - reg * bi[t]));
                    red_add_f32(p.B + jt[t], lr * (-z - reg * bj[t]));
                }
            } else {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const float uf = fu[t].v[e], vi = fi[t].v[e], vj = fj[t].v[e];
                    fu[t].v[e] = uf + lr * (z * (vi - vj) - reg * uf);
                    fi[t].v[e] = vi + lr * (z * uf - reg * vi);
                    fj[t].v[e] = vj + lr * (-z * uf - reg * vj);
                }
                row_store<G, NPL, VEC>(fu[t], pu, lg, n_units);
                row_store<G, NPL, VEC>(fi[t], pi, lg, n_units);
                row_store<G, NPL, VEC>(fj[t], pj, lg, n_units);
                if (p.use_bias && lg == 0) {
                    __stcg(p.B + it[t], bi[t] + lr * (z - reg * bi[t]));
                    __stcg(p.B + jt[t], bj[t] + lr * (-z - reg * bj[t]));
                }
            }
        }
    }

    // ---- epoch statistics: one count per group (its lane 0), block-reduced, two atomics per block
    __shared__ unsigned int sh_stats[2];
    if (threadIdx.x < 2) sh_stats[threadIdx.x] = 0;
    __syncthreads();
    unsigned int c = (lg == 0) ? n_correct : 0u, sk = (lg == 0) ? n_skipped : 0u;
    c = __reduce_add_sync(0xffffffffu, c);
    sk = __reduce_add_sync(0xffffffffu, sk);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&sh_stats[0], c);
        atomicAdd(&sh_stats[1], sk);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(p.stats + 0, (unsigned long long)sh_stats[0]);
        atomicAdd(p.stats + 1, (unsigned long long)sh_stats[1]);
    }
}

// ---------------------------------------------------------------------------------------
// Chunked variant (the default): the per-sample bookkeeping that every lane of a group used
// to compute redundantly (Philox, range reduction, pair gather, key hash, bucket probe) is done
// ONCE PER LANE FOR G DIFFERENT SAMPLES -- lane l of a group resolves sample (chunk*G + l) --
// so a group has G independent metadata gathers in flight at once and pays 1/G of those
// instructions per sample.  The G resolved triplets are then broadcast one by one with warp
// shuffles and applied by the whole group (row gathers of sample t+1 are issued before the
// arithmetic of sample t).
template <int G, int NPL, bool VEC, bool ATOMIC, int MINB, int DEPTH>
__global__ void __launch_bounds__(256, MINB) bpr_hogwild_chunk_kernel(const BprParams p)
{
    using Frag = RowFrag<NPL, VEC>;
    constexpr int E = NPL * Frag::W;
    const int lane = threadIdx.x & 31;
    const int lg = lane & (G - 1);
    const int gbase = lane & ~(G - 1);
    const unsigned gmask = group_mask<G>();
    const int n_units = VEC ? p.k / 4 : p.k;
    const int64_t groups_per_block = blockDim.x / G;
    const int64_t n_groups = (int64_t)gridDim.x * groups_per_block;
    const int64_t gid = (int64_t)blockIdx.x * groups_per_block + threadIdx.x / G;
    const int64_t n_chunks = (p.n_samples + G - 1) / G;
    const size_t k = (size_t)p.k;
    const float lr = p.lr, reg = p.reg;

    unsigned int n_correct = 0, n_skipped = 0;

    for (int64_t c = gid; c < n_chunks; c += n_groups) {
        // ---- phase 1: this lane's own sample
        const int64_t sl = c * G + lg;
        int mlive = sl < p.n_samples;
        const uint64_t s = p.sample_base + (uint64_t)sl;
        const Philox4 r = philox4x32_10((uint32_t)s, (uint32_t)(s >> 32), p.epoch_lo, p.epoch_hi, p.seed_lo, p.seed_hi);
        int64_t i_lo, i_len, j_lo, j_len;
        law_ranges(p.law, s, i_lo, i_len, j_lo, j_len);
        const int64_t ii = i_lo + (int64_t)range64(r.x, r.y, (uint64_t)i_len);
        const int32_t mj = p.neg_weighted ? __ldg(p.pairs + range64(r.z, r.w, (uint64_t)p.nnz)).y     // recom_wbpr.pyx:131
                                          : (int32_t)(j_lo + (int64_t)range64(r.z, r.w, (uint64_t)j_len));
        const int2 pr = __ldg(p.pairs + ii);
        const int32_t mu = pr.x, mi = pr.y;
        {
            const uint64_t key = ((uint64_t)(uint32_t)mu << 32) | (uint32_t)mj;
            uint64_t bb = mix64(key) & p.bucket_mask;
            bool found, full;
            do {
                const ulonglong2 b0 = __ldg(reinterpret_cast<const ulonglong2*>(p.table + 4 * bb));
                const ulonglong2 b1 = __ldg(reinterpret_cast<const ulonglong2*>(p.table + 4 * bb) + 1);
                found = (b0.x == key) | (b0.y == key) | (b1.x == key) | (b1.y == key);
                full = (b1.y != TABLE_EMPTY);
                bb = (bb + 1) & p.bucket_mask;
            } while (!found && full);              // rare: the bucket overflowed into the next one
            if (mlive && found) { mlive = 0; ++n_skipped; }          // recom_bpr.pyx:241-243
        }
        // ---- phase 2: apply the G samples one after the other, DEPTH row-gathers ahead
        constexpr int NSLOT = DEPTH + 1;
        Frag fu[NSLOT], fi[NSLOT], fj[NSLOT];
        float bi[NSLOT], bj[NSLOT];
        int32_t cu[NSLOT], ci[NSLOT], cj[NSLOT];
        int cl[NSLOT];
        auto fetch = [&](int t, int slot) {
            cu[slot] = __shfl_sync(gmask, mu, gbase + t);
            ci[slot] = __shfl_sync(gmask, mi, gbase + t);
            cj[slot] = __shfl_sync(gmask, mj, gbase + t);
            cl[slot] = __shfl_sync(gmask, mlive, gbase + t);
            if (cl[slot]) {
                row_load<G, NPL, VEC>(fu[slot], p.U + (size_t)cu[slot] * k, lg, n_units);
                row_load<G, NPL, VEC>(fi[slot], p.V + (size_t)ci[slot] * k, lg, n_units);
                row_load<G, NPL, VEC>(fj[slot], p.V + (size_t)cj[slot] * k, lg, n_units);
                bi[slot] = __ldcg(p.B + ci[slot]);
                bj[slot] = __ldcg(p.B + cj[slot]);
            }
        };
#pragma unroll
        for (int t = 0; t < DEPTH; ++t)
            if (t < G) fetch(t, t % NSLOT);
#pragma unroll
        for (int t = 0; t < G; ++t) {
            const int cur = t % NSLOT;
            if (t + DEPTH < G) fetch(t + DEPTH, (t + DEPTH) % NSLOT);
            if (!cl[cur]) continue;                 // group-uniform
            float part = 0.f;
#pragma unroll
            for (int e = 0; e < E; ++e) part = fmaf(fu[cur].v[e], fi[cur].v[e] - fj[cur].v[e], part);
            const float score = (bi[cur] - bj[cur]) + group_sum<G>(part);      // recom_bpr.pyx:249-251
            float z;
            if (p.hinge) {                              // recom_mmmf.pyx:137-139
                if (score > 0.f) { ++n_correct; continue; }
                z = 1.f;
            } else {
                z = bpr_z(score, p.exact_exp);
                n_correct += (z < .5f);
            }
            float* pu = p.U + (size_t)cu[cur] * k;
            float* pi = p.V + (size_t)ci[cur] * k;
            float* pj = p.V + (size_t)cj[cur] * k;
            if (ATOMIC) {
                Frag du, di, dj;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const float uf = fu[cur].v[e], vi = fi[cur].v[e], vj = fj[cur].v[e];
                    du.v[e] = lr * (z * (vi - vj) - reg * uf);
                    di.v[e] = lr * (z * uf - reg * vi);
                    dj.v[e] = lr * (-z * uf - reg * vj);
                }
                if (!(p.debug_skip & 1)) row_red_add<G, NPL, VEC>(du, pu, lg, n_units);
                if (!(p.debug_skip & 2)) row_red_add<G, NPL, VEC>(di, pi, lg, n_units);
                if (!(p.debug_skip & 4)) row_red_add<G, NPL, VEC>(dj, pj, lg, n_units);
                if (p.use_bias && lg == 0) {
                    red_add_f32(p.B + ci[cur], lr * (z - reg * bi[cur]));
                    red_add_f32(p.B + cj[cur], lr * (-z - reg * bj[cur]));
                }
            } else {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const float uf = fu[cur].v[e], vi = fi[cur].v[e], vj = fj[cur].v[e];
                    fu[cur].v[e] = uf + lr * (z * (vi - vj) - reg * uf);
                    fi[cur].v[e] = vi + lr * (z * uf - reg * vi);
                    fj[cur].v[e] = vj + lr * (-z * uf - reg * vj);
                }
                row_store<G, NPL, VEC>(fu[cur], pu, lg, n_units);
                row_store<G, NPL, VEC>(fi[cur], pi, lg, n_units);
                row_store<G, NPL, VEC>(fj[cur], pj, lg, n_units);
                if (p.use_bias && lg == 0) {
                    __stcg(p.B + ci[cur], bi[cur] + lr * (z - reg * bi[cur]));
                    __stcg(p.B + cj[cur], bj[cur] + lr * (-z - reg * bj[cur]));
                }
            }
        }
    }

    __shared__ unsigned int sh_stats[2];
    if (threadIdx.x < 2) sh_stats[threadIdx.x] = 0;
    __syncthreads();
    unsigned int cc = (lg == 0) ? n_correct : 0u, sk = n_skipped;     // skips were counted per lane
    cc = __reduce_add_sync(0xffffffffu, cc);
    sk = __reduce_add_sync(0xffffffffu, sk);
    if (lane == 0) {
        atomicAdd(&sh_stats[0], cc);
        atomicAdd(&sh_stats[1], sk);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(p.stats + 0, (unsigned long long)sh_stats[0]);
        atomicAdd(p.stats + 1, (unsigned long long)sh_stats[1]);
    }
}

// ---------------------------------------------------------------------------------------
// Streamed variant (the default for k % 4 == 0, k <= 128): the chunked kernel above keeps the rows of the samples in
// flight in REGISTERS (one sample ahead: 24 registers), is fully unrolled over the G samples of a chunk (190 KB of code:
// 17 % of its stall samples were instruction-cache misses, ncu r02) and exposes the two dependent DRAM gathers of the
// sampling (pair -> bucket) once per chunk.  Here
//   * the factor rows of the next D samples are staged in SHARED MEMORY with cp.async (LDGSTS.BYPASS, L2-coherent like
//     the ld.global.cg they replace): every lane copies and later reads back only its own 16-byte column, so no barrier
//     is needed, no register is held by a row in flight, and D = 4 samples (6 KB per warp at k = 128) are in flight
//     per group instead of 2;
//   * the sampling of the NEXT chunk (Philox, pair gather, membership bucket) is issued while the current chunk's
//     samples are applied, one step per quarter of the chunk, so its latency is off the critical path;
//   * the loop over the chunk is a real loop (unrolled by 2), the per-sample integer work is cut down (triplet packed
//     in three shuffles, deltas as (lr z) x - (lr reg) y): ~100 warp instructions per sample instead of ~200.
__device__ __forceinline__ void cp_async_16(uint32_t dst_smem, const void* src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst_smem), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }
__device__ __forceinline__ float4 lds_f4(uint32_t addr)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}

// sampling of one chunk, in three steps so that it can be spread over the previous chunk's sample loop
struct ChunkMeta {
    int32_t u, i, j;        // this lane's sample of the chunk (u < 0: not live -- out of range or skipped)
    uint64_t key, bucket;
    ulonglong2 b0, b1;      // the membership bucket in flight
    int2 pr;                // the pair in flight
    int in_range;
};

template <int G>
__device__ __forceinline__ void meta_step_a(const BprParams& p, ChunkMeta& m, int64_t chunk, int lg)
{
    const int64_t sl = chunk * G + lg;
    m.in_range = sl < p.n_samples;
    const uint64_t s = p.sample_base + (uint64_t)sl;
    const Philox4 r = philox4x32_10((uint32_t)s, (uint32_t)(s >> 32), p.epoch_lo, p.epoch_hi, p.seed_lo, p.seed_hi);
    int64_t i_lo, i_len, j_lo, j_len;
    law_ranges(p.law, s, i_lo, i_len, j_lo, j_len);
    const int64_t ii = i_lo + (int64_t)range64(r.x, r.y, (uint64_t)i_len);
    m.j = p.neg_weighted ? __ldg(p.pairs + range64(r.z, r.w, (uint64_t)p.nnz)).y     // recom_wbpr.pyx:131
                         : (int32_t)(j_lo + (int64_t)range64(r.z, r.w, (uint64_t)j_len));
    m.pr = __ldg(p.pairs + ii);
}
__device__ __forceinline__ void meta_step_b(const BprParams& p, ChunkMeta& m)
{
    m.u = m.pr.x; m.i = m.pr.y;
    m.key = ((uint64_t)(uint32_t)m.u << 32) | (uint32_t)m.j;
    m.bucket = mix64(m.key) & p.bucket_mask;
    m.b0 = __ldg(reinterpret_cast<const ulonglong2*>(p.table + 4 * m.bucket));
    m.b1 = __ldg(reinterpret_cast<const ulonglong2*>(p.table + 4 * m.bucket) + 1);
}
// returns 1 when the sample was skipped (has_non_zero(u, j), recom_bpr.pyx:241-243); marks dead samples with u = ~u
__device__ __forceinline__ int meta_step_c(const BprParams& p, ChunkMeta& m)
{
    bool found = (m.b0.x == m.key) | (m.b0.y == m.key) | (m.b1.x == m.key) | (m.b1.y == m.key);
    bool full = (m.b1.y != TABLE_EMPTY);
    uint64_t bb = m.bucket;
    while (!found && full) {                    // rare: the bucket overflowed into the next one
        bb = (bb + 1) & p.bucket_mask;
        const ulonglong2 c0 = __ldg(reinterpret_cast<const ulonglong2*>(p.table + 4 * bb));
        const ulonglong2 c1 = __ldg(reinterpret_cast<const ulonglong2*>(p.table + 4 * bb) + 1);
        found = (c0.x == m.key) | (c0.y == m.key) | (c1.x == m.key) | (c1.y == m.key);
        full = (c1.y != TABLE_EMPTY);
    }
    const int skipped = m.in_range && found;
    if (!m.in_range || found) m.u = ~m.u;      // u >= 0 always: the complement is negative = "not live"
    return skipped;
}

template <int G, bool ATOMIC, int D, int MINB>
__global__ void __launch_bounds__(256, MINB) bpr_hogwild_stream_kernel(const BprParams p)
{
    extern __shared__ __align__(16) unsigned char stream_smem[];
    constexpr int SLOT = 3 * G * 16;            // bytes of one sample's three rows (G lanes x 16 B each)
    const int lane = threadIdx.x & 31;
    const int lg = lane & (G - 1);
    const int gbase = lane & ~(G - 1);
    const unsigned gmask = group_mask<G>();
    const int n_units = p.k / 4;                // float4 units of a row (<= G)
    const bool col = lg < n_units;              // this lane owns a column of the rows
    const int64_t groups_per_block = blockDim.x / G;
    const int64_t n_groups = (int64_t)gridDim.x * groups_per_block;
    const int64_t gid = (int64_t)blockIdx.x * groups_per_block + threadIdx.x / G;
    const int64_t n_chunks = (p.n_samples + G - 1) / G;
    const size_t k = (size_t)p.k;
    const float lr = p.lr, lrreg = p.lr * p.reg;
    // this lane's 16-byte column of the group's D slots: slot s, row r (0 = U, 1 = V+, 2 = V-) at my_s + s*SLOT + r*G*16
    const uint32_t my_s = (uint32_t)__cvta_generic_to_shared(stream_smem) + (uint32_t)(threadIdx.x / G) * (D * SLOT) + lg * 16;

    unsigned int n_correct = 0, n_skipped = 0;
    ChunkMeta cur, nxt;
    cur.u = cur.i = cur.j = -1;
    int64_t c = gid;
    if (c < n_chunks) {
        meta_step_a<G>(p, cur, c, lg);
        meta_step_b(p, cur);
        n_skipped += meta_step_c(p, cur);
    }
    for (; c < n_chunks; c += n_groups) {
        const int64_t cn = c + n_groups;
        const bool has_next = cn < n_chunks;
        nxt = cur;
        float bslot = 0.f;                      // lane 2s / 2s+1 of the group: B[i] / B[j] of the sample in slot s
        // rows (and biases) of sample t of the chunk -> slot t % D; one commit group per sample, live or not
        auto issue = [&](int t) {
            const int32_t su = __shfl_sync(gmask, cur.u, gbase + t);
            const int32_t si = __shfl_sync(gmask, cur.i, gbase + t);
            const int32_t sj = __shfl_sync(gmask, cur.j, gbase + t);
            if (su >= 0) {
                const int s = t % D;
                if (col) {
                    const uint32_t dst = my_s + s * SLOT;
                    cp_async_16(dst, p.U + (size_t)su * k + lg * 4);
                    cp_async_16(dst + G * 16, p.V + (size_t)si * k + lg * 4);
                    cp_async_16(dst + 2 * G * 16, p.V + (size_t)sj * k + lg * 4);
                }
                if (lg == 2 * s) bslot = __ldcg(p.B + si);
                if (lg == 2 * s + 1) bslot = __ldcg(p.B + sj);
            }
            cp_async_commit();
        };
#pragma unroll
        for (int t = 0; t < D; ++t) issue(t);
#pragma unroll 2
        for (int t = 0; t < G; ++t) {
            // ---- the next chunk's sampling, one step per quarter of this chunk
            if (has_next) {
                if (t == 0) meta_step_a<G>(p, nxt, cn, lg);
                else if (t == G / 4) meta_step_b(p, nxt);
                else if (t == (3 * G) / 4) n_skipped += meta_step_c(p, nxt);
            }
            // ---- sample t: rows have landed in slot t % D
            cp_async_wait<D - 1>();
            const int s = t % D;
            const int32_t su = __shfl_sync(gmask, cur.u, gbase + t);
            const int32_t si = __shfl_sync(gmask, cur.i, gbase + t);
            const int32_t sj = __shfl_sync(gmask, cur.j, gbase + t);
            const float bi = __shfl_sync(gmask, bslot, gbase + 2 * s);
            const float bj = __shfl_sync(gmask, bslot, gbase + 2 * s + 1);
            float4 u4 = make_float4(0.f, 0.f, 0.f, 0.f), vi4 = u4, vj4 = u4;
            if (su >= 0 && col) {
                const uint32_t src = my_s + s * SLOT;
                u4 = lds_f4(src); vi4 = lds_f4(src + G * 16); vj4 = lds_f4(src + 2 * G * 16);
            }
            if (t + D < G) issue(t + D); else cp_async_commit();      // refill the slot just read (same lane, same bytes)
            if (su < 0) continue;                   // group-uniform: skipped / out of range
            const float dx = vi4.x - vj4.x, dy = vi4.y - vj4.y, dz = vi4.z - vj4.z, dw = vi4.w - vj4.w;
            float part = u4.x * dx;
            part = fmaf(u4.y, dy, part); part = fmaf(u4.z, dz, part); part = fmaf(u4.w, dw, part);
            const float score = (bi - bj) + group_sum<G>(part);       // recom_bpr.pyx:249-251
            float z;
            if (p.hinge) {                              // recom_mmmf.pyx:137-139
                if (score > 0.f) { ++n_correct; continue; }
                z = 1.f;
            } else {
                z = bpr_z(score, p.exact_exp);
                n_correct += (z < .5f);
            }
            const float a = lr * z;                     // delta = lr (z x - reg y) = a x - lrreg y
            float* pu = p.U + (size_t)su * k + lg * 4;
            float* pi = p.V + (size_t)si * k + lg * 4;
            float* pj = p.V + (size_t)sj * k + lg * 4;
            if (col) {
                if (ATOMIC) {
                    if (!(p.debug_skip & 1))
                        red_add_v4(pu, fmaf(a, dx, -lrreg * u4.x), fmaf(a, dy, -lrreg * u4.y), fmaf(a, dz, -lrreg * u4.z), fmaf(a, dw, -lrreg * u4.w));
                    if (!(p.debug_skip & 2))
                        red_add_v4(pi, fmaf(a, u4.x, -lrreg * vi4.x), fmaf(a, u4.y, -lrreg * vi4.y), fmaf(a, u4.z, -lrreg * vi4.z), fmaf(a, u4.w, -lrreg * vi4.w));
                    if (!(p.debug_skip & 4))
                        red_add_v4(pj, fmaf(-a, u4.x, -lrreg * vj4.x), fmaf(-a, u4.y, -lrreg * vj4.y), fmaf(-a, u4.z, -lrreg * vj4.z), fmaf(-a, u4.w, -lrreg * vj4.w));
                } else {
                    __stcg(reinterpret_cast<float4*>(pu), make_float4(u4.x + fmaf(a, dx, -lrreg * u4.x), u4.y + fmaf(a, dy, -lrreg * u4.y),
                                                                      u4.z + fmaf(a, dz, -lrreg * u4.z), u4.w + fmaf(a, dw, -lrreg * u4.w)));
                    __stcg(reinterpret_cast<float4*>(pi), make_float4(vi4.x + fmaf(a, u4.x, -lrreg * vi4.x), vi4.y + fmaf(a, u4.y, -lrreg * vi4.y),
                                                                      vi4.z + fmaf(a, u4.z, -lrreg * vi4.z), vi4.w + fmaf(a, u4.w, -lrreg * vi4.w)));
                    __stcg(reinterpret_cast<float4*>(pj), make_float4(vj4.x + fmaf(-a, u4.x, -lrreg * vj4.x), vj4.y + fmaf(-a, u4.y, -lrreg * vj4.y),
                                                                      vj4.z + fmaf(-a, u4.z, -lrreg * vj4.z), vj4.w + fmaf(-a, u4.w, -lrreg * vj4.w)));
                }
            }
            if (p.use_bias && lg == 0) {
                if (ATOMIC) {
                    red_add_f32(p.B + si, a - lrreg * bi);
                    red_add_f32(p.B + sj, -a - lrreg * bj);
                } else {
                    __stcg(p.B + si, bi + (a - lrreg * bi));
                    __stcg(p.B + sj, bj + (-a - lrreg * bj));
                }
            }
        }
        cur = nxt;
    }
    cp_async_wait<0>();

    __shared__ unsigned int sh_stats[2];
    if (threadIdx.x < 2) sh_stats[threadIdx.x] = 0;
    __syncthreads();
    unsigned int cc = (lg == 0) ? n_correct : 0u, sk = n_skipped;     // skips were counted per lane
    cc = __reduce_add_sync(0xffffffffu, cc);
    sk = __reduce_add_sync(0xffffffffu, sk);
    if (lane == 0) {
        atomicAdd(&sh_stats[0], cc);
        atomicAdd(&sh_stats[1], sk);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(p.stats + 0, (unsigned long long)sh_stats[0]);
        atomicAdd(p.stats + 1, (unsigned long long)sh_stats[1]);
    }
}

// ---------------------------------------------------------------------------------------
// Parity mode: one warp, serial-equivalent.  Unfused f32 arithmetic in the operation order
// of recom_bpr.pyx:249-267 (the dot is a lane-strided partial sum + shuffle tree).
struct ReplayParams {
    const int64_t* __restrict__ i_index;
    const int32_t* __restrict__ j_id;
    int64_t n_samples;
    const int32_t* __restrict__ indptr;
    const int32_t* __restrict__ indices;
    const int32_t* __restrict__ coo_row;
    float* U;
    float* V;
    float* B;
    int k;
    float lr, reg;
    int use_bias;
    int hinge;
    unsigned long long* stats;
};

__global__ void __launch_bounds__(32) bpr_replay_kernel(const ReplayParams p)
{
    const int lane = threadIdx.x;
    const size_t k = (size_t)p.k;
    unsigned long long n_correct = 0, n_skipped = 0;
    for (int64_t base = 0; base < p.n_samples; base += 32) {
        // metadata of 32 consecutive samples, one per lane (read-only inputs => order-free)
        const int64_t s = base + lane;
        int32_t mu = 0, mi = 0, mj = 0;
        bool mskip = true;
        if (s < p.n_samples) {
            const int64_t ii = p.i_index[s];
            mj = p.j_id[s];
            mu = __ldg(p.coo_row + ii);
            mi = __ldg(p.indices + ii);
            mskip = row_contains(p.indices, __ldg(p.indptr + mu), __ldg(p.indptr + mu + 1), mj);
        }
        const int n_here = (int)min((int64_t)32, p.n_samples - base);
        for (int t = 0; t < n_here; ++t) {
            const bool skip = __shfl_sync(0xffffffffu, (int)mskip, t) != 0;
            if (skip) { ++n_skipped; continue; }
            const int32_t u = __shfl_sync(0xffffffffu, mu, t);
            const int32_t i = __shfl_sync(0xffffffffu, mi, t);
            const int32_t j = __shfl_sync(0xffffffffu, mj, t);
            float* pu = p.U + (size_t)u * k;
            float* pi = p.V + (size_t)i * k;
            float* pj = p.V + (size_t)j * k;
            const float bi = __ldcg(p.B + i), bj = __ldcg(p.B + j);
            float part = 0.f;
            for (int f = lane; f < p.k; f += 32)
                part = __fadd_rn(part, __fmul_rn(__ldcg(pu + f), __fsub_rn(__ldcg(pi + f), __ldcg(pj + f))));
            const float score = __fadd_rn(__fsub_rn(bi, bj), group_sum<32>(part));
            float z;
            if (p.hinge) {                              // recom_mmmf.pyx:137-139 (warp-uniform)
                if (score > 0.f) { ++n_correct; continue; }
                z = 1.f;
            } else {
                z = (float)(1.0 / (1.0 + exp((double)score)));
                n_correct += (z < .5f);
            }
            const float lr = p.lr, reg = p.reg;
            for (int f = lane; f < p.k; f += 32) {
                const float uf = __ldcg(pu + f), vi = __ldcg(pi + f), vj = __ldcg(pj + f);
                __stcg(pu + f, __fadd_rn(uf, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, __fsub_rn(vi, vj)), __fmul_rn(reg, uf)))));
                __stcg(pi + f, __fadd_rn(vi, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, uf), __fmul_rn(reg, vi)))));
                __stcg(pj + f, __fadd_rn(vj, __fmul_rn(lr, __fsub_rn(__fmul_rn(-z, uf), __fmul_rn(reg, vj)))));
            }
            if (p.use_bias && lane == 0) {
                __stcg(p.B + i, __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(z, __fmul_rn(reg, bi)))));
                __stcg(p.B + j, __fadd_rn(bj, __fmul_rn(lr, __fsub_rn(-z, __fmul_rn(reg, bj)))));
            }
            __syncwarp();   // order lane 0's bias stores before the next sample's reads
        }
    }
    if (lane == 0) {
        atomicAdd(p.stats + 0, n_correct);
        atomicAdd(p.stats + 1, n_skipped);
    }
}

// ---------------------------------------------------------------------------------------
// b200_bpr_prepare: CSR -> (pairs, membership table).  One warp per user row (lanes stride over the row's
// interactions): the user id is the row index, no search; the cost is the random 8-byte CAS per interaction.
__global__ void bpr_prepare_kernel(const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                   int64_t n_users, int64_t nnz, int2* __restrict__ pairs,
                                   unsigned long long* __restrict__ table, uint64_t bucket_mask)
{
    const int lane = threadIdx.x & 31;
    const int64_t wstride = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < n_users; u += wstride) {
        const int64_t lo = __ldg(indptr + u), hi = __ldg(indptr + u + 1);
        for (int64_t e = lo + lane; e < hi; e += 32) {
            const int32_t i = __ldg(indices + e);
            pairs[e] = make_int2((int32_t)u, i);                    // COO row = user_ids of recom_bpr.pyx:154-161
            const unsigned long long key = ((unsigned long long)(uint32_t)u << 32) | (uint32_t)i;
            uint64_t b = mix64(key) & bucket_mask;
            for (;;) {
                bool done = false;
                for (int sl = 0; sl < 4 && !done; ++sl) {
                    const unsigned long long old = atomicCAS(table + 4 * b + sl, TABLE_EMPTY, key);
                    done = (old == TABLE_EMPTY) || (old == key);
                }
                if (done) break;
                b = (b + 1) & bucket_mask;
            }
        }
    }
    (void)nnz;
}

static int64_t table_buckets_for(int64_t nnz)
{
    int64_t b = 1;
    while (b * 2 < nnz) b <<= 1;     // 4 slots per bucket => load factor in (0.25, 0.5]
    return b;
}

struct HogwildTune {
    int S, threads, blocks_per_sm;
};
static HogwildTune read_tune()
{
    HogwildTune t{0, 256, 0};
    if (const char* e = getenv("B200_BPR_TUNE")) sscanf(e, "%d,%d,%d", &t.S, &t.threads, &t.blocks_per_sm);
    if (t.threads != 64 && t.threads != 128 && t.threads != 256) t.threads = 256;
    return t;
}

// ---------------------------------------------------------------------------------------
// Parity mode, windowed: one CTA of 32 warps.  32 consecutive samples are resolved at a time (one per
// warp) and executed in dependency order: a sample may run as soon as no EARLIER still-pending sample
// of the window touches one of its rows (its user row, or either of its two item rows).  Samples that
// share no row commute exactly, so the result is bit-identical to bpr_replay_kernel (strictly serial)
// while independent samples run in parallel -- on a matrix with thousands of rows a window needs 1-3
// rounds instead of 32 serial updates.
__global__ void __launch_bounds__(1024) bpr_replay_window_kernel(const ReplayParams p)
{
    __shared__ int m_u[1024], m_i[1024], m_j[1024];
    __shared__ unsigned char m_todo[1024];
    __shared__ int s_u[32], s_i[32], s_j[32], s_pending[32];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t k = (size_t)p.k;
    unsigned long long n_correct = 0, n_skipped = 0;
    for (int64_t base0 = 0; base0 < p.n_samples; base0 += 1024) {
        // ---- resolve 1024 samples at once, one per THREAD (read-only inputs => order-free): the ~10
        //      dependent gathers of (u, i, skip test) are paid once per 32 windows
        __syncthreads();
        {
            const int64_t s = base0 + threadIdx.x;
            int32_t mu = 0, mi = 0, mj = 0;
            bool todo = false;
            if (s < p.n_samples) {
                const int64_t ii = p.i_index[s];
                mj = p.j_id[s];
                mu = __ldg(p.coo_row + ii);
                mi = __ldg(p.indices + ii);
                todo = !row_contains(p.indices, __ldg(p.indptr + mu), __ldg(p.indptr + mu + 1), mj);
                if (!todo) ++n_skipped;             // counted per thread, summed at the end
            }
            m_u[threadIdx.x] = mu; m_i[threadIdx.x] = mi; m_j[threadIdx.x] = mj; m_todo[threadIdx.x] = todo ? 1 : 0;
        }
        __syncthreads();
        const int n_win = (int)min((int64_t)32, (p.n_samples - base0 + 31) / 32);
      for (int win = 0; win < n_win; ++win) {
        const int slot = win * 32 + w;              // this warp's sample of the window
        const int32_t mu = m_u[slot], mi = m_i[slot], mj = m_j[slot];
        bool todo = m_todo[slot] != 0;
        __syncthreads();                            // previous window fully retired
        if (lane == 0) { s_u[w] = mu; s_i[w] = mi; s_j[w] = mj; s_pending[w] = todo ? 1 : 0; }
        for (;;) {
            if (!__syncthreads_or(todo)) break;     // also publishes the state written in the last round
            bool run = false;
            if (todo) {
                bool conflict = false;
                if (lane < w && s_pending[lane]) {
                    const int ou = s_u[lane], oi = s_i[lane], oj = s_j[lane];
                    conflict = (ou == mu) | (oi == mi) | (oi == mj) | (oj == mi) | (oj == mj);
                }
                run = !__any_sync(0xffffffffu, conflict);
            }
            __syncthreads();                        // everybody has read the snapshot of s_pending
            if (run) {
                float* pu = p.U + (size_t)mu * k;
                float* pi = p.V + (size_t)mi * k;
                float* pj = p.V + (size_t)mj * k;
                const float bi = __ldcg(p.B + mi), bj = __ldcg(p.B + mj);
                // the first RC elements per lane stay in registers between the dot and the update (k <= 128:
                // the rows are read from L2 once per sample instead of twice)
                constexpr int RC = 4;
                float ru[RC], ri[RC], rj[RC];
                float part = 0.f;
#pragma unroll
                for (int t = 0; t < RC; ++t) {
                    const int f = lane + 32 * t;
                    ru[t] = ri[t] = rj[t] = 0.f;
                    if (f < p.k) { ru[t] = __ldcg(pu + f); ri[t] = __ldcg(pi + f); rj[t] = __ldcg(pj + f); }
                }
#pragma unroll
                for (int t = 0; t < RC; ++t)
                    if (lane + 32 * t < p.k) part = __fadd_rn(part, __fmul_rn(ru[t], __fsub_rn(ri[t], rj[t])));
                for (int f = lane + 32 * RC; f < p.k; f += 32)
                    part = __fadd_rn(part, __fmul_rn(__ldcg(pu + f), __fsub_rn(__ldcg(pi + f), __ldcg(pj + f))));
                const float score = __fadd_rn(__fsub_rn(bi, bj), group_sum<32>(part));
                float z = 1.f;
                bool update = true;
                if (p.hinge) {                      // recom_mmmf.pyx:137-139
                    if (score > 0.f) { ++n_correct; update = false; }
                } else {
                    z = (float)(1.0 / (1.0 + exp((double)score)));
                    n_correct += (z < .5f);
                }
                if (update) {
                    const float lr = p.lr, reg = p.reg;
#pragma unroll
                    for (int t = 0; t < RC; ++t) {
                        const int f = lane + 32 * t;
                        if (f < p.k) {
                            const float uf = ru[t], vi = ri[t], vj = rj[t];
                            __stcg(pu + f, __fadd_rn(uf, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, __fsub_rn(vi, vj)), __fmul_rn(reg, uf)))));
                            __stcg(pi + f, __fadd_rn(vi, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, uf), __fmul_rn(reg, vi)))));
                            __stcg(pj + f, __fadd_rn(vj, __fmul_rn(lr, __fsub_rn(__fmul_rn(-z, uf), __fmul_rn(reg, vj)))));
                        }
                    }
                    for (int f = lane + 32 * RC; f < p.k; f += 32) {
                        const float uf = __ldcg(pu + f), vi = __ldcg(pi + f), vj = __ldcg(pj + f);
                        __stcg(pu + f, __fadd_rn(uf, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, __fsub_rn(vi, vj)), __fmul_rn(reg, uf)))));
                        __stcg(pi + f, __fadd_rn(vi, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, uf), __fmul_rn(reg, vi)))));
                        __stcg(pj + f, __fadd_rn(vj, __fmul_rn(lr, __fsub_rn(__fmul_rn(-z, uf), __fmul_rn(reg, vj)))));
                    }
                    if (p.use_bias && lane == 0) {
                        __stcg(p.B + mi, __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(z, __fmul_rn(reg, bi)))));
                        __stcg(p.B + mj, __fadd_rn(bj, __fmul_rn(lr, __fsub_rn(-z, __fmul_rn(reg, bj)))));
                    }
                }
                todo = false;
                if (lane == 0) s_pending[w] = 0;
            }
        }
      }
    }
    // correct: one count per warp (lane 0); skipped: one count per resolving thread
    const unsigned long long sk = __reduce_add_sync(0xffffffffu, (unsigned)n_skipped);
    if (lane == 0) {
        atomicAdd(p.stats + 0, n_correct);
        atomicAdd(p.stats + 1, sk);
    }
}

// ---------------------------------------------------------------------------------------
// Parity mode, scheduled: one CTA of 32 warps, dependencies resolved over whole PHASES of 1024 samples.
// The windowed kernel above only looks 32 samples ahead; the stream's own critical path is 3-4x shorter than what
// 32-sample windows allow (tools/replay_levels.py).  Here every thread owns one sample of the phase and, round by round,
//   (A) every pending sample puts its index into the slots of its three rows in two direct-mapped "earliest pending
//       toucher" tables (atomicMin; user rows and item rows apart);
//   (B) a sample that holds all three of its slots has no earlier pending sample on any of its rows: it is READY.  Hash
//       collisions only make a sample wait (the earliest pending sample of the phase always wins its slots: progress);
//   (C) the ready samples are compacted into a queue and executed, one per warp at a time, in parallel -- they touch
//       pairwise-disjoint rows, and every earlier sample that shares a row with one of them has already been applied,
//       so the result is the serial one BIT FOR BIT (same per-sample arithmetic as bpr_replay_kernel).
// SMEM_MODEL: U, V and B are loaded into shared memory for the whole epoch when they fit (ML-100K sized problems: the
// case the seeded mode exists for), so a sample's rows cost ~30 cycles instead of an L2 round trip.
struct SchedShared {
    int m_u[1024], m_i[1024], m_j[1024];
    unsigned int tab_u[4096], tab_i[4096];
    unsigned short queue[1024];
    unsigned char pending[1024];
    int q_n;
};

__device__ __forceinline__ unsigned int sched_slot(int row) { return ((unsigned int)row * 2654435761u) >> 20; }

template <bool SMEM_MODEL>
__global__ void __launch_bounds__(1024) bpr_replay_sched_kernel(const ReplayParams p, int64_t n_users, int64_t n_items)
{
    extern __shared__ __align__(16) unsigned char sched_dyn[];
    SchedShared& sh = *reinterpret_cast<SchedShared*>(sched_dyn);
    float* sU = reinterpret_cast<float*>(sched_dyn + ((sizeof(SchedShared) + 15) & ~(size_t)15));
    float* sV = sU + (SMEM_MODEL ? n_users * p.k : 0);
    float* sB = sV + (SMEM_MODEL ? n_items * p.k : 0);
    const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
    const size_t k = (size_t)p.k;
    if (SMEM_MODEL) {
        for (int64_t x = tid; x < n_users * p.k; x += 1024) sU[x] = __ldcg(p.U + x);
        for (int64_t x = tid; x < n_items * p.k; x += 1024) sV[x] = __ldcg(p.V + x);
        for (int64_t x = tid; x < n_items; x += 1024) sB[x] = __ldcg(p.B + x);
    }
    for (int x = tid; x < 4096; x += 1024) { sh.tab_u[x] = 0xffffffffu; sh.tab_i[x] = 0xffffffffu; }
    if (tid == 0) sh.q_n = 0;
    __syncthreads();
    float* const Ub = SMEM_MODEL ? sU : p.U;
    float* const Vb = SMEM_MODEL ? sV : p.V;
    float* const Bb = SMEM_MODEL ? sB : p.B;
    auto ld = [&](const float* a) { return SMEM_MODEL ? *a : __ldcg(a); };
    auto st = [&](float* a, float v) { if (SMEM_MODEL) *a = v; else __stcg(a, v); };
    unsigned long long n_correct = 0, n_skipped = 0;
    for (int64_t base0 = 0; base0 < p.n_samples; base0 += 1024) {
        // ---- resolve the phase's samples, one per thread (read-only inputs: order-free)
        const int64_t s = base0 + tid;
        int32_t mu = 0, mi = 0, mj = 0;
        bool pend = false;
        if (s < p.n_samples) {
            const int64_t ii = p.i_index[s];
            mj = p.j_id[s];
            mu = __ldg(p.coo_row + ii);
            mi = __ldg(p.indices + ii);
            pend = !row_contains(p.indices, __ldg(p.indptr + mu), __ldg(p.indptr + mu + 1), mj);
            if (!pend) ++n_skipped;
        }
        sh.m_u[tid] = mu; sh.m_i[tid] = mi; sh.m_j[tid] = mj;
        const unsigned int hu = sched_slot(mu), hi = sched_slot(mi), hj = sched_slot(mj);
        for (;;) {
            if (!__syncthreads_or(pend)) break;                  // also orders the previous round's row writes
            // (A) earliest pending toucher of every row slot
            if (pend) {
                atomicMin(&sh.tab_u[hu], (unsigned int)tid);
                atomicMin(&sh.tab_i[hi], (unsigned int)tid);
                atomicMin(&sh.tab_i[hj], (unsigned int)tid);
            }
            __syncthreads();
            // (B) ready = holds all its slots
            const bool ready = pend && sh.tab_u[hu] == (unsigned int)tid && sh.tab_i[hi] == (unsigned int)tid
                               && sh.tab_i[hj] == (unsigned int)tid;
            const unsigned int bal = __ballot_sync(0xffffffffu, ready);
            int wbase = 0;
            if (lane == 0 && bal) wbase = atomicAdd(&sh.q_n, __popc(bal));
            wbase = __shfl_sync(0xffffffffu, wbase, 0);
            __syncthreads();                                       // every table read is done: slots may be reset
            if (pend) { sh.tab_u[hu] = 0xffffffffu; sh.tab_i[hi] = 0xffffffffu; sh.tab_i[hj] = 0xffffffffu; }
            if (ready) {
                sh.queue[wbase + __popc(bal & ((1u << lane) - 1u))] = (unsigned short)tid;
                pend = false;
            }
            __syncthreads();
            // (C) execute the ready samples, one per warp at a time (any order: they share no row)
            const int n_ready = sh.q_n;
            for (int q = w; q < n_ready; q += 32) {
                const int t = sh.queue[q];
                const int32_t u = sh.m_u[t], i = sh.m_i[t], j = sh.m_j[t];
                float* pu = Ub + (size_t)u * k;
                float* pi = Vb + (size_t)i * k;
                float* pj = Vb + (size_t)j * k;
                const float bi = ld(Bb + i), bj = ld(Bb + j);
                constexpr int RC = 4;                              // k <= 128: rows stay in registers between dot and update
                float ru[RC], ri[RC], rj[RC];
                float part = 0.f;
#pragma unroll
                for (int x = 0; x < RC; ++x) {
                    const int f = lane + 32 * x;
                    ru[x] = ri[x] = rj[x] = 0.f;
                    if (f < p.k) { ru[x] = ld(pu + f); ri[x] = ld(pi + f); rj[x] = ld(pj + f); }
                }
#pragma unroll
                for (int x = 0; x < RC; ++x)
                    if (lane + 32 * x < p.k) part = __fadd_rn(part, __fmul_rn(ru[x], __fsub_rn(ri[x], rj[x])));
                for (int f = lane + 32 * RC; f < p.k; f += 32)
                    part = __fadd_rn(part, __fmul_rn(ld(pu + f), __fsub_rn(ld(pi + f), ld(pj + f))));
                const float score = __fadd_rn(__fsub_rn(bi, bj), group_sum<32>(part));
                float z = 1.f;
                bool update = true;
                if (p.hinge) {                                     // recom_mmmf.pyx:137-139
                    if (score > 0.f) { ++n_correct; update = false; }
                } else {
                    z = (float)(1.0 / (1.0 + exp((double)score)));
                    n_correct += (z < .5f);
                }
                if (update) {
                    const float lr = p.lr, reg = p.reg;
#pragma unroll
                    for (int x = 0; x < RC; ++x) {
                        const int f = lane + 32 * x;
                        if (f < p.k) {
                            const float uf = ru[x], vi = ri[x], vj = rj[x];
                            st(pu + f, __fadd_rn(uf, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, __fsub_rn(vi, vj)), __fmul_rn(reg, uf)))));
                            st(pi + f, __fadd_rn(vi, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, uf), __fmul_rn(reg, vi)))));
                            st(pj + f, __fadd_rn(vj, __fmul_rn(lr, __fsub_rn(__fmul_rn(-z, uf), __fmul_rn(reg, vj)))));
                        }
                    }
                    for (int f = lane + 32 * RC; f < p.k; f += 32) {
                        const float uf = ld(pu + f), vi = ld(pi + f), vj = ld(pj + f);
                        st(pu + f, __fadd_rn(uf, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, __fsub_rn(vi, vj)), __fmul_rn(reg, uf)))));
                        st(pi + f, __fadd_rn(vi, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, uf), __fmul_rn(reg, vi)))));
                        st(pj + f, __fadd_rn(vj, __fmul_rn(lr, __fsub_rn(__fmul_rn(-z, uf), __fmul_rn(reg, vj)))));
                    }
                    if (p.use_bias && lane == 0) {
                        st(Bb + i, __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(z, __fmul_rn(reg, bi)))));
                        st(Bb + j, __fadd_rn(bj, __fmul_rn(lr, __fsub_rn(-z, __fmul_rn(reg, bj)))));
                    }
                }
            }
            __syncthreads();                                       // queue consumed
            if (tid == 0) sh.q_n = 0;
        }
    }
    __syncthreads();
    if (SMEM_MODEL) {
        for (int64_t x = tid; x < n_users * p.k; x += 1024) p.U[x] = sU[x];
        for (int64_t x = tid; x < n_items * p.k; x += 1024) p.V[x] = sV[x];
        for (int64_t x = tid; x < n_items; x += 1024) p.B[x] = sB[x];
    }
    // correct: one count per warp (lane 0 counted for the whole warp); skipped: one count per resolving thread
    const unsigned long long sk = __reduce_add_sync(0xffffffffu, (unsigned)n_skipped);
    if (lane == 0) {
        atomicAdd(p.stats + 0, n_correct);
        atomicAdd(p.stats + 1, sk);
    }
}

template <int G, int NPL, bool VEC, bool ATOMIC, int S, int MINB>
static int launch_hogwild_s(const BprParams& p, cudaStream_t st, const HogwildTune& tune)
{
    auto kern = bpr_hogwild_kernel<G, NPL, VEC, ATOMIC, S, MINB>;
    const int threads = tune.threads;
    int occ = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, 0));
    if (occ < 1) occ = 1;
    if (tune.blocks_per_sm > 0 && tune.blocks_per_sm < occ) occ = tune.blocks_per_sm;
    const int64_t groups_per_block = threads / G;
    int64_t want = (p.n_samples + groups_per_block * S - 1) / (groups_per_block * S);
    int64_t grid = (int64_t)sm_count() * occ;
    if (want < grid) grid = want;
    // Hogwild staleness bound: never run more samples concurrently than a quarter of the rows
    // of the smaller factor matrix (with fewer rows than in-flight samples every update would
    // be computed from a stale row and the epoch degenerates into one huge-batch step)
    const int64_t cap = (p.max_groups + groups_per_block * S - 1) / (groups_per_block * S);
    if (cap < grid) grid = cap;
    if (grid < 1) grid = 1;
    kern<<<(unsigned)grid, threads, 0, st>>>(p); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

template <int G, int NPL, bool VEC, bool ATOMIC, int MINB, int DEPTH>
static int launch_hogwild_chunk(const BprParams& p, cudaStream_t st, const HogwildTune& tune)
{
    auto kern = bpr_hogwild_chunk_kernel<G, NPL, VEC, ATOMIC, MINB, DEPTH>;
    const int threads = tune.threads;
    int occ = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, 0));
    if (occ < 1) occ = 1;
    if (tune.blocks_per_sm > 0 && tune.blocks_per_sm < occ) occ = tune.blocks_per_sm;
    const int64_t groups_per_block = threads / G;
    const int64_t n_chunks = (p.n_samples + G - 1) / G;
    int64_t want = (n_chunks + groups_per_block - 1) / groups_per_block;
    int64_t grid = (int64_t)sm_count() * occ;
    if (want < grid) grid = want;
    const int64_t cap = (p.max_groups + groups_per_block - 1) / groups_per_block;     // staleness bound
    if (cap < grid) grid = cap;
    if (grid < 1) grid = 1;
    kern<<<(unsigned)grid, threads, 0, st>>>(p); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

template <int G, bool ATOMIC, int D, int MINB>
static int launch_hogwild_stream(const BprParams& p, cudaStream_t st, const HogwildTune& tune)
{
    auto kern = bpr_hogwild_stream_kernel<G, ATOMIC, D, MINB>;
    const int threads = 256;
    const size_t smem = (size_t)(threads / G) * D * (3 * G * 16);
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
    if (occ < 1) occ = 1;
    if (tune.blocks_per_sm > 0 && tune.blocks_per_sm < occ) occ = tune.blocks_per_sm;
    const int64_t groups_per_block = threads / G;
    const int64_t n_chunks = (p.n_samples + G - 1) / G;
    int64_t want = (n_chunks + groups_per_block - 1) / groups_per_block;
    int64_t grid = (int64_t)sm_count() * occ;
    if (want < grid) grid = want;
    // staleness bound (see launch_hogwild_s): a group has D samples in flight
    const int64_t cap = (p.max_groups / D + groups_per_block - 1) / groups_per_block;
    if (cap < grid) grid = cap;
    if (grid < 1) grid = 1;
    kern<<<(unsigned)grid, threads, smem, st>>>(p); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

template <int G, int NPL, bool VEC, bool ATOMIC>
static int launch_hogwild(const BprParams& p, cudaStream_t st)
{
    // samples in flight per group: bounded by the register footprint of the 3*S row fragments
    constexpr int E = NPL * (VEC ? 4 : 1);
    const HogwildTune tune = read_tune();
    if constexpr (VEC && NPL == 1 && G >= 16) {
        // one float4 per lane (k % 4 == 0, 52 <= k <= 128): rows staged in shared memory, 2 samples in flight per group.
        // 16-lane groups (k <= 64, V L2-resident at configs[1]) stay on the register-staged chunk kernel.
        if (tune.S == 0 && G >= 32) return launch_hogwild_stream<G, ATOMIC, 2, 4>(p, st, tune);
        if (tune.S == 2) return launch_hogwild_stream<G, ATOMIC, 2, 4>(p, st, tune);          // A/B: force the streamed kernels
        if (tune.S == 4) return launch_hogwild_stream<G, ATOMIC, 4, 4>(p, st, tune);
    }
    if constexpr (E <= 8) {
        // 16-lane groups run two row-gathers ahead at 3 blocks/SM; 32-lane groups (k = 128: 512-byte rows, V beyond the
        // L2 at 1 M items) one gather ahead at 4 resident blocks (60 registers).  B200_BPR_TUNE selects the others.
        if (tune.S == 0 || tune.S == 64) {       // (64 = the register-staged chunk kernel where the streamed one is the default)
            if (G >= 32) return launch_hogwild_chunk<G, NPL, VEC, ATOMIC, 4, 1>(p, st, tune);
            return launch_hogwild_chunk<G, NPL, VEC, ATOMIC, 3, 2>(p, st, tune);
        }
        if (tune.S == 32) {              // the other combinations, for A/B runs
            if (G >= 32) return launch_hogwild_chunk<G, NPL, VEC, ATOMIC, 3, 1>(p, st, tune);
            return launch_hogwild_chunk<G, NPL, VEC, ATOMIC, 4, 1>(p, st, tune);
        }
    }
    if constexpr (E <= 4) {
        return launch_hogwild_s<G, NPL, VEC, ATOMIC, 1, 5>(p, st, tune);      // register-only variant (B200_BPR_TUNE=1,...)
    } else {
        return launch_hogwild_s<G, NPL, VEC, ATOMIC, 1, hogwild_min_blocks<NPL, VEC, 1>()>(p, st, tune);
    }
}

// ---------------------------------------------------------------------------------------
// Deterministic throughput mode (B200_BPR_DETERMINISTIC): the epoch's samples run in rounds of at most DET_ROUND.  Every
// sample of a round reads the factors as the previous round left them (bpr_det_grad_kernel writes nothing but the
// accumulators), and the round's updates are summed in 2^-40 fixed point with integer atomics -- exact, so their order
// does not matter -- before bpr_det_apply_kernel adds each touched element's sum once.  The result depends on the
// seed and the sample law only, not on thread timing: a run repeats bit for bit.  A round is about as many samples as
// the Hogwild kernels keep in flight, so the updates of a popular row are summed against a similar staleness.
constexpr int64_t DET_ROUND = 16384;
constexpr double DET_SCALE = 1099511627776.0;       // 2^40

struct DetAcc {
    unsigned long long* U;      // [n_users * k]  fixed-point sums of the round
    unsigned long long* V;      // [n_neg * k]
    unsigned long long* B;      // [n_neg]
};

// An update that is not finite or beyond the fixed-point range (|d| >= 2^22) cannot be summed: the element it belongs to
// becomes NaN at once, so a diverging model shows NaN as under the Hogwild kernels instead of saturated sums.
__device__ __forceinline__ void det_add(unsigned long long* a, float* x, float d)
{
    if (!(fabsf(d) < 4194304.f)) {
        atomicExch(reinterpret_cast<unsigned int*>(x), 0x7fc00000u);
        return;
    }
    const long long q = __double2ll_rn((double)d * DET_SCALE);
    if (q) atomicAdd(a, (unsigned long long)q);
}
// the element's sum is taken (and cleared) by exactly one of the samples that touched it
__device__ __forceinline__ void det_apply(unsigned long long* a, float* x)
{
    const long long q = (long long)atomicExch(a, 0ull);
    if (q) atomicAdd(x, (float)((double)q * (1.0 / DET_SCALE)));
}

// (u, i) and j of epoch-local sample s: the law of the Hogwild kernels
__device__ __forceinline__ void det_draw(const BprParams& p, int64_t s_local, int32_t& u, int32_t& i, int32_t& j)
{
    const uint64_t s = p.sample_base + (uint64_t)s_local;
    const Philox4 r = philox4x32_10((uint32_t)s, (uint32_t)(s >> 32), p.epoch_lo, p.epoch_hi, p.seed_lo, p.seed_hi);
    int64_t i_lo, i_len, j_lo, j_len;
    law_ranges(p.law, s, i_lo, i_len, j_lo, j_len);
    const int64_t ii = i_lo + (int64_t)range64(r.x, r.y, (uint64_t)i_len);
    j = p.neg_weighted ? __ldg(p.pairs + range64(r.z, r.w, (uint64_t)p.nnz)).y
                       : (int32_t)(j_lo + (int64_t)range64(r.z, r.w, (uint64_t)j_len));
    const int2 pr = __ldg(p.pairs + ii);
    u = pr.x;
    i = pr.y;
}

// one warp per sample of [s_begin, s_end): skip test, score, z, the three row updates into the accumulators
__global__ void __launch_bounds__(256) bpr_det_grad_kernel(const BprParams p, const DetAcc a, int64_t s_begin, int64_t s_end)
{
    const int lane = threadIdx.x & 31;
    const int64_t s_loc = s_begin + ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
    unsigned int n_correct = 0, n_skipped = 0;
    if (s_loc < s_end) {
        int32_t u, i, j;
        det_draw(p, s_loc, u, i, j);
        // has_non_zero(u, j)  (recom_bpr.pyx:241-243) = key (u, j) in the table
        const uint64_t key = ((uint64_t)(uint32_t)u << 32) | (uint32_t)j;
        uint64_t bb = mix64(key) & p.bucket_mask;
        bool hit = false;
        for (;;) {
            const unsigned long long sl = (lane < 4) ? __ldg(p.table + 4 * bb + lane) : 0ull;
            const unsigned h = __ballot_sync(0xffffffffu, lane < 4 && sl == key);
            const unsigned f = __ballot_sync(0xffffffffu, lane == 3 && sl != TABLE_EMPTY);
            if (h) { hit = true; break; }
            if (!f) break;
            bb = (bb + 1) & p.bucket_mask;
        }
        if (hit) {
            n_skipped = 1;
        } else {
            const size_t k = (size_t)p.k;
            const float* pu = p.U + (size_t)u * k;
            const float* pi = p.V + (size_t)i * k;
            const float* pj = p.V + (size_t)j * k;
            float part = 0.f;
            for (int e = lane; e < p.k; e += 32) part = fmaf(__ldcg(pu + e), __ldcg(pi + e) - __ldcg(pj + e), part);
            const float bi = __ldcg(p.B + i), bj = __ldcg(p.B + j);
            const float score = (bi - bj) + group_sum<32>(part);
            float z = 1.f;
            bool update = true;
            if (p.hinge) {
                if (score > 0.f) { n_correct = 1; update = false; }
            } else {
                z = bpr_z(score, p.exact_exp);
                n_correct = (z < .5f);
            }
            if (update) {
                const float lr = p.lr, reg = p.reg;
                for (int e = lane; e < p.k; e += 32) {
                    const float uf = __ldcg(pu + e), vi = __ldcg(pi + e), vj = __ldcg(pj + e);
                    det_add(a.U + (size_t)u * k + e, p.U + (size_t)u * k + e, lr * (z * (vi - vj) - reg * uf));
                    det_add(a.V + (size_t)i * k + e, p.V + (size_t)i * k + e, lr * (z * uf - reg * vi));
                    det_add(a.V + (size_t)j * k + e, p.V + (size_t)j * k + e, lr * (-z * uf - reg * vj));
                }
                if (p.use_bias && lane == 0) {
                    det_add(a.B + i, p.B + i, lr * (z - reg * bi));
                    det_add(a.B + j, p.B + j, lr * (-z - reg * bj));
                }
            }
        }
    }
    __shared__ unsigned int sh_stats[2];
    if (threadIdx.x < 2) sh_stats[threadIdx.x] = 0;
    __syncthreads();
    if (lane == 0 && (n_correct | n_skipped)) {
        atomicAdd(&sh_stats[0], n_correct);
        atomicAdd(&sh_stats[1], n_skipped);
    }
    __syncthreads();
    if (threadIdx.x == 0 && (sh_stats[0] | sh_stats[1])) {
        atomicAdd(p.stats + 0, (unsigned long long)sh_stats[0]);
        atomicAdd(p.stats + 1, (unsigned long long)sh_stats[1]);
    }
}

// one warp per sample of the same round: the summed updates of its rows, each element applied once
__global__ void __launch_bounds__(256) bpr_det_apply_kernel(const BprParams p, const DetAcc a, int64_t s_begin, int64_t s_end)
{
    const int lane = threadIdx.x & 31;
    const int64_t s_loc = s_begin + ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
    if (s_loc >= s_end) return;
    int32_t u, i, j;
    det_draw(p, s_loc, u, i, j);
    const size_t k = (size_t)p.k;
    for (int e = lane; e < p.k; e += 32) {
        det_apply(a.U + (size_t)u * k + e, p.U + (size_t)u * k + e);
        det_apply(a.V + (size_t)i * k + e, p.V + (size_t)i * k + e);
        det_apply(a.V + (size_t)j * k + e, p.V + (size_t)j * k + e);
    }
    if (p.use_bias && lane == 0) {
        det_apply(a.B + i, p.B + i);
        det_apply(a.B + j, p.B + j);
    }
}

static int bpr_epoch_deterministic(const BprParams& p, int64_t n_users, cudaStream_t st)
{
    const int64_t round = p.max_groups < DET_ROUND ? p.max_groups : DET_ROUND;
    const size_t nu = (size_t)n_users * p.k, nv = (size_t)p.n_neg * p.k;
    const size_t bytes = (nu + nv + (size_t)p.n_neg) * sizeof(unsigned long long);
    void* buf = nullptr;
    B200_CUDA(cudaMallocAsync(&buf, bytes, st));
    DetAcc a;
    a.U = static_cast<unsigned long long*>(buf);
    a.V = a.U + nu;
    a.B = a.V + nv;
    cudaError_t e = cudaMemsetAsync(buf, 0, bytes, st);      // the apply kernel leaves every sum it takes at zero
    const unsigned grid = (unsigned)((round * 32 + 255) / 256);
    for (int64_t s0 = 0; s0 < p.n_samples && e == cudaSuccess; s0 += round) {
        const int64_t s1 = s0 + round < p.n_samples ? s0 + round : p.n_samples;
        const unsigned g = (unsigned)(((s1 - s0) * 32 + 255) / 256);
        bpr_det_grad_kernel<<<g < grid ? g : grid, 256, 0, st>>>(p, a, s0, s1);
        bpr_det_apply_kernel<<<g < grid ? g : grid, 256, 0, st>>>(p, a, s0, s1);
        ::b200::count_launch(2);
        e = cudaGetLastError();
    }
    const cudaError_t f = cudaFreeAsync(buf, st);
    if (e != cudaSuccess) return cuda_fail(e, "bpr_det_grad_kernel / bpr_det_apply_kernel", __FILE__, __LINE__);
    B200_CUDA(f);
    return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" int64_t b200_bpr_table_slots(int64_t nnz)
{
    return nnz <= 0 ? 4 : table_buckets_for(nnz) * 4;
}

extern "C" int b200_bpr_prepare(const int32_t* indptr, const int32_t* indices, int64_t n_users, int64_t nnz,
                                int32_t* pairs, uint64_t* table, int64_t table_slots, void* stream)
{
    B200_REQUIRE(indptr && indices && pairs && table, "b200_bpr_prepare: null pointer argument");
    B200_REQUIRE(n_users >= 0 && nnz >= 0, "b200_bpr_prepare: bad sizes");
    B200_REQUIRE(table_slots == b200_bpr_table_slots(nnz), "b200_bpr_prepare: table_slots=%lld, expected %lld",
                 (long long)table_slots, (long long)b200_bpr_table_slots(nnz));
    B200_REQUIRE((((uintptr_t)pairs) & 7) == 0 && (((uintptr_t)table) & 31) == 0, "b200_bpr_prepare: pairs/table misaligned");
    cudaStream_t st = (cudaStream_t)stream;
    B200_CUDA(cudaMemsetAsync(table, 0xff, (size_t)table_slots * sizeof(uint64_t), st));
    if (nnz == 0) return B200_OK;
    const uint64_t mask = (uint64_t)(table_slots / 4) - 1;
    int64_t grid = (n_users + 7) / 8;                               // 8 warps (rows) per block
    if (grid > (int64_t)sm_count() * 32) grid = (int64_t)sm_count() * 32;
    if (grid < 1) grid = 1;
    bpr_prepare_kernel<<<(unsigned)grid, 256, 0, st>>>(indptr, indices, n_users, nnz, reinterpret_cast<int2*>(pairs),
                                                       reinterpret_cast<unsigned long long*>(table), mask); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

// Windows of the interaction list / blocks of the items of 40 MB of rows each, so that the rows one run of the epoch
// touches are a small slice of the whole model instead of all of it; 1 / 1 when the matrix is within two parts.
// The part size fixes the sample order of a blocked epoch; it was chosen for a 126 MB L2 and is kept on the H100's
// 50 MB L2 (where only one part at a time can stay resident), so that a seed keeps drawing the same epochs.
extern "C" int b200_bpr_block_plan(int64_t n_users, int64_t n_neg, int k, uint32_t* n_windows, uint32_t* n_blocks)
{
    B200_REQUIRE(n_users >= 1 && n_neg >= 1 && k >= 1 && n_windows && n_blocks, "b200_bpr_block_plan: bad argument");
    double part = 40.0 * 1024 * 1024;
    if (const char* e = getenv("B200_BPR_PART_MB")) {          // dev knob: bytes of rows per window / item block
        const double mb = atof(e);
        if (mb >= 1.0 && mb <= 4096.0) part = mb * 1024 * 1024;
    }
    const double ub = (double)n_users * k * 4, vb = (double)n_neg * k * 4;
    uint32_t wn = 1, bn = 1;
    if (ub + vb > 2 * part) {
        wn = (uint32_t)((ub + part - 1) / part);
        bn = (uint32_t)((vb + part - 1) / part);
        if (wn < 1) wn = 1;
        if (bn < 1) bn = 1;
    }
    *n_windows = wn; *n_blocks = bn;
    return B200_OK;
}

extern "C" int b200_bpr_epoch(const int32_t* pairs, const uint64_t* table, int64_t table_slots,
                              int64_t nnz, int64_t n_users, int64_t n_neg, int64_t n_samples,
                              float* U, float* V, float* B, int k,
                              float lr, float reg, int use_bias,
                              uint64_t seed, uint64_t epoch, uint64_t sample_base,
                              unsigned flags, int64_t* stats, void* stream)
{
    B200_REQUIRE(pairs && table && U && V && B && stats, "b200_bpr_epoch: null pointer argument");
    B200_REQUIRE(k >= 1 && k <= 1024, "b200_bpr_epoch: k=%d out of range [1, 1024]", k);
    B200_REQUIRE(nnz >= 0 && n_users >= 1 && n_neg >= 1 && n_samples >= 0, "b200_bpr_epoch: bad sizes nnz=%lld n_users=%lld n_neg=%lld n_samples=%lld",
                 (long long)nnz, (long long)n_users, (long long)n_neg, (long long)n_samples);
    B200_REQUIRE(table_slots == b200_bpr_table_slots(nnz), "b200_bpr_epoch: table_slots=%lld does not match nnz=%lld",
                 (long long)table_slots, (long long)nnz);
    if (n_samples == 0 || nnz == 0) return B200_OK;
    const RowLayout L = pick_layout(k);
    B200_REQUIRE(L.npl <= 8, "b200_bpr_epoch: k=%d not supported (scalar rows are limited to k <= 256)", k);
    if (L.vec) {
        B200_REQUIRE((((uintptr_t)U | (uintptr_t)V) & 15) == 0, "b200_bpr_epoch: U/V must be 16-byte aligned");
    }
    BprParams p;
    p.pairs = reinterpret_cast<const int2*>(pairs);
    p.table = reinterpret_cast<const unsigned long long*>(table);
    p.bucket_mask = (uint64_t)(table_slots / 4) - 1;
    p.nnz = nnz; p.n_neg = n_neg; p.n_samples = n_samples;
    {
        int64_t rows = n_users < n_neg ? n_users : n_neg;
        p.max_groups = rows / 4 < 16 ? 16 : rows / 4;
        if (flags & B200_SGD_UNBOUNDED) p.max_groups = INT64_MAX / 1024;
    }
    p.neg_weighted = (flags & B200_BPR_NEG_WEIGHTED) ? 1 : 0;
    p.hinge = (flags & B200_BPR_LOSS_HINGE) ? 1 : 0;
    {
        uint32_t wn = 1, bn = 1;
        if (flags & B200_BPR_BLOCKED) {
            const int rc = b200_bpr_block_plan(n_users, n_neg, k, &wn, &bn);
            if (rc) return rc;
            if (p.neg_weighted) bn = 1;      // WBPR negatives follow the interaction list: only the user side is blocked
        }
        p.law = make_law(nnz, n_neg, wn, bn, epoch);
        if (wn > 1 || bn > 1) {              // the staleness cap counts the rows of ONE window / block
            int64_t rows = (n_users / wn) < (n_neg / bn) ? (n_users / wn) : (n_neg / bn);
            const int64_t cap = rows / 4 < 16 ? 16 : rows / 4;
            if (!(flags & B200_SGD_UNBOUNDED) && cap < p.max_groups) p.max_groups = cap;
        }
    }
    p.debug_skip = 0;
    if (const char* e = getenv("B200_BPR_DEBUG_SKIP")) p.debug_skip = atoi(e);
    p.U = U; p.V = V; p.B = B; p.k = k; p.lr = lr; p.reg = reg; p.use_bias = use_bias;
    if (p.hinge) p.use_bias = 1;          // MMMF always trains the item biases (recom_mmmf.pyx:149-152)
    p.seed_lo = (uint32_t)seed; p.seed_hi = (uint32_t)(seed >> 32);
    p.epoch_lo = (uint32_t)epoch; p.epoch_hi = (uint32_t)(epoch >> 32);
    p.sample_base = sample_base;
    p.stats = reinterpret_cast<unsigned long long*>(stats);
    cudaStream_t st = (cudaStream_t)stream;
    const bool atomic = flags & B200_SGD_ATOMIC;
    p.exact_exp = (flags & B200_SGD_EXACT_EXP) ? 1 : 0;
    if (flags & B200_BPR_DETERMINISTIC) return bpr_epoch_deterministic(p, n_users, st);
#define CALL(G_, NPL_, VEC_)                                                                      \
    do {                                                                                          \
        const int rc = atomic ? launch_hogwild<G_, NPL_, VEC_, true>(p, st)                       \
                              : launch_hogwild<G_, NPL_, VEC_, false>(p, st);                     \
        if (rc) return rc;                                                                        \
    } while (0)
    B200_DISPATCH_LAYOUT(L, CALL);
#undef CALL
    return B200_OK;
}

static int bpr_replay_launch(ReplayParams& p, int64_t n_users, int64_t n_items, cudaStream_t st)
{
    const char* mode = getenv("B200_REPLAY_SERIAL");          // dev knob: 1 = strictly serial warp, 2 = 32-sample windows
    ::b200::count_launch();
    if (mode && mode[0] == '1') { bpr_replay_kernel<<<1, 32, 0, st>>>(p); B200_CUDA(cudaGetLastError()); return B200_OK; }
    if (mode && mode[0] == '2') { bpr_replay_window_kernel<<<1, 1024, 0, st>>>(p); B200_CUDA(cudaGetLastError()); return B200_OK; }
    const size_t fixed = (sizeof(SchedShared) + 15) & ~(size_t)15;
    size_t model = 0;
    if (n_users > 0 && n_items > 0) model = ((size_t)(n_users + n_items) * p.k + (size_t)n_items) * sizeof(float);
    const size_t limit = 227 * 1024 - 1024;
    if (model > 0 && fixed + model <= limit && !(mode && mode[0] == '3')) {      // 3 = scheduled kernel on the global factors
        const size_t smem = fixed + model;
        B200_CUDA(cudaFuncSetAttribute(bpr_replay_sched_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        bpr_replay_sched_kernel<true><<<1, 1024, smem, st>>>(p, n_users, n_items);
    } else {
        B200_CUDA(cudaFuncSetAttribute(bpr_replay_sched_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fixed));
        bpr_replay_sched_kernel<false><<<1, 1024, fixed, st>>>(p, 0, 0);
    }
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_bpr_epoch_replay2(const int64_t* i_index, const int32_t* j_id, int64_t n_samples,
                                      const int32_t* indptr, const int32_t* indices, const int32_t* coo_row,
                                      int64_t n_users, int64_t n_items,
                                      float* U, float* V, float* B, int k,
                                      float lr, float reg, int use_bias, unsigned flags,
                                      int64_t* stats, void* stream)
{
    B200_REQUIRE(i_index && j_id && indptr && indices && coo_row && U && V && B && stats,
                 "b200_bpr_epoch_replay: null pointer argument");
    B200_REQUIRE(k >= 1, "b200_bpr_epoch_replay: k=%d", k);
    if (n_samples <= 0) return B200_OK;
    ReplayParams p;
    p.i_index = i_index; p.j_id = j_id; p.n_samples = n_samples;
    p.indptr = indptr; p.indices = indices; p.coo_row = coo_row;
    p.U = U; p.V = V; p.B = B; p.k = k; p.lr = lr; p.reg = reg; p.use_bias = use_bias;
    p.hinge = (flags & B200_BPR_LOSS_HINGE) ? 1 : 0;
    if (p.hinge) p.use_bias = 1;
    p.stats = reinterpret_cast<unsigned long long*>(stats);
    return bpr_replay_launch(p, n_users, n_items, (cudaStream_t)stream);
}

extern "C" int b200_bpr_epoch_replay(const int64_t* i_index, const int32_t* j_id, int64_t n_samples,
                                     const int32_t* indptr, const int32_t* indices, const int32_t* coo_row,
                                     float* U, float* V, float* B, int k,
                                     float lr, float reg, int use_bias, unsigned flags,
                                     int64_t* stats, void* stream)
{
    return b200_bpr_epoch_replay2(i_index, j_id, n_samples, indptr, indices, coo_row, 0, 0, U, V, B, k, lr, reg, use_bias,
                                  flags, stats, stream);
}
