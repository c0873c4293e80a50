// BPR SGD epochs for sm_90a.
//
// Replaces BPR._fit_sgd (reference: cornac/models/bpr/recom_bpr.pyx:208-269) with
//   * throughput mode (Hogwild): persistent grids in which every G-lane group draws its own (u, i+, j-) triplets from
//     the CSR matrix with a counter-based RNG, gathers the three factor rows with L2-only loads, reduces the pairwise
//     dot with warp shuffles and scatters the update back (plain stores = the reference's lock-free Hogwild, or
//     red.global.add when B200_SGD_ATOMIC is set).  launch_hogwild picks one kernel per row layout:
//     bpr_hogwild_stream_kernel, bpr_hogwild_chunk_kernel or bpr_hogwild_kernel.
//   * deterministic mode: bpr_det_grad_kernel + bpr_det_apply_kernel, the same law and updates in fixed rounds.
//   * parity mode: bpr_replay_sched_kernel applies an explicit sample stream with the same result as the sequential
//     seeded reference (num_threads = 1, recom_bpr.pyx:132-133); bpr_replay_kernel (one warp, strictly serial) is the
//     reference it is checked against.
//
// HBM-bound integer/gather work: no tensor cores here by design (DESIGN.md, K1).
#include <stdlib.h>

#include <algorithm>

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

// key of the pair (u, i) in the membership table
__device__ __forceinline__ uint64_t pair_key(int32_t u, int32_t i)
{
    return ((uint64_t)(uint32_t)u << 32) | (uint32_t)i;
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

// z of a sample and its count as correctly ranked.  MMMF (recom_mmmf.pyx:137-139) does not update a correctly ranked
// pair (returns false) and uses z = 1 otherwise.
template <class Count>
__device__ __forceinline__ bool sample_z(int hinge, int exact, float score, float& z, Count& n_correct)
{
    if (hinge) {
        if (score > 0.f) { ++n_correct; return false; }
        z = 1.f;
    } else {
        z = bpr_z(score, exact);
        n_correct += (z < .5f);
    }
    return true;
}

// ---------------------------------------------------------------------------------------
// Pieces shared by the throughput kernels.

// Sample s_local of the epoch (the law of common.cuh): its interaction index ii and its negative j.  A WBPR negative is
// the item of a uniformly drawn interaction (recom_wbpr.pyx:131).  The caller gathers pairs[ii] itself, where the
// latency of that load fits its schedule.
__device__ __forceinline__ void draw_sample(const BprParams& p, int64_t s_local, int64_t& ii, int32_t& j)
{
    const uint64_t s = p.sample_base + (uint64_t)s_local;
    const Philox4 r = philox4x32_10((uint32_t)s, (uint32_t)(s >> 32), p.epoch_lo, p.epoch_hi, p.seed_lo, p.seed_hi);
    int64_t i_lo, i_len, j_lo, j_len;
    law_ranges(p.law, s, i_lo, i_len, j_lo, j_len);
    ii = i_lo + (int64_t)range64(r.x, r.y, (uint64_t)i_len);
    j = p.neg_weighted ? __ldg(p.pairs + range64(r.z, r.w, (uint64_t)p.nnz)).y
                       : (int32_t)(j_lo + (int64_t)range64(r.z, r.w, (uint64_t)j_len));
}

// has_non_zero(u, j) (recom_bpr.pyx:241-243) by one lane: `key` in `bucket` (two 16-byte loads) or in the buckets it
// overflowed into
__device__ __forceinline__ bool bucket_has(const unsigned long long* table, uint64_t mask, uint64_t key, uint64_t bucket)
{
    bool found, full;
    do {
        const ulonglong2 b0 = __ldg(reinterpret_cast<const ulonglong2*>(table + 4 * bucket));
        const ulonglong2 b1 = __ldg(reinterpret_cast<const ulonglong2*>(table + 4 * bucket) + 1);
        found = (b0.x == key) | (b0.y == key) | (b1.x == key) | (b1.y == key);
        full = (b1.y != TABLE_EMPTY);
        bucket = (bucket + 1) & mask;
    } while (!found && full);              // rare: the bucket overflowed into the next one
    return found;
}

// The same test by a G-lane group: lanes 0-3 read the four slots of a bucket, 8 bytes each
template <int G>
__device__ __forceinline__ bool group_has(const unsigned long long* table, uint64_t mask, uint64_t key, uint64_t bucket,
                                          int lg)
{
    const unsigned gmask = group_mask<G>();
    for (;;) {
        const unsigned long long sl = (lg < 4) ? __ldg(table + 4 * bucket + lg) : 0ull;
        const unsigned hit = __ballot_sync(gmask, lg < 4 && sl == key) & gmask;
        const unsigned full = __ballot_sync(gmask, lg == 3 && sl != TABLE_EMPTY) & gmask;
        if (hit) return true;
        if (!full) return false;
        bucket = (bucket + 1) & mask;      // rare: the bucket overflowed into the next one
    }
}

// Block epilogue: the block's (correct, skipped) counts added to the epoch statistics with two atomics.  Every thread
// passes its own share, so a count kept by the whole group goes in from one lane of the group only.
__device__ __forceinline__ void flush_stats(unsigned int correct, unsigned int skipped, unsigned long long* stats)
{
    __shared__ unsigned int sh_stats[2];
    if (threadIdx.x < 2) sh_stats[threadIdx.x] = 0;
    __syncthreads();
    correct = __reduce_add_sync(0xffffffffu, correct);
    skipped = __reduce_add_sync(0xffffffffu, skipped);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&sh_stats[0], correct);
        atomicAdd(&sh_stats[1], skipped);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(stats + 0, (unsigned long long)sh_stats[0]);
        atomicAdd(stats + 1, (unsigned long long)sh_stats[1]);
    }
}

// The SGD step of sample (u, i, j) from the group's fragments of its rows (recom_bpr.pyx:253-267): red.add of the
// deltas (ATOMIC) or plain stores of the updated rows and biases
template <int G, int NPL, bool VEC, bool ATOMIC>
__device__ __forceinline__ void frag_update(const BprParams& p, RowFrag<NPL, VEC>& fu, RowFrag<NPL, VEC>& fi,
                                            RowFrag<NPL, VEC>& fj, float bi, float bj, int32_t u, int32_t i, int32_t j,
                                            float z, int lg, int n_units)
{
    constexpr int E = NPL * RowFrag<NPL, VEC>::W;
    const float lr = p.lr, reg = p.reg;
    const size_t k = (size_t)p.k;
    float* pu = p.U + (size_t)u * k;
    float* pi = p.V + (size_t)i * k;
    float* pj = p.V + (size_t)j * k;
    if (ATOMIC) {
        RowFrag<NPL, VEC> du, di, dj;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const float uf = fu.v[e], vi = fi.v[e], vj = fj.v[e];
            du.v[e] = lr * (z * (vi - vj) - reg * uf);
            di.v[e] = lr * (z * uf - reg * vi);
            dj.v[e] = lr * (-z * uf - reg * vj);
        }
        row_red_add<G, NPL, VEC>(du, pu, lg, n_units);
        row_red_add<G, NPL, VEC>(di, pi, lg, n_units);
        row_red_add<G, NPL, VEC>(dj, pj, lg, n_units);
        if (p.use_bias && lg == 0) {
            red_add_f32(p.B + i, lr * (z - reg * bi));
            red_add_f32(p.B + j, lr * (-z - reg * bj));
        }
    } else {
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const float uf = fu.v[e], vi = fi.v[e], vj = fj.v[e];
            fu.v[e] = uf + lr * (z * (vi - vj) - reg * uf);
            fi.v[e] = vi + lr * (z * uf - reg * vi);
            fj.v[e] = vj + lr * (-z * uf - reg * vj);
        }
        row_store<G, NPL, VEC>(fu, pu, lg, n_units);
        row_store<G, NPL, VEC>(fi, pi, lg, n_units);
        row_store<G, NPL, VEC>(fj, pj, lg, n_units);
        if (p.use_bias && lg == 0) {
            __stcg(p.B + i, bi + lr * (z - reg * bi));
            __stcg(p.B + j, bj + lr * (-z - reg * bj));
        }
    }
}

// ---------------------------------------------------------------------------------------
// One sample per G-lane group, rows in registers: the layouts with 16 or 32 floats of a row per lane (k > 256).
template <int G, int NPL, bool VEC, bool ATOMIC, int MINB>
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

    for (int64_t s = gid; s < p.n_samples; s += n_groups) {
        // ---- draw the triplet (every lane of the group computes the same values); the negative row does not depend on
        //      the interaction gather, so it goes out first
        int64_t ii;
        int32_t j;
        draw_sample(p, s, ii, j);
        const int2 pr = __ldg(p.pairs + ii);
        Frag fu, fi, fj;
        row_load<G, NPL, VEC>(fj, p.V + (size_t)j * k, lg, n_units);
        const float bj = __ldcg(p.B + j);
        // ---- user row, positive row and the membership bucket (has_non_zero(u, j), recom_bpr.pyx:241-243), all in
        //      flight together
        const int32_t u = pr.x, i = pr.y;
        row_load<G, NPL, VEC>(fu, p.U + (size_t)u * k, lg, n_units);
        row_load<G, NPL, VEC>(fi, p.V + (size_t)i * k, lg, n_units);
        const float bi = __ldcg(p.B + i);
        const uint64_t key = pair_key(u, j);
        const bool skip = group_has<G>(p.table, p.bucket_mask, key, mix64(key) & p.bucket_mask, lg);
        n_skipped += skip;
        // ---- score, z, update (recom_bpr.pyx:249-267)
        float part = 0.f;
#pragma unroll
        for (int e = 0; e < E; ++e) part = fmaf(fu.v[e], fi.v[e] - fj.v[e], part);
        const float score = (bi - bj) + group_sum<G>(part);
        if (skip) continue;     // group-uniform
        float z;
        if (!sample_z(p.hinge, p.exact_exp, score, z, n_correct)) continue;
        frag_update<G, NPL, VEC, ATOMIC>(p, fu, fi, fj, bi, bj, u, i, j, z, lg, n_units);
    }
    flush_stats(lg == 0 ? n_correct : 0u, lg == 0 ? n_skipped : 0u, p.stats);      // one count per group
}

// ---------------------------------------------------------------------------------------
// Chunked kernel (the layouts with up to 8 floats of a row per lane, but for the one of the streamed kernel below): the
// per-sample bookkeeping that every lane of a group would compute redundantly (Philox, range reduction, pair gather, key
// hash, bucket probe) is done ONCE PER LANE FOR G DIFFERENT SAMPLES -- lane l of a group resolves sample (chunk*G + l) --
// so a group has G independent metadata gathers in flight at once and pays 1/G of those instructions per sample.  The G
// resolved triplets are then broadcast one by one with warp shuffles and applied by the whole group, DEPTH row-gathers
// ahead of the arithmetic: groups of fewer than 32 lanes two gathers ahead at 3 resident blocks per SM, 32-lane groups one
// ahead at 4.
template <int G, int NPL, bool VEC, bool ATOMIC, int MINB = (G < 32 ? 3 : 4), int DEPTH = (G < 32 ? 2 : 1)>
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

    unsigned int n_correct = 0, n_skipped = 0;

    for (int64_t c = gid; c < n_chunks; c += n_groups) {
        // ---- phase 1: this lane's own sample
        const int64_t sl = c * G + lg;
        int mlive = sl < p.n_samples;
        int64_t ii;
        int32_t mj;
        draw_sample(p, sl, ii, mj);
        const int2 pr = __ldg(p.pairs + ii);
        const int32_t mu = pr.x, mi = pr.y;
        {
            const uint64_t key = pair_key(mu, mj);
            const bool found = bucket_has(p.table, p.bucket_mask, key, mix64(key) & p.bucket_mask);
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
            if (!sample_z(p.hinge, p.exact_exp, score, z, n_correct)) continue;
            frag_update<G, NPL, VEC, ATOMIC>(p, fu[cur], fi[cur], fj[cur], bi[cur], bj[cur], cu[cur], ci[cur], cj[cur], z,
                                             lg, n_units);
        }
    }
    flush_stats(lg == 0 ? n_correct : 0u, n_skipped, p.stats);      // skips were counted per lane
}

// ---------------------------------------------------------------------------------------
// Streamed kernel (k % 4 == 0, 64 < k <= 128: 32-lane groups, one float4 of a row per lane): the chunked kernel above keeps
// the rows of the samples in flight in REGISTERS, is fully unrolled over the G samples of a chunk (190 KB of code: 17 % of
// its stall samples were instruction-cache misses, ncu r02) and exposes the two dependent DRAM gathers of the sampling
// (pair -> bucket) once per chunk.  Here
//   * the factor rows of the next D samples are staged in SHARED MEMORY with cp.async (LDGSTS.BYPASS, L2-coherent like
//     the ld.global.cg they replace): every lane copies and later reads back only its own 16-byte column, so no barrier
//     is needed and no register is held by a row in flight;
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
    int64_t ii;
    draw_sample(p, sl, ii, m.j);
    m.pr = __ldg(p.pairs + ii);
}
__device__ __forceinline__ void meta_step_b(const BprParams& p, ChunkMeta& m)
{
    m.u = m.pr.x; m.i = m.pr.y;
    m.key = pair_key(m.u, m.j);
    m.bucket = mix64(m.key) & p.bucket_mask;
    m.b0 = __ldg(reinterpret_cast<const ulonglong2*>(p.table + 4 * m.bucket));
    m.b1 = __ldg(reinterpret_cast<const ulonglong2*>(p.table + 4 * m.bucket) + 1);
}
// returns 1 when the sample was skipped (has_non_zero(u, j), recom_bpr.pyx:241-243); marks dead samples with u = ~u
__device__ __forceinline__ int meta_step_c(const BprParams& p, ChunkMeta& m)
{
    bool found = (m.b0.x == m.key) | (m.b0.y == m.key) | (m.b1.x == m.key) | (m.b1.y == m.key);
    if (!found && m.b1.y != TABLE_EMPTY)        // rare: the bucket overflowed into the next one
        found = bucket_has(p.table, p.bucket_mask, m.key, (m.bucket + 1) & p.bucket_mask);
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
            if (!sample_z(p.hinge, p.exact_exp, score, z, n_correct)) continue;
            const float a = lr * z;                     // delta = lr (z x - reg y) = a x - lrreg y
            float* pu = p.U + (size_t)su * k + lg * 4;
            float* pi = p.V + (size_t)si * k + lg * 4;
            float* pj = p.V + (size_t)sj * k + lg * 4;
            if (col) {
                if (ATOMIC) {
                    red_add_v4(pu, fmaf(a, dx, -lrreg * u4.x), fmaf(a, dy, -lrreg * u4.y), fmaf(a, dz, -lrreg * u4.z), fmaf(a, dw, -lrreg * u4.w));
                    red_add_v4(pi, fmaf(a, u4.x, -lrreg * vi4.x), fmaf(a, u4.y, -lrreg * vi4.y), fmaf(a, u4.z, -lrreg * vi4.z), fmaf(a, u4.w, -lrreg * vi4.w));
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
    flush_stats(lg == 0 ? n_correct : 0u, n_skipped, p.stats);      // skips were counted per lane
}

// ---------------------------------------------------------------------------------------
// Parity mode: the sample stream is applied with the result of the strictly serial loop, bit for bit.
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

// One sample (u, i, j) on one warp: unfused f32 arithmetic in the operation order of recom_bpr.pyx:249-267 (the dot is a
// lane-strided partial sum over f = lane, lane + 32, ... + shuffle tree).  The first RC elements per lane stay in
// registers between the dot and the update (k <= 128: the rows are read once per sample instead of twice).  ld / st
// read and write the factors U, V, B: in global memory or an on-chip copy.  Returns 1 when the sample counts as
// correctly ranked (every lane returns the same).
template <class Ld, class St>
__device__ __forceinline__ int replay_sample(const ReplayParams& p, float* U, float* V, float* B, int32_t u, int32_t i,
                                             int32_t j, int lane, Ld ld, St st)
{
    const size_t k = (size_t)p.k;
    float* pu = U + (size_t)u * k;
    float* pi = V + (size_t)i * k;
    float* pj = V + (size_t)j * k;
    const float bi = ld(B + i), bj = ld(B + j);
    constexpr int RC = 4;
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
    float z;
    int correct = 0;
    if (sample_z(p.hinge, 1, score, z, correct)) {
        const float lr = p.lr, reg = p.reg;
        auto step = [&](int f, float uf, float vi, float vj) {
            st(pu + f, __fadd_rn(uf, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, __fsub_rn(vi, vj)), __fmul_rn(reg, uf)))));
            st(pi + f, __fadd_rn(vi, __fmul_rn(lr, __fsub_rn(__fmul_rn(z, uf), __fmul_rn(reg, vi)))));
            st(pj + f, __fadd_rn(vj, __fmul_rn(lr, __fsub_rn(__fmul_rn(-z, uf), __fmul_rn(reg, vj)))));
        };
#pragma unroll
        for (int x = 0; x < RC; ++x)
            if (lane + 32 * x < p.k) step(lane + 32 * x, ru[x], ri[x], rj[x]);
        for (int f = lane + 32 * RC; f < p.k; f += 32) {
            const float uf = ld(pu + f), vi = ld(pi + f), vj = ld(pj + f);
            step(f, uf, vi, vj);
        }
        if (p.use_bias && lane == 0) {
            st(B + i, __fadd_rn(bi, __fmul_rn(lr, __fsub_rn(z, __fmul_rn(reg, bi)))));
            st(B + j, __fadd_rn(bj, __fmul_rn(lr, __fsub_rn(-z, __fmul_rn(reg, bj)))));
        }
    }
    return correct;
}

// The strictly serial reference: one warp, the samples one after the other
__global__ void __launch_bounds__(32) bpr_replay_kernel(const ReplayParams p)
{
    const int lane = threadIdx.x;
    auto ld = [](const float* a) { return __ldcg(a); };
    auto st = [](float* a, float v) { __stcg(a, v); };
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
            n_correct += replay_sample(p, p.U, p.V, p.B, u, i, j, lane, ld, st);
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
            const unsigned long long key = pair_key((int32_t)u, i);
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

// ---------------------------------------------------------------------------------------
// Parity mode, scheduled: one CTA of 32 warps, dependencies resolved over whole PHASES of 1024 samples.
// The stream's critical path is far shorter than its length (tools/replay_levels.py).  Every thread owns one sample of
// the phase and, round by round,
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
                n_correct += replay_sample(p, Ub, Vb, Bb, sh.m_u[t], sh.m_i[t], sh.m_j[t], lane, ld, st);
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

// Persistent grid of 256-thread blocks of G-lane groups: as many blocks as are resident on the device at once, but no
// more than `units` units of work (one per group and grid-stride step) need, and no more groups than `max_groups`.  That
// is the Hogwild staleness bound: never run more samples concurrently than a quarter of the rows of the smaller factor
// matrix (with fewer rows than in-flight samples every update would be computed from a stale row and the epoch
// degenerates into one huge-batch step).
template <class Kern>
static int launch_persistent(Kern kern, const BprParams& p, int G, int64_t units, int64_t max_groups, size_t smem,
                             cudaStream_t st)
{
    constexpr int threads = 256;
    int occ = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
    if (occ < 1) occ = 1;
    const int64_t groups_per_block = threads / G;
    const int64_t want = (units + groups_per_block - 1) / groups_per_block;
    const int64_t cap = (max_groups + groups_per_block - 1) / groups_per_block;
    int64_t grid = (int64_t)sm_count() * occ;
    if (want < grid) grid = want;
    if (cap < grid) grid = cap;
    if (grid < 1) grid = 1;
    kern<<<(unsigned)grid, threads, smem, st>>>(p); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

// One kernel per row layout (pick_layout), E floats of a row per lane.  The launch shapes were chosen on B200 and have
// not been re-tuned on the H100.
template <int G, int NPL, bool VEC, bool ATOMIC>
static int launch_hogwild(const BprParams& p, cudaStream_t st)
{
    constexpr int E = NPL * (VEC ? 4 : 1);
    const int64_t n_chunks = (p.n_samples + G - 1) / G;
    if constexpr (VEC && NPL == 1 && G == 32) {
        // one float4 per lane (k % 4 == 0, 64 < k <= 128): rows staged in shared memory, D samples in flight per group
        constexpr int D = 2;
        auto kern = bpr_hogwild_stream_kernel<G, ATOMIC, D, 4>;
        const size_t smem = (size_t)(256 / G) * D * (3 * G * 16);
        B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        return launch_persistent(kern, p, G, n_chunks, p.max_groups / D, smem, st);
    } else if constexpr (E <= 8) {
        return launch_persistent(bpr_hogwild_chunk_kernel<G, NPL, VEC, ATOMIC>, p, G, n_chunks, p.max_groups, 0, st);
    } else {
        // 16 or 32 floats per lane: the resident blocks per SM the register allocator is asked to make room for (the
        // kernel is latency-bound on dependent gathers, so samples in flight per SM is the lever)
        return launch_persistent(bpr_hogwild_kernel<G, NPL, VEC, ATOMIC, (E <= 16 ? 2 : 1)>, p, G, p.n_samples,
                                 p.max_groups, 0, st);
    }
}

// ---------------------------------------------------------------------------------------
// Deterministic throughput mode (B200_BPR_DETERMINISTIC): the epoch's samples run in rounds of at most DET_ROUND.  Every
// sample of a round reads the factors as the previous round left them, and each element of a row gets ONE update per
// round, x <- x + (float)(Q 2^-40), where Q is the exact (wrapping int64) sum of the round's 2^-40 fixed-point deltas of
// that element -- so the order in which the samples run does not matter and a run repeats bit for bit.  A round is about
// as many samples as the Hogwild kernels keep in flight, so the updates of a popular row are summed against a similar
// staleness.  Per round r the work is split in three phases, ordered by kernel boundaries on one stream only:
//   plan   (in the first CTAs of bpr_det_grad_kernel of round r - 1; a prologue launch of bpr_det_apply_kernel plans
//          round 0): one thread per sample draws it, runs the skip test, writes its record {u, i, j, live} and counts the
//          touches of its three rows; the touch that makes a row SHARED (count 1 -> 2) gives it a slot of a compact
//          accumulator (which row gets which slot depends on timing, but the sums are exact integers, so it does not
//          change the result);
//   grad   (bpr_det_grad_kernel): one warp per record computes score, z and the deltas.  A row the sample is the only
//          toucher of is read by no other sample of the round, so the warp adds its deltas to it at once; the deltas of a
//          shared row go into the row's slot with integer atomics;
//   apply  (bpr_det_apply_kernel): one warp per slot adds the slot's sums to its row and clears the slot.
// A live sample never touches one item row twice (j == i means (u, j) is an interaction: the sample is skipped), so a
// row touched once receives exactly one term.  The plan state is double-buffered by round parity: the plan of round
// r + 1 reads only the inputs and writes only the other parity, whose last users (grad and apply of round r - 1) have
// completed, so it shares nothing with the grad and apply of round r.
constexpr int64_t DET_ROUND = 16384;
constexpr double DET_SCALE = 1099511627776.0;       // 2^40
constexpr unsigned DET_ITEM = 0x80000000u;          // row_of_slot tag of an item row (user rows carry their id alone)

struct DetPlan {
    int4* rec;                      // [round] {u, i, j, live} of the round's samples
    unsigned int* cnt_u;            // [n_users] touches of the row in the round (reset to 0 by the round's grad / apply)
    unsigned int* cnt_v;            // [n_neg]
    unsigned int* slot_u;           // [n_users] accumulator slot of a shared row (valid while its count is >= 2)
    unsigned int* slot_v;           // [n_neg]
    unsigned int* row_of_slot;      // [cap] the row of each slot: user id, or item id | DET_ITEM
};

struct DetState {
    DetPlan plan[2];                // by round parity
    unsigned long long* acc;        // [cap][k + 1] 2^-40 fixed-point sums of the shared rows; column k = the item bias
    unsigned int* n_shared;         // [rounds] slots taken by each round
    unsigned int cap;               // slots of a round's row_of_slot
    float d_max;                    // bound on |d| that keeps every round sum in range (det_delta_bound)
};

// Largest |d| a delta may have in rounds of R samples: 2^(22 - ceil(log2 R)), 256 at R = 16384.  A live sample touches
// each row at most once (one user row; i != j), so an element takes at most R terms per round and |Q| <= 2^62: the
// int64 sum cannot wrap into a finite, wrong value.
static float det_delta_bound(int64_t R)
{
    int c = 0;
    while (((int64_t)1 << c) < R) ++c;
    return ldexpf(1.f, 22 - c);
}

// x + d as the global f32 atomic add computes it (round to nearest, subnormal inputs and results flushed to zero)
__device__ __forceinline__ float det_fadd(float x, float d)
{
    float r;
    asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(x), "f"(d));
    return r;
}

// Where a sample's delta for one element of a row goes: straight into the factor x when the sample is the row's only
// toucher in the round (a == nullptr), else into the row's accumulator slot a.
struct DetDst {
    float* x;
    unsigned long long* a;
};

// An update that is not finite or not below the round's bound d_max cannot be summed: the element it belongs to becomes
// NaN at once, so a diverging model shows NaN as under the Hogwild kernels instead of wrapped sums.
__device__ __forceinline__ void det_put(const DetDst& t, int e, float d, float x, float d_max)
{
    if (!(fabsf(d) < d_max)) {
        __stcg(t.x + e, __int_as_float(0x7fc00000));
        return;
    }
    const long long q = __double2ll_rn((double)d * DET_SCALE);
    if (!q) return;
    if (t.a) atomicAdd(t.a + e, (unsigned long long)q);
    else __stcg(t.x + e, det_fadd(x, (float)((double)q * (1.0 / DET_SCALE))));
}

// the slot's sum q of one element added to the factor's value v, the slot left at zero
__device__ __forceinline__ void det_apply(unsigned long long* a, float* x, long long q, float v)
{
    if (!q) return;
    __stcg(a, 0ull);
    __stcg(x, det_fadd(v, (float)((double)q * (1.0 / DET_SCALE))));
}

// Programmatic dependent launch: the per-round launches of an epoch may start while the launch before them still runs.
// Every CTA calls this before its first access to state an earlier launch writes: it waits until the launch before has
// completed and its writes are visible, and only then lets the next launch start.  So when launch N + 1 starts, every
// CTA of launch N has passed its wait, and launch N - 1 has completed.  (Without a programmatic dependency the wait
// returns at once.)
__device__ __forceinline__ void det_pdl_sync()
{
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// Plan of sample s0 + t (t < n) into nx, its shared rows taking slots from *n_shared; returns 1 when the sample is
// skipped.  Every lane of the warp calls it: the draw and the two gathers read only inputs and run before det_pdl_sync,
// so they overlap the launch before; the touch counters, slots and records of nx come after it.
__device__ __forceinline__ unsigned det_plan(const BprParams& p, const DetPlan& nx, unsigned int* n_shared, int64_t t,
                                             int64_t s0, int64_t n)
{
    int2 pr = make_int2(0, 0);
    int32_t j = 0;
    bool skip = false;
    if (t < n) {
        int64_t ii;
        draw_sample(p, s0 + t, ii, j);
        pr = __ldg(p.pairs + ii);
        const uint64_t key = pair_key(pr.x, j);
        skip = bucket_has(p.table, p.bucket_mask, key, mix64(key) & p.bucket_mask);      // recom_bpr.pyx:241-243
    }
    det_pdl_sync();
    unsigned cu = 0, ci = 0, cj = 0;
    if (t < n) {
        __stcg(nx.rec + t, make_int4(pr.x, pr.y, j, !skip));
        if (!skip) {
            // the three counts (independent round trips); the touch that takes a count from 1 to 2 makes the row shared
            cu = atomicAdd(nx.cnt_u + pr.x, 1u);
            ci = atomicAdd(nx.cnt_v + pr.y, 1u);
            cj = atomicAdd(nx.cnt_v + j, 1u);
        }
    }
    // the warp takes the slots of all its shared rows (0-3 per lane) with one atomic: lane l's first slot is the base plus
    // the rows of lanes < l, counted from the two bits of each lane's number
    const bool su = cu == 1u, si = ci == 1u, sj = cj == 1u;
    const unsigned m = (unsigned)su + (unsigned)si + (unsigned)sj;
    const unsigned b0 = __ballot_sync(0xffffffffu, m & 1u), b1 = __ballot_sync(0xffffffffu, m & 2u);
    if (b0 | b1) {
        const int lane = threadIdx.x & 31;
        unsigned base = 0;
        if (lane == 0) base = atomicAdd(n_shared, (unsigned)__popc(b0) + 2u * (unsigned)__popc(b1));
        const unsigned below = (1u << lane) - 1u;
        unsigned s = __shfl_sync(0xffffffffu, base, 0) + (unsigned)__popc(b0 & below) + 2u * (unsigned)__popc(b1 & below);
        if (su) { nx.slot_u[pr.x] = s; nx.row_of_slot[s++] = (unsigned)pr.x; }
        if (si) { nx.slot_v[pr.y] = s; nx.row_of_slot[s++] = (unsigned)pr.y | DET_ITEM; }
        if (sj) { nx.slot_v[j] = s; nx.row_of_slot[s] = (unsigned)j | DET_ITEM; }
    }
    return skip ? 1u : 0u;
}

// the row's destination in the grad kernel
__device__ __forceinline__ DetDst det_dst(float* x, const unsigned int* cnt, const unsigned int* slot, int32_t row,
                                          unsigned long long* acc, int k)
{
    DetDst t{x, nullptr};
    // the slot is read beside the count, not after it: one round trip (a row touched once has a stale or unset slot,
    // which is not used)
    const unsigned c = __ldcg(cnt + row), s = __ldcg(slot + row);
    if (c >= 2u) t.a = acc + (size_t)s * (size_t)(k + 1);
    return t;
}

// Block epilogue of the deterministic kernels: (correct, skipped) added to the epoch statistics, only when non-zero
__device__ __forceinline__ void det_flush_stats(unsigned int correct, unsigned int skipped, unsigned long long* stats)
{
    __shared__ unsigned int sh_stats[2];
    if (threadIdx.x < 2) sh_stats[threadIdx.x] = 0;
    __syncthreads();
    correct = __reduce_add_sync(0xffffffffu, correct);
    skipped = __reduce_add_sync(0xffffffffu, skipped);
    if ((threadIdx.x & 31) == 0 && (correct | skipped)) {
        atomicAdd(&sh_stats[0], correct);
        atomicAdd(&sh_stats[1], skipped);
    }
    __syncthreads();
    if (threadIdx.x == 0 && (sh_stats[0] | sh_stats[1])) {
        atomicAdd(stats + 0, (unsigned long long)sh_stats[0]);
        atomicAdd(stats + 1, (unsigned long long)sh_stats[1]);
    }
}

// Grad of round r (parity par, n records) and plan of round r + 1 (next_n samples from epoch-local next_s0 into parity
// par ^ 1).  The first ceil(next_n / 256) CTAs plan, one sample per thread.  CTAs are expected (not guaranteed) to be
// dispatched in blockIdx order, so the plan's chains of dependent gathers and atomics overlap the grad CTAs; the result
// does not depend on it.  The other CTAs run one warp per record: score, z, and the three row updates.  Lane l owns the elements l, l + 32, ...; the first DET_RC of them stay in registers between the dot and the
// update.
constexpr int DET_RC = 4;

__global__ void __launch_bounds__(256, 4) bpr_det_grad_kernel(const BprParams p, const DetState d, int64_t r, int par,
                                                              int64_t n, int64_t next_s0, int64_t next_n)
{
    const int lane = threadIdx.x & 31;
    const unsigned plan_ctas = (unsigned)((next_n + 255) / 256);
    if (blockIdx.x < plan_ctas) {
        const DetPlan nx = par ? d.plan[0] : d.plan[1];
        const unsigned skipped = det_plan(p, nx, d.n_shared + (r + 1), (int64_t)blockIdx.x * blockDim.x + threadIdx.x,
                                          next_s0, next_n);
        det_flush_stats(0u, skipped, p.stats);
        return;
    }
    det_pdl_sync();
    const int64_t w = ((int64_t)(blockIdx.x - plan_ctas) * blockDim.x + threadIdx.x) / 32;
    const DetPlan pl = par ? d.plan[1] : d.plan[0];
    unsigned int n_correct = 0;
    if (w < n) {
        const int4 rec = __ldcg(pl.rec + w);
        if (rec.w) {
            const int32_t u = rec.x, i = rec.y, j = rec.z;
            const int k = p.k;
            float* pu = p.U + (size_t)u * k;
            float* pi = p.V + (size_t)i * k;
            float* pj = p.V + (size_t)j * k;
            float ru[DET_RC], ri[DET_RC], rj[DET_RC];
#pragma unroll
            for (int x = 0; x < DET_RC; ++x) {
                const int e = lane + 32 * x;
                ru[x] = ri[x] = rj[x] = 0.f;
                if (e < k) { ru[x] = __ldcg(pu + e); ri[x] = __ldcg(pi + e); rj[x] = __ldcg(pj + e); }
            }
            const float bi = __ldcg(p.B + i), bj = __ldcg(p.B + j);
            const DetDst du = det_dst(pu, pl.cnt_u, pl.slot_u, u, d.acc, k);
            const DetDst di = det_dst(pi, pl.cnt_v, pl.slot_v, i, d.acc, k);
            const DetDst dj = det_dst(pj, pl.cnt_v, pl.slot_v, j, d.acc, k);
            float part = 0.f;
#pragma unroll
            for (int x = 0; x < DET_RC; ++x)
                if (lane + 32 * x < k) part = fmaf(ru[x], ri[x] - rj[x], part);
            for (int e = lane + 32 * DET_RC; e < k; e += 32) part = fmaf(__ldcg(pu + e), __ldcg(pi + e) - __ldcg(pj + e), part);
            const float score = (bi - bj) + group_sum<32>(part);
            float z;
            if (sample_z(p.hinge, p.exact_exp, score, z, n_correct)) {
                const float lr = p.lr, reg = p.reg;
                const float d_max = d.d_max;
                auto step = [&](int e, float uf, float vi, float vj) {
                    det_put(du, e, lr * (z * (vi - vj) - reg * uf), uf, d_max);
                    det_put(di, e, lr * (z * uf - reg * vi), vi, d_max);
                    det_put(dj, e, lr * (-z * uf - reg * vj), vj, d_max);
                };
#pragma unroll
                for (int x = 0; x < DET_RC; ++x)
                    if (lane + 32 * x < k) step(lane + 32 * x, ru[x], ri[x], rj[x]);
                for (int e = lane + 32 * DET_RC; e < k; e += 32) step(e, __ldcg(pu + e), __ldcg(pi + e), __ldcg(pj + e));
                if (p.use_bias && lane == 0) {
                    det_put(DetDst{p.B + i, di.a ? di.a + k : nullptr}, 0, lr * (z - reg * bi), bi, d_max);
                    det_put(DetDst{p.B + j, dj.a ? dj.a + k : nullptr}, 0, lr * (-z - reg * bj), bj, d_max);
                }
            }
            // a row touched once is reset by its only toucher, after every lane has read its count
            __syncwarp();
            if (lane == 0) {
                if (!du.a) pl.cnt_u[u] = 0u;
                if (!di.a) pl.cnt_v[i] = 0u;
                if (!dj.a) pl.cnt_v[j] = 0u;
            }
        }
    }
    det_flush_stats(lane == 0 ? n_correct : 0u, 0u, p.stats);      // one count per warp
}

// Apply of round r (parity par): warps grid-stride over the round's slots.  The epoch's prologue launch (r < 0) has
// nothing to apply and plans round 0 instead, one sample per thread (next_n samples from epoch-local 0 into parity 0).
__global__ void __launch_bounds__(256) bpr_det_apply_kernel(const BprParams p, const DetState d, int64_t r, int par,
                                                            int64_t next_n)
{
    const int lane = threadIdx.x & 31;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < 0) {
        det_flush_stats(0u, det_plan(p, d.plan[0], d.n_shared, t, 0, next_n), p.stats);
        return;
    }
    det_pdl_sync();
    const DetPlan pl = par ? d.plan[1] : d.plan[0];
    const int k = p.k;
    const unsigned n_warps = gridDim.x * (blockDim.x / 32);
    // the warp's first slot's row is read beside the round's slot count, before it is known to be one of the round's
    const unsigned s0 = (unsigned)(t / 32);
    unsigned tag = s0 < d.cap ? __ldcg(pl.row_of_slot + s0) : 0u;
    const unsigned n_sh = __ldcg(d.n_shared + r);
    for (unsigned s = s0; s < n_sh; s += n_warps) {
        if (s != s0) tag = __ldcg(pl.row_of_slot + s);
        const int32_t row = (int32_t)(tag & ~DET_ITEM);
        const bool item = tag & DET_ITEM;
        float* x = (item ? p.V : p.U) + (size_t)row * k;
        unsigned long long* a = d.acc + (size_t)s * (size_t)(k + 1);
        // the bias sum and value are read with the first elements
        const bool bias = lane == 0 && item && p.use_bias;
        long long qb = 0;
        float vb = 0.f;
        if (bias) { qb = (long long)__ldcg(a + k); vb = __ldcg(p.B + row); }
        for (int e0 = 0; e0 < k; e0 += 32 * DET_RC) {       // DET_RC elements per lane in flight at once
            long long q[DET_RC];
            float v[DET_RC];
#pragma unroll
            for (int c = 0; c < DET_RC; ++c) {
                const int e = e0 + lane + 32 * c;
                q[c] = 0;
                if (e < k) { q[c] = (long long)__ldcg(a + e); v[c] = __ldcg(x + e); }
            }
#pragma unroll
            for (int c = 0; c < DET_RC; ++c) {
                const int e = e0 + lane + 32 * c;
                if (e < k) det_apply(a + e, x + e, q[c], v[c]);
            }
        }
        if (bias) det_apply(a + k, p.B + row, qb, vb);
        if (lane == 0) (item ? pl.cnt_v : pl.cnt_u)[row] = 0u;
    }
}

static int bpr_epoch_deterministic(const BprParams& p, int64_t n_users, cudaStream_t st)
{
    const int64_t round = p.max_groups < DET_ROUND ? p.max_groups : DET_ROUND;
    const int64_t n_rounds = (p.n_samples + round - 1) / round;
    const int64_t cap = 3 * round / 2;                 // a shared row takes >= 2 of the round's <= 3 round touches
    const size_t n_rows = (size_t)n_users + (size_t)p.n_neg;
    // one stream-ordered buffer: records | accumulators, slot counts, touch counters (zeroed) | slots
    const size_t rec_b = 2 * (size_t)round * sizeof(int4);
    const size_t acc_b = (size_t)cap * (size_t)(p.k + 1) * sizeof(unsigned long long);
    const size_t zero_b = acc_b + (size_t)n_rounds * sizeof(unsigned int) + 2 * n_rows * sizeof(unsigned int);
    const size_t bytes = rec_b + zero_b + 2 * (n_rows + (size_t)cap) * sizeof(unsigned int);
    char* buf = nullptr;
    B200_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&buf), bytes, st));
    DetState d;
    d.d_max = det_delta_bound(round);
    d.cap = (unsigned)cap;
    d.acc = reinterpret_cast<unsigned long long*>(buf + rec_b);
    d.n_shared = reinterpret_cast<unsigned int*>(buf + rec_b + acc_b);
    unsigned int* cnt = d.n_shared + n_rounds;
    unsigned int* slot = cnt + 2 * n_rows;
    unsigned int* ros = slot + 2 * n_rows;
    for (int q = 0; q < 2; ++q) {
        DetPlan& pl = d.plan[q];
        pl.rec = reinterpret_cast<int4*>(buf) + q * round;
        pl.cnt_u = cnt + q * n_rows;
        pl.cnt_v = pl.cnt_u + n_users;
        pl.slot_u = slot + q * n_rows;
        pl.slot_v = pl.slot_u + n_users;
        pl.row_of_slot = ros + q * cap;
    }
    cudaError_t e = cudaMemsetAsync(buf + rec_b, 0, zero_b, st);      // every round leaves counters and slots at zero
    auto blocks = [](int64_t threads) { return (unsigned)((threads + 255) / 256); };
    // apply grid: one resident grid of warps for the shared rows, capped by the slots a round can have
    const unsigned apply_grid = (unsigned)std::min<int64_t>((int64_t)sm_count() * (2048 / 256), blocks(cap * 32));
    if (e == cudaSuccess) {
        bpr_det_apply_kernel<<<blocks(std::min(round, p.n_samples)), 256, 0, st>>>(p, d, -1, 0, std::min(round, p.n_samples));
        ::b200::count_launch();
        e = cudaGetLastError();
    }
    // the rounds' launches start while the launch before them runs (programmatic dependent launch, det_pdl_sync); the
    // prologue above and whatever follows the epoch on the stream stay fully stream-ordered
    cudaLaunchAttribute pdl;
    pdl.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    pdl.val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(256);
    cfg.stream = st;
    cfg.attrs = &pdl;
    cfg.numAttrs = 1;
    for (int64_t r = 0; r < n_rounds && e == cudaSuccess; ++r) {
        const int64_t s0 = r * round;
        const int64_t n = std::min(round, p.n_samples - s0);
        const int64_t next_n = r + 1 < n_rounds ? std::min(round, p.n_samples - s0 - round) : 0;
        const int par = (int)(r & 1);
        cfg.gridDim = dim3(blocks(next_n) + blocks(n * 32));
        e = cudaLaunchKernelEx(&cfg, bpr_det_grad_kernel, p, d, r, par, n, s0 + round, next_n);
        if (e != cudaSuccess) break;
        cfg.gridDim = dim3(apply_grid);
        e = cudaLaunchKernelEx(&cfg, bpr_det_apply_kernel, p, d, r, par, (int64_t)0);
        ::b200::count_launch(2);
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
    const char* mode = getenv("B200_REPLAY_SERIAL");          // dev knob: 1 = the strictly serial reference kernel
    ::b200::count_launch();
    if (mode && mode[0] == '1') { bpr_replay_kernel<<<1, 32, 0, st>>>(p); B200_CUDA(cudaGetLastError()); return B200_OK; }
    const size_t fixed = (sizeof(SchedShared) + 15) & ~(size_t)15;
    size_t model = 0;
    if (n_users > 0 && n_items > 0) model = ((size_t)(n_users + n_items) * p.k + (size_t)n_items) * sizeof(float);
    const size_t limit = 227 * 1024 - 1024;
    const bool on_chip = model > 0 && fixed + model <= limit;
    auto kern = on_chip ? bpr_replay_sched_kernel<true> : bpr_replay_sched_kernel<false>;
    const size_t smem = on_chip ? fixed + model : fixed;
    B200_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<1, 1024, smem, st>>>(p, on_chip ? n_users : 0, on_chip ? n_items : 0);
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
