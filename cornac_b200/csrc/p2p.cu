// Multi-GPU item-replica exchange over NVLink peer memory: make-delta + all-reduce + apply in ONE kernel.
//
// No reference counterpart (the reference is a single process, SURVEY.md 2.5).  After an epoch every rank's replica x_r of
// the item factors differs from the common epoch-start value s by that rank's local changes; the exchange sets every
// replica to   s + sum_r (x_r - s).   b200_delta_make -> NCCL all-reduce -> b200_delta_apply does that with three passes
// over local HBM around the collective.  Here the ranks map each other's replicas (CUDA IPC, one process per GPU) and
// every rank OWNS one contiguous slice of the vector: it reads that slice of every peer's replica straight over
// NVLink (ld.volatile: peer lines are cached in the local L1 only, B300_MICROARCH "NVLink"), adds the deltas to its
// snapshot of the slice in rank order (so the result is deterministic and bit-equal on all ranks), and stores the new
// values into EVERY replica -- reduce-scatter, apply and all-gather fused, each byte crossing NVLink once each way, no
// delta buffers, snapshots only of the owned slice (n / world floats).
// Cross-GPU ordering: a flag word per (phase, rank) in every rank's flag buffer, written by the peers with system-scope
// release stores and polled with system-scope acquire loads; waits are bounded (a missing peer sets an error word
// instead of hanging the GPU).
#include <cuda.h>

#include "common.cuh"

namespace b200 {
namespace p2p {

constexpr int MAX_WORLD = 8;
constexpr int THREADS = 256;

struct Peers {
    float* x[MAX_WORLD];            // replica of every rank (own pointer at [rank])
    unsigned int* flags[MAX_WORLD]; // flag buffer of every rank: [2 phases][MAX_WORLD], + [16] done counter, [17] error
};

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v)
{
    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p)
{
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 ld_volatile_f4(const float* p)
{
    float4 v;
    asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ float ld_volatile_f(const float* p)
{
    float v;
    asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

// wait until every rank has published `seq` in this rank's flag row `phase`; false on timeout (~4 s)
__device__ bool wait_all(const unsigned int* my_flags, int phase, int world, unsigned int seq)
{
    const long long t0 = clock64();
    for (int r = 0; r < world; ++r) {
        while ((int)(ld_acquire_sys(my_flags + phase * MAX_WORLD + r) - seq) < 0) {
            if (clock64() - t0 > 8000000000ll) return false;
            __nanosleep(200);
        }
    }
    return true;
}

// mean_touched: new = snap + (sum_r d_r) / #{r : d_r != 0}  (d_r = x_r - snap) instead of snap + sum_r d_r.  The plain sum is the
// single-process step count only while the ranks change DIFFERENT rows; a row every rank trains (a popular item) is moved
// `world` times too far and the epochs oscillate with growing amplitude from 4 ranks on (tools/sim_localsgd.py).  The mean over
// the ranks that changed an element is a convex combination of their local results: stable at any world size, and equal to the
// sum wherever one rank alone touched the element.
// peers_aligned: every replica pointer is 16-byte aligned (the host checks them; a view at a storage offset is not), else
// the whole slice takes the scalar loop.
__global__ void __launch_bounds__(THREADS) item_exchange_kernel(const Peers P, int rank, int world, float* __restrict__ snap,
                                                                int64_t n, int64_t lo, int64_t hi, unsigned int seq, int mean_touched,
                                                                int peers_aligned)
{
    unsigned int* my_flags = P.flags[rank];
    __shared__ int ok_s;
    // ---- phase 0: everybody's epoch is complete (their replicas are final) before anyone reads them
    if (threadIdx.x == 0) {
        if (blockIdx.x == 0) {
            __threadfence_system();
            for (int r = 0; r < world; ++r) st_release_sys(P.flags[r] + 0 * MAX_WORLD + rank, seq);
        }
        ok_s = wait_all(my_flags, 0, world, seq) ? 1 : 0;
        if (!ok_s) my_flags[17] = 1;
    }
    __syncthreads();
    if (ok_s) {
        // ---- owned slice [lo, hi): new = snap + sum_r (x_r - snap), stored into every replica and the snapshot
        const int64_t len = hi - lo;
        const bool vec = peers_aligned && ((lo & 3) == 0) && ((reinterpret_cast<uintptr_t>(snap) & 15) == 0);
        const int64_t n4 = vec ? len / 4 : 0;
        const int64_t stride = (int64_t)gridDim.x * THREADS;
        for (int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x; i < n4; i += stride) {
            const float4 s = *reinterpret_cast<const float4*>(snap + 4 * i);
            float4 acc = s;
            float4 v[MAX_WORLD];
#pragma unroll
            for (int r = 0; r < MAX_WORLD; ++r)
                if (r < world) v[r] = ld_volatile_f4(P.x[r] + lo + 4 * i);       // all peers' loads in flight together
            float4 d = make_float4(0.f, 0.f, 0.f, 0.f), c = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int r = 0; r < MAX_WORLD; ++r) {
                if (r < world) {
                    const float dx = v[r].x - s.x, dy = v[r].y - s.y, dz = v[r].z - s.z, dw = v[r].w - s.w;
                    d.x += dx; d.y += dy; d.z += dz; d.w += dw;
                    c.x += dx != 0.f ? 1.f : 0.f; c.y += dy != 0.f ? 1.f : 0.f; c.z += dz != 0.f ? 1.f : 0.f; c.w += dw != 0.f ? 1.f : 0.f;
                }
            }
            if (mean_touched) {
                if (c.x > 1.f) d.x /= c.x;
                if (c.y > 1.f) d.y /= c.y;
                if (c.z > 1.f) d.z /= c.z;
                if (c.w > 1.f) d.w /= c.w;
            }
            acc.x += d.x; acc.y += d.y; acc.z += d.z; acc.w += d.w;
#pragma unroll
            for (int r = 0; r < MAX_WORLD; ++r)
                if (r < world) *reinterpret_cast<float4*>(P.x[r] + lo + 4 * i) = acc;
            *reinterpret_cast<float4*>(snap + 4 * i) = acc;
        }
        for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * THREADS + threadIdx.x; i < len; i += stride) {
            const float s = snap[i];
            float d = 0.f, c = 0.f;
            for (int r = 0; r < world; ++r) {
                const float dx = ld_volatile_f(P.x[r] + lo + i) - s;
                d += dx;
                c += dx != 0.f ? 1.f : 0.f;
            }
            if (mean_touched && c > 1.f) d /= c;
            const float acc = s + d;
            for (int r = 0; r < world; ++r) P.x[r][lo + i] = acc;
            snap[i] = acc;
        }
    }
    // ---- phase 1: my stores into the peers are complete; leave only when theirs into my replica are
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int done = atomicAdd(my_flags + 16, 1u);
        if (done == gridDim.x - 1) {                    // the last block of this rank
            my_flags[16] = 0;
            __threadfence_system();
            for (int r = 0; r < world; ++r) st_release_sys(P.flags[r] + 1 * MAX_WORLD + rank, seq);
            if (!wait_all(my_flags, 1, world, seq)) my_flags[17] = 1;
        }
    }
    (void)n;
}

}  // namespace p2p
}  // namespace b200

using namespace b200;

// ---- CUDA IPC plumbing (host): export the allocation that contains a device pointer, open a peer's
extern "C" int b200_ipc_export(const void* dev_ptr, void* handle64_out, int64_t* offset_out)
{
    B200_REQUIRE(dev_ptr && handle64_out && offset_out, "b200_ipc_export: null argument");
    CUdeviceptr base = 0;
    size_t size = 0;
    // the driver entry point is resolved at run time: the library must load (and answer host-only calls) on machines
    // without libcuda.so.1
    typedef CUresult (*get_range_fn)(CUdeviceptr*, size_t*, CUdeviceptr);
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    B200_CUDA(cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &qres));
    B200_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, "b200_ipc_export: cuMemGetAddressRange is not available");
    const CUresult r = reinterpret_cast<get_range_fn>(fn)(&base, &size, (CUdeviceptr)dev_ptr);
    if (r != CUDA_SUCCESS) {
        set_error("b200_ipc_export: cuMemGetAddressRange failed (%d)", (int)r);
        return B200_ERR_CUDA;
    }
    cudaIpcMemHandle_t h;
    B200_CUDA(cudaIpcGetMemHandle(&h, (void*)base));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    memcpy(handle64_out, &h, 64);
    *offset_out = (int64_t)((CUdeviceptr)dev_ptr - base);
    return B200_OK;
}

extern "C" int b200_ipc_open(const void* handle64, int64_t offset, void** mapped_out)
{
    B200_REQUIRE(handle64 && mapped_out && offset >= 0, "b200_ipc_open: bad argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    void* base = nullptr;
    B200_CUDA(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    *mapped_out = static_cast<char*>(base) + offset;
    return B200_OK;
}

extern "C" int b200_ipc_close(void* mapped, int64_t offset)
{
    if (!mapped) return B200_OK;
    B200_CUDA(cudaIpcCloseMemHandle(static_cast<char*>(mapped) - offset));
    return B200_OK;
}

extern "C" int b200_item_exchange(int rank, int world, void* const* x_peers, void* const* flag_peers, float* snapshot_slice,
                                  int64_t n, uint32_t seq, int mean_touched, void* stream)
{
    B200_REQUIRE(world >= 1 && world <= p2p::MAX_WORLD && rank >= 0 && rank < world, "b200_item_exchange: rank %d / world %d", rank, world);
    B200_REQUIRE(x_peers && flag_peers && snapshot_slice && n >= 0 && seq != 0, "b200_item_exchange: bad argument");
    p2p::Peers P;
    int peers_aligned = 1;
    for (int r = 0; r < p2p::MAX_WORLD; ++r) {
        P.x[r] = r < world ? static_cast<float*>(x_peers[r]) : nullptr;
        P.flags[r] = r < world ? static_cast<unsigned int*>(flag_peers[r]) : nullptr;
        B200_REQUIRE(r >= world || (P.x[r] && P.flags[r]), "b200_item_exchange: missing peer pointer %d", r);
        if (r < world && (reinterpret_cast<uintptr_t>(P.x[r]) & 15) != 0) peers_aligned = 0;
    }
    // slices are cut at multiples of 4 floats so that every slice of an aligned replica keeps 16-byte alignment
    const int64_t per = ((n + world - 1) / world + 3) & ~(int64_t)3;
    int64_t lo = per * rank, hi = lo + per;
    if (lo > n) lo = n;
    if (hi > n) hi = n;
    int64_t blocks = ((hi - lo) / 4 + p2p::THREADS - 1) / p2p::THREADS;
    const int64_t cap = (int64_t)sm_count() * 4;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    p2p::item_exchange_kernel<<<(unsigned)blocks, p2p::THREADS, 0, (cudaStream_t)stream>>>(P, rank, world, snapshot_slice, n, lo, hi, seq,
                                                                                       mean_touched, peers_aligned);
    ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

// [lo, hi) of the slice rank `rank` owns (the host needs it to keep the snapshot)
extern "C" int b200_item_exchange_slice(int rank, int world, int64_t n, int64_t* lo_out, int64_t* hi_out)
{
    B200_REQUIRE(world >= 1 && rank >= 0 && rank < world && lo_out && hi_out && n >= 0, "b200_item_exchange_slice: bad argument");
    const int64_t per = ((n + world - 1) / world + 3) & ~(int64_t)3;
    int64_t lo = per * rank, hi = lo + per;
    if (lo > n) lo = n;
    if (hi > n) hi = n;
    *lo_out = lo; *hi_out = hi;
    return B200_OK;
}
