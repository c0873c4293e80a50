// Library plumbing: error text, device info, the CSC map of a sparse matrix, the multi-GPU delta kernels.
#include <stdarg.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <vector>

#include "common.cuh"

namespace b200 {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line)
{
    const char* base = strrchr(file, '/');
    set_error("CUDA error %d (%s) at %s:%d in `%s`", (int)e, cudaGetErrorString(e), base ? base + 1 : file, line, what);
    return B200_ERR_CUDA;
}

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count()
{
    static thread_local int cached_dev = -1, cached = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached = n;
        cached_dev = dev;
    }
    return cached;
}

__global__ void delta_make_kernel(const float4* __restrict__ x, const float4* __restrict__ snap, float4* __restrict__ delta,
                                  int64_t n4, const float* xs, const float* ss, float* ds, int64_t n)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 a = x[i], b = snap[i];
        delta[i] = make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
    }
    for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) ds[i] = xs[i] - ss[i];
}

__global__ void delta_apply_kernel(float4* __restrict__ x, float4* __restrict__ snap, const float4* __restrict__ delta,
                                   int64_t n4, float* xs, float* ss, const float* ds, int64_t n)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 b = snap[i], d = delta[i];
        const float4 r = make_float4(b.x + d.x, b.y + d.y, b.z + d.z, b.w + d.w);
        x[i] = r;
        snap[i] = r;
    }
    for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float r = ss[i] + ds[i];
        xs[i] = r;
        ss[i] = r;
    }
}

}  // namespace b200

using namespace b200;

extern "C" const char* b200_last_error(void) { return g_err; }
extern "C" int b200_abi_version(void) { return 3; }
extern "C" int64_t b200_kernel_launches(void) { return (int64_t)g_launches.load(std::memory_order_relaxed); }

extern "C" int b200_device_info(int* sms, int* cc_major, int* cc_minor)
{
    int dev = 0;
    B200_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    B200_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (sms) *sms = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return B200_OK;
}

extern "C" int b200_csc_map(const int32_t* indptr, const int32_t* indices, int64_t n_rows, int64_t n_cols, int64_t nnz,
                            int32_t* csc_ptr, int32_t* csc_pos)
{
    B200_REQUIRE(nnz >= 0 && nnz < (1ll << 31) && n_rows >= 0 && n_cols >= 0 && n_rows < (1ll << 31) &&
                     n_cols < (1ll << 31),
                 "b200_csc_map: bad sizes n_rows=%lld n_cols=%lld nnz=%lld", (long long)n_rows, (long long)n_cols,
                 (long long)nnz);
    B200_REQUIRE(indptr && csc_ptr && (nnz == 0 || (indices && csc_pos)), "b200_csc_map: null pointer argument");
    B200_REQUIRE(indptr[0] == 0 && indptr[n_rows] == nnz, "b200_csc_map: indptr spans [%d, %d], expected [0, %lld]",
                 indptr[0], indptr[n_rows], (long long)nnz);
    for (int64_t r = 0; r < n_rows; ++r)
        B200_REQUIRE(indptr[r] <= indptr[r + 1], "b200_csc_map: indptr decreases at row %lld", (long long)r);
    std::fill(csc_ptr, csc_ptr + n_cols + 1, 0);
    for (int64_t j = 0; j < nnz; ++j) {
        const int32_t c = indices[j];
        B200_REQUIRE(c >= 0 && c < n_cols, "b200_csc_map: entry %lld has column %d outside [0, %lld)", (long long)j, c,
                     (long long)n_cols);
        ++csc_ptr[c + 1];
    }
    for (int64_t c = 0; c < n_cols; ++c) csc_ptr[c + 1] += csc_ptr[c];
    std::vector<int32_t> next(csc_ptr, csc_ptr + n_cols);       // counting sort: stable, rows ascending in a column
    for (int64_t j = 0; j < nnz; ++j) csc_pos[next[indices[j]]++] = (int32_t)j;
    return B200_OK;
}

static inline bool aligned16(const void* a, const void* b, const void* c)
{
    return ((((uintptr_t)a) | ((uintptr_t)b) | ((uintptr_t)c)) & 15) == 0;
}

extern "C" int b200_delta_make(const float* x, const float* snapshot, float* delta, int64_t n, void* stream)
{
    B200_REQUIRE(x && snapshot && delta && n >= 0, "b200_delta_make: bad argument");
    if (n == 0) return B200_OK;
    const int64_t n4 = aligned16(x, snapshot, delta) ? n / 4 : 0;
    const int grid = sm_count() * 8;
    delta_make_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const float4*)x, (const float4*)snapshot, (float4*)delta, n4,
                                                              x, snapshot, delta, n); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_delta_apply(float* x, float* snapshot, const float* delta, int64_t n, void* stream)
{
    B200_REQUIRE(x && snapshot && delta && n >= 0, "b200_delta_apply: bad argument");
    if (n == 0) return B200_OK;
    const int64_t n4 = aligned16(x, snapshot, delta) ? n / 4 : 0;
    const int grid = sm_count() * 8;
    delta_apply_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((float4*)x, (float4*)snapshot, (const float4*)delta, n4,
                                                               x, snapshot, delta, n); ::b200::count_launch();
    B200_CUDA(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_bpr_draw_host2(uint64_t seed, uint64_t epoch, uint64_t sample_base, int64_t n,
                                   int64_t nnz, int64_t n_neg, uint32_t n_windows, uint32_t n_blocks,
                                   int64_t* out_i_index, int32_t* out_j_id)
{
    B200_REQUIRE(n >= 0 && nnz >= 1 && n_neg >= 1 && (n == 0 || (out_i_index && out_j_id)), "b200_bpr_draw_host: bad argument");
    const SampleLaw law = make_law(nnz, n_neg, n_windows, n_blocks, epoch);
    for (int64_t t = 0; t < n; ++t) {
        const uint64_t s = sample_base + (uint64_t)t;
        const Philox4 r = philox4x32_10((uint32_t)s, (uint32_t)(s >> 32), (uint32_t)epoch, (uint32_t)(epoch >> 32),
                                        (uint32_t)seed, (uint32_t)(seed >> 32));
        int64_t i_lo, i_len, j_lo, j_len;
        law_ranges(law, s, i_lo, i_len, j_lo, j_len);
        out_i_index[t] = i_lo + (int64_t)range64(r.x, r.y, (uint64_t)i_len);
        out_j_id[t] = (int32_t)(j_lo + (int64_t)range64(r.z, r.w, (uint64_t)j_len));
    }
    return B200_OK;
}

extern "C" int b200_bpr_draw_host(uint64_t seed, uint64_t epoch, uint64_t sample_base, int64_t n,
                                  int64_t nnz, int64_t n_neg, int64_t* out_i_index, int32_t* out_j_id)
{
    return b200_bpr_draw_host2(seed, epoch, sample_base, n, nnz, n_neg, 1, 1, out_i_index, out_j_id);
}
