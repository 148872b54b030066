// Shared host/device helpers of libhaphic_b200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>
#include <new>
#include <vector>

#include "../../include/haphic_b200.h"

// ---------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------
void hh_set_error(const char* fmt, ...);

#define HH_CUDA(expr)                                                                         \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            hh_set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return (_e == cudaErrorMemoryAllocation) ? HH_ERR_NOMEM : HH_ERR_CUDA;            \
        }                                                                                     \
    } while (0)

#define HH_CHECK(expr)                                                                        \
    do {                                                                                      \
        int _rc = (expr);                                                                     \
        if (_rc != HH_OK) return _rc;                                                         \
    } while (0)

#define HH_REQUIRE(cond, code, ...)                                                           \
    do {                                                                                      \
        if (!(cond)) {                                                                        \
            hh_set_error(__VA_ARGS__);                                                        \
            return (code);                                                                    \
        }                                                                                     \
    } while (0)

// launch + count + check
#define HH_LAUNCH(ctx, kernel, grid, block, smem, ...)                                        \
    do {                                                                                      \
        kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);                      \
        (ctx)->launches++;                                                                    \
        HH_CUDA(cudaGetLastError());                                                          \
    } while (0)

struct hh_ctx {
    int device;
    int sm_count;
    size_t smem_optin;      // max dynamic shared memory per block
    size_t l2_bytes;
    cudaStream_t stream;
    int64_t launches;
    // small pinned scratch for flag / counter read-back
    uint64_t* h_scratch;    // pinned, 64 x u64
    uint64_t* d_scratch;    // device, 64 x u64
    // workspace cache: the multi-GB transients of a pass (partition regions, operand planes of the tensor-core GEMM)
    // come from blocks that stay with the context and are handed out best-fit, so every pass finds the blocks of the
    // previous one instead of re-shaping the stream-ordered pool (all use is ordered on `stream`)
    struct ws_block {
        void* p;
        size_t bytes;
        bool used;
        uint64_t tick;      // last release (least recently used blocks go first when the cache is trimmed)
    };
    std::vector<ws_block>* ws;
    uint64_t ws_tick;
};

void* hh_ws_alloc_bytes(hh_ctx* ctx, size_t bytes);
bool hh_ws_release(hh_ctx* ctx, void* p);
void hh_ws_free_ptr(hh_ctx* ctx, void* p);
template <typename T>
static inline int hh_ws_alloc(hh_ctx* ctx, T** p, size_t count) {
    *p = reinterpret_cast<T*>(hh_ws_alloc_bytes(ctx, (count ? count : 1) * sizeof(T)));
    return *p ? HH_OK : HH_ERR_NOMEM;
}
template <typename T>
static inline void hh_ws_free(hh_ctx* ctx, T*& p) {
    if (p) hh_ws_free_ptr(ctx, (void*)p);
    p = nullptr;
}

// Every ABI entry point opens an hh_scope: device selected, and device buffers come from the
// stream-ordered memory pool of the context's stream (cudaMallocAsync / cudaFreeAsync; the pool keeps
// freed blocks, so the multi-GB tables of one pass are reused by the next without cudaMalloc cost).
extern thread_local hh_ctx* hh_tls_ctx;
struct hh_scope {
    hh_ctx* prev;
    explicit hh_scope(hh_ctx* c) : prev(hh_tls_ctx) {
        hh_tls_ctx = c;
        if (c) cudaSetDevice(c->device);
    }
    ~hh_scope() { hh_tls_ctx = prev; }
};

// Large buffers (>= HH_WS_MIN bytes) come from the context's workspace cache (best fit, blocks stay with the context):
// the stream-ordered pool re-shapes itself when the sequence of multi-GB requests changes from pass to pass, which cost
// up to a second per step; small ones from the pool.
#define HH_WS_MIN ((size_t)32 << 20)
template <typename T>
static inline int hh_dmalloc(T** p, size_t count) {
    *p = nullptr;
    if (count == 0) count = 1;
    if (hh_tls_ctx && count * sizeof(T) >= HH_WS_MIN) {
        *p = reinterpret_cast<T*>(hh_ws_alloc_bytes(hh_tls_ctx, count * sizeof(T)));
        return *p ? HH_OK : HH_ERR_NOMEM;
    }
    cudaError_t e = hh_tls_ctx ? cudaMallocAsync((void**)p, count * sizeof(T), hh_tls_ctx->stream)
                               : cudaMalloc((void**)p, count * sizeof(T));
    if (e != cudaSuccess) {
        hh_set_error("cudaMalloc of %zu bytes failed: %s", count * sizeof(T), cudaGetErrorString(e));
        cudaGetLastError();
        return HH_ERR_NOMEM;
    }
    return HH_OK;
}
template <typename T>
static inline void hh_dfree(T*& p) {
    if (p) {
        if (hh_ws_release(hh_tls_ctx, (void*)p)) {       // also looks through the other contexts of the process
        } else if (hh_tls_ctx) {
            cudaFreeAsync((void*)p, hh_tls_ctx->stream);
        } else {
            cudaFree((void*)p);
        }
    }
    p = nullptr;
}

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
#define HH_FULL_MASK 0xffffffffu

__device__ __forceinline__ int hh_lane() { return threadIdx.x & 31; }
__device__ __forceinline__ int hh_warp() { return threadIdx.x >> 5; }

__device__ __forceinline__ double hh_warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(HH_FULL_MASK, v, o);
    return v;
}
__device__ __forceinline__ int hh_warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(HH_FULL_MASK, v, o);
    return v;
}
__device__ __forceinline__ unsigned long long hh_warp_sum(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(HH_FULL_MASK, v, o);
    return v;
}
// inclusive prefix sum over the lanes of a warp: lane i gets v(0) + ... + v(i)
template <typename T>
__device__ __forceinline__ T hh_warp_incl_scan(T v) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T t = __shfl_up_sync(HH_FULL_MASK, v, o);
        if (hh_lane() >= o) v += t;
    }
    return v;
}
__device__ __forceinline__ float hh_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(HH_FULL_MASK, v, o));
    return v;
}

// streaming 128-bit load that does not pollute L1 (records are read exactly once)
__device__ __forceinline__ int4 hh_ld_stream(const int4* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ unsigned long long hh_ld_stream_u64(const unsigned long long* p) {
    unsigned long long r;
    asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ float4 hh_ld_stream_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

// Exclusive prefix, in place, of the n <= 8 x 512 counts c[] of a tile, by its 512 threads; returns their sum.  s_wtot is
// shared scratch of 16 words.  Barriers on entry (c[] is complete) and on exit (the prefix is visible).
__device__ __forceinline__ unsigned int hh_tile_scan(unsigned int* c, int n, unsigned int* s_wtot) {
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const int per = (n + 511) >> 9, lo = threadIdx.x * per;
    __syncthreads();
    unsigned int sum = 0;
    for (int k = 0; k < per; ++k)
        if (lo + k < n) sum += c[lo + k];
    unsigned int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned int t = __shfl_up_sync(HH_FULL_MASK, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_wtot[wv] = incl;
    __syncthreads();
    unsigned int run = incl - sum, all = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        const unsigned int t = s_wtot[k];
        run += (k < wv) ? t : 0u;
        all += t;
    }
    for (int k = 0; k < per; ++k) {
        if (lo + k < n) {
            const unsigned int t = c[lo + k];
            c[lo + k] = run;
            run += t;
        }
    }
    __syncthreads();
    return all;
}

// CTAs of `kernel` (at `threads` threads and `smem` bytes of dynamic shared memory) that the GPU holds at once: the grid of
// a persistent kernel whose CTAs each loop over a fixed share of the work, so that none waits for another to exit
template <typename K>
static inline int hh_resident_grid(hh_ctx* ctx, K kernel, int threads, size_t smem, int* grid) {
    int per_sm = 0;
    HH_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
    HH_REQUIRE(per_sm > 0, HH_ERR_CUDA, "a kernel of %d threads and %zu bytes of shared memory does not fit an SM", threads, smem);
    *grid = ctx->sm_count * per_sm;
    return HH_OK;
}

// single-CTA exclusive scan of n ints (n up to a few million): out[i] = sum_{k<i} in[k], out[n] = total
__global__ void hh_k_scan_small(const int* __restrict__ in, int64_t* __restrict__ out, int n);
// multi-block stream compaction support
int hh_exclusive_scan_i32(hh_ctx* ctx, const int* d_in, int64_t* d_out, int n);
