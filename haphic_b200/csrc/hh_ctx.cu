// Context, error string, small utilities of libhaphic_b200.
#include "hh_common.cuh"

#include <mutex>
static thread_local char g_err[1024] = "";
static std::mutex g_ctx_mutex;
static std::vector<hh_ctx*> g_ctx_list;      // live contexts: a buffer may be released under another context's scope
thread_local hh_ctx* hh_tls_ctx = nullptr;

void hh_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" int hh_version(void) { return HH_VERSION; }
extern "C" const char* hh_last_error(void) { return g_err; }

extern "C" int hh_ctx_create(int device, hh_ctx** out) {
    HH_REQUIRE(out != nullptr, HH_ERR_ARG, "hh_ctx_create: out is NULL");
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        hh_set_error("hh_ctx_create: no CUDA device available (%s); this library has no CPU fallback",
                     e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
        cudaGetLastError();
        return HH_ERR_CUDA;
    }
    HH_REQUIRE(device >= 0 && device < count, HH_ERR_ARG, "hh_ctx_create: device %d out of range [0,%d)", device, count);
    HH_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    HH_CUDA(cudaGetDeviceProperties(&prop, device));
    HH_REQUIRE(prop.major == 9 && prop.minor == 0, HH_ERR_UNSUPPORTED,
               "hh_ctx_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only", device,
               prop.major, prop.minor);
    hh_ctx* c = new (std::nothrow) hh_ctx();
    HH_REQUIRE(c != nullptr, HH_ERR_NOMEM, "hh_ctx_create: out of host memory");
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    c->smem_optin = prop.sharedMemPerBlockOptin;
    c->l2_bytes = (size_t)prop.l2CacheSize;
    c->launches = 0;
    c->stream = nullptr;
    c->h_scratch = nullptr;
    c->d_scratch = nullptr;
    c->ws = new std::vector<hh_ctx::ws_block>();
    c->ws_tick = 0;
    HH_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    {   // keep freed device memory in the pool: a pass re-allocates the same multi-GB buffers
        cudaMemPool_t pool;
        HH_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
        unsigned long long keep = ~0ull;
        HH_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    }
    HH_CUDA(cudaMallocHost((void**)&c->h_scratch, 64 * sizeof(uint64_t)));
    HH_CUDA(cudaMalloc((void**)&c->d_scratch, 64 * sizeof(uint64_t)));
    {
        std::lock_guard<std::mutex> g(g_ctx_mutex);
        g_ctx_list.push_back(c);
    }
    *out = c;
    return HH_OK;
}

extern "C" int hh_ctx_destroy(hh_ctx* c) {
    if (!c) return HH_OK;
    {
        std::lock_guard<std::mutex> g(g_ctx_mutex);
        for (size_t k = 0; k < g_ctx_list.size(); ++k)
            if (g_ctx_list[k] == c) {
                g_ctx_list.erase(g_ctx_list.begin() + (long)k);
                break;
            }
    }
    cudaSetDevice(c->device);
    if (c->stream) {
        cudaStreamSynchronize(c->stream);
        cudaStreamDestroy(c->stream);
    }
    if (c->h_scratch) cudaFreeHost(c->h_scratch);
    if (c->d_scratch) cudaFree(c->d_scratch);
    if (c->ws) {
        for (size_t k = 0; k < c->ws->size(); ++k) cudaFree((*c->ws)[k].p);
        delete c->ws;
    }
    delete c;
    return HH_OK;
}

// best fit among the cached blocks that are not much larger than the request; otherwise a new block
void* hh_ws_alloc_bytes(hh_ctx* c, size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    int best = -1;
    for (size_t k = 0; k < c->ws->size(); ++k) {
        const hh_ctx::ws_block& b = (*c->ws)[k];
        if (b.used || b.bytes < bytes || b.bytes > 2 * bytes + (64u << 20)) continue;
        if (best < 0 || b.bytes < (*c->ws)[(size_t)best].bytes) best = (int)k;
    }
    if (best >= 0) {
        (*c->ws)[(size_t)best].used = true;
        return (*c->ws)[(size_t)best].p;
    }
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) {
        // out of memory: give the unused cached blocks back and try once more
        cudaGetLastError();
        cudaStreamSynchronize(c->stream);
        for (size_t k = 0; k < c->ws->size();) {
            if (!(*c->ws)[k].used) {
                cudaFree((*c->ws)[k].p);
                c->ws->erase(c->ws->begin() + (long)k);
            } else {
                ++k;
            }
        }
        e = cudaMalloc(&p, bytes);
    }
    if (e != cudaSuccess) {
        hh_set_error("workspace allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
        cudaGetLastError();
        return nullptr;
    }
    hh_ctx::ws_block nb;
    nb.p = p;
    nb.bytes = bytes;
    nb.used = true;
    nb.tick = 0;
    c->ws->push_back(nb);
    return p;
}

// give a block back to the cache; false if `p` is not a workspace block.  Unused blocks beyond HH_WS_KEEP bytes are freed,
// least recently used first, so that other allocators of the process (torch) keep finding memory.
static bool ws_mark_free(hh_ctx* c, void* p) {
    if (!c || !c->ws) return false;
    for (size_t k = 0; k < c->ws->size(); ++k)
        if ((*c->ws)[k].p == p) {
            (*c->ws)[k].used = false;
            (*c->ws)[k].tick = ++c->ws_tick;
            return true;
        }
    return false;
}

bool hh_ws_release(hh_ctx* c, void* p) {
    bool found = ws_mark_free(c, p);
    if (!found) {
        // released under another context's scope (or none): look through every live context
        std::lock_guard<std::mutex> g(g_ctx_mutex);
        for (size_t k = 0; k < g_ctx_list.size() && !found; ++k)
            if (g_ctx_list[k] != c && ws_mark_free(g_ctx_list[k], p)) {
                found = true;
                c = g_ctx_list[k];
            }
    }
    if (!found) return false;
    const size_t keep = (size_t)72 << 30;
    for (;;) {
        size_t idle = 0;
        int oldest = -1;
        for (size_t k = 0; k < c->ws->size(); ++k) {
            const hh_ctx::ws_block& b = (*c->ws)[k];
            if (b.used) continue;
            idle += b.bytes;
            if (oldest < 0 || b.tick < (*c->ws)[(size_t)oldest].tick) oldest = (int)k;
        }
        if (idle <= keep || oldest < 0) break;
        cudaStreamSynchronize(c->stream);
        cudaFree((*c->ws)[(size_t)oldest].p);
        c->ws->erase(c->ws->begin() + oldest);
    }
    return true;
}

void hh_ws_free_ptr(hh_ctx* c, void* p) { hh_ws_release(c, p); }

// What the next large allocations can get: the small-allocation pool hands its unused memory back first (cudaMalloc of a
// workspace block does not draw on it), and the idle workspace blocks count as free because a failed allocation releases them.
extern "C" int hh_ctx_mem_available(hh_ctx* c, size_t* bytes) {
    HH_REQUIRE(c && bytes, HH_ERR_ARG, "hh_ctx_mem_available: NULL argument");
    HH_CUDA(cudaSetDevice(c->device));
    HH_CUDA(cudaStreamSynchronize(c->stream));
    cudaMemPool_t pool;
    HH_CUDA(cudaDeviceGetDefaultMemPool(&pool, c->device));
    HH_CUDA(cudaMemPoolTrimTo(pool, 0));
    size_t free_b = 0, total_b = 0;
    HH_CUDA(cudaMemGetInfo(&free_b, &total_b));
    for (size_t k = 0; k < c->ws->size(); ++k)
        if (!(*c->ws)[k].used) free_b += (*c->ws)[k].bytes;
    *bytes = free_b;
    return HH_OK;
}

extern "C" int hh_ctx_sync(hh_ctx* c) {
    HH_REQUIRE(c != nullptr, HH_ERR_ARG, "hh_ctx_sync: ctx is NULL");
    HH_CUDA(cudaSetDevice(c->device));
    HH_CUDA(cudaStreamSynchronize(c->stream));
    return HH_OK;
}

extern "C" void* hh_ctx_stream(hh_ctx* c) { return c ? (void*)c->stream : nullptr; }
extern "C" int hh_ctx_device(hh_ctx* c) { return c ? c->device : -1; }
extern "C" int hh_ctx_sm_count(hh_ctx* c) { return c ? c->sm_count : 0; }
extern "C" int64_t hh_ctx_launches(hh_ctx* c) { return c ? c->launches : 0; }

// ---------------------------------------------------------------------------------------------
// single-CTA exclusive scan (1024 threads, tiles of 1024 with a running carry)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) hh_k_scan_small(const int* __restrict__ in, int64_t* __restrict__ out, int n) {
    __shared__ int64_t warp_tot[32];
    __shared__ int64_t carry_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        int i = base + threadIdx.x;
        int64_t v = (i < n) ? (int64_t)in[i] : 0;
        int64_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int64_t t = __shfl_up_sync(HH_FULL_MASK, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int64_t w = warp_tot[lane];
            int64_t wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int64_t t = __shfl_up_sync(HH_FULL_MASK, wi, o);
                if (lane >= o) wi += t;
            }
            warp_tot[lane] = wi - w;   // exclusive prefix of warp totals
        }
        __syncthreads();
        int64_t carry = carry_s;
        int64_t excl = carry + warp_tot[warp] + incl - v;
        if (i < n) out[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) out[n] = carry_s;
}

int hh_exclusive_scan_i32(hh_ctx* ctx, const int* d_in, int64_t* d_out, int n) {
    HH_LAUNCH(ctx, hh_k_scan_small, 1, 1024, 0, d_in, d_out, n);
    return HH_OK;
}
