// dict_to_matrix (scripts/HapHiC_cluster.py:310-373) on the GPU: from the compact link table to a
// symmetric fp32 CSC with self loops, in the reference's first-seen index order.  With a haplotype array the
// inter-haplotype entries are reduced first (reduce_inter_hap_HiC_links, 695-707; hh_flank_value).
#include "hh_common.cuh"
#include "hh_internal.cuh"
#include <algorithm>

__global__ void hh_k_set_tail(const int32_t* __restrict__ tail, int n_tail, int n_linked, const uint8_t* __restrict__ keep,
                              int32_t* __restrict__ index, int n_ctg, int* __restrict__ err) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tail) return;
    const int c = tail[t];
    if (c < 0 || c >= n_ctg || !keep[c] || index[c] >= 0) {
        atomicExch(err, 1);
        return;
    }
    index[c] = n_linked + t;
}

// every kept fragment must have an index by now, every dropped one must not
__global__ void hh_k_check_index(const int32_t* __restrict__ index, const uint8_t* __restrict__ keep, int n_ctg, int n,
                                 int* __restrict__ err) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_ctg) return;
    const int ix = index[c];
    if (keep[c] ? (ix < 0 || ix >= n) : (ix >= 0)) atomicExch(err, 2);
}

__global__ void hh_k_fill_i32(int* __restrict__ p, int v, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// column counts from the degrees the index pass accumulated: a linked fragment's column holds its entries and the self
// loop; the tail columns keep the self loop the fill gave them
__global__ void hh_k_mat_colcnt(const int32_t* __restrict__ index, const int32_t* __restrict__ deg, int n_ctg, int self_loop,
                                int* __restrict__ colcnt) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_ctg) return;
    const int ix = index[c];
    if (ix >= 0) colcnt[ix] = deg[c] + self_loop;
}

// Each self loop takes slot 0 of its column (362-364); the cursors start at 1, so no atomic is needed here
__global__ void hh_k_mat_self_loops(int n, const int64_t* __restrict__ colptr, int32_t* __restrict__ row, float* __restrict__ val) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    const int64_t q = colptr[c];
    row[q] = c;
    val[q] = 1.0f;
}

// ---------------------------------------------------------------------------------------------
// Placement of the passing entries, in two passes through a staging list laid out like the CSC.  The matrix columns are
// cut into groups of C = 2^cbits consecutive columns (hh_mat_cbits: at most 4096 groups).  A staged half-entry is 8 bytes,
// {row << cbits | column - g·C, fp32 value}, and group g's staging run is the part of its CSC extent that the self loops
// leave, [colptr[g·C] + sl·(columns of g), colptr[(g+1)·C]).
//   hh_k_mat_group   tiles of compact entries: both halves of every passing entry, counted per group in shared memory,
//                    one global reservation per (tile, group), stored run by run from a staged copy of the tile
//   hh_k_mat_chunks  one CTA: the groups' staging cursors and the list of chunks (at most HH_MAT_CHUNK staged records,
//                    inside one group)
//   hh_k_mat_place   persistent CTAs, one chunk at a time: a counting sort of the chunk over its group's columns in
//                    shared memory, one cursor atomic per (chunk, column), rows and values stored in column runs
// Few groups keep the staging runs long; chunks of 8192 records keep the placement's write front at one group's columns.
// ---------------------------------------------------------------------------------------------
#define HH_MAT_TILE 4096           // compact entries per tile of hh_k_mat_group (512 threads x 8): 2 x 4096 half-entries
#define HH_MAT_CHUNK 8192          // staged records per chunk of hh_k_mat_place (512 threads x 16)
#define HH_MAT_MAX_N (1 << 22)     // bits(n) + cbits <= 32: the staged word holds the row and the column in the group

struct hh_mat_chunk {
    long long start;               // first staged record
    int len;                       // records, 1 .. HH_MAT_CHUNK
    int group;
};

// columns per group: C = 2^cbits with cbits = max(8, bits(n) - 12), so at most 4096 groups
static int hh_mat_cbits(int n) {
    int bits = 0;
    while (((int64_t)1 << bits) < n) ++bits;
    return std::max(8, bits - 12);
}

// shared memory of hh_k_mat_group: the staged tile, the group of every staged record, then per group its reservation
// and count
static size_t hh_mat_group_smem(int ngroups) {
    return (size_t)2 * HH_MAT_TILE * (sizeof(uint2) + sizeof(uint16_t)) + (size_t)ngroups * (sizeof(unsigned long long) + sizeof(unsigned int));
}

__global__ void __launch_bounds__(512, 2)
hh_k_mat_group(const uint32_t* __restrict__ compact, int64_t nnz, const int32_t* __restrict__ index,
               const unsigned long long* __restrict__ ctg_tot, int normalize, const int32_t* __restrict__ hap, double w,
               const int32_t* __restrict__ ul_path, const int32_t* __restrict__ ul_parent, int cbits, int ngroups,
               unsigned long long* __restrict__ gcur, uint2* __restrict__ stage) {
    constexpr int ITEMS = HH_MAT_TILE / 512;
    extern __shared__ uint2 s_mat_mem[];
    uint2* s_stage = s_mat_mem;                                               // the tile's half-entries, ordered by group
    uint16_t* s_grp = reinterpret_cast<uint16_t*>(s_stage + 2 * HH_MAT_TILE);  // the group of each staged one
    unsigned long long* s_base = reinterpret_cast<unsigned long long*>(s_grp + 2 * HH_MAT_TILE);
    unsigned int* s_cnt = reinterpret_cast<unsigned int*>(s_base + ngroups);  // half-entries per group, then their prefix
    __shared__ unsigned int s_wtot[16];
    const uint32_t cmask = (1u << cbits) - 1u;
    const int64_t tiles = (nnz + HH_MAT_TILE - 1) / HH_MAT_TILE;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        for (int k = threadIdx.x; k < ngroups; k += 512) s_cnt[k] = 0;
        __syncthreads();
        // The words of the tile's entries are loaded together, then the matrix indices of their ends; ii[k] = -1 marks an
        // entry that does not pass.  Shared cursors over the scanned counts give the staged places, so no rank is held.
        int ii[ITEMS], jj[ITEMS];
        float v[ITEMS];
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            const int64_t e = t * HH_MAT_TILE + (int64_t)k * 512 + threadIdx.x;
            ii[k] = -1;
            if (e < nnz) {
                const uint32_t* p = compact + e * HH_E_WORDS;
                const uint32_t fl = p[HH_E_FLANK], ci = p[HH_E_I], cj = p[HH_E_J];
                if (fl) {
                    ii[k] = (int)ci;
                    jj[k] = (int)cj;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            if (ii[k] < 0) continue;
            ii[k] = index[ii[k]];
            jj[k] = index[jj[k]];
        }
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            if (ii[k] < 0 || jj[k] < 0) {                // 329-330
                ii[k] = -1;
                continue;
            }
            double x;
            if (!hh_flank_value(compact + (t * HH_MAT_TILE + (int64_t)k * 512 + threadIdx.x) * HH_E_WORDS, ctg_tot, normalize, hap,
                                w, ul_path, ul_parent, &x)) {
                ii[k] = -1;
                continue;
            }
            v[k] = (float)x;                             // coo_matrix(dtype=float32) (368)
            // (row ii, column jj) and its diagonal mirror (351-353)
            atomicAdd(&s_cnt[jj[k] >> cbits], 1u);
            atomicAdd(&s_cnt[ii[k] >> cbits], 1u);
        }
        __syncthreads();
        for (int k = threadIdx.x; k < ngroups; k += 512)
            if (s_cnt[k]) s_base[k] = atomicAdd(gcur + k, (unsigned long long)s_cnt[k]);
        const unsigned int n_tile = hh_tile_scan(s_cnt, ngroups, s_wtot);
        // staged record e of group g goes to s_base[g] + e; s_cnt becomes the staging cursors
        for (int k = threadIdx.x; k < ngroups; k += 512) s_base[k] -= s_cnt[k];
        __syncthreads();
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            if (ii[k] < 0) continue;
            const uint32_t a = (uint32_t)ii[k], b = (uint32_t)jj[k];
            const unsigned int qa = atomicAdd(&s_cnt[b >> cbits], 1u);
            s_stage[qa] = make_uint2(a << cbits | (b & cmask), __float_as_uint(v[k]));
            s_grp[qa] = (uint16_t)(b >> cbits);
            const unsigned int qb = atomicAdd(&s_cnt[a >> cbits], 1u);
            s_stage[qb] = make_uint2(b << cbits | (a & cmask), __float_as_uint(v[k]));
            s_grp[qb] = (uint16_t)(a >> cbits);
        }
        __syncthreads();
        for (unsigned int e = threadIdx.x; e < n_tile; e += 512) stage[s_base[s_grp[e]] + e] = s_stage[e];
        __syncthreads();
    }
}

// One CTA of 512 threads: gcur[g] = the start of group g's staging run, and the chunk list (*n_chunks chunks, those of
// one group consecutive)
__global__ void __launch_bounds__(512)
hh_k_mat_chunks(const int64_t* __restrict__ colptr, int n, int cbits, int ngroups, int sl, unsigned long long* __restrict__ gcur,
                hh_mat_chunk* __restrict__ chunk, unsigned int* __restrict__ n_chunks) {
    __shared__ unsigned int s_off[4096];                // chunks per group, then their exclusive prefix
    __shared__ unsigned int s_wtot[16];
    for (int g = threadIdx.x; g < ngroups; g += 512) {
        const int lo = g << cbits, hi = min(n, lo + (1 << cbits));
        const int64_t s = colptr[lo] + (int64_t)sl * (hi - lo);
        gcur[g] = (unsigned long long)s;
        s_off[g] = (unsigned int)((colptr[hi] - s + HH_MAT_CHUNK - 1) / HH_MAT_CHUNK);
    }
    const unsigned int total = hh_tile_scan(s_off, ngroups, s_wtot);
    for (unsigned int c = threadIdx.x; c < total; c += 512) {
        int g = 0;                                      // the last group whose chunks start at or before c
        for (int step = 2048; step > 0; step >>= 1)
            if (g + step < ngroups && s_off[g + step] <= c) g += step;
        const int lo = g << cbits, hi = min(n, lo + (1 << cbits));
        const int64_t s = colptr[lo] + (int64_t)sl * (hi - lo) + (int64_t)(c - s_off[g]) * HH_MAT_CHUNK;
        chunk[c] = hh_mat_chunk{s, (int)min((int64_t)HH_MAT_CHUNK, colptr[hi] - s), g};
    }
    if (threadIdx.x == 0) *n_chunks = total;
}

__global__ void __launch_bounds__(512, 2)
hh_k_mat_place(const uint2* __restrict__ stage, const hh_mat_chunk* __restrict__ chunk, const unsigned int* __restrict__ n_chunks,
               int cbits, const int64_t* __restrict__ colptr, int* __restrict__ cursor, int32_t* __restrict__ row,
               float* __restrict__ val) {
    constexpr int ITEMS = HH_MAT_CHUNK / 512;
    extern __shared__ uint2 s_mat_mem[];
    uint2* s_rec = s_mat_mem;                           // the chunk, ordered by column
    __shared__ unsigned int s_cnt[1024];                // records per column, their prefix, then the placement cursors
    __shared__ long long s_base[1024];                  // CSC position of the column's run, minus its first staged slot
    __shared__ unsigned int s_wtot[16];
    const int ncol = 1 << cbits;
    const uint32_t cmask = (uint32_t)ncol - 1u;
    const unsigned int total = *n_chunks;
    for (unsigned int c = blockIdx.x; c < total; c += gridDim.x) {
        const hh_mat_chunk ch = chunk[c];
        for (int k = threadIdx.x; k < ncol; k += 512) s_cnt[k] = 0;
        __syncthreads();
        uint2 r[ITEMS];
#pragma unroll
        for (int k = 0; k < ITEMS; ++k)
            if (k * 512 + (int)threadIdx.x < ch.len) r[k] = stage[ch.start + k * 512 + threadIdx.x];
#pragma unroll
        for (int k = 0; k < ITEMS; ++k)
            if (k * 512 + (int)threadIdx.x < ch.len) atomicAdd(&s_cnt[r[k].x & cmask], 1u);
        __syncthreads();
        const int col0 = ch.group << cbits;
        for (int k = threadIdx.x; k < ncol; k += 512)
            if (s_cnt[k]) s_base[k] = colptr[col0 + k] + atomicAdd(cursor + col0 + k, (int)s_cnt[k]);
        hh_tile_scan(s_cnt, ncol, s_wtot);
        for (int k = threadIdx.x; k < ncol; k += 512) s_base[k] -= s_cnt[k];
        __syncthreads();
#pragma unroll
        for (int k = 0; k < ITEMS; ++k)
            if (k * 512 + (int)threadIdx.x < ch.len) s_rec[atomicAdd(&s_cnt[r[k].x & cmask], 1u)] = r[k];
        __syncthreads();
        for (int e = threadIdx.x; e < ch.len; e += 512) {
            const uint2 x = s_rec[e];
            const long long q = s_base[x.x & cmask] + e;
            row[q] = (int32_t)(x.x >> cbits);
            val[q] = __uint_as_float(x.y);
        }
        __syncthreads();
    }
}

static int matrix_alloc(hh_ctx* ctx, int32_t n, int64_t nnz, hh_matrix** out) {
    hh_matrix* m = new (std::nothrow) hh_matrix();
    HH_REQUIRE(m != nullptr, HH_ERR_NOMEM, "hh_matrix: out of host memory");
    memset(m, 0, sizeof(*m));
    m->ctx = ctx;
    m->n = n;
    m->nnz = nnz;
    int rc;
    if ((rc = hh_dmalloc(&m->d_colptr, (size_t)n + 1)) != HH_OK || (rc = hh_dmalloc(&m->d_row, (size_t)nnz)) != HH_OK ||
        (rc = hh_dmalloc(&m->d_val, (size_t)nnz)) != HH_OK) {
        hh_matrix_destroy(m);
        return rc;
    }
    *out = m;
    return HH_OK;
}

extern "C" int hh_matrix_from_links(hh_links* lk, const uint8_t* keep, const int32_t* tail, int32_t n_tail,
                                    int normalize_by_nlinks, int add_self_loops, hh_matrix** out) {
    return hh_matrix_from_links_phased(lk, keep, tail, n_tail, normalize_by_nlinks, add_self_loops, nullptr, 0.0, out);
}

extern "C" int hh_matrix_from_links_phased(hh_links* lk, const uint8_t* keep, const int32_t* tail, int32_t n_tail,
                                           int normalize_by_nlinks, int add_self_loops, const int32_t* hap, double w,
                                           hh_matrix** out) {
    return hh_matrix_from_links_ex(lk, keep, tail, n_tail, normalize_by_nlinks, add_self_loops, hap, w, nullptr, nullptr, out);
}

extern "C" int hh_matrix_from_links_ex(hh_links* lk, const uint8_t* keep, const int32_t* tail, int32_t n_tail, int normalize_by_nlinks,
                                       int add_self_loops, const int32_t* hap, double w, const int32_t* ul_path,
                                       const int32_t* ul_parent, hh_matrix** out) {
    HH_REQUIRE(lk && keep && out, HH_ERR_ARG, "hh_matrix_from_links: NULL argument");
    hh_scope _scope(hh_links_ctx(lk));
    HH_REQUIRE(n_tail >= 0 && (tail || n_tail == 0), HH_ERR_ARG, "hh_matrix_from_links: bad tail");
    HH_REQUIRE(!ul_path == !ul_parent, HH_ERR_ARG, "hh_matrix_from_links_ex: give both ul_path and ul_parent, or neither");
    HH_REQUIRE(hh_links_finished(lk), HH_ERR_STATE, "hh_matrix_from_links: call hh_links_finish first");
    *out = nullptr;
    hh_ctx* ctx = hh_links_ctx(lk);
    HH_CUDA(cudaSetDevice(ctx->device));
    const int n_ctg = hh_links_n_ctg(lk);
    // the first-seen indices, degrees and passing count for this keep mask: reused when hh_links_linked_index_phased
    // computed them from the same arguments, recomputed (with one sync) otherwise
    int32_t n_linked = 0;
    HH_CHECK(hh_links_linked_index_phased(lk, keep, normalize_by_nlinks, hap, w, nullptr, &n_linked));
    const int32_t* d_hap = hh_links_hap_dev(lk);
    const int32_t* d_index = hh_links_index_dev(lk, &n_linked);
    int64_t n_pass = 0;
    const int32_t* d_deg = hh_links_degree_dev(lk, &n_pass);
    const uint8_t* d_keep = hh_links_keep_dev(lk);
    // a tail longer than the unlinked fragments must repeat or list a linked / absent id: refused before the matrix is sized
    HH_REQUIRE(n_tail <= n_ctg - n_linked, HH_ERR_ARG,
               "hh_matrix_from_links: tail lists an id that is dropped, linked, repeated or out of range");
    const int n = n_linked + n_tail;
    HH_REQUIRE(n > 0, HH_ERR_ARG, "hh_matrix_from_links: empty fragment set");
    HH_REQUIRE(n <= HH_MAT_MAX_N, HH_ERR_ARG, "hh_matrix_from_links: %d fragments in the matrix, at most %d are supported", n,
               HH_MAT_MAX_N);
    const int sl = add_self_loops ? 1 : 0;
    const int64_t nnz = 2 * n_pass + (int64_t)sl * n;      // known before any sync: the matrix is allocated up front
    int* d_err = reinterpret_cast<int*>(ctx->d_scratch + 10);
    int32_t* d_tail = nullptr;
    int32_t* d_ul = nullptr;
    int* d_cnt = nullptr;
    uint2* d_stage = nullptr;
    unsigned long long* d_gcur = nullptr;
    hh_mat_chunk* d_chunk = nullptr;
    unsigned int* d_nchunk = nullptr;
    hh_matrix* m = nullptr;
    int rc = [&]() -> int {
        HH_CHECK(matrix_alloc(ctx, n, nnz, &m));
        // the matrix gets its own copy of the index, and the tail goes there: the table's index stays reusable
        HH_CHECK(hh_dmalloc(&m->d_index, (size_t)n_ctg));
        m->n_index = n_ctg;
        HH_CUDA(cudaMemcpyAsync(m->d_index, d_index, (size_t)n_ctg * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
        HH_CUDA(cudaMemsetAsync(d_err, 0, sizeof(int), ctx->stream));
        if (n_tail) {
            HH_CHECK(hh_dmalloc(&d_tail, (size_t)n_tail));
            HH_CUDA(cudaMemcpyAsync(d_tail, tail, (size_t)n_tail * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
            HH_LAUNCH(ctx, hh_k_set_tail, (n_tail + 255) / 256, 256, 0, d_tail, n_tail, n_linked, d_keep, m->d_index, n_ctg, d_err);
        }
        HH_LAUNCH(ctx, hh_k_check_index, (n_ctg + 255) / 256, 256, 0, m->d_index, d_keep, n_ctg, n, d_err);
        HH_CHECK(hh_dmalloc(&d_cnt, (size_t)n));
        HH_LAUNCH(ctx, hh_k_fill_i32, (n + 255) / 256, 256, 0, d_cnt, sl, n);
        HH_LAUNCH(ctx, hh_k_mat_colcnt, (n_ctg + 255) / 256, 256, 0, d_index, d_deg, n_ctg, sl, d_cnt);
        HH_CHECK(hh_exclusive_scan_i32(ctx, d_cnt, m->d_colptr, n));
        int* d_cursor = d_cnt;                             // the counts are scanned: the buffer becomes the column cursors
        HH_LAUNCH(ctx, hh_k_fill_i32, (n + 255) / 256, 256, 0, d_cursor, sl, n);
        if (sl) HH_LAUNCH(ctx, hh_k_mat_self_loops, (n + 255) / 256, 256, 0, n, m->d_colptr, m->d_row, m->d_val);
        int64_t nnz_c = 0;
        const uint32_t* compact = hh_links_compact(lk, &nnz_c);
        if (ul_path && n_pass) {
            HH_CHECK(hh_dmalloc(&d_ul, (size_t)n_ctg * 2));
            HH_CUDA(cudaMemcpyAsync(d_ul, ul_path, (size_t)n_ctg * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
            HH_CUDA(cudaMemcpyAsync(d_ul + n_ctg, ul_parent, (size_t)n_ctg * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
        }
        if (n_pass) {
            const int cbits = hh_mat_cbits(n), ngroups = (n + (1 << cbits) - 1) >> cbits;
            const int64_t max_chunks = (nnz + HH_MAT_CHUNK - 1) / HH_MAT_CHUNK + ngroups;
            HH_CHECK(hh_ws_alloc(ctx, &d_stage, (size_t)nnz));
            HH_CHECK(hh_dmalloc(&d_gcur, (size_t)ngroups));
            HH_CHECK(hh_dmalloc(&d_chunk, (size_t)max_chunks));
            HH_CHECK(hh_dmalloc(&d_nchunk, 1));
            HH_LAUNCH(ctx, hh_k_mat_chunks, 1, 512, 0, m->d_colptr, n, cbits, ngroups, sl, d_gcur, d_chunk, d_nchunk);
            const size_t smem1 = hh_mat_group_smem(ngroups), smem2 = (size_t)HH_MAT_CHUNK * sizeof(uint2);
            int grid = 0;
            HH_CUDA(cudaFuncSetAttribute(hh_k_mat_group, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
            HH_CHECK(hh_resident_grid(ctx, hh_k_mat_group, 512, smem1, &grid));
            grid = (int)std::min<int64_t>((nnz_c + HH_MAT_TILE - 1) / HH_MAT_TILE, grid);
            HH_LAUNCH(ctx, hh_k_mat_group, grid, 512, smem1, compact, nnz_c, d_index, hh_links_ctg_totals(lk), normalize_by_nlinks,
                      d_hap, w, d_ul, d_ul ? d_ul + n_ctg : nullptr, cbits, ngroups, d_gcur, d_stage);
            HH_CUDA(cudaFuncSetAttribute(hh_k_mat_place, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
            HH_CHECK(hh_resident_grid(ctx, hh_k_mat_place, 512, smem2, &grid));
            grid = (int)std::min<int64_t>(max_chunks, grid);
            HH_LAUNCH(ctx, hh_k_mat_place, grid, 512, smem2, d_stage, d_chunk, d_nchunk, cbits, m->d_colptr, d_cursor, m->d_row,
                      m->d_val);
        }
        HH_CUDA(cudaMemcpyAsync(ctx->h_scratch + 10, d_err, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        const int err = *reinterpret_cast<int*>(ctx->h_scratch + 10);
        HH_REQUIRE(err == 0, HH_ERR_ARG,
                   err == 1 ? "hh_matrix_from_links: tail lists an id that is dropped, linked, repeated or out of range"
                            : "hh_matrix_from_links: keep mask and tail do not cover the fragment set exactly");
        return HH_OK;
    }();
    hh_dfree(d_tail);
    hh_dfree(d_ul);
    hh_dfree(d_cnt);
    hh_ws_free(ctx, d_stage);
    hh_dfree(d_gcur);
    hh_dfree(d_chunk);
    hh_dfree(d_nchunk);
    if (rc != HH_OK) {
        hh_matrix_destroy(m);
        return rc;
    }
    *out = m;
    return HH_OK;
}

extern "C" int hh_matrix_from_csc(hh_ctx* ctx, int32_t n, const int64_t* indptr, const int32_t* indices, const float* data,
                                  hh_matrix** out) {
    HH_REQUIRE(ctx && indptr && out, HH_ERR_ARG, "hh_matrix_from_csc: NULL argument");
    hh_scope _scope(ctx);
    HH_REQUIRE(n > 0, HH_ERR_ARG, "hh_matrix_from_csc: n must be positive");
    *out = nullptr;
    HH_REQUIRE(indptr[0] == 0, HH_ERR_ARG, "hh_matrix_from_csc: indptr[0] must be 0");
    for (int32_t c = 0; c < n; ++c)
        HH_REQUIRE(indptr[c + 1] >= indptr[c] && indptr[c + 1] - indptr[c] <= n, HH_ERR_ARG,
                   "hh_matrix_from_csc: column %d has an invalid extent", c);
    const int64_t nnz = indptr[n];
    HH_REQUIRE(nnz == 0 || (indices && data), HH_ERR_ARG, "hh_matrix_from_csc: NULL indices/data");
    for (int64_t e = 0; e < nnz; ++e)
        HH_REQUIRE(indices[e] >= 0 && indices[e] < n, HH_ERR_ARG, "hh_matrix_from_csc: row index out of range at entry %lld",
                   (long long)e);
    HH_CUDA(cudaSetDevice(ctx->device));
    hh_matrix* m = nullptr;
    HH_CHECK(matrix_alloc(ctx, n, nnz, &m));
    int rc = [&]() -> int {
        HH_CUDA(cudaMemcpyAsync(m->d_colptr, indptr, ((size_t)n + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
        if (nnz) {
            HH_CUDA(cudaMemcpyAsync(m->d_row, indices, (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
            HH_CUDA(cudaMemcpyAsync(m->d_val, data, (size_t)nnz * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        }
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        return HH_OK;
    }();
    if (rc != HH_OK) {
        hh_matrix_destroy(m);
        return rc;
    }
    *out = m;
    return HH_OK;
}

extern "C" int hh_matrix_info(hh_matrix* m, int32_t* n, int64_t* nnz) {
    HH_REQUIRE(m != nullptr, HH_ERR_ARG, "hh_matrix_info: NULL handle");
    if (n) *n = m->n;
    if (nnz) *nnz = m->nnz;
    return HH_OK;
}

extern "C" int hh_matrix_destroy(hh_matrix* m) {
    if (!m) return HH_OK;
    hh_scope _scope(m->ctx);
    cudaSetDevice(m->ctx->device);
    cudaStreamSynchronize(m->ctx->stream);
    hh_dfree(m->d_colptr);
    hh_dfree(m->d_row);
    hh_dfree(m->d_val);
    hh_dfree(m->d_index);
    delete m;
    return HH_OK;
}
