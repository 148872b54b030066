// Reassignment statistics over the full links (output_statistics, HapHiC_cluster.py:2245-2478): the (contig, group) link
// sums that parse_link_dict (2245-2258) accumulates, each contig's groups ranked by them, and the best-group link, density
// and density ratio.  The links are integer counts, or ints and Python floats after a fractional --phasing_weight or a
// link scaling.  The statistics files hold the repr of fp64 results, so every sum here is the serial chain of adds the
// reference makes, in its order:
//   * a segment (contig, group) is summed with sequential fp64 adds over its directed entries in visiting order, from 0.
//     Integer prefixes are exact in fp64 (counts are uint32, every sum stays far below 2^53), so this is Python's
//     int + int / int + float chain bit for bit.
//   * `others` adds the densities of ranked[1:] in rank order with CPython >= 3.12 sum()'s Neumaier compensation.
// No tree reduction: a short chain runs on one lane; a long one (more than 32 terms) on a whole warp, which loads 32 terms
// at a time and hands them to the accumulator in order through shuffles (every lane carries the same accumulator).
#include <algorithm>

#include <cub/cub.cuh>

#include "hh_internal.cuh"

struct hh_stats {
    hh_ctx* ctx;
    int32_t n_ctg;
    int64_t m;              // entries; 2m directed positions (first end of entry e at 2e, second end at 2e + 1)
    int32_t* d_ki;          // [m]
    int32_t* d_kj;          // [m]
    double* d_val;          // [m] exact integers or the reduced floats
    uint8_t* d_flt;         // [m] 1 = the value is a Python float
    // ranking of the last hh_stats_rank: nseg (contig, group) segments in (contig, rank) order
    int32_t* d_gid;         // [n_ctg] group of every contig, -1 = ungrouped
    int64_t nseg;
    int32_t* d_c;
    int32_t* d_g;
    double* d_sum;
    uint8_t* d_isf;
    int64_t* d_beg;         // [n_ctg] ranked list of contig c = [d_beg[c], d_end[c])
    int64_t* d_end;
    bool ranked;
};

static const int HH_ST_SHORT = 32;   // chains up to this length run on one lane

static inline int hh_bit_len(uint64_t x) { return x ? 64 - __builtin_clzll(x) : 1; }

// sort key of every directed position: contig * ng + group of the other end; links to ungrouped contigs get `sentinel`
// (= n_ctg * ng, after every real key).  Counts the real ones.
__global__ void __launch_bounds__(256)
hh_k_stats_keys(const int32_t* __restrict__ ki, const int32_t* __restrict__ kj, int64_t m, const int32_t* __restrict__ gid,
                int64_t ng, uint64_t sentinel, uint64_t* __restrict__ key, uint32_t* __restrict__ pos,
                unsigned long long* __restrict__ n_valid) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int mine = 0;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < 2 * m; p += stride) {
        const int64_t e = p >> 1;
        const int32_t a = ki[e], b = kj[e];
        const int32_t c = (p & 1) ? b : a, o = (p & 1) ? a : b;
        const int32_t g = gid[o];
        key[p] = g >= 0 ? (uint64_t)c * (uint64_t)ng + (uint64_t)g : sentinel;
        pos[p] = (uint32_t)p;
        mine += g >= 0;
    }
    mine = hh_warp_sum(mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(n_valid, (unsigned long long)mine);
}

// segment s = (contig, group): its positions are pos_s[off[s] .. off[s] + cnt[s]) in visiting order (the radix sort is
// stable and the positions went in ascending).  One warp per 32 consecutive segments.
__global__ void __launch_bounds__(256)
hh_k_stats_seg_sums(const uint64_t* __restrict__ ukey, const uint32_t* __restrict__ pos_s, const int64_t* __restrict__ off,
                    const int64_t* __restrict__ cnt, int64_t nseg, int64_t ng, const double* __restrict__ val,
                    const uint8_t* __restrict__ flt, int32_t* __restrict__ seg_c, int32_t* __restrict__ seg_g,
                    double* __restrict__ sum, uint8_t* __restrict__ isf, uint32_t* __restrict__ first) {
    const int lane = threadIdx.x & 31;
    const int64_t base = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32;
    const int64_t s = base + lane;
    bool lng = false;
    if (s < nseg) {
        const int64_t lo = off[s], n = cnt[s];
        seg_c[s] = (int32_t)(ukey[s] / (uint64_t)ng);
        seg_g[s] = (int32_t)(ukey[s] % (uint64_t)ng);
        first[s] = pos_s[lo];
        lng = n > HH_ST_SHORT;
        if (!lng) {
            double acc = 0.0;
            uint8_t f = 0;
            for (int64_t k = 0; k < n; ++k) {
                const uint32_t e = pos_s[lo + k] >> 1;
                acc = __dadd_rn(acc, val[e]);
                f |= flt[e];
            }
            sum[s] = acc;
            isf[s] = f;
        }
    }
    unsigned todo = __ballot_sync(HH_FULL_MASK, lng);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int64_t t = base + src;
        const int64_t lo = off[t], n = cnt[t];
        double acc = 0.0;
        bool f = false;
        for (int64_t b = 0; b < n; b += 32) {
            double x = 0.0;
            int fl = 0;
            if (b + lane < n) {
                const uint32_t e = pos_s[lo + b + lane] >> 1;
                x = val[e];
                fl = flt[e];
            }
            const int len = (int)(n - b < 32 ? n - b : 32);
            for (int k = 0; k < len; ++k) acc = __dadd_rn(acc, __shfl_sync(HH_FULL_MASK, x, k));
            f |= __any_sync(HH_FULL_MASK, fl) != 0;
        }
        if (lane == 0) {
            sum[t] = acc;
            isf[t] = f ? 1 : 0;
        }
    }
}

// descending sum as an ascending key: sums are positive, so their bit patterns order like the values
__global__ void hh_k_stats_sum_key(const double* __restrict__ sum, const uint32_t* __restrict__ idx, int64_t n,
                                   uint64_t* __restrict__ key) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) key[k] = ~(uint64_t)__double_as_longlong(sum[idx[k]]);
}

__global__ void hh_k_stats_iota(uint32_t* __restrict__ p, int64_t n) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) p[k] = (uint32_t)k;
}

template <typename T>
__global__ void hh_k_stats_gather(const T* __restrict__ src, const uint32_t* __restrict__ idx, int64_t n, T* __restrict__ dst) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) dst[k] = src[idx[k]];
}

__global__ void hh_k_stats_bounds(const int32_t* __restrict__ c, int64_t n, int64_t* __restrict__ beg, int64_t* __restrict__ end) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (k == 0 || c[k - 1] != c[k]) beg[c[k]] = k;
    if (k == n - 1 || c[k + 1] != c[k]) end[c[k]] = k + 1;
}

// one term of sum(): CPython >= 3.12 (bltinmodule.c, builtin_sum_impl) adds floats with Neumaier's compensation
__device__ __forceinline__ void hh_sum_add(double& f, double& comp, double x, int compensated) {
    const double t = __dadd_rn(f, x);
    if (compensated) comp = __dadd_rn(comp, fabs(f) >= fabs(x) ? __dadd_rn(__dsub_rn(f, t), x) : __dadd_rn(__dsub_rn(x, t), f));
    f = t;
}

// cal_link_density (2271-2276): links / RE of the group, or / (RE of the group + RE of the contig - 1) for another group
__device__ __forceinline__ double hh_density(double links, int32_t g, int32_t own, const int64_t* __restrict__ group_re,
                                             int64_t ctg_re) {
    const int64_t d = g == own ? group_re[g] : group_re[g] + ctg_re - 1;
    return __ddiv_rn(links, (double)d);
}

// Per contig: the best group's links and density, the mean density of the others (sum over ranked[1:] / (n_groups - 1))
// and the ratio.  One warp per 32 consecutive contigs, as hh_k_stats_seg_sums.
__global__ void __launch_bounds__(256)
hh_k_stats_best(const int64_t* __restrict__ beg, const int64_t* __restrict__ end, int32_t n_ctg, const int32_t* __restrict__ g_of,
                const double* __restrict__ sum, const uint8_t* __restrict__ isf, const int32_t* __restrict__ gid,
                const int64_t* __restrict__ group_re, const int64_t* __restrict__ ctg_re, int32_t n_groups, int compensated,
                uint8_t* __restrict__ has, double* __restrict__ top_links, uint8_t* __restrict__ top_float,
                double* __restrict__ top_dens, double* __restrict__ others, double* __restrict__ ratio) {
    const int lane = threadIdx.x & 31;
    const int64_t base = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32;
    const int64_t c = base + lane;
    int64_t lo = 0, n = 0;
    if (c < n_ctg) {
        lo = beg[c];
        n = end[c] - lo;
    }
    const bool lng = n > HH_ST_SHORT;
    double acc = 0.0, comp = 0.0;
    if (c < n_ctg && !lng) {
        for (int64_t k = 1; k < n; ++k) hh_sum_add(acc, comp, hh_density(sum[lo + k], g_of[lo + k], gid[c], group_re, ctg_re[c]),
                                                  compensated);
    }
    unsigned todo = __ballot_sync(HH_FULL_MASK, lng);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int64_t t = base + src;
        const int64_t tlo = beg[t], tn = end[t] - tlo;
        double a = 0.0, cp = 0.0;
        for (int64_t b = 1; b < tn; b += 32) {
            double x = 0.0;
            if (b + lane < tn) x = hh_density(sum[tlo + b + lane], g_of[tlo + b + lane], gid[t], group_re, ctg_re[t]);
            const int len = (int)(tn - b < 32 ? tn - b : 32);
            for (int k = 0; k < len; ++k) hh_sum_add(a, cp, __shfl_sync(HH_FULL_MASK, x, k), compensated);
        }
        if (lane == src) {
            acc = a;
            comp = cp;
        }
    }
    if (c >= n_ctg) return;
    has[c] = n > 0;
    if (n == 0) {
        top_links[c] = top_dens[c] = others[c] = ratio[c] = 0.0;
        top_float[c] = 0;
        return;
    }
    // "add the compensation if it is non-zero and finite" (builtin_sum_impl, end of the float loop)
    if (compensated && comp != 0.0 && isfinite(comp)) acc = __dadd_rn(acc, comp);
    const double d0 = hh_density(sum[lo], g_of[lo], gid[c], group_re, ctg_re[c]);
    const double o = n_groups > 1 ? __ddiv_rn(acc, (double)(n_groups - 1)) : 0.0;
    top_links[c] = sum[lo];
    top_float[c] = isf[lo];
    top_dens[c] = d0;
    others[c] = o;
    ratio[c] = __ddiv_rn(d0, o);     // inf / nan when o == 0: the caller writes 1000000 then
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static inline unsigned hh_blocks(int64_t n, int t = 256) { return (unsigned)std::max<int64_t>(1, (n + t - 1) / t); }

static void stats_free_ranking(hh_stats* st) {
    hh_dfree(st->d_c);
    hh_dfree(st->d_g);
    hh_dfree(st->d_sum);
    hh_dfree(st->d_isf);
    st->nseg = 0;
    st->ranked = false;
}

extern "C" int hh_stats_create(hh_ctx* ctx, int32_t n_ctg, const int32_t* key_i, const int32_t* key_j, const double* values,
                               const uint8_t* is_float, int64_t n_entries, hh_stats** out) {
    HH_REQUIRE(ctx && out && n_ctg > 0 && n_entries >= 0, HH_ERR_ARG, "hh_stats_create: bad argument");
    HH_REQUIRE(n_entries == 0 || (key_i && key_j && values && is_float), HH_ERR_ARG, "hh_stats_create: NULL entry array");
    // the run-length encoding of the sorted positions counts in int
    HH_REQUIRE(2 * n_entries <= (int64_t)INT32_MAX, HH_ERR_UNSUPPORTED, "hh_stats_create: %lld entries (at most 2^30 - 1)",
               (long long)n_entries);
    *out = nullptr;
    hh_scope _scope(ctx);
    hh_stats* st = new (std::nothrow) hh_stats();
    HH_REQUIRE(st, HH_ERR_NOMEM, "hh_stats_create: out of host memory");
    st->ctx = ctx;
    st->n_ctg = n_ctg;
    st->m = n_entries;
    const int rc = [&]() -> int {
        const size_t m = (size_t)n_entries;
        HH_CHECK(hh_dmalloc(&st->d_ki, m));
        HH_CHECK(hh_dmalloc(&st->d_kj, m));
        HH_CHECK(hh_dmalloc(&st->d_val, m));
        HH_CHECK(hh_dmalloc(&st->d_flt, m));
        HH_CHECK(hh_dmalloc(&st->d_gid, (size_t)n_ctg));
        HH_CHECK(hh_dmalloc(&st->d_beg, (size_t)n_ctg));
        HH_CHECK(hh_dmalloc(&st->d_end, (size_t)n_ctg));
        if (m) {
            HH_CUDA(cudaMemcpyAsync(st->d_ki, key_i, m * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
            HH_CUDA(cudaMemcpyAsync(st->d_kj, key_j, m * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
            HH_CUDA(cudaMemcpyAsync(st->d_val, values, m * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
            HH_CUDA(cudaMemcpyAsync(st->d_flt, is_float, m, cudaMemcpyHostToDevice, ctx->stream));
        }
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        return HH_OK;
    }();
    if (rc != HH_OK) {
        hh_stats_destroy(st);
        return rc;
    }
    *out = st;
    return HH_OK;
}

extern "C" int hh_stats_rank(hh_stats* st, const int32_t* group, int32_t n_groups, int64_t* n_ranked) {
    HH_REQUIRE(st && group && n_groups > 0, HH_ERR_ARG, "hh_stats_rank: bad argument");
    hh_scope _scope(st->ctx);
    hh_ctx* ctx = st->ctx;
    stats_free_ranking(st);
    const int64_t P = 2 * st->m;
    const uint64_t ng = (uint64_t)n_groups;
    const uint64_t sentinel = (uint64_t)st->n_ctg * ng;
    HH_CUDA(cudaMemcpyAsync(st->d_gid, group, (size_t)st->n_ctg * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    HH_CUDA(cudaMemsetAsync(st->d_beg, 0, (size_t)st->n_ctg * sizeof(int64_t), ctx->stream));
    HH_CUDA(cudaMemsetAsync(st->d_end, 0, (size_t)st->n_ctg * sizeof(int64_t), ctx->stream));
    if (P == 0) {
        if (n_ranked) *n_ranked = 0;
        st->ranked = true;
        return HH_OK;
    }
    uint64_t *d_key = nullptr, *d_key_s = nullptr;
    uint32_t *d_pos = nullptr, *d_pos_s = nullptr, *d_first = nullptr;
    int64_t *d_cnt = nullptr, *d_off = nullptr;
    int32_t *d_sc = nullptr, *d_sg = nullptr;
    double* d_ssum = nullptr;
    uint8_t *d_sisf = nullptr, *d_tmp = nullptr;
    unsigned long long* d_n = nullptr;
    const int rc = [&]() -> int {
        HH_CHECK(hh_dmalloc(&d_key, (size_t)P));
        HH_CHECK(hh_dmalloc(&d_key_s, (size_t)P));
        HH_CHECK(hh_dmalloc(&d_pos, (size_t)P));
        HH_CHECK(hh_dmalloc(&d_pos_s, (size_t)P));
        HH_CHECK(hh_dmalloc(&d_n, 2));
        HH_CUDA(cudaMemsetAsync(d_n, 0, 2 * sizeof(unsigned long long), ctx->stream));
        HH_LAUNCH(ctx, hh_k_stats_keys, (unsigned)std::min<int64_t>(hh_blocks(P), (int64_t)ctx->sm_count * 8), 256, 0, st->d_ki,
                  st->d_kj, st->m, st->d_gid, (int64_t)ng, sentinel, d_key, d_pos, d_n);
        const int key_bits = hh_bit_len(sentinel);
        size_t tmp_bytes = 0, b = 0;
        HH_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, d_key, d_key_s, d_pos, d_pos_s, P, 0, key_bits, ctx->stream));
        tmp_bytes = std::max(tmp_bytes, b);
        HH_CUDA(cub::DeviceRunLengthEncode::Encode(nullptr, b, d_key_s, d_key, d_off, d_n + 1, (int)P, ctx->stream));
        tmp_bytes = std::max(tmp_bytes, b);
        HH_CHECK(hh_dmalloc(&d_tmp, tmp_bytes));
        HH_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_key, d_key_s, d_pos, d_pos_s, P, 0, key_bits, ctx->stream));
        unsigned long long h_n[2];
        HH_CUDA(cudaMemcpyAsync(h_n, d_n, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        const int64_t nvalid = (int64_t)h_n[0];
        if (nvalid == 0) return HH_OK;
        // segments: the runs of equal keys among the real ones (unique keys overwrite d_key, the lengths go to d_cnt)
        HH_CHECK(hh_dmalloc(&d_cnt, (size_t)nvalid));
        HH_CHECK(hh_dmalloc(&d_off, (size_t)nvalid));
        b = tmp_bytes;
        HH_CUDA(cub::DeviceRunLengthEncode::Encode(d_tmp, b, d_key_s, d_key, d_cnt, d_n + 1, (int)nvalid, ctx->stream));
        HH_CUDA(cudaMemcpyAsync(h_n + 1, d_n + 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        const int64_t nseg = (int64_t)h_n[1];
        HH_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, d_cnt, d_off, nseg, ctx->stream));
        if (b > tmp_bytes) {
            hh_dfree(d_tmp);
            tmp_bytes = b;
            HH_CHECK(hh_dmalloc(&d_tmp, tmp_bytes));
        }
        HH_CUDA(cub::DeviceScan::ExclusiveSum(d_tmp, b, d_cnt, d_off, nseg, ctx->stream));
        HH_CHECK(hh_dmalloc(&d_sc, (size_t)nseg));
        HH_CHECK(hh_dmalloc(&d_sg, (size_t)nseg));
        HH_CHECK(hh_dmalloc(&d_ssum, (size_t)nseg));
        HH_CHECK(hh_dmalloc(&d_sisf, (size_t)nseg));
        HH_CHECK(hh_dmalloc(&d_first, (size_t)nseg));
        HH_LAUNCH(ctx, hh_k_stats_seg_sums, hh_blocks(nseg), 256, 0, d_key, d_pos_s, d_off, d_cnt, nseg, (int64_t)ng, st->d_val,
                  st->d_flt, d_sc, d_sg, d_ssum, d_sisf, d_first);
        // rank: three stable radix sorts of the segment indices, least significant key first -- first visit ascending, sum
        // descending, contig ascending (Python's stable sorted(..., reverse=True) per contig)
        uint32_t* idx_a = d_pos;               // P >= nseg entries each: the position arrays are free again
        uint32_t* idx_b = d_pos_s;
        uint32_t* key32 = reinterpret_cast<uint32_t*>(d_off);        // offsets are consumed: nseg x 8 bytes of room
        uint32_t* key32_s = reinterpret_cast<uint32_t*>(d_cnt);
        uint64_t* key64 = d_key;
        uint64_t* key64_s = d_key_s;
        HH_LAUNCH(ctx, hh_k_stats_iota, hh_blocks(nseg), 256, 0, idx_a, nseg);
        const int pos_bits = hh_bit_len((uint64_t)P), ctg_bits = hh_bit_len((uint64_t)st->n_ctg);
        HH_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, key32, key32_s, idx_a, idx_b, nseg, 0, pos_bits, ctx->stream));
        size_t need = b;
        HH_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, key64, key64_s, idx_a, idx_b, nseg, 0, 64, ctx->stream));
        need = std::max(need, b);
        if (need > tmp_bytes) {
            hh_dfree(d_tmp);
            tmp_bytes = need;
            HH_CHECK(hh_dmalloc(&d_tmp, tmp_bytes));
        }
        HH_CUDA(cudaMemcpyAsync(key32, d_first, (size_t)nseg * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
        b = tmp_bytes;
        HH_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, b, key32, key32_s, idx_a, idx_b, nseg, 0, pos_bits, ctx->stream));
        HH_LAUNCH(ctx, hh_k_stats_sum_key, hh_blocks(nseg), 256, 0, d_ssum, idx_b, nseg, key64);
        b = tmp_bytes;
        HH_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, b, key64, key64_s, idx_b, idx_a, nseg, 0, 64, ctx->stream));
        HH_LAUNCH(ctx, hh_k_stats_gather<uint32_t>, hh_blocks(nseg), 256, 0, reinterpret_cast<const uint32_t*>(d_sc), idx_a, nseg,
                  key32);
        b = tmp_bytes;
        HH_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, b, key32, key32_s, idx_a, idx_b, nseg, 0, ctg_bits, ctx->stream));
        HH_CHECK(hh_dmalloc(&st->d_c, (size_t)nseg));
        HH_CHECK(hh_dmalloc(&st->d_g, (size_t)nseg));
        HH_CHECK(hh_dmalloc(&st->d_sum, (size_t)nseg));
        HH_CHECK(hh_dmalloc(&st->d_isf, (size_t)nseg));
        HH_LAUNCH(ctx, hh_k_stats_gather<int32_t>, hh_blocks(nseg), 256, 0, d_sc, idx_b, nseg, st->d_c);
        HH_LAUNCH(ctx, hh_k_stats_gather<int32_t>, hh_blocks(nseg), 256, 0, d_sg, idx_b, nseg, st->d_g);
        HH_LAUNCH(ctx, hh_k_stats_gather<double>, hh_blocks(nseg), 256, 0, d_ssum, idx_b, nseg, st->d_sum);
        HH_LAUNCH(ctx, hh_k_stats_gather<uint8_t>, hh_blocks(nseg), 256, 0, d_sisf, idx_b, nseg, st->d_isf);
        HH_LAUNCH(ctx, hh_k_stats_bounds, hh_blocks(nseg), 256, 0, st->d_c, nseg, st->d_beg, st->d_end);
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        st->nseg = nseg;
        return HH_OK;
    }();
    hh_dfree(d_key);
    hh_dfree(d_key_s);
    hh_dfree(d_pos);
    hh_dfree(d_pos_s);
    hh_dfree(d_first);
    hh_dfree(d_cnt);
    hh_dfree(d_off);
    hh_dfree(d_sc);
    hh_dfree(d_sg);
    hh_dfree(d_ssum);
    hh_dfree(d_sisf);
    hh_dfree(d_tmp);
    hh_dfree(d_n);
    if (rc != HH_OK) {
        stats_free_ranking(st);
        return rc;
    }
    st->ranked = true;
    if (n_ranked) *n_ranked = st->nseg;
    return HH_OK;
}

extern "C" int hh_stats_fetch_ranked(hh_stats* st, int32_t* ctg, int32_t* group, double* links, uint8_t* is_float) {
    HH_REQUIRE(st != nullptr, HH_ERR_ARG, "hh_stats_fetch_ranked: NULL handle");
    HH_REQUIRE(st->ranked, HH_ERR_STATE, "hh_stats_fetch_ranked: call hh_stats_rank first");
    hh_scope _scope(st->ctx);
    cudaStream_t s = st->ctx->stream;
    const size_t n = (size_t)st->nseg;
    if (n) {
        if (ctg) HH_CUDA(cudaMemcpyAsync(ctg, st->d_c, n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        if (group) HH_CUDA(cudaMemcpyAsync(group, st->d_g, n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        if (links) HH_CUDA(cudaMemcpyAsync(links, st->d_sum, n * sizeof(double), cudaMemcpyDeviceToHost, s));
        if (is_float) HH_CUDA(cudaMemcpyAsync(is_float, st->d_isf, n, cudaMemcpyDeviceToHost, s));
    }
    HH_CUDA(cudaStreamSynchronize(s));
    return HH_OK;
}

extern "C" int hh_stats_best(hh_stats* st, const int64_t* group_re, int32_t n_groups, const int64_t* ctg_re, int compensated,
                             uint8_t* has, double* top_links, uint8_t* top_is_float, double* top_density, double* others,
                             double* ratio) {
    HH_REQUIRE(st && group_re && ctg_re && n_groups > 0, HH_ERR_ARG, "hh_stats_best: bad argument");
    HH_REQUIRE(has && top_links && top_is_float && top_density && others && ratio, HH_ERR_ARG, "hh_stats_best: NULL output");
    HH_REQUIRE(st->ranked, HH_ERR_STATE, "hh_stats_best: call hh_stats_rank first");
    hh_scope _scope(st->ctx);
    hh_ctx* ctx = st->ctx;
    const int32_t n = st->n_ctg;
    int64_t *d_gre = nullptr, *d_cre = nullptr;
    uint8_t* d_u8 = nullptr;      // has, top_is_float
    double* d_f = nullptr;        // top_links, top_density, others, ratio
    const int rc = [&]() -> int {
        HH_CHECK(hh_dmalloc(&d_gre, (size_t)n_groups));
        HH_CHECK(hh_dmalloc(&d_cre, (size_t)n));
        HH_CHECK(hh_dmalloc(&d_u8, (size_t)n * 2));
        HH_CHECK(hh_dmalloc(&d_f, (size_t)n * 4));
        HH_CUDA(cudaMemcpyAsync(d_gre, group_re, (size_t)n_groups * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
        HH_CUDA(cudaMemcpyAsync(d_cre, ctg_re, (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
        HH_LAUNCH(ctx, hh_k_stats_best, hh_blocks(n), 256, 0, st->d_beg, st->d_end, n, st->d_g, st->d_sum, st->d_isf, st->d_gid,
                  d_gre, d_cre, n_groups, compensated, d_u8, d_f, d_u8 + n, d_f + n, d_f + 2 * (size_t)n, d_f + 3 * (size_t)n);
        uint8_t* u8[2] = {has, top_is_float};
        double* f[4] = {top_links, top_density, others, ratio};
        for (int k = 0; k < 2; ++k)
            HH_CUDA(cudaMemcpyAsync(u8[k], d_u8 + (size_t)k * n, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
        for (int k = 0; k < 4; ++k)
            HH_CUDA(cudaMemcpyAsync(f[k], d_f + (size_t)k * n, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        return HH_OK;
    }();
    hh_dfree(d_gre);
    hh_dfree(d_cre);
    hh_dfree(d_u8);
    hh_dfree(d_f);
    return rc;
}

extern "C" int hh_stats_destroy(hh_stats* st) {
    if (!st) return HH_OK;
    hh_scope _scope(st->ctx);
    cudaStreamSynchronize(st->ctx->stream);
    stats_free_ranking(st);
    hh_dfree(st->d_ki);
    hh_dfree(st->d_kj);
    hh_dfree(st->d_val);
    hh_dfree(st->d_flt);
    hh_dfree(st->d_gid);
    hh_dfree(st->d_beg);
    hh_dfree(st->d_end);
    delete st;
    return HH_OK;
}
