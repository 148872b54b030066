// Assembly correction (`--correct_nrounds`) on the GPU: the Hi-C coverage pass, breakpoint detection, contig breaking
// and the remapping of the record stream of scripts/HapHiC_cluster.py (v1.0.7):
//   parse_pairs_for_correction / parse_bam_for_correction (1300-1398)   hh_correct_add
//   detect_break_points (943-1014)                                        hh_correct_round
//   break_and_update_ctgs, coverage and link parts (1063-1113, 1151-1153, 1176-1178)
//                                                                        hh_correct_round (rounds that are not last)
//   convert_ctg of the *_for_correction generators (1401-1536)           hh_correct_remap
// The name / fa_dict / break-table bookkeeping stays on the host (haphic_b200/correct.py).
//
// Integer arithmetic throughout; every update is an integer add, so the results do not depend on the order in which
// records or links are processed and are bit-identical to the reference's numpy arrays.
//
// Fragments.  Every fragment ever examined has an id: 0 .. n_ctg-1 are the contigs (FASTA order), the pieces of the
// fragments broken in a round get the next ids, in the order of the broken fragments and left to right.  A fragment is
// a slice [off, off + nbins) of ONE coverage buffer: a contig owns len//res + 1 bins, and the reference's piece coverage
// `cov[start//res : point//res]` (and `cov[start//res:]` for the last piece) tiles the parent's slice exactly, so a
// piece is only a new (off, nbins) on the parent's bins.  Spanning links are subtracted from the parent before the
// slicing (1092) -- through the same buffer -- so nothing is ever copied.
#include "hh_common.cuh"
#include <cub/cub.cuh>
#include <limits.h>

struct hh_correct {
    hh_ctx* ctx;
    int32_t n_ctg;
    int64_t res;
    int64_t total_bins;
    int32_t* d_cov;          // [total_bins]
    int32_t* d_diff;         // [total_bins + 1] difference array (coverage pass, spanning-link subtraction)
    int32_t* d_sorted;       // [total_bins] segment-sorted copy of the examined slices (medians)
    int32_t* d_bp_bin;       // [total_bins] breakpoint candidates of a fragment at its own offset
    int32_t* d_bp_cov;       // [total_bins]
    bool cov_ready;          // the coverage pass has been turned into d_cov
    // fragment table, capacity f_cap
    int32_t n_frag, f_cap;
    int64_t* d_f_off;        // first bin in the coverage buffer
    int32_t* d_f_nbins;
    int64_t* d_f_len;        // fa_dict[frag][1]
    int64_t* d_f_start;      // 1-based start on the source contig (pos_shift, 1038-1044: 1 for unbroken contigs)
    int32_t* d_act_pos;      // [f_cap] position of a fragment in the examined list (valid for examined fragments)
    // fragments under examination (ctg_cov_dict keys, in dict order)
    int32_t n_active;
    int32_t* d_active;       // [n_active]
    int32_t* d_cnt;          // [n_active + 1] breakpoints of every examined fragment (+ scan slot)
    int32_t* d_bpos;         // [n_active + 1] exclusive scan of d_cnt
    int32_t* d_pcnt;         // [n_active + 1] pieces of every examined fragment (cnt + 1 or 0)
    int32_t* d_pbase;        // [n_active + 1] exclusive scan of d_pcnt
    std::vector<int32_t> breaks;   // (fragment, bin, coverage) of the last round's breakpoints, examined-list order
    // link store: ctg_link_pos_dict as (fragment, lo, hi); fragment -1 = dropped
    int64_t n_links, l_cap;
    int32_t* d_l_frag;
    int32_t* d_l_lo;
    int32_t* d_l_hi;
    unsigned long long* d_counter;
    // remap layout (hh_correct_set_layout)
    int32_t* d_src_base;     // [n_ctg + 1]
    int64_t* d_piece_start;  // [n_pieces] ascending per source contig
    int32_t* d_piece_id;
    int32_t n_pieces;
    // staging for host records
    int4* d_stage;
    int64_t stage_cap;
    void* d_cub;
    size_t cub_bytes;
};

// Python semantics of a slice bound on an array of n elements (negative = from the end, clamped to [0, n])
__device__ __forceinline__ int64_t hh_pyslice(int64_t i, int64_t n) {
    if (i < 0) {
        i += n;
        if (i < 0) i = 0;
    }
    return i > n ? n : i;
}
__device__ __forceinline__ int64_t hh_floordiv(int64_t a, int64_t b) {
    int64_t q = a / b;
    return (q * b != a && ((a < 0) != (b < 0))) ? q - 1 : q;
}

// ---------------------------------------------------------------------------------------------
// coverage pass (1334-1342 / 1388-1396): `cov[ref][lo//res : hi//res + 1] += 1` and `ctg_link_pos_dict[ref] += (lo, hi)`
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
hh_k_correct_cov(const int4* __restrict__ rec, int64_t n_rec, int32_t n_ctg, int64_t res, const int64_t* __restrict__ f_off,
                 const int32_t* __restrict__ f_nbins, int32_t* __restrict__ diff, int32_t* __restrict__ l_frag,
                 int32_t* __restrict__ l_lo, int32_t* __restrict__ l_hi, unsigned long long* __restrict__ counter) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); i0 < n_rec; i0 += stride) {
        const int64_t i = i0 + lane;
        int4 r = make_int4(-1, 0, -2, 0);
        if (i < n_rec) r = hh_ld_stream(rec + i);
        // same contig (1327 / `refid == mrefid`), contig in the FASTA (1331 / 1385)
        const bool keep = r.x == r.z && (unsigned)r.x < (unsigned)n_ctg;
        const int lo = min(r.y, r.w), hi = max(r.y, r.w);
        if (keep) {
            const int64_t nb = f_nbins[r.x], off = f_off[r.x];
            const int64_t s = hh_pyslice(hh_floordiv(lo, res), nb), e = hh_pyslice(hh_floordiv(hi, res) + 1, nb);
            if (s < e) {                 // numpy drops what lies past the end of the array
                atomicAdd(diff + off + s, 1);
                atomicAdd(diff + off + e, -1);
            }
        }
        // warp-aggregated reservation in the link store (the order of the links does not matter)
        const unsigned m = __ballot_sync(HH_FULL_MASK, keep);
        if (m == 0) continue;
        const int leader = __ffs(m) - 1;
        unsigned long long base = 0;
        if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(m));
        base = __shfl_sync(HH_FULL_MASK, base, leader);
        if (keep) {
            const int64_t slot = (int64_t)base + __popc(m & ((1u << lane) - 1u));
            l_frag[slot] = r.x;
            l_lo[slot] = lo;
            l_hi[slot] = hi;
        }
    }
}

__global__ void hh_k_correct_add_scan(int32_t* __restrict__ cov, const int32_t* __restrict__ scan, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        cov[i] += scan[i];
}

__global__ void hh_k_correct_segments(const int32_t* __restrict__ active, int32_t n_active, const int64_t* __restrict__ f_off,
                                      const int32_t* __restrict__ f_nbins, int32_t* __restrict__ seg_begin,
                                      int32_t* __restrict__ seg_end) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_active) return;
    const int f = active[i];
    seg_begin[i] = (int32_t)f_off[f];
    seg_end[i] = (int32_t)(f_off[f] + f_nbins[f]);
}

// ---------------------------------------------------------------------------------------------
// detect_break_points (943-1014), one thread per examined fragment.  The high-coverage runs are the `portion` union of
// closed(n*res, (n+1)*res) (965): touching closed intervals merge, so a run is a maximal stretch of consecutive high bins.
// One left-to-right pass keeps the minimum / first zero of the bins since the end of the last LARGE run; a snapshot taken
// where the current run starts is the valley statistic once that run turns out to be large (small high runs inside a
// valley belong to it, 981).  Candidates go to bp_*[off + k]; the final breakpoints overwrite them in place.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
hh_k_correct_detect(const int32_t* __restrict__ active, int32_t n_active, const int64_t* __restrict__ f_off,
                    const int32_t* __restrict__ f_nbins, const int64_t* __restrict__ f_len, const int32_t* __restrict__ cov,
                    const int32_t* __restrict__ sorted, int64_t res, double median_cov_ratio, double region_len_ratio,
                    int64_t min_region_cutoff, int32_t* __restrict__ bp_bin, int32_t* __restrict__ bp_cov,
                    int32_t* __restrict__ cnt) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_active) return;
    const int f = active[a];
    const int64_t off = f_off[f];
    const int32_t n = f_nbins[f];
    cnt[a] = 0;
    if (n <= 0) return;
    // numpy.median: the middle value, or the float64 mean of the two middle values
    const double med = (n & 1) ? (double)sorted[off + n / 2]
                               : ((double)sorted[off + n / 2 - 1] + (double)sorted[off + n / 2]) / 2.0;
    if (med == 0.0) return;                                        // 954
    const double cov_cutoff = med * median_cov_ratio;              // 959
    const double lcut = (double)f_len[f] * region_len_ratio;       // 960: max(min_region_cutoff, len * ratio)
    const double region_cutoff = (double)min_region_cutoff >= lcut ? (double)min_region_cutoff : lcut;
    int n_runs = 0, n_large = 0, n_valley = 0;
    int prev_end = -1;                                             // bin after the last large run
    int vz = -1, vmin = INT_MAX, varg = -1;                        // valley statistics since prev_end
    int sz = -1, smin = INT_MAX, sarg = -1;                        // ... snapshot where the current run began
    bool in_run = false;
    int run_s = 0;
    for (int i = 0; i <= n; ++i) {
        const int c = i < n ? cov[off + i] : 0;
        const bool high = i < n && (double)c >= cov_cutoff;
        if (in_run && !high) {                                     // run [run_s, i) ends
            in_run = false;
            ++n_runs;
            if ((double)((int64_t)(i - run_s) * res) >= region_cutoff) {     // 973
                ++n_large;
                if (prev_end >= 0) {                               // valley between two large runs: first zero, else argmin
                    bp_bin[off + n_valley] = sz >= 0 ? sz : sarg;
                    bp_cov[off + n_valley] = sz >= 0 ? 0 : smin;
                    ++n_valley;
                }
                prev_end = i;
                vz = -1;
                vmin = INT_MAX;
                varg = -1;
            }
        }
        if (i == n) break;
        if (high && !in_run) {
            in_run = true;
            run_s = i;
            sz = vz;
            smin = vmin;
            sarg = varg;
        }
        if (prev_end >= 0) {
            if (c == 0 && vz < 0) vz = i;
            if (c < vmin) {
                vmin = c;
                varg = i;
            }
        }
    }
    if (n_runs < 2 || n_large < 2) return;                        // 968, 977
    bool any_zero = false;
    for (int k = 0; k < n_valley; ++k) any_zero = any_zero || bp_cov[off + k] == 0;
    if (any_zero) {                                                // 1003-1005: every zero candidate, left to right
        int m = 0;
        for (int k = 0; k < n_valley; ++k) {
            if (bp_cov[off + k] == 0) {
                bp_bin[off + m] = bp_bin[off + k];
                bp_cov[off + m] = 0;
                ++m;
            }
        }
        cnt[a] = m;
    } else {                                                       // 1008: stable sort by coverage -> leftmost minimum
        int best = 0;
        for (int k = 1; k < n_valley; ++k)
            if (bp_cov[off + k] < bp_cov[off + best]) best = k;
        bp_bin[off] = bp_bin[off + best];
        bp_cov[off] = bp_cov[off + best];
        cnt[a] = 1;
    }
}

__global__ void hh_k_correct_piece_counts(const int32_t* __restrict__ cnt, int32_t n_active, int32_t* __restrict__ pcnt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_active) pcnt[i] = cnt[i] ? cnt[i] + 1 : 0;
    if (i == n_active) pcnt[i] = 0;
}

// compact (fragment, bin, coverage) list of the round, examined-list order
__global__ void hh_k_correct_compact(const int32_t* __restrict__ active, int32_t n_active, const int64_t* __restrict__ f_off,
                                     const int32_t* __restrict__ cnt, const int32_t* __restrict__ bpos,
                                     const int32_t* __restrict__ bp_bin, const int32_t* __restrict__ bp_cov,
                                     int32_t* __restrict__ out) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_active || cnt[a] == 0) return;
    const int f = active[a];
    const int64_t off = f_off[f];
    for (int k = 0; k < cnt[a]; ++k) {
        int32_t* o = out + 3 * (int64_t)(bpos[a] + k);
        o[0] = f;
        o[1] = bp_bin[off + k];
        o[2] = bp_cov[off + k];
    }
}

// break_and_update_ctgs, piece table (1122-1182): piece j of a fragment broken at bins b_1 < ... < b_k covers the bins
// [b_j, b_{j+1}) of the parent (b_0 = 0, b_{k+1} = nbins) and the bases [b_j*res, b_{j+1}*res) (the last one up to the
// parent's length).  The pieces become the next examined list.
__global__ void hh_k_correct_pieces(const int32_t* __restrict__ active, int32_t n_active, const int32_t* __restrict__ cnt,
                                    const int32_t* __restrict__ pbase, const int32_t* __restrict__ bp_bin, int64_t res,
                                    int32_t n_frag, int64_t* __restrict__ f_off, int32_t* __restrict__ f_nbins,
                                    int64_t* __restrict__ f_len, int64_t* __restrict__ f_start, int32_t* __restrict__ act_pos,
                                    int32_t* __restrict__ next_active) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_active || cnt[a] == 0) return;
    const int f = active[a];
    const int64_t off = f_off[f], len = f_len[f], start = f_start[f];
    const int32_t nb = f_nbins[f];
    const int k = cnt[a];
    int32_t prev = 0;
    for (int j = 0; j <= k; ++j) {
        const int32_t next = j < k ? bp_bin[off + j] : nb;
        const int id = n_frag + pbase[a] + j;
        f_off[id] = off + prev;
        f_nbins[id] = next - prev;
        f_len[id] = (j < k ? (int64_t)next * res : len) - (int64_t)prev * res;
        f_start[id] = start + (int64_t)prev * res;
        act_pos[id] = pbase[a] + j;
        next_active[pbase[a] + j] = id;
        prev = next;
    }
}

// break_and_update_ctgs, links (1079-1113).  A link of a fragment that was not broken takes no further part (1195-1197).
// Non-zero breakpoint (there is exactly one): a link whose closed(lo, hi) overlaps closed(bp, bp + res) is subtracted from
// the parent's coverage over [lo//res, hi//res] (1089-1092) and dropped.  Every other link moves to the piece holding both
// ends, at shifted coordinates (pos_shift, 1036-1052).  pos_shift names a piece of a fragment that does not start at 1 with
// an unshifted upper bound unless it is the last piece (1050): such links are filed under a name no fragment has, i.e.
// dropped here.  Ends in two pieces are dropped (1099).
// Not reproduced: in the reference such a wrong name '{raw}:{p+start}-{next_p}' is a plain dict key, and a later round
// could create a real fragment of exactly that name (piece j broken again at a multiple of res that equals its shift);
// the stale links would then count in that fragment two rounds later.  It needs five or more rounds and that exact
// geometry; here those links are gone for good.
__global__ void __launch_bounds__(256)
hh_k_correct_links(int64_t n_links, int32_t* __restrict__ l_frag, int32_t* __restrict__ l_lo, int32_t* __restrict__ l_hi,
                   const int32_t* __restrict__ act_pos, const int32_t* __restrict__ cnt, const int32_t* __restrict__ pbase,
                   const int64_t* __restrict__ f_off, const int32_t* __restrict__ f_nbins, const int64_t* __restrict__ f_start,
                   const int32_t* __restrict__ bp_bin, const int32_t* __restrict__ bp_cov, int64_t res, int32_t n_frag,
                   int32_t* __restrict__ diff) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_links; t += (int64_t)gridDim.x * blockDim.x) {
        const int f = l_frag[t];
        if (f < 0) continue;
        const int a = act_pos[f];
        const int k = cnt[a];
        if (k == 0) {
            l_frag[t] = -1;
            continue;
        }
        const int64_t off = f_off[f];
        const int64_t lo = l_lo[t], hi = l_hi[t];
        if (bp_cov[off] != 0) {
            const int64_t bp = (int64_t)bp_bin[off] * res;
            if (lo <= bp + res && hi >= bp) {
                const int64_t nb = f_nbins[f];
                const int64_t s = hh_pyslice(hh_floordiv(lo, res), nb), e = hh_pyslice(hh_floordiv(hi, res) + 1, nb);
                if (s < e) {
                    atomicAdd(diff + off + s, -1);
                    atomicAdd(diff + off + e, 1);
                }
                l_frag[t] = -1;
                continue;
            }
        }
        int ji = 0, jj = 0;
        for (int m = 0; m < k; ++m) {
            const int64_t p = (int64_t)bp_bin[off + m] * res;
            ji += p <= lo;
            jj += p <= hi;
        }
        if (lo < 0 || ji != jj || (f_start[f] != 1 && ji < k)) {
            l_frag[t] = -1;
            continue;
        }
        const int64_t p = ji ? (int64_t)bp_bin[off + ji - 1] * res : 0;
        l_frag[t] = n_frag + pbase[a] + ji;
        l_lo[t] = (int32_t)(lo - p);
        l_hi[t] = (int32_t)(hi - p);
    }
}

// convert_ctg (1405-1411): the piece with the largest start <= pos, at pos - start.  Unbroken contigs only change id
// (fa_dict is re-ordered); ids outside the FASTA stay as they are.
__global__ void __launch_bounds__(256)
hh_k_correct_remap(const int4* rec, int4* out, int64_t n_rec, int32_t n_ctg,
                   const int32_t* __restrict__ src_base, const int64_t* __restrict__ piece_start,
                   const int32_t* __restrict__ piece_id) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rec; i += (int64_t)gridDim.x * blockDim.x) {
        int4 r = rec[i];                           // (rec may alias out)
        int* end[2][2] = {{&r.x, &r.y}, {&r.z, &r.w}};
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const int c = *end[s][0];
            if ((unsigned)c >= (unsigned)n_ctg) continue;
            int lo = src_base[c], hi = src_base[c + 1] - 1;
            const int64_t pos = *end[s][1];
            while (lo < hi) {                     // last piece whose start <= pos
                const int mid = (lo + hi + 1) >> 1;
                if (piece_start[mid] <= pos) lo = mid;
                else hi = mid - 1;
            }
            *end[s][0] = piece_id[lo];
            *end[s][1] = (int)(pos - piece_start[lo]);
        }
        out[i] = r;
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int hh_grid(hh_ctx* ctx, int64_t n, int block) {
    const int64_t want = (n + block - 1) / block;
    const int64_t cap = (int64_t)ctx->sm_count * 8;
    return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

template <typename T>
static int hh_grow(T** p, int64_t used, int64_t cap_new) {
    T* q = nullptr;
    HH_CHECK(hh_dmalloc(&q, (size_t)cap_new));
    if (*p && used) HH_CUDA(cudaMemcpyAsync(q, *p, (size_t)used * sizeof(T), cudaMemcpyDeviceToDevice, hh_tls_ctx->stream));
    hh_dfree(*p);
    *p = q;
    return HH_OK;
}

static int hh_cub_reserve(hh_correct* cr, size_t bytes) {
    if (bytes <= cr->cub_bytes) return HH_OK;
    char* p = (char*)cr->d_cub;
    hh_dfree(p);
    cr->d_cub = nullptr;
    HH_CHECK(hh_dmalloc(&p, bytes));
    cr->d_cub = p;
    cr->cub_bytes = bytes;
    return HH_OK;
}

static int hh_correct_exclusive_scan(hh_correct* cr, const int32_t* in, int32_t* out, int n) {
    size_t bytes = 0;
    HH_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, n, cr->ctx->stream));
    HH_CHECK(hh_cub_reserve(cr, bytes));
    HH_CUDA(cub::DeviceScan::ExclusiveSum(cr->d_cub, bytes, in, out, n, cr->ctx->stream));
    return HH_OK;
}

// d_cov += inclusive_scan(d_diff); d_diff is cleared for the next use
static int hh_correct_apply_diff(hh_correct* cr) {
    hh_ctx* ctx = cr->ctx;
    const int n = (int)cr->total_bins;
    size_t bytes = 0;
    HH_CUDA(cub::DeviceScan::InclusiveSum(nullptr, bytes, cr->d_diff, cr->d_sorted, n, ctx->stream));
    HH_CHECK(hh_cub_reserve(cr, bytes));
    HH_CUDA(cub::DeviceScan::InclusiveSum(cr->d_cub, bytes, cr->d_diff, cr->d_sorted, n, ctx->stream));
    HH_LAUNCH(ctx, hh_k_correct_add_scan, hh_grid(ctx, n, 256), 256, 0, cr->d_cov, cr->d_sorted, (int64_t)n);
    HH_CUDA(cudaMemsetAsync(cr->d_diff, 0, (size_t)(n + 1) * sizeof(int32_t), ctx->stream));
    return HH_OK;
}

static void hh_correct_free(hh_correct* cr) {
    hh_dfree(cr->d_cov);
    hh_dfree(cr->d_diff);
    hh_dfree(cr->d_sorted);
    hh_dfree(cr->d_bp_bin);
    hh_dfree(cr->d_bp_cov);
    hh_dfree(cr->d_f_off);
    hh_dfree(cr->d_f_nbins);
    hh_dfree(cr->d_f_len);
    hh_dfree(cr->d_f_start);
    hh_dfree(cr->d_act_pos);
    hh_dfree(cr->d_active);
    hh_dfree(cr->d_cnt);
    hh_dfree(cr->d_bpos);
    hh_dfree(cr->d_pcnt);
    hh_dfree(cr->d_pbase);
    hh_dfree(cr->d_l_frag);
    hh_dfree(cr->d_l_lo);
    hh_dfree(cr->d_l_hi);
    hh_dfree(cr->d_counter);
    hh_dfree(cr->d_src_base);
    hh_dfree(cr->d_piece_start);
    hh_dfree(cr->d_piece_id);
    hh_dfree(cr->d_stage);
    char* p = (char*)cr->d_cub;
    hh_dfree(p);
}

static int hh_correct_alloc_active(hh_correct* cr, int32_t n) {
    hh_dfree(cr->d_active);
    hh_dfree(cr->d_cnt);
    hh_dfree(cr->d_bpos);
    hh_dfree(cr->d_pcnt);
    hh_dfree(cr->d_pbase);
    HH_CHECK(hh_dmalloc(&cr->d_active, (size_t)n + 1));
    HH_CHECK(hh_dmalloc(&cr->d_cnt, (size_t)n + 1));
    HH_CHECK(hh_dmalloc(&cr->d_bpos, (size_t)n + 1));
    HH_CHECK(hh_dmalloc(&cr->d_pcnt, (size_t)n + 1));
    HH_CHECK(hh_dmalloc(&cr->d_pbase, (size_t)n + 1));
    HH_CUDA(cudaMemsetAsync(cr->d_cnt, 0, ((size_t)n + 1) * sizeof(int32_t), hh_tls_ctx->stream));
    cr->n_active = n;
    return HH_OK;
}

extern "C" {

// parse_pairs_for_correction / parse_bam_for_correction (1307-1311, 1370-1374): one int32 array of len//res + 1 bins per
// contig.  The whole coverage buffer is addressed with int32 offsets: at most 2^31 - 1 bins in all.
int hh_correct_create(hh_ctx* ctx, int32_t n_ctg, const int64_t* ctg_len, int64_t resolution, hh_correct** out) {
    HH_REQUIRE(ctx && ctg_len && out && n_ctg > 0 && resolution > 0, HH_ERR_ARG, "hh_correct_create: bad arguments");
    hh_scope sc(ctx);
    std::vector<int64_t> off(n_ctg), len(ctg_len, ctg_len + n_ctg), start(n_ctg, 1);
    std::vector<int32_t> nb(n_ctg), act(n_ctg), pos(n_ctg);
    int64_t total = 0;
    for (int32_t c = 0; c < n_ctg; ++c) {
        HH_REQUIRE(ctg_len[c] >= 0, HH_ERR_ARG, "hh_correct_create: negative contig length");
        off[c] = total;
        nb[c] = (int32_t)(ctg_len[c] / resolution + 1);
        total += nb[c];
        act[c] = c;
        pos[c] = c;
    }
    HH_REQUIRE(total < INT_MAX, HH_ERR_ARG, "hh_correct_create: %lld coverage bins exceed the int32 range",
               (long long)total);
    hh_correct* cr = new (std::nothrow) hh_correct();
    HH_REQUIRE(cr, HH_ERR_NOMEM, "hh_correct_create: out of host memory");
    cr->ctx = ctx;
    cr->n_ctg = n_ctg;
    cr->res = resolution;
    cr->total_bins = total;
    cr->n_frag = n_ctg;
    cr->f_cap = n_ctg;
    int rc = HH_OK;
#define HH_TRY(expr)                  \
    do {                              \
        rc = (expr);                  \
        if (rc != HH_OK) goto fail;   \
    } while (0)
    HH_TRY(hh_dmalloc(&cr->d_cov, (size_t)total));
    HH_TRY(hh_dmalloc(&cr->d_diff, (size_t)total + 1));
    HH_TRY(hh_dmalloc(&cr->d_sorted, (size_t)total));
    HH_TRY(hh_dmalloc(&cr->d_bp_bin, (size_t)total));
    HH_TRY(hh_dmalloc(&cr->d_bp_cov, (size_t)total));
    HH_TRY(hh_dmalloc(&cr->d_f_off, (size_t)n_ctg));
    HH_TRY(hh_dmalloc(&cr->d_f_nbins, (size_t)n_ctg));
    HH_TRY(hh_dmalloc(&cr->d_f_len, (size_t)n_ctg));
    HH_TRY(hh_dmalloc(&cr->d_f_start, (size_t)n_ctg));
    HH_TRY(hh_dmalloc(&cr->d_act_pos, (size_t)n_ctg));
    HH_TRY(hh_dmalloc(&cr->d_counter, 1));
    HH_TRY(hh_correct_alloc_active(cr, n_ctg));
#undef HH_TRY
    {
        cudaStream_t s = ctx->stream;
        cudaError_t e = cudaSuccess;
        if (e == cudaSuccess) e = cudaMemsetAsync(cr->d_cov, 0, (size_t)total * sizeof(int32_t), s);
        if (e == cudaSuccess) e = cudaMemsetAsync(cr->d_diff, 0, ((size_t)total + 1) * sizeof(int32_t), s);
        if (e == cudaSuccess) e = cudaMemsetAsync(cr->d_counter, 0, sizeof(unsigned long long), s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(cr->d_f_off, off.data(), n_ctg * sizeof(int64_t), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(cr->d_f_nbins, nb.data(), n_ctg * sizeof(int32_t), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(cr->d_f_len, len.data(), n_ctg * sizeof(int64_t), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(cr->d_f_start, start.data(), n_ctg * sizeof(int64_t), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(cr->d_active, act.data(), n_ctg * sizeof(int32_t), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaMemcpyAsync(cr->d_act_pos, pos.data(), n_ctg * sizeof(int32_t), cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);     // the host vectors die on return
        if (e != cudaSuccess) {
            hh_set_error("hh_correct_create: %s", cudaGetErrorString(e));
            rc = HH_ERR_CUDA;
            goto fail;
        }
    }
    *out = cr;
    return HH_OK;
fail:
    hh_correct_free(cr);
    delete cr;
    return rc;
}

// one batch of records {ctg_a, pos_a, ctg_b, pos_b} (0-based) for the coverage pass (1321-1342 / 1380-1396); records of
// two contigs or of contigs outside the FASTA are ignored, so the whole read1 stream may be passed
int hh_correct_add(hh_correct* cr, const int32_t* rec, int64_t n_rec, int mem) {
    HH_REQUIRE(cr && (rec || n_rec == 0) && n_rec >= 0, HH_ERR_ARG, "hh_correct_add: bad arguments");
    HH_REQUIRE(!cr->cov_ready, HH_ERR_STATE, "hh_correct_add: the rounds have started");
    if (n_rec == 0) return HH_OK;
    hh_ctx* ctx = cr->ctx;
    hh_scope sc(ctx);
    if (cr->n_links + n_rec > cr->l_cap) {
        int64_t cap = cr->l_cap ? cr->l_cap : (1 << 20);
        while (cap < cr->n_links + n_rec) cap *= 2;
        HH_CHECK(hh_grow(&cr->d_l_frag, cr->n_links, cap));
        HH_CHECK(hh_grow(&cr->d_l_lo, cr->n_links, cap));
        HH_CHECK(hh_grow(&cr->d_l_hi, cr->n_links, cap));
        cr->l_cap = cap;
    }
    const int4* d_rec = reinterpret_cast<const int4*>(rec);
    if (mem == HH_MEM_HOST) {
        if (n_rec > cr->stage_cap) {
            hh_dfree(cr->d_stage);
            HH_CHECK(hh_dmalloc(&cr->d_stage, (size_t)n_rec));
            cr->stage_cap = n_rec;
        }
        HH_CUDA(cudaMemcpyAsync(cr->d_stage, rec, (size_t)n_rec * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
        d_rec = cr->d_stage;
    }
    HH_LAUNCH(ctx, hh_k_correct_cov, hh_grid(ctx, n_rec, 256), 256, 0, d_rec, n_rec, cr->n_ctg, cr->res, cr->d_f_off,
              cr->d_f_nbins, cr->d_diff, cr->d_l_frag, cr->d_l_lo, cr->d_l_hi, cr->d_counter);
    unsigned long long n_links = 0;
    HH_CUDA(cudaMemcpyAsync(&n_links, cr->d_counter, sizeof(n_links), cudaMemcpyDeviceToHost, ctx->stream));
    HH_CUDA(cudaStreamSynchronize(ctx->stream));
    cr->n_links = (int64_t)n_links;
    return HH_OK;
}

// One round of correct_assembly (1210-1243): detect_break_points on every fragment under examination, then -- unless
// last_round -- the coverage / link updates of break_and_update_ctgs, after which the pieces are the fragments under
// examination (their ids: n_frag, n_frag + 1, ... in breakpoint-list order, left to right).
int hh_correct_round(hh_correct* cr, double median_cov_ratio, double region_len_ratio, int64_t min_region_cutoff,
                     int last_round, hh_correct_round_info* info) {
    HH_REQUIRE(cr && info, HH_ERR_ARG, "hh_correct_round: bad arguments");
    hh_ctx* ctx = cr->ctx;
    hh_scope sc(ctx);
    cudaStream_t s = ctx->stream;
    if (!cr->cov_ready) {
        HH_CHECK(hh_correct_apply_diff(cr));
        cr->cov_ready = true;
    }
    memset(info, 0, sizeof(*info));
    const int32_t na = cr->n_active;
    info->n_examined = na;
    info->n_frag = cr->n_frag;
    if (na == 0) return HH_OK;
    // medians: segmented sort of a copy of the examined slices
    int32_t *seg_b = nullptr, *seg_e = nullptr;
    HH_CHECK(hh_dmalloc(&seg_b, (size_t)na));
    HH_CHECK(hh_dmalloc(&seg_e, (size_t)na));
    HH_LAUNCH(ctx, hh_k_correct_segments, (na + 255) / 256, 256, 0, cr->d_active, na, cr->d_f_off, cr->d_f_nbins, seg_b, seg_e);
    size_t bytes = 0;
    HH_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, bytes, cr->d_cov, cr->d_sorted, (int)cr->total_bins, na, seg_b, seg_e, s));
    HH_CHECK(hh_cub_reserve(cr, bytes));
    HH_CUDA(cub::DeviceSegmentedSort::SortKeys(cr->d_cub, bytes, cr->d_cov, cr->d_sorted, (int)cr->total_bins, na, seg_b, seg_e, s));
    HH_LAUNCH(ctx, hh_k_correct_detect, (na + 127) / 128, 128, 0, cr->d_active, na, cr->d_f_off, cr->d_f_nbins, cr->d_f_len,
              cr->d_cov, cr->d_sorted, cr->res, median_cov_ratio, region_len_ratio, min_region_cutoff, cr->d_bp_bin,
              cr->d_bp_cov, cr->d_cnt);
    hh_dfree(seg_b);
    hh_dfree(seg_e);
    HH_CHECK(hh_correct_exclusive_scan(cr, cr->d_cnt, cr->d_bpos, na + 1));
    HH_LAUNCH(ctx, hh_k_correct_piece_counts, (na + 1 + 255) / 256, 256, 0, cr->d_cnt, na, cr->d_pcnt);
    HH_CHECK(hh_correct_exclusive_scan(cr, cr->d_pcnt, cr->d_pbase, na + 1));
    int32_t totals[2];
    HH_CUDA(cudaMemcpyAsync(&totals[0], cr->d_bpos + na, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    HH_CUDA(cudaMemcpyAsync(&totals[1], cr->d_pbase + na, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    HH_CUDA(cudaStreamSynchronize(s));
    const int32_t n_breaks = totals[0], n_pieces = totals[1];
    info->n_breaks = n_breaks;
    info->n_broken = n_pieces - n_breaks;          // a broken fragment has one piece more than breakpoints
    info->n_links = cr->n_links;
    cr->breaks.assign(3 * (size_t)n_breaks, 0);
    if (n_breaks == 0) return HH_OK;
    int32_t* brk = nullptr;
    HH_CHECK(hh_dmalloc(&brk, 3 * (size_t)n_breaks));
    HH_LAUNCH(ctx, hh_k_correct_compact, (na + 127) / 128, 128, 0, cr->d_active, na, cr->d_f_off, cr->d_cnt, cr->d_bpos,
              cr->d_bp_bin, cr->d_bp_cov, brk);
    HH_CUDA(cudaMemcpyAsync(cr->breaks.data(), brk, 3 * (size_t)n_breaks * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    HH_CUDA(cudaStreamSynchronize(s));
    hh_dfree(brk);
    if (last_round) return HH_OK;                  // 1233-1236: the last round only updates fa_dict and the break tables
    if ((int64_t)cr->n_frag + n_pieces > cr->f_cap) {
        int64_t cap = (int64_t)cr->f_cap * 2;
        if (cap < (int64_t)cr->n_frag + n_pieces) cap = (int64_t)cr->n_frag + n_pieces;
        HH_REQUIRE(cap < INT_MAX, HH_ERR_CAPACITY, "hh_correct_round: too many fragments");
        HH_CHECK(hh_grow(&cr->d_f_off, cr->n_frag, cap));
        HH_CHECK(hh_grow(&cr->d_f_nbins, cr->n_frag, cap));
        HH_CHECK(hh_grow(&cr->d_f_len, cr->n_frag, cap));
        HH_CHECK(hh_grow(&cr->d_f_start, cr->n_frag, cap));
        HH_CHECK(hh_grow(&cr->d_act_pos, cr->n_frag, cap));
        cr->f_cap = (int32_t)cap;
    }
    int32_t* next_active = nullptr;
    HH_CHECK(hh_dmalloc(&next_active, (size_t)n_pieces));
    HH_LAUNCH(ctx, hh_k_correct_pieces, (na + 127) / 128, 128, 0, cr->d_active, na, cr->d_cnt, cr->d_pbase, cr->d_bp_bin,
              cr->res, cr->n_frag, cr->d_f_off, cr->d_f_nbins, cr->d_f_len, cr->d_f_start, cr->d_act_pos, next_active);
    if (cr->n_links)
        HH_LAUNCH(ctx, hh_k_correct_links, hh_grid(ctx, cr->n_links, 256), 256, 0, cr->n_links, cr->d_l_frag, cr->d_l_lo,
                  cr->d_l_hi, cr->d_act_pos, cr->d_cnt, cr->d_pbase, cr->d_f_off, cr->d_f_nbins, cr->d_f_start, cr->d_bp_bin,
                  cr->d_bp_cov, cr->res, cr->n_frag, cr->d_diff);
    HH_CHECK(hh_correct_apply_diff(cr));
    // only the pieces are examined in the next round (1192-1197)
    HH_CHECK(hh_correct_alloc_active(cr, n_pieces));
    HH_CUDA(cudaMemcpyAsync(cr->d_active, next_active, (size_t)n_pieces * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    HH_CUDA(cudaStreamSynchronize(s));
    hh_dfree(next_active);
    cr->n_frag += n_pieces;
    return HH_OK;
}

int hh_correct_fetch_breaks(hh_correct* cr, int32_t* frag, int32_t* bin, int32_t* cov) {
    HH_REQUIRE(cr, HH_ERR_ARG, "hh_correct_fetch_breaks: bad arguments");
    const size_t n = cr->breaks.size() / 3;
    for (size_t k = 0; k < n; ++k) {
        if (frag) frag[k] = cr->breaks[3 * k];
        if (bin) bin[k] = cr->breaks[3 * k + 1];
        if (cov) cov[k] = cr->breaks[3 * k + 2];
    }
    return HH_OK;
}

int hh_correct_info(hh_correct* cr, int32_t* n_active, int64_t* active_bins, int64_t* n_links) {
    HH_REQUIRE(cr, HH_ERR_ARG, "hh_correct_info: bad arguments");
    hh_scope sc(cr->ctx);
    if (n_active) *n_active = cr->n_active;
    if (n_links) *n_links = cr->n_links;
    if (active_bins) {
        std::vector<int32_t> act(cr->n_active), nb(cr->f_cap);
        HH_CUDA(cudaMemcpyAsync(act.data(), cr->d_active, act.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, cr->ctx->stream));
        HH_CUDA(cudaMemcpyAsync(nb.data(), cr->d_f_nbins, (size_t)cr->n_frag * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                cr->ctx->stream));
        HH_CUDA(cudaStreamSynchronize(cr->ctx->stream));
        int64_t t = 0;
        for (int32_t f : act) t += nb[f];
        *active_bins = t;
    }
    return HH_OK;
}

int hh_correct_fetch_cov(hh_correct* cr, int32_t* frag, int32_t* nbins, int32_t* cov) {
    HH_REQUIRE(cr && frag && nbins && cov, HH_ERR_ARG, "hh_correct_fetch_cov: bad arguments");
    hh_scope sc(cr->ctx);
    cudaStream_t s = cr->ctx->stream;
    if (!cr->cov_ready) {
        HH_CHECK(hh_correct_apply_diff(cr));
        cr->cov_ready = true;
    }
    std::vector<int64_t> off(cr->n_frag);
    std::vector<int32_t> nb(cr->n_frag);
    HH_CUDA(cudaMemcpyAsync(frag, cr->d_active, (size_t)cr->n_active * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    HH_CUDA(cudaMemcpyAsync(off.data(), cr->d_f_off, off.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    HH_CUDA(cudaMemcpyAsync(nb.data(), cr->d_f_nbins, nb.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    HH_CUDA(cudaStreamSynchronize(s));
    int64_t at = 0;
    for (int32_t a = 0; a < cr->n_active; ++a) {
        const int32_t f = frag[a];
        nbins[a] = nb[f];
        HH_CUDA(cudaMemcpyAsync(cov + at, cr->d_cov + off[f], (size_t)nb[f] * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        at += nb[f];
    }
    HH_CUDA(cudaStreamSynchronize(s));
    return HH_OK;
}

// The piece table of the corrected assembly (final_break_pos_dict / final_break_frag_dict, decided on the host): source
// contig c owns the entries [src_base[c], src_base[c+1]), ascending starts; an unbroken contig has one entry (start 0)
// holding its id in the corrected fa_dict.
int hh_correct_set_layout(hh_correct* cr, const int32_t* src_base, const int64_t* piece_start, const int32_t* piece_id,
                          int32_t n_pieces) {
    HH_REQUIRE(cr && src_base && piece_start && piece_id && n_pieces > 0, HH_ERR_ARG, "hh_correct_set_layout: bad arguments");
    for (int32_t c = 0; c < cr->n_ctg; ++c)
        HH_REQUIRE(src_base[c] < src_base[c + 1], HH_ERR_ARG, "hh_correct_set_layout: contig %d has no piece", c);
    HH_REQUIRE(src_base[0] == 0 && src_base[cr->n_ctg] == n_pieces, HH_ERR_ARG, "hh_correct_set_layout: bad src_base");
    hh_scope sc(cr->ctx);
    cudaStream_t s = cr->ctx->stream;
    hh_dfree(cr->d_src_base);
    hh_dfree(cr->d_piece_start);
    hh_dfree(cr->d_piece_id);
    HH_CHECK(hh_dmalloc(&cr->d_src_base, (size_t)cr->n_ctg + 1));
    HH_CHECK(hh_dmalloc(&cr->d_piece_start, (size_t)n_pieces));
    HH_CHECK(hh_dmalloc(&cr->d_piece_id, (size_t)n_pieces));
    HH_CUDA(cudaMemcpyAsync(cr->d_src_base, src_base, ((size_t)cr->n_ctg + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    HH_CUDA(cudaMemcpyAsync(cr->d_piece_start, piece_start, (size_t)n_pieces * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    HH_CUDA(cudaMemcpyAsync(cr->d_piece_id, piece_id, (size_t)n_pieces * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    HH_CUDA(cudaStreamSynchronize(s));
    cr->n_pieces = n_pieces;
    return HH_OK;
}

// records of the original stream -> records in the corrected name space (rec_in and rec_out both in `mem`; may alias)
int hh_correct_remap(hh_correct* cr, const int32_t* rec_in, int32_t* rec_out, int64_t n_rec, int mem) {
    HH_REQUIRE(cr && n_rec >= 0 && (n_rec == 0 || (rec_in && rec_out)), HH_ERR_ARG, "hh_correct_remap: bad arguments");
    HH_REQUIRE(cr->n_pieces > 0, HH_ERR_STATE, "hh_correct_remap: hh_correct_set_layout has not been called");
    if (n_rec == 0) return HH_OK;
    hh_ctx* ctx = cr->ctx;
    hh_scope sc(ctx);
    const int4* d_in = reinterpret_cast<const int4*>(rec_in);
    int4* d_out = reinterpret_cast<int4*>(rec_out);
    if (mem == HH_MEM_HOST) {
        if (n_rec > cr->stage_cap) {
            hh_dfree(cr->d_stage);
            HH_CHECK(hh_dmalloc(&cr->d_stage, (size_t)n_rec));
            cr->stage_cap = n_rec;
        }
        HH_CUDA(cudaMemcpyAsync(cr->d_stage, rec_in, (size_t)n_rec * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
        d_in = d_out = cr->d_stage;
    }
    HH_LAUNCH(ctx, hh_k_correct_remap, hh_grid(ctx, n_rec, 256), 256, 0, d_in, d_out, n_rec, cr->n_ctg, cr->d_src_base,
              cr->d_piece_start, cr->d_piece_id);
    if (mem == HH_MEM_HOST)
        HH_CUDA(cudaMemcpyAsync(rec_out, cr->d_stage, (size_t)n_rec * sizeof(int4), cudaMemcpyDeviceToHost, ctx->stream));
    HH_CUDA(cudaStreamSynchronize(ctx->stream));
    return HH_OK;
}

int hh_correct_destroy(hh_correct* cr) {
    if (!cr) return HH_OK;
    hh_scope sc(cr->ctx);
    hh_correct_free(cr);
    cudaStreamSynchronize(cr->ctx->stream);
    delete cr;
    return HH_OK;
}

}  // extern "C"
