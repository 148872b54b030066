// Link counting on the GPU: the per-read-pair loop of parse_alignments_for_ctgs
// (scripts/HapHiC_cluster.py:1596-1655) as a warp-aggregated atomic histogram over an
// open-addressing hash table keyed by the (name-ordered) contig pair.
//
// Per record (16 B, one 128-bit streaming load) the kernel
//   * drops ctg_a == ctg_b (generator filter, 1582 / 2862) and ids outside the FASTA (1625),
//   * orders the two ends by contig NAME rank (1629),
//   * evaluates is_flank on both 1-based coordinates and the Nx membership (1636, 299-307),
//   * evaluates the head/tail halves `coord*2 > len` (404-416),
//   * groups equal keys inside the warp with match.any so one lane issues the atomics for the
//     whole group (coordinate- or name-sorted inputs collapse 32 records into one update),
//   * updates {full, flank, HT, TH, TT} counters and the first-seen stream indices (dict
//     insertion order of full_link_dict / flank_link_dict) of the key's slot, and the two
//     per-fragment totals (ctg_link_dict, 1638-1639).
// hh_links_finish orders the distinct keys by first appearance with a scatter + stream
// compaction (no sort): order[first_full] = slot, then compact.
#include "hh_common.cuh"
#include "hh_internal.cuh"
#include <cub/cub.cuh>
#include <stdlib.h>
#include <algorithm>
#include <vector>

#define HH_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull
#define HH_NONE32 0xFFFFFFFFu

struct __align__(32) hh_slot {
    uint32_t first_full, first_flank, full, flank, ht, th, tt, pad;
};

struct hh_partset {
    void* buf;                       // [npart][pcap] records: hh_nrec when narrow, else int4 (see "partition records")
    bool narrow;
    unsigned long long* cursor;      // [npart] records written to every region (may exceed pcap: the excess went to the spill list)
    uint64_t pcap;                   // records per partition region
    int64_t sized_for, sent;         // records the set was sized for / sent to it so far
};

struct hh_links {
    hh_ctx* ctx;
    int32_t n_ctg;                   // key space: contigs, or fragments (contigs / bins) in fragment mode
    int64_t flank_bp;
    int32_t* d_len;                  // [n_ctg] lengths of the key-space objects
    int32_t* d_rank;                 // [n_ctg] name rank of the key-space objects
    uint8_t* d_nx;
    // fragment mode (parse_alignments, HapHiC_cluster.py:1658-1752): records name SOURCE contigs, keys are fragments
    int32_t n_src;                   // number of source contigs (= n_ctg in contig mode)
    int32_t* d_src_rank;             // [n_src] name rank of the source contigs
    int32_t* d_fbase;                // [n_src + 1] first fragment id of every contig (more than one fragment = split into bins)
    int64_t bin_size;
    unsigned long long* d_ctg;       // [n_ctg] per-fragment flank-link totals
    uint64_t* d_keys;                // [cap]
    hh_slot* d_vals;                 // [cap]
    uint64_t cap;                    // power of two
    unsigned long long* d_counters;  // [0] distinct keys  [1] records used  [2] overflow flag  [3] nnz_flank
                                     // [4] largest first-seen index merged from a peer
    int64_t n_records, stream_end;
    int64_t known_unique, since_known;   // growth bookkeeping (see ensure_capacity)
    bool finished;
    bool ordered;                    // d_compact is in dict insertion order (false after hh_links_finish_partition / hh_links_adopt)
    int64_t nnz, nnz_flank, n_used;
    int64_t peer_used;               // records counted by merged peers
    uint32_t* d_compact;             // [nnz][HH_E_WORDS]  {i, j, full, flank, first_full, first_flank, HT, TH, TT}
    // host staging (double-buffered H2D)
    int4* d_stage[2];
    cudaEvent_t ev_copied[2], ev_consumed[2];
    cudaStream_t copy_stream;
    int64_t stage_records;
    // partitioned counting (contig mode, long streams; see "partition, then aggregate" below)
    int mode;                        // 0 undecided, 1 direct (one big hash table), 2 partitioned
    int npart_log;                   // log2 of the number of partitions
    int kbits;                       // bits of j in the pair key (i << kbits) | j: the least with 2^kbits >= n_ctg
    std::vector<int32_t> set_bytes;  // record bytes of every partition set opened (hh_links_record_bytes)
    int32_t bucket_bytes;            // record bytes of the bucket buffer of the finish, 0 before it
    uint64_t scap;                   // slots of a shared-memory table, or of the fallback's global table when one ran
    int64_t agg_buckets, agg_smem, agg_fallback;   // buckets at finish / counted in shared memory / by the fallback
    uint64_t spill_cap;
    std::vector<hh_partset> psets;   // partition buffers; normally one set, a new one when a later add call outgrows it
    int4* d_spill;                   // wide records of partitions whose region overflowed (skewed keys)
    unsigned long long* d_spill_cursor;
    int64_t capacity_hint;
    // dict_to_matrix support
    int32_t* d_index;                // [n_ctg] matrix index of linked fragments (hh_links_linked_index)
    int32_t n_linked;
    uint8_t* d_keep;
    int32_t* d_hap;                  // [n_ctg] haplotype of every fragment (allocated on the first phased call)
    bool phased;                     // the last hh_links_linked_index_phased got a haplotype array
    int32_t* d_deg;                  // [n_ctg] entries of the (reduced) flank dict that touch each kept fragment
    int64_t n_pass;                  // entries of that dict between kept fragments: the matrix has 2 n_pass off-diagonal entries
    // what d_index / d_deg / n_pass were computed from: the index is reused while all of it is unchanged
    uint64_t gen;                    // bumped whenever d_compact or d_ctg is rewritten (finish, adopt, merge)
    bool ix_valid;
    uint64_t ix_gen;
    int ix_normalize;
    double ix_w;
    std::vector<uint8_t> ix_keep;
    std::vector<int32_t> ix_hap;     // empty: unphased
    // contig pairs joined by ultra-long reads (hh_links_set_ul_pairs): keys (i << 32 | j) ascending, the HT slot of each
    unsigned long long* d_ul_key = nullptr;
    int32_t* d_ul_slot = nullptr;
    int64_t n_ul = 0;
};

__device__ __forceinline__ uint64_t hh_mix64(uint64_t k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return k;
}

// find-or-insert; returns slot index, sets *inserted.  Returns cap (invalid) if the table is full.
__device__ __forceinline__ uint64_t hh_probe_insert(uint64_t* __restrict__ keys, uint64_t cap, uint64_t key, bool* inserted) {
    const uint64_t mask = cap - 1;
    uint64_t slot = hh_mix64(key) & mask;
    *inserted = false;
    for (uint64_t probes = 0; probes < cap; ++probes) {
        uint64_t k = *((volatile uint64_t*)(keys + slot));
        if (k == key) return slot;
        if (k == HH_EMPTY_KEY) {
            unsigned long long prev = atomicCAS((unsigned long long*)(keys + slot), (unsigned long long)HH_EMPTY_KEY,
                                                (unsigned long long)key);
            if (prev == HH_EMPTY_KEY) {
                *inserted = true;
                return slot;
            }
            if (prev == key) return slot;
        }
        slot = (slot + 1) & mask;
    }
    return cap;
}

__global__ void hh_k_links_init(uint64_t* __restrict__ keys, hh_slot* __restrict__ vals, uint64_t cap) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += stride) {
        keys[s] = HH_EMPTY_KEY;
        uint4* v = reinterpret_cast<uint4*>(vals + s);
        v[0] = make_uint4(HH_NONE32, HH_NONE32, 0u, 0u);
        v[1] = make_uint4(0u, 0u, 0u, 0u);
    }
}

// ---------------------------------------------------------------------------------------------
// What a record means: the ordered pair of key-space objects it links and three flags.  The partition records carry
// the flags in the low bits of their .w.
// ---------------------------------------------------------------------------------------------
#define HH_F_FLANK 1u              // both ends in a flank region of an Nx member (flank_link_dict)
#define HH_F_TI 2u                 // end i in the tail half of its object
#define HH_F_TJ 4u                 // end j in the tail half of its object

struct hh_pair {
    int a, b;                        // key-space ids, in key order
    unsigned flags;                  // HH_F_*
};

__device__ __forceinline__ uint64_t hh_pair_key(int a, int b) { return ((uint64_t)(uint32_t)a << 32) | (uint64_t)(uint32_t)b; }

__device__ __forceinline__ void hh_swap_ends(int& a, int& b, int& pa, int& pb) {
    int t = a; a = b; b = t;
    t = pa; pa = pb; pb = t;
}

// the ordered pair (a, b) with its 0-based positions -> *out
__device__ __forceinline__ void hh_pair_flags(int a, int b, int pa, int pb, const int32_t* __restrict__ ctg_len,
                                              const uint8_t* __restrict__ in_nx, int64_t flank_bp, hh_pair* out) {
    const int64_t coord_i = (int64_t)pa + 1, coord_j = (int64_t)pb + 1;   // 1-based
    const int64_t li = ctg_len[a], lj = ctg_len[b];
    const bool fi = (flank_bp == 0) || (coord_i <= flank_bp) || (coord_i > li - flank_bp);   // is_flank, 299-307
    const bool fj = (flank_bp == 0) || (coord_j <= flank_bp) || (coord_j > lj - flank_bp);
    out->a = a;
    out->b = b;
    out->flags = ((fi && fj && in_nx[a] && in_nx[b]) ? HH_F_FLANK : 0u)                         // 1636
                 | ((coord_i * 2 > li) ? HH_F_TI : 0u) | ((coord_j * 2 > lj) ? HH_F_TJ : 0u);   // 404-416
}

// contig mode: false = the record is not counted (same contig: generator filter, 1582 / 2862; ids outside the FASTA, 1625)
__device__ __forceinline__ bool hh_classify_contig(int4 r, int32_t n_ctg, const int32_t* __restrict__ ctg_len,
                                                   const int32_t* __restrict__ name_rank, const uint8_t* __restrict__ in_nx,
                                                   int64_t flank_bp, hh_pair* out) {
    int a = r.x, b = r.z, pa = r.y, pb = r.w;
    if (a == b || (unsigned)a >= (unsigned)n_ctg || (unsigned)b >= (unsigned)n_ctg) return false;
    if (name_rank[a] > name_rank[b]) hh_swap_ends(a, b, pa, pb);      // sorted(((ref,pos+1),(mref,mpos+1))), 1629
    hh_pair_flags(a, b, pa, pb, ctg_len, in_nx, flank_bp, out);
    return true;
}

// floor(x / d) for d > 0 (Python's //): bin number - 1 of the 0-based position x, ceil((x + 1) / d) - 1, for any x
__device__ __forceinline__ int64_t hh_floor_div(int64_t x, int64_t d) { return x >= 0 ? x / d : -((-x + d - 1) / d); }

// convert_frags (1662-1670) for one end on a split contig: the contig's first fragment f and the position p become the bin
// and the position inside it.  false = the position names a bin that does not exist
__device__ __forceinline__ bool hh_to_bin(int& f, int& p, int nbins, int64_t bin_size) {
    const int64_t nb = ((int64_t)p + 1 + bin_size - 1) / bin_size;
    const bool exists = p >= 0 && nb >= 1 && nb <= (int64_t)nbins;
    f += (int)(nb - 1);
    p = (int)((int64_t)p - (nb - 1) * bin_size);
    return exists;
}

// fragment mode (1696-1720): records name source contigs; a contig with several fragments is split into bins of bin_size
// bp.  ctg_len / name_rank / in_nx describe the fragments; ids are checked against fbase.  idx = the record's stream index.
__device__ __forceinline__ bool hh_classify_frag(int4 r, int32_t n_src, const int32_t* __restrict__ src_rank,
                                                 const int32_t* __restrict__ fbase, int64_t bin_size, const int32_t* __restrict__ ctg_len,
                                                 const int32_t* __restrict__ name_rank, const uint8_t* __restrict__ in_nx,
                                                 int64_t flank_bp, uint32_t idx, unsigned long long* __restrict__ counters,
                                                 hh_pair* out) {
    int a = r.x, b = r.z, pa = r.y, pb = r.w;
    if ((unsigned)a >= (unsigned)n_src || (unsigned)b >= (unsigned)n_src) return false;
    if (a == b && fbase[a + 1] - fbase[a] <= 1) return false;        // intra-contig pairs only matter for split contigs (1699)
    // sorted(((ref, pos+1), (mref, mpos+1))): by contig name, then by coordinate (1707)
    if (src_rank[a] > src_rank[b] || (a == b && pa > pb)) hh_swap_ends(a, b, pa, pb);
    int fa = fbase[a], fb = fbase[b];
    const int na = fbase[a + 1] - fa, nb = fbase[b + 1] - fb;
    // a position outside the contig (.pairs position 0, or beyond the last bin) names a bin that does not exist: the
    // reference dies with a KeyError on frag_len_dict['ctg_binK'] (1723); here the record is refused and hh_links_finish
    // reports it.  Both ends of an intra-contig record in the same bin number -- existing or not -- are one fragment, which
    // the reference skips (1715) before that lookup.
    if (a == b && hh_floor_div((int64_t)pa, bin_size) == hh_floor_div((int64_t)pb, bin_size)) return false;
    bool bad = false;
    if (na > 1) bad = !hh_to_bin(fa, pa, na, bin_size);
    if (nb > 1) bad = !hh_to_bin(fb, pb, nb, bin_size) || bad;
    if (bad) {
        atomicAdd(counters + 5, 1ull);
        atomicMax(counters + 6, (unsigned long long)idx + 1ull);
        return false;
    }
    if (fa == fb) return false;                                       // intra-bin links are not considered (1715)
    if ((na > 1 || nb > 1) && name_rank[fa] > name_rank[fb]) hh_swap_ends(fa, fb, pa, pb);   // sort by bin name (1719-1720)
    hh_pair_flags(fa, fb, pa, pb, ctg_len, in_nx, flank_bp, out);
    return true;
}

// ---------------------------------------------------------------------------------------------
// Folding a warp's records by key: the lanes that hold the same key form a group (match.any), and the group's lowest
// lane -- its leader -- gets the group's counts and first-seen indices and updates the key's slot alone.  Coordinate- or
// name-sorted inputs collapse 32 records into one update.
// ---------------------------------------------------------------------------------------------
struct hh_group {
    bool leader;
    uint32_t first_all, first_flank;     // smallest stream index of the group's records / of its flank records
    unsigned full, flank, ht, th, tt;    // records of the group per counter
};

// Called by all 32 lanes; a lane without a record (ok = false) joins no group.
__device__ __forceinline__ hh_group hh_warp_fold(bool ok, uint64_t key, uint32_t idx, unsigned flags) {
    const int lane = threadIdx.x & 31;
    if (!ok) key = HH_EMPTY_KEY - 1 - (uint64_t)lane;      // unique per lane: never groups, never a real key
    const unsigned peers = __match_any_sync(HH_FULL_MASK, key);
    const bool fl = ok && (flags & HH_F_FLANK), ti = (flags & HH_F_TI) != 0, tj = (flags & HH_F_TJ) != 0;
    hh_group g;
    g.first_all = __reduce_min_sync(peers, ok ? idx : HH_NONE32);
    g.first_flank = __reduce_min_sync(peers, fl ? idx : HH_NONE32);
    const unsigned b_fl = __ballot_sync(HH_FULL_MASK, fl);
    const unsigned b_ht = __ballot_sync(HH_FULL_MASK, ok && !ti && tj);
    const unsigned b_th = __ballot_sync(HH_FULL_MASK, ok && ti && !tj);
    const unsigned b_tt = __ballot_sync(HH_FULL_MASK, ok && ti && tj);
    g.leader = ok && lane == (__ffs(peers) - 1);
    g.full = __popc(peers);
    g.flank = __popc(peers & b_fl);
    g.ht = __popc(peers & b_ht);
    g.th = __popc(peers & b_th);
    g.tt = __popc(peers & b_tt);
    return g;
}

// A group's update of a slot of a global table: plain 32-bit reductions (fire and forget).
__device__ __forceinline__ void hh_slot_update(hh_slot* v, const hh_group& g) {
    atomicAdd(&v->full, g.full);
    atomicMin(&v->first_full, g.first_all);
    if (g.flank) {
        atomicAdd(&v->flank, g.flank);
        atomicMin(&v->first_flank, g.first_flank);
    }
    if (g.ht) atomicAdd(&v->ht, g.ht);
    if (g.th) atomicAdd(&v->th, g.th);
    if (g.tt) atomicAdd(&v->tt, g.tt);
}

__device__ __forceinline__ void hh_entry_store(uint32_t* __restrict__ o, uint64_t key, uint32_t full, uint32_t flank, uint32_t first_full,
                                               uint32_t first_flank, uint32_t ht, uint32_t th, uint32_t tt) {
    o[HH_E_I] = (uint32_t)(key >> 32);
    o[HH_E_J] = (uint32_t)key;
    o[HH_E_FULL] = full;
    o[HH_E_FLANK] = flank;
    o[HH_E_FIRST_FULL] = first_full;
    o[HH_E_FIRST_FLANK] = first_flank;
    o[HH_E_HT] = ht;
    o[HH_E_TH] = th;
    o[HH_E_TT] = tt;
}

// entry of a slot of a global table: v0 = {first_full, first_flank, full, flank}, v1 = {ht, th, tt, pad}
__device__ __forceinline__ void hh_entry_store(uint32_t* __restrict__ o, uint64_t key, uint4 v0, uint4 v1) {
    hh_entry_store(o, key, v0.z, v0.w, v0.x, v0.y, v1.x, v1.y, v1.z);
}

// Rank of this thread's `cnt` live items among those of its 256-thread block, in thread order, and the block's count.
// s_wtot is shared scratch of 8 words; the first barrier makes a call safe right after the previous one was used.
__device__ __forceinline__ unsigned int hh_block_rank(unsigned int cnt, unsigned int* s_wtot, unsigned int* total) {
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    unsigned int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned int t = __shfl_up_sync(HH_FULL_MASK, incl, o);
        if (lane >= o) incl += t;
    }
    __syncthreads();
    if (lane == 31) s_wtot[wv] = incl;
    __syncthreads();
    unsigned int before = 0, all = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const unsigned int t = s_wtot[k];
        before += (k < wv) ? t : 0u;
        all += t;
    }
    *total = all;
    return before + incl - cnt;
}

// load, classify, fold, probe, update
__global__ void __launch_bounds__(256)
hh_k_links_insert(const int4* __restrict__ rec, int64_t n_rec, uint32_t stream_off, int32_t n_ctg,
                  const int32_t* __restrict__ ctg_len, const int32_t* __restrict__ name_rank,
                  const uint8_t* __restrict__ in_nx, int64_t flank_bp, uint64_t* __restrict__ keys,
                  hh_slot* __restrict__ vals, uint64_t cap, unsigned long long* __restrict__ ctg_links,
                  unsigned long long* __restrict__ counters, const int32_t* __restrict__ src_rank,
                  const int32_t* __restrict__ fbase, int64_t bin_size, int32_t n_src, const uint32_t* __restrict__ pos) {
    __shared__ unsigned int s_new, s_used, s_over;
    if (threadIdx.x == 0) {
        s_new = 0;
        s_used = 0;
        s_over = 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int my_new = 0, my_used = 0;
    // warp-uniform loop bounds: every lane of a warp runs the same number of trips
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); i0 < n_rec; i0 += stride) {
        const int64_t i = i0 + lane;
        bool ok = i < n_rec;
        hh_pair p = {0, 0, 0u};
        uint32_t idx = HH_NONE32;
        if (ok) {
            const int4 r = hh_ld_stream(rec + i);
            // stream position of the record: implicit (contiguous shard) or carried along (routed records, any order)
            idx = pos ? pos[i] : stream_off + (uint32_t)i;
            ok = fbase == nullptr ? hh_classify_contig(r, n_ctg, ctg_len, name_rank, in_nx, flank_bp, &p)
                                  : hh_classify_frag(r, n_src, src_rank, fbase, bin_size, ctg_len, name_rank, in_nx, flank_bp, idx,
                                                     counters, &p);
        }
        if (ok) my_used++;
        const uint64_t key = hh_pair_key(p.a, p.b);
        const hh_group g = hh_warp_fold(ok, key, idx, p.flags);
        if (g.leader) {
            bool inserted;
            const uint64_t slot = hh_probe_insert(keys, cap, key, &inserted);
            if (slot >= cap) {
                s_over = 1;
            } else {
                if (inserted) my_new++;
                hh_slot_update(vals + slot, g);
                if (g.flank) {
                    atomicAdd(ctg_links + p.a, (unsigned long long)g.flank);
                    atomicAdd(ctg_links + p.b, (unsigned long long)g.flank);
                }
            }
        }
    }
    if (my_new) atomicAdd(&s_new, my_new);
    if (my_used) atomicAdd(&s_used, my_used);
    __syncthreads();
    if (threadIdx.x == 0) {
        if (s_new) atomicAdd(counters + 0, (unsigned long long)s_new);
        if (s_used) atomicAdd(counters + 1, (unsigned long long)s_used);
        if (s_over) atomicExch(counters + 2, 1ull);
    }
}

// ---------------------------------------------------------------------------------------------
// Partition, then aggregate.  One big hash table costs every record a random DRAM sector for the key and another
// read-modify-write for the counters (the table is two orders of magnitude larger than L2).  For long streams the
// records are therefore split twice by the high bits of the key hash: into 2^npart_log partition regions while they
// stream in, and at finish into 2^bucket_log buckets (the next hash bits, links_bucket_log) laid out densely.  A bucket
// (about 1.3k records at the benchmark's 200M records) is then sorted by pair in shared memory, its runs are reduced, and
// it is emitted as compact entries (9 words, the hh_links_adopt list format).  Integer adds and mins only: the result is identical to
// the direct path.
//   hh_k_part_scatter   record -> partition record (ends ordered by name rank, is_flank / head-tail evaluated once)
//   hh_k_part_hist      records per bucket (shared-memory histogram of a region's sub-buckets per tile)
//   hh_k_part_scatter2  the same pass again: every record to its place in the dense bucket buffer
//   hh_k_bucket_count   persistent CTAs: count one bucket at a time in shared memory (sort by pair, reduce the runs),
//                       emit its entries
//   hh_k_part_step      fallback for the buckets shared memory does not take: gathered, then counted in batches of
//                       about 2^19 records through global scratch tables
// ---------------------------------------------------------------------------------------------
#define HH_PART_TILE 4096          // wide records per tile of the scatter kernels (512 threads x 8), and spill records per tile
#define HH_PART_MAX 1024

// ---- partition records ------------------------------------------------------------------------------------------------
// Every usable record crosses device memory four times between the scatter and the count, so its width sets the cost of
// those passes.  Two formats:
//   wide   int4 {i, j, stream index, flags | partition << 8}: any key space and stream index (the partition is only
//          read by the scatter that wrote it, and is absent from records converted from the narrow format);
//   narrow hh_nrec, 8 bytes: high word the pair key (i << kbits) | j, low word flags << 29 | stream index.  It holds
//          what the count needs while kbits <= 16 (at most 65,536 objects) and stream indices are below 2^29.  Its
//          partition is not stored: the region it sits in implies it, and hh_bucket_of recomputes it from the key.
// A partition set is narrow when the call that opens it can use the narrow format (links_narrow); the bucket buffer of
// the finish is narrow when the whole stream can.  The spill list, shared by all sets and rarely used, stays wide.
#define HH_NREC_KBITS 16
#define HH_NREC_ZBITS 29
#define HH_NREC_ZEND (1ll << HH_NREC_ZBITS)     // narrow records carry stream indices below this

struct __align__(8) hh_nrec {
    unsigned long long v;
};

__device__ __forceinline__ int4 hh_ld_rec(const int4* p) { return hh_ld_stream(p); }
__device__ __forceinline__ hh_nrec hh_ld_rec(const hh_nrec* p) { return hh_nrec{hh_ld_stream_u64(&p->v)}; }

__device__ __forceinline__ uint32_t hh_rec_i(int4 r, int) { return (uint32_t)r.x; }
__device__ __forceinline__ uint32_t hh_rec_j(int4 r, int) { return (uint32_t)r.y; }
__device__ __forceinline__ uint32_t hh_rec_z(int4 r) { return (uint32_t)r.z; }
__device__ __forceinline__ unsigned hh_rec_flags(int4 r) { return (unsigned)r.w & 7u; }
__device__ __forceinline__ uint32_t hh_rec_i(hh_nrec r, int kbits) { return (uint32_t)(r.v >> 32) >> kbits; }
__device__ __forceinline__ uint32_t hh_rec_j(hh_nrec r, int kbits) { return (uint32_t)(r.v >> 32) & ((1u << kbits) - 1u); }
__device__ __forceinline__ uint32_t hh_rec_z(hh_nrec r) { return (uint32_t)r.v & (uint32_t)(HH_NREC_ZEND - 1); }
__device__ __forceinline__ unsigned hh_rec_flags(hh_nrec r) { return (uint32_t)r.v >> HH_NREC_ZBITS; }

__device__ __forceinline__ hh_nrec hh_nrec_make(uint32_t i, uint32_t j, uint32_t z, unsigned flags, int kbits) {
    return hh_nrec{((unsigned long long)((i << kbits) | j) << 32) | ((unsigned long long)flags << HH_NREC_ZBITS) | z};
}

// *d = s in the format of d
__device__ __forceinline__ void hh_rec_put(int4* d, int4 s, int) { *d = s; }
__device__ __forceinline__ void hh_rec_put(hh_nrec* d, hh_nrec s, int) { *d = s; }
__device__ __forceinline__ void hh_rec_put(int4* d, hh_nrec s, int kbits) {
    *d = make_int4((int)hh_rec_i(s, kbits), (int)hh_rec_j(s, kbits), (int)hh_rec_z(s), (int)hh_rec_flags(s));
}
__device__ __forceinline__ void hh_rec_put(hh_nrec* d, int4 s, int kbits) {
    *d = hh_nrec_make(hh_rec_i(s, kbits), hh_rec_j(s, kbits), hh_rec_z(s), hh_rec_flags(s), kbits);
}

__device__ __forceinline__ void hh_rec_set_z(int4* r, uint32_t z) { r->z = (int)z; }
__device__ __forceinline__ void hh_rec_set_z(hh_nrec* r, uint32_t z) { r->v = (r->v & ~(unsigned long long)(HH_NREC_ZEND - 1)) | z; }

// The scatter kernels stage a tile's records in dynamic shared memory, ordered by destination (partition, or sub-bucket),
// so that consecutive threads store the consecutive records of one run: a warp store then covers a few contiguous
// stretches instead of 32 lines.  64 KiB per CTA beside 12 or 32 KiB of static arrays: two CTAs per SM, as the
// registers x 512 threads allow anyway.
#define HH_STAGE_SMEM ((size_t)HH_PART_TILE * sizeof(int4))

// A bucket (or a partition: bucket_log = npart_log) is the top bucket_log bits of hh_mix64(key).
template <typename R>
__device__ __forceinline__ uint32_t hh_bucket_of(R r, int bucket_log, int kbits) {
    return (uint32_t)(hh_mix64(hh_pair_key((int)hh_rec_i(r, kbits), (int)hh_rec_j(r, kbits))) >> (64 - bucket_log));
}

// partition records of the scatter, and the partition of a staged one
__device__ __forceinline__ void hh_part_rec(int4* o, const hh_pair& pr, uint32_t z, unsigned p, int) {
    *o = make_int4(pr.a, pr.b, (int)z, (int)(pr.flags | (p << 8)));
}
__device__ __forceinline__ void hh_part_rec(hh_nrec* o, const hh_pair& pr, uint32_t z, unsigned, int kbits) {
    *o = hh_nrec_make((uint32_t)pr.a, (uint32_t)pr.b, z, pr.flags, kbits);
}
__device__ __forceinline__ unsigned hh_part_of(int4 r, int, int) { return (unsigned)r.w >> 8; }
__device__ __forceinline__ unsigned hh_part_of(hh_nrec r, int npart_log, int kbits) { return hh_bucket_of(r, npart_log, kbits); }

// records per tile of hh_k_part_scatter: the 64 KiB of staging, 512 threads x 8 wide or 16 narrow records (a run of a
// partition is then about 128 B long at 512 partitions either way)
template <typename R>
__host__ __device__ constexpr int hh_scatter_tile() { return (int)(HH_STAGE_SMEM / sizeof(R)); }

template <typename R>
__global__ void __launch_bounds__(512, 2)
hh_k_part_scatter(const int4* __restrict__ rec, int64_t n_rec, uint32_t stream_off, int32_t n_ctg, const int32_t* __restrict__ ctg_len,
                  const int32_t* __restrict__ name_rank, const uint8_t* __restrict__ in_nx, int64_t flank_bp, int npart_log, int kbits,
                  R* __restrict__ pbuf, uint64_t pcap, unsigned long long* __restrict__ cursor, int4* __restrict__ spill,
                  uint64_t spill_cap, unsigned long long* __restrict__ spill_cursor, unsigned long long* __restrict__ counters) {
    constexpr int TILE = hh_scatter_tile<R>(), ITEMS = TILE / 512;
    extern __shared__ int4 s_stage_mem[];
    R* s_stage = reinterpret_cast<R*>(s_stage_mem);  // TILE records, ordered by partition
    __shared__ unsigned int s_cnt[HH_PART_MAX];      // records of the tile per partition, then their exclusive prefix
    __shared__ unsigned long long s_base[HH_PART_MAX];
    __shared__ unsigned int s_wtot[16];
    __shared__ unsigned int s_used;
    const int npart = 1 << npart_log;
    const int64_t tiles = (n_rec + TILE - 1) / TILE;
    unsigned int my_used = 0;
    if (threadIdx.x == 0) s_used = 0;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        for (int k = threadIdx.x; k < npart; k += 512) s_cnt[k] = 0;
        __syncthreads();
        // Until it is staged, a record holds partition << 13 | its rank in the tile's run of that partition (< 2^13) in
        // place of its stream index, which its place in the tile implies: no registers beside the records.
        R out[ITEMS];
        uint32_t live = 0;                              // bit k: out[k] holds a record
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            const int64_t i = t * TILE + (int64_t)k * 512 + threadIdx.x;
            if (i < n_rec) {
                hh_pair pr;
                if (hh_classify_contig(hh_ld_stream(rec + i), n_ctg, ctg_len, name_rank, in_nx, flank_bp, &pr)) {
                    const unsigned p = (unsigned)(hh_mix64(hh_pair_key(pr.a, pr.b)) >> (64 - npart_log));
                    hh_part_rec(&out[k], pr, (p << 13) | atomicAdd(&s_cnt[p], 1u), p, kbits);
                    live |= 1u << k;
                    my_used++;
                }
            }
        }
        __syncthreads();
        for (int k = threadIdx.x; k < npart; k += 512)
            if (s_cnt[k]) s_base[k] = atomicAdd(cursor + k, (unsigned long long)s_cnt[k]);
        const unsigned int n_tile = hh_tile_scan(s_cnt, npart, s_wtot);
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            if (!((live >> k) & 1u)) continue;
            const uint32_t at = hh_rec_z(out[k]);
            hh_rec_set_z(&out[k], stream_off + (uint32_t)(t * TILE + k * 512 + threadIdx.x));
            s_stage[s_cnt[at >> 13] + (at & 0x1FFFu)] = out[k];
        }
        __syncthreads();
        // staged record e is number e - s_cnt[p] of the tile's run in partition p
        for (unsigned int e = threadIdx.x; e < n_tile; e += 512) {
            const R r = s_stage[e];
            const unsigned int p = hh_part_of(r, npart_log, kbits);
            const unsigned long long q = s_base[p] + (e - s_cnt[p]);
            if (q < pcap) {
                pbuf[(size_t)p * (size_t)pcap + (size_t)q] = r;
            } else {
                // the region of this partition is full (a few pairs own a large share of the stream): spill list
                const unsigned long long sq = atomicAdd(spill_cursor, 1ull);
                if (sq < spill_cap) hh_rec_put(spill + sq, r, kbits);
                else atomicExch(counters + 2, 3ull);
            }
        }
        __syncthreads();
    }
    my_used = (unsigned)hh_warp_sum((int)my_used);
    if ((threadIdx.x & 31) == 0 && my_used) atomicAdd(&s_used, my_used);
    __syncthreads();
    if (threadIdx.x == 0 && s_used) atomicAdd(counters + 1, (unsigned long long)s_used);
}

// ---- level 2: buckets -------------------------------------------------------------------------------------------------
// A bucket is the top bucket_log bits of hh_mix64(key): the partition (top npart_log bits) and below it a sub-bucket.
#define HH_AGG_MEAN 2048           // buckets hold at most this many records on average (links_bucket_log)
#define HH_SUB_MAX_LOG 12          // at most 2^12 sub-buckets per partition region: the shared histograms of hist / scatter2
#define HH_AGG_SLOTS 2048          // the largest table of the fallback rule (tsize in hh_k_bucket_count)
#define HH_AGG_LIST (HH_AGG_SLOTS / 4 * 3)   // the largest distinct-pair limit: entries of a bucket's aggregate list
#define HH_AGG_THREADS 256
#define HH_AGG_HOT 32              // a bucket with more than HH_AGG_HOT x the mean records skips shared memory (links_hot_records)

// Records per bucket.  The virtual tiles are `tpr` tiles of every region (those past the region's fill exit at once),
// then the spill list; a region tile histograms its 2^(bucket_log - npart_log) sub-buckets in shared memory and adds them
// with one global atomic per sub-bucket.  Spill records (rare) go straight to their bucket.
template <typename R>
__global__ void __launch_bounds__(512)
hh_k_part_hist(const R* __restrict__ pbuf, uint64_t pcap, const unsigned long long* __restrict__ cursor, int npart_log, int kbits,
               int64_t tpr, const int4* __restrict__ spill, int64_t n_spill, int bucket_log, unsigned int* __restrict__ bcnt) {
    constexpr int TILE = HH_PART_TILE, ITEMS = TILE / 512;
    __shared__ unsigned int s_cnt[1 << HH_SUB_MAX_LOG];
    const int sub_log = bucket_log - npart_log, nsub = 1 << sub_log;
    const int64_t region_tiles = ((int64_t)1 << npart_log) * tpr;
    const int64_t tiles = region_tiles + (n_spill + HH_PART_TILE - 1) / HH_PART_TILE;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        if (t >= region_tiles) {
            const int64_t base = (t - region_tiles) * HH_PART_TILE;
            for (int k = threadIdx.x; k < HH_PART_TILE; k += 512)
                if (base + k < n_spill) atomicAdd(bcnt + hh_bucket_of(hh_ld_rec(spill + base + k), bucket_log, kbits), 1u);
            continue;
        }
        const int p = (int)(t / tpr);
        const uint64_t start = (uint64_t)(t % tpr) * TILE;
        const uint64_t fill = min((uint64_t)cursor[p], pcap);
        if (start >= fill) continue;                    // block-uniform
        for (int k = threadIdx.x; k < nsub; k += 512) s_cnt[k] = 0;
        __syncthreads();
        const R* reg = pbuf + (size_t)p * (size_t)pcap;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            const uint64_t i = start + (uint64_t)k * 512 + threadIdx.x;
            if (i < fill) atomicAdd(&s_cnt[hh_bucket_of(hh_ld_rec(reg + i), bucket_log, kbits) & (nsub - 1)], 1u);
        }
        __syncthreads();
        for (int k = threadIdx.x; k < nsub; k += 512)
            if (s_cnt[k]) atomicAdd(bcnt + ((size_t)p << sub_log) + k, s_cnt[k]);
        __syncthreads();
    }
}

// The pass of hh_k_part_hist again: every record goes to boff[bucket] + its rank, in the bucket buffer's format D.  Ranks
// inside a tile come from shared memory, one global atomic per (tile, sub-bucket) reserves the tile's run; bfill counts
// what each bucket received.  A region tile is staged in shared memory ordered by sub-bucket and stored run by run.
template <typename R, typename D>
__global__ void __launch_bounds__(512, 2)
hh_k_part_scatter2(const R* __restrict__ pbuf, uint64_t pcap, const unsigned long long* __restrict__ cursor, int npart_log, int kbits,
                   int64_t tpr, const int4* __restrict__ spill, int64_t n_spill, int bucket_log, const int64_t* __restrict__ boff,
                   unsigned int* __restrict__ bfill, D* __restrict__ out, uint64_t n_out, unsigned long long* __restrict__ counters) {
    constexpr int TILE = HH_PART_TILE, ITEMS = TILE / 512;
    extern __shared__ int4 s_stage_mem[];
    R* s_stage = reinterpret_cast<R*>(s_stage_mem);      // TILE records, ordered by sub-bucket
    __shared__ unsigned int s_cnt[1 << HH_SUB_MAX_LOG];  // records of the tile per sub-bucket, then their exclusive prefix
    __shared__ unsigned int s_base[1 << HH_SUB_MAX_LOG];
    __shared__ unsigned int s_wtot[16];
    const int sub_log = bucket_log - npart_log, nsub = 1 << sub_log;
    const int64_t region_tiles = ((int64_t)1 << npart_log) * tpr;
    const int64_t tiles = region_tiles + (n_spill + HH_PART_TILE - 1) / HH_PART_TILE;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        if (t >= region_tiles) {
            const int64_t base = (t - region_tiles) * HH_PART_TILE;
            for (int k = threadIdx.x; k < HH_PART_TILE; k += 512) {
                if (base + k >= n_spill) break;
                const int4 r = hh_ld_rec(spill + base + k);
                const uint32_t b = hh_bucket_of(r, bucket_log, kbits);
                const uint64_t q = (uint64_t)boff[b] + atomicAdd(bfill + b, 1u);
                if (q < n_out) hh_rec_put(out + q, r, kbits);
                else atomicExch(counters + 2, 6ull);
            }
            continue;
        }
        const int p = (int)(t / tpr);
        const uint64_t start = (uint64_t)(t % tpr) * TILE;
        const uint64_t fill = min((uint64_t)cursor[p], pcap);
        if (start >= fill) continue;                    // block-uniform
        for (int k = threadIdx.x; k < nsub; k += 512) s_cnt[k] = 0;
        __syncthreads();
        const R* reg = pbuf + (size_t)p * (size_t)pcap;
        R r[ITEMS];
        uint32_t at[ITEMS];                             // sub-bucket << 16 | rank in the tile (both < 2^13), ~0 = none
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            const uint64_t i = start + (uint64_t)k * 512 + threadIdx.x;
            at[k] = HH_NONE32;
            if (i < fill) {
                r[k] = hh_ld_rec(reg + i);
                const uint32_t sub = hh_bucket_of(r[k], bucket_log, kbits) & (nsub - 1);
                at[k] = (sub << 16) | atomicAdd(&s_cnt[sub], 1u);
            }
        }
        __syncthreads();
        for (int k = threadIdx.x; k < nsub; k += 512)
            if (s_cnt[k]) s_base[k] = atomicAdd(bfill + ((size_t)p << sub_log) + k, s_cnt[k]);
        const unsigned int n_tile = hh_tile_scan(s_cnt, nsub, s_wtot);
#pragma unroll
        for (int k = 0; k < ITEMS; ++k)
            if (at[k] != HH_NONE32) s_stage[s_cnt[at[k] >> 16] + (at[k] & 0xFFFFu)] = r[k];
        __syncthreads();
        // staged record e is number e - s_cnt[sub] of the tile's run in its sub-bucket
        for (unsigned int e = threadIdx.x; e < n_tile; e += 512) {
            const R rec = s_stage[e];
            const uint32_t sub = hh_bucket_of(rec, bucket_log, kbits) & (nsub - 1);
            const size_t b = ((size_t)p << sub_log) + sub;
            const uint64_t q = (uint64_t)boff[b] + s_base[sub] + (e - s_cnt[sub]);
            if (q < n_out) hh_rec_put(out + q, rec, kbits);
            else atomicExch(counters + 2, 6ull);
        }
        __syncthreads();
    }
}

// Count every bucket in shared memory.  Persistent CTAs take buckets from an atomic queue (agg[0]) and read a bucket in
// chunks of S = 256 x ITEMS records.  A chunk is sorted by its exact pair key (i << kbits) | j (block radix sort over the
// 2 kbits key bits; payload: the record's place in the chunk and its flags), the runs of equal keys are reduced by one
// segmented block scan, and the runs are merged into the bucket's aggregate list, a key-sorted SoA list in shared memory
// of at most HH_AGG_LIST entries: a run whose key is on the list adds to its entry, the new ones are placed by their rank
// among the new keys plus their lower bound on the list (merge path).  The fallback rule: with tsize the power of two
// >= 1.5 x the bucket's records (256 .. HH_AGG_SLOTS), a bucket with more than tsize / 4 x 3 distinct pairs (checked
// after every chunk; the count only grows) goes on the fallback list (agg[1] entries), as does a bucket of more than `hot`
// records.  Nothing leaves the CTA before the bucket has counted completely.  A completed bucket reserves its entries with
// one global atomic and writes them word by word (consecutive threads, consecutive words), with the per-fragment totals
// and nnz_flank.  agg[2] counts completed buckets.
#define HH_PK_FLANK 12             // a run's counters packed 12 bits each (a chunk has at most 2048 < 2^12 records)
#define HH_PK_HT 24
#define HH_PK_TH 36
#define HH_PK_TT 48
#define HH_PK_MASK 0xFFFull
#define HH_PK_HEAD (1ull << 63)    // a run starts at this record

struct hh_run {
    unsigned long long c;            // full | flank << 12 | HT << 24 | TH << 36 | TT << 48 | head << 63
    uint32_t first_full, first_flank;
};

// segmented sum / min: a head on the right starts over
struct hh_run_op {
    __device__ __forceinline__ hh_run operator()(const hh_run& a, const hh_run& b) const {
        if (b.c & HH_PK_HEAD) return b;
        return hh_run{a.c + b.c, min(a.first_full, b.first_full), min(a.first_flank, b.first_flank)};
    }
};

template <typename K>
__device__ __forceinline__ int hh_lower_bound(const K* a, int n, K k) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// 32-bit keys up to 65,536 objects: chunks of 2048 records; 64-bit keys: 1280.  Three CTAs per SM (80 registers).
template <typename K, int ITEMS>
struct hh_bc_smem {
    typedef cub::BlockRadixSort<K, HH_AGG_THREADS, ITEMS, uint32_t> sort_t;
    typedef cub::BlockScan<hh_run, HH_AGG_THREADS> run_scan_t;
    typedef cub::BlockScan<unsigned int, HH_AGG_THREADS> cnt_scan_t;
    K key[HH_AGG_LIST];                              // the aggregate list, ascending keys
    uint32_t val[HH_E_WORDS - 2][HH_AGG_LIST];       // its counters, word w of an entry in val[w - 2]
    uint32_t z[HH_AGG_THREADS * ITEMS];              // stream index of the chunk's records
    union {
        typename sort_t::TempStorage sort;
        struct {
            K first[HH_AGG_THREADS], last[HH_AGG_THREADS];   // every thread's first / last key after the sort
        } edge;
        K fresh[HH_AGG_THREADS * ITEMS];             // the chunk's keys that are not on the list, ascending
    } u;
    typename run_scan_t::TempStorage run_scan;
    typename cnt_scan_t::TempStorage cnt_scan;
    unsigned long long base;
    int bucket;
};

template <typename K, int ITEMS, typename R>
__global__ void __launch_bounds__(HH_AGG_THREADS, 3)
hh_k_bucket_count(const R* __restrict__ rec, const int64_t* __restrict__ boff, int nbuckets, uint64_t hot, int kbits,
                  uint32_t* __restrict__ compact, uint64_t compact_cap, unsigned long long* __restrict__ ctg_links,
                  unsigned long long* __restrict__ counters, unsigned long long* __restrict__ agg, uint32_t* __restrict__ fallback) {
    typedef hh_bc_smem<K, ITEMS> smem_t;
    constexpr int S = HH_AGG_THREADS * ITEMS;
    extern __shared__ __align__(16) unsigned char hh_agg_smem[];
    smem_t& sm = *reinterpret_cast<smem_t*>(hh_agg_smem);
    const int t = threadIdx.x;
    const K jmask = ((K)1 << kbits) - 1;
    const hh_run none = {HH_PK_HEAD, HH_NONE32, HH_NONE32};
    unsigned int nfl = 0, n_done = 0;
    for (;;) {
        __syncthreads();                            // the previous bucket is finished with every shared variable
        if (t == 0) sm.bucket = (int)atomicAdd(agg + 0, 1ull);
        __syncthreads();
        const int bk = sm.bucket;
        if (bk >= nbuckets) break;
        const int64_t lo = boff[bk], n = boff[bk + 1] - lo;
        if ((uint64_t)n > hot) {
            if (t == 0) fallback[atomicAdd(agg + 1, 1ull)] = (uint32_t)bk;
            continue;
        }
        int tsize = HH_AGG_THREADS;
        while (tsize < HH_AGG_SLOTS && (int64_t)tsize * 2 < n * 3) tsize <<= 1;
        const int limit = tsize / 4 * 3;
        int na = 0;                                 // entries on the aggregate list (block-uniform)
        bool abandon = false;
        for (int64_t c0 = 0; c0 < n; c0 += S) {
            const int m = (int)min((int64_t)S, n - c0);
            // ---- load (striped: a warp reads consecutive records) and sort.  Padding sorts last: a real key has i != j,
            // so its 2 kbits are never all ones.
            K key[ITEMS];
            uint32_t pay[ITEMS];                    // place in the chunk | flags << 11 | (merge: 1 + lower bound of a new run) << 16
            __syncthreads();                        // the previous chunk is finished with z and the list
#pragma unroll
            for (int q = 0; q < ITEMS; ++q) {
                const int l = q * HH_AGG_THREADS + t;
                key[q] = ~(K)0;
                pay[q] = 0;
                if (l < m) {
                    const R r = hh_ld_rec(rec + lo + c0 + l);
                    key[q] = ((K)hh_rec_i(r, kbits) << kbits) | (K)hh_rec_j(r, kbits);
                    pay[q] = (uint32_t)l | (hh_rec_flags(r) << 11);
                    sm.z[l] = hh_rec_z(r);
                }
            }
            typename smem_t::sort_t(sm.u.sort).Sort(key, pay, 0, 2 * kbits);
            // ---- reduce: thread t holds sorted places t * ITEMS + q
            __syncthreads();
            sm.u.edge.first[t] = key[0];
            sm.u.edge.last[t] = key[ITEMS - 1];
            __syncthreads();
            const K prev = t > 0 ? sm.u.edge.last[t - 1] : ~(K)0;
            const K next = t + 1 < HH_AGG_THREADS ? sm.u.edge.first[t + 1] : ~(K)0;
            auto item = [&](int q) -> hh_run {
                const int pos = t * ITEMS + q;
                if (pos >= m) return none;
                const unsigned f = (pay[q] >> 11) & 7u;
                const uint32_t z = sm.z[pay[q] & 0x7FFu];
                const bool fl = f & HH_F_FLANK, ti = f & HH_F_TI, tj = f & HH_F_TJ;
                hh_run r;
                const bool head = pos == 0 || key[q] != (q ? key[q - 1] : prev);
                r.c = 1ull | ((unsigned long long)head << 63) | ((unsigned long long)fl << HH_PK_FLANK) | ((unsigned long long)(!ti && tj) << HH_PK_HT) |
                      ((unsigned long long)(ti && !tj) << HH_PK_TH) | ((unsigned long long)(ti && tj) << HH_PK_TT);
                r.first_full = z;
                r.first_flank = fl ? z : HH_NONE32;
                return r;
            };
            const hh_run_op op;
            hh_run acc = item(0);
#pragma unroll
            for (int q = 1; q < ITEMS; ++q) acc = op(acc, item(q));
            hh_run carry;                           // the open run of the threads before this one
            typename smem_t::run_scan_t(sm.run_scan).ExclusiveScan(acc, carry, hh_run{0ull, HH_NONE32, HH_NONE32}, op);
            // ---- merge, step 1: runs whose key is on the list add to its entry; the others are new
            unsigned int nnew = 0;
            hh_run run = carry;
#pragma unroll
            for (int q = 0; q < ITEMS; ++q) {
                run = op(run, item(q));
                const int pos = t * ITEMS + q;
                if (pos < m && (pos + 1 == m || key[q] != (q + 1 < ITEMS ? key[q + 1] : next))) {
                    const int lb = hh_lower_bound(sm.key, na, key[q]);
                    if (lb < na && sm.key[lb] == key[q]) {
                        sm.val[HH_E_FULL - 2][lb] += (uint32_t)(run.c & HH_PK_MASK);
                        sm.val[HH_E_FLANK - 2][lb] += (uint32_t)((run.c >> HH_PK_FLANK) & HH_PK_MASK);
                        sm.val[HH_E_FIRST_FULL - 2][lb] = min(sm.val[HH_E_FIRST_FULL - 2][lb], run.first_full);
                        sm.val[HH_E_FIRST_FLANK - 2][lb] = min(sm.val[HH_E_FIRST_FLANK - 2][lb], run.first_flank);
                        sm.val[HH_E_HT - 2][lb] += (uint32_t)((run.c >> HH_PK_HT) & HH_PK_MASK);
                        sm.val[HH_E_TH - 2][lb] += (uint32_t)((run.c >> HH_PK_TH) & HH_PK_MASK);
                        sm.val[HH_E_TT - 2][lb] += (uint32_t)((run.c >> HH_PK_TT) & HH_PK_MASK);
                    } else {
                        pay[q] |= (uint32_t)(lb + 1) << 16;
                        nnew++;
                    }
                }
            }
            unsigned int rank, fresh;
            typename smem_t::cnt_scan_t(sm.cnt_scan).ExclusiveSum(nnew, rank, fresh);
            if (na + (int)fresh > limit) {
                abandon = true;
                break;
            }
            if (fresh == 0) continue;
            // ---- merge, step 2: an entry of the list moves up by the new keys below it.  Destinations are >= sources, so
            // groups of 256 entries move from the top down, each read completely before it is written.
            if (na) {
                unsigned int r = rank;
#pragma unroll
                for (int q = 0; q < ITEMS; ++q)
                    if (pay[q] >> 16) sm.u.fresh[r++] = key[q];
                __syncthreads();
                for (int hi = na; hi > 0; hi -= HH_AGG_THREADS) {
                    const int a = hi - HH_AGG_THREADS + t;
                    K k = 0;
                    uint32_t v[HH_E_WORDS - 2];
                    int d = a;                      // stays: no entry, or one that does not move
                    if (a >= 0) {
                        k = sm.key[a];
#pragma unroll
                        for (int w = 0; w < HH_E_WORDS - 2; ++w) v[w] = sm.val[w][a];
                        d = a + hh_lower_bound(sm.u.fresh, (int)fresh, k);
                    }
                    __syncthreads();
                    if (d > a) {
                        sm.key[d] = k;
#pragma unroll
                        for (int w = 0; w < HH_E_WORDS - 2; ++w) sm.val[w][d] = v[w];
                    }
                    __syncthreads();
                }
            }
            // ---- merge, step 3: the new runs, reduced again (fewer registers than keeping them), take the places left free
            run = carry;
#pragma unroll
            for (int q = 0; q < ITEMS; ++q) {
                run = op(run, item(q));
                if ((pay[q] >> 16) == 0) continue;
                const int d = (int)(pay[q] >> 16) - 1 + (int)rank++;
                const hh_run& o = run;
                sm.key[d] = key[q];
                sm.val[HH_E_FULL - 2][d] = (uint32_t)(o.c & HH_PK_MASK);
                sm.val[HH_E_FLANK - 2][d] = (uint32_t)((o.c >> HH_PK_FLANK) & HH_PK_MASK);
                sm.val[HH_E_FIRST_FULL - 2][d] = o.first_full;
                sm.val[HH_E_FIRST_FLANK - 2][d] = o.first_flank;
                sm.val[HH_E_HT - 2][d] = (uint32_t)((o.c >> HH_PK_HT) & HH_PK_MASK);
                sm.val[HH_E_TH - 2][d] = (uint32_t)((o.c >> HH_PK_TH) & HH_PK_MASK);
                sm.val[HH_E_TT - 2][d] = (uint32_t)((o.c >> HH_PK_TT) & HH_PK_MASK);
            }
            na += (int)fresh;
        }
        if (abandon) {
            if (t == 0) fallback[atomicAdd(agg + 1, 1ull)] = (uint32_t)bk;
            continue;
        }
        // ---- emit: entry e of the list is entry base + e, word w of it is compact word base x 9 + w
        __syncthreads();
        if (t == 0) sm.base = na ? atomicAdd(counters + 0, (unsigned long long)na) : 0ull;
        __syncthreads();
        const unsigned long long base = sm.base;
        for (int w = t; w < na * HH_E_WORDS; w += HH_AGG_THREADS) {
            const int e = w / HH_E_WORDS, f = w - e * HH_E_WORDS;
            const uint32_t x = f == HH_E_I ? (uint32_t)(sm.key[e] >> kbits)
                             : f == HH_E_J ? (uint32_t)(sm.key[e] & jmask) : sm.val[f - 2][e];
            if (base + e < compact_cap) compact[base * HH_E_WORDS + w] = x;
            else atomicExch(counters + 2, 5ull);
        }
        for (int e = t; e < na; e += HH_AGG_THREADS) {
            const uint32_t flank = sm.val[HH_E_FLANK - 2][e];
            if (flank) {
                nfl++;
                atomicAdd(ctg_links + (uint32_t)(sm.key[e] >> kbits), (unsigned long long)flank);    // ctg_link_dict (1638-1639)
                atomicAdd(ctg_links + (uint32_t)(sm.key[e] & jmask), (unsigned long long)flank);
            }
        }
        n_done++;
    }
    nfl = (unsigned)hh_warp_sum((int)nfl);
    if ((t & 31) == 0 && nfl) atomicAdd(counters + 3, (unsigned long long)nfl);
    if (t == 0 && n_done) atomicAdd(agg + 2, (unsigned long long)n_done);
}

// ---- fallback: the global scratch table ------------------------------------------------------------------------------
// The listed buckets are gathered into one dense list and counted in batches of about HH_FB_BATCH records, so that the
// number of launches grows with the records that fall back and not with the buckets.  Buckets are functions of the key,
// so the keys of different buckets never meet and a batch may hold any number of them.
#define HH_FB_BATCH (1 << 19)      // records per fallback batch: two 2^20-slot scratch tables of 42 MB at load <= 0.5

// dst[pre[k] + r] = src[src_off[k] + r], as a wide record, for the nf listed buckets (pre = exclusive prefix of their
// record counts)
template <typename R>
__global__ void hh_k_gather_buckets(const R* __restrict__ src, const int64_t* __restrict__ src_off, const int64_t* __restrict__ pre,
                                    int nf, int kbits, int4* __restrict__ dst) {
    const int64_t total = pre[nf];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        int lo = 0, hi = nf - 1;                   // the last bucket that starts at or before i
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (pre[mid] <= i) lo = mid;
            else hi = mid - 1;
        }
        hh_rec_put(dst + i, hh_ld_rec(src + src_off[lo] + (i - pre[lo])), kbits);
    }
}

// count `n` bucket records ({i, j, stream index, flags}) into a scratch table
__device__ __forceinline__ void hh_part_count(const int4* __restrict__ prec, int64_t n, uint64_t* __restrict__ keys,
                                              hh_slot* __restrict__ vals, uint64_t cap, unsigned long long* __restrict__ counters) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); i0 < n; i0 += stride) {
        const int64_t i = i0 + lane;
        const bool ok = i < n;
        int4 r = make_int4(0, 0, 0, 0);
        if (ok) r = hh_ld_stream(prec + i);
        const uint64_t key = hh_pair_key(r.x, r.y);
        const hh_group g = hh_warp_fold(ok, key, (uint32_t)r.z, (unsigned)r.w);
        if (g.leader) {
            bool inserted;
            const uint64_t slot = hh_probe_insert(keys, cap, key, &inserted);
            if (slot >= cap) atomicExch(counters + 2, 4ull);
            else hh_slot_update(vals + slot, g);
        }
    }
}

// count one bucket into the scratch table (ckeys), or emit the table (ekeys)
__global__ void __launch_bounds__(256)
hh_k_part_step(const int4* __restrict__ prec, int64_t n, uint64_t* __restrict__ ckeys, hh_slot* __restrict__ cvals,
               uint64_t* __restrict__ ekeys, hh_slot* __restrict__ evals, uint64_t cap, uint32_t* __restrict__ compact,
               uint64_t compact_cap, unsigned long long* __restrict__ ctg_links, unsigned long long* __restrict__ counters) {
    // ---- emit the table of the previous bucket: live slots -> compact entries, per-fragment totals; slots are cleared.
    // A CTA takes 512 consecutive slots, two per thread: the keys are loaded together (one memory round trip instead
    // of one per slot), the live ones are ranked by a block scan, the output positions of the whole CTA are reserved with
    // ONE atomic on the global cursor, then the values are read together and written.
    if (ekeys != nullptr) {
        __shared__ unsigned int s_wtot[8];
        __shared__ unsigned long long s_base;
        unsigned int nfl = 0;
        constexpr int E = 2;
        for (uint64_t r0 = (uint64_t)blockIdx.x * (256ull * E); r0 < cap; r0 += (uint64_t)gridDim.x * (256ull * E)) {
            uint64_t key[E];
            unsigned int cnt = 0;
#pragma unroll
            for (int q = 0; q < E; ++q) {
                const uint64_t sl = r0 + (uint64_t)q * 256ull + threadIdx.x;
                key[q] = (sl < cap) ? ekeys[sl] : HH_EMPTY_KEY;
                cnt += (key[q] != HH_EMPTY_KEY) ? 1u : 0u;
            }
            unsigned int total;
            const unsigned int rank = hh_block_rank(cnt, s_wtot, &total);     // its first barrier: the last trip has read s_base
            if (threadIdx.x == 0) s_base = total ? atomicAdd(counters + 0, (unsigned long long)total) : 0ull;
            __syncthreads();
            if (cnt) {
                unsigned long long pos = s_base + rank;
                uint4 v0[E], v1[E];
#pragma unroll
                for (int q = 0; q < E; ++q) {
                    if (key[q] != HH_EMPTY_KEY) {
                        const uint4* vp = reinterpret_cast<const uint4*>(evals + (r0 + (uint64_t)q * 256ull + threadIdx.x));
                        v0[q] = vp[0];       // {first_full, first_flank, full, flank}
                        v1[q] = vp[1];       // {ht, th, tt, pad}
                    }
                }
#pragma unroll
                for (int q = 0; q < E; ++q) {
                    if (key[q] == HH_EMPTY_KEY) continue;
                    const uint64_t sl = r0 + (uint64_t)q * 256ull + threadIdx.x;
                    if (pos < compact_cap) hh_entry_store(compact + pos * HH_E_WORDS, key[q], v0[q], v1[q]);
                    else atomicExch(counters + 2, 5ull);
                    pos++;
                    if (v0[q].w) {
                        nfl++;
                        atomicAdd(ctg_links + (uint32_t)(key[q] >> 32), (unsigned long long)v0[q].w);      // ctg_link_dict (1638-1639)
                        atomicAdd(ctg_links + (uint32_t)key[q], (unsigned long long)v0[q].w);
                    }
                    ekeys[sl] = HH_EMPTY_KEY;
                    uint4* vw = reinterpret_cast<uint4*>(evals + sl);
                    vw[0] = make_uint4(HH_NONE32, HH_NONE32, 0u, 0u);
                    vw[1] = make_uint4(0u, 0u, 0u, 0u);
                }
            }
        }
        nfl = (unsigned)hh_warp_sum((int)nfl);
        if ((threadIdx.x & 31) == 0 && nfl) atomicAdd(counters + 3, (unsigned long long)nfl);
    }
    // ---- count the current bucket
    if (ckeys != nullptr && n > 0) hh_part_count(prec, n, ckeys, cvals, cap, counters);
}

// re-insert every live slot of the old table into a (larger) new one
__global__ void hh_k_links_rehash(const uint64_t* __restrict__ okeys, const hh_slot* __restrict__ ovals, uint64_t ocap,
                                  uint64_t* __restrict__ keys, hh_slot* __restrict__ vals, uint64_t cap,
                                  unsigned long long* __restrict__ counters) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < ocap; s += stride) {
        const uint64_t k = okeys[s];
        if (k == HH_EMPTY_KEY) continue;
        bool inserted;
        const uint64_t slot = hh_probe_insert(keys, cap, k, &inserted);
        if (slot >= cap) {
            atomicExch(counters + 2, 1ull);
            continue;
        }
        const uint4* src = reinterpret_cast<const uint4*>(ovals + s);
        uint4* dst = reinterpret_cast<uint4*>(vals + slot);
        dst[0] = src[0];
        dst[1] = src[1];
    }
}

// merge a peer's export (9 x u32 per entry) into this table
__global__ void hh_k_links_merge(const uint32_t* __restrict__ ent, int64_t n_ent, uint64_t* __restrict__ keys,
                                 hh_slot* __restrict__ vals, uint64_t cap, unsigned long long* __restrict__ counters) {
    __shared__ unsigned int s_new;
    if (threadIdx.x == 0) s_new = 0;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int my_new = 0, my_last = 0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_ent; e += stride) {
        const uint32_t* p = ent + e * HH_E_WORDS;
        const uint64_t key = ((uint64_t)p[HH_E_I] << 32) | (uint64_t)p[HH_E_J];
        bool inserted;
        const uint64_t slot = hh_probe_insert(keys, cap, key, &inserted);
        if (slot >= cap) {
            atomicExch(counters + 2, 1ull);
            continue;
        }
        if (inserted) my_new++;
        hh_slot* v = vals + slot;
        atomicAdd(&v->full, p[HH_E_FULL]);
        if (p[HH_E_FLANK]) atomicAdd(&v->flank, p[HH_E_FLANK]);
        atomicMin(&v->first_full, p[HH_E_FIRST_FULL]);
        atomicMin(&v->first_flank, p[HH_E_FIRST_FLANK]);
        my_last = max(my_last, p[HH_E_FIRST_FULL]);
        if (p[HH_E_HT]) atomicAdd(&v->ht, p[HH_E_HT]);
        if (p[HH_E_TH]) atomicAdd(&v->th, p[HH_E_TH]);
        if (p[HH_E_TT]) atomicAdd(&v->tt, p[HH_E_TT]);
    }
    if (my_new) atomicAdd(&s_new, my_new);
    my_last = __reduce_max_sync(HH_FULL_MASK, my_last);
    if ((threadIdx.x & 31) == 0 && my_last) atomicMax(counters + 4, (unsigned long long)my_last);
    __syncthreads();
    if (threadIdx.x == 0 && s_new) atomicAdd(counters + 0, (unsigned long long)s_new);
}

__global__ void hh_k_add_u64(unsigned long long* __restrict__ dst, const int64_t* __restrict__ src, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] += (unsigned long long)src[i];
}

// ---------------------------------------------------------------------------------------------
// multi-GPU routing: every contig pair has ONE owner rank, so the partition tables are disjoint and no
// counter is ever reduced across ranks
// ---------------------------------------------------------------------------------------------
#define HH_MAX_WORLD 64

__device__ __forceinline__ int hh_owner(int a, int b, int world) {
    const uint32_t lo = (uint32_t)min(a, b), hi = (uint32_t)max(a, b);
    return (int)(hh_mix64(((uint64_t)lo << 32) | (uint64_t)hi) % (uint64_t)world);
}

// destination of a record, -1 = can never be used (same contig in contig mode, ids outside the FASTA)
__device__ __forceinline__ int hh_route_dest(const int4 r, int n_src, bool contig_mode, int world) {
    if ((unsigned)r.x >= (unsigned)n_src || (unsigned)r.z >= (unsigned)n_src) return -1;
    if (contig_mode && r.x == r.z) return -1;
    return hh_owner(r.x, r.z, world);
}

__global__ void __launch_bounds__(256)
hh_k_route_count(const int4* __restrict__ rec, int64_t n_rec, int n_src, int contig_mode, int world,
                 unsigned long long* __restrict__ counts) {
    __shared__ unsigned int s_cnt[HH_MAX_WORLD];
    if (threadIdx.x < HH_MAX_WORLD) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rec; i += stride) {
        const int d = hh_route_dest(hh_ld_stream(rec + i), n_src, contig_mode != 0, world);
        if (d >= 0) atomicAdd(&s_cnt[d], 1u);
    }
    __syncthreads();
    if (threadIdx.x < world && s_cnt[threadIdx.x]) atomicAdd(counts + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

// scatter into the destination groups; cursor[d] starts at the group's base.  One tile of 256 records per trip:
// shared-memory ranks inside the tile, one global atomic per destination and tile.
__global__ void __launch_bounds__(256)
hh_k_route_scatter(const int4* __restrict__ rec, int64_t n_rec, uint32_t stream_off, int n_src, int contig_mode, int world,
                   unsigned long long* __restrict__ cursor, int4* __restrict__ rec_out, uint32_t* __restrict__ pos_out) {
    __shared__ unsigned int s_cnt[HH_MAX_WORLD];
    __shared__ unsigned long long s_base[HH_MAX_WORLD];
    const int64_t tiles = (n_rec + 255) / 256;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        if (threadIdx.x < HH_MAX_WORLD) s_cnt[threadIdx.x] = 0;
        __syncthreads();
        const int64_t i = t * 256 + threadIdx.x;
        int4 r = make_int4(-1, 0, -1, 0);
        int d = -1;
        unsigned int my = 0;
        if (i < n_rec) {
            r = hh_ld_stream(rec + i);
            d = hh_route_dest(r, n_src, contig_mode != 0, world);
            if (d >= 0) my = atomicAdd(&s_cnt[d], 1u);
        }
        __syncthreads();
        if (threadIdx.x < world && s_cnt[threadIdx.x])
            s_base[threadIdx.x] = atomicAdd(cursor + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
        __syncthreads();
        if (d >= 0) {
            const unsigned long long q = s_base[d] + my;
            rec_out[q] = r;
            pos_out[q] = stream_off + (uint32_t)i;
        }
        __syncthreads();
    }
}

// order[s] = s for live slots (unordered compaction of a partition table re-uses the compaction kernels)
__global__ void hh_k_links_mark_slots(const uint64_t* __restrict__ keys, uint64_t cap, uint32_t* __restrict__ order) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += stride)
        order[s] = (keys[s] == HH_EMPTY_KEY) ? HH_NONE32 : (uint32_t)s;
}

// adopted (unordered) entry list -> order[first_full] = entry index; and the flank count
__global__ void hh_k_list_scatter_order(const uint32_t* __restrict__ ent, int64_t nnz, uint32_t* __restrict__ order, int64_t stream_end,
                                        unsigned long long* __restrict__ counters) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        const uint32_t f = ent[e * HH_E_WORDS + HH_E_FIRST_FULL];
        if ((int64_t)f < stream_end) order[f] = (uint32_t)e;
        else atomicExch(counters + 2, 2ull);
    }
}

__global__ void hh_k_list_count_flank(const uint32_t* __restrict__ ent, int64_t nnz, unsigned long long* __restrict__ counters) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int c = 0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride)
        c += ent[e * HH_E_WORDS + HH_E_FLANK] ? 1u : 0u;
    c = hh_warp_sum((int)c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(counters + 3, (unsigned long long)c);
}

// order[first_full] = slot
__global__ void hh_k_links_scatter_order(const uint64_t* __restrict__ keys, const hh_slot* __restrict__ vals, uint64_t cap,
                                         uint32_t* __restrict__ order, int64_t stream_end,
                                         unsigned long long* __restrict__ counters) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += stride) {
        if (keys[s] == HH_EMPTY_KEY) continue;
        const uint32_t f = vals[s].first_full;
        if ((int64_t)f < stream_end) order[f] = (uint32_t)s;
        else atomicExch(counters + 2, 2ull);
    }
}

#define HH_CMP_TILE 2048   // elements per block in the compaction kernels (256 threads x 8)

__global__ void __launch_bounds__(256)
hh_k_compact_count(const uint32_t* __restrict__ order, int64_t n, int* __restrict__ block_cnt) {
    __shared__ int s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * HH_CMP_TILE + (int64_t)threadIdx.x * 8;
    int c = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int64_t e = base + k;
        if (e < n && order[e] != HH_NONE32) c++;
    }
    c = hh_warp_sum(c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) block_cnt[blockIdx.x] = s_cnt;
}

__global__ void __launch_bounds__(256)
hh_k_compact_gather(const uint32_t* __restrict__ order, int64_t n, const int64_t* __restrict__ block_off,
                    const uint64_t* __restrict__ keys, const hh_slot* __restrict__ vals,
                    uint32_t* __restrict__ compact, unsigned long long* __restrict__ counters) {
    __shared__ unsigned int s_wtot[8];
    __shared__ unsigned int s_flank;
    if (threadIdx.x == 0) s_flank = 0;
    const int64_t base = (int64_t)blockIdx.x * HH_CMP_TILE + (int64_t)threadIdx.x * 8;
    uint32_t slot[8];
    unsigned int c = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int64_t e = base + k;
        slot[k] = (e < n) ? order[e] : HH_NONE32;
        if (slot[k] != HH_NONE32) c++;
    }
    unsigned int total;
    int64_t q = block_off[blockIdx.x] + hh_block_rank(c, s_wtot, &total);
    unsigned int nfl = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (slot[k] == HH_NONE32) continue;
        uint32_t* o = compact + q * HH_E_WORDS;
        q++;
        if (keys == nullptr) {
            // source is an entry list (hh_links_adopt): plain copy of the words
            const uint32_t* src = reinterpret_cast<const uint32_t*>(vals) + (size_t)slot[k] * HH_E_WORDS;
#pragma unroll
            for (int w = 0; w < HH_E_WORDS; ++w) o[w] = src[w];
            continue;
        }
        const uint4* v = reinterpret_cast<const uint4*>(vals + slot[k]);
        const uint4 v0 = v[0], v1 = v[1];
        hh_entry_store(o, keys[slot[k]], v0, v1);
        if (v0.w) nfl++;
    }
    if (nfl) atomicAdd(&s_flank, nfl);
    __syncthreads();
    if (threadIdx.x == 0 && s_flank) atomicAdd(counters + 3, (unsigned long long)s_flank);
}

// ---------------------------------------------------------------------------------------------
// dict_to_matrix index assignment (327-349): first touch of each fragment in flank-dict order.  An entry that the
// phasing reduction deleted is not in the dict and touches nothing.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
hh_k_touch(const uint32_t* __restrict__ compact, int64_t nnz, const uint8_t* __restrict__ keep,
           const unsigned long long* __restrict__ ctg_tot, int normalize, const int32_t* __restrict__ hap, double w,
           unsigned long long* __restrict__ touch, int* __restrict__ deg, unsigned long long* __restrict__ n_pass) {
    __shared__ unsigned int s_pass;
    if (threadIdx.x == 0) s_pass = 0;
    __syncthreads();
    unsigned int my_pass = 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        const uint32_t* p = compact + e * HH_E_WORDS;
        if (p[HH_E_FLANK] == 0) continue;              // no flank link
        const uint32_t i = p[HH_E_I], j = p[HH_E_J];
        if (!keep[i] || !keep[j]) continue;            // 329-330
        double x;
        if (!hh_flank_value(p, ctg_tot, normalize, hap, w, nullptr, nullptr, &x)) continue;   // not in flank_link_dict
        const unsigned long long t = (unsigned long long)p[HH_E_FIRST_FLANK] * 2ull;
        // touch values only fall, so a value read from L2 that is already below t makes the atomic a no-op; most are
        if (t < __ldcg(touch + i)) atomicMin(touch + i, t);
        if (t + 1ull < __ldcg(touch + j)) atomicMin(touch + j, t + 1ull);
        atomicAdd(deg + i, 1);                          // the column counts of the matrix (hh_matrix_from_links_phased)
        atomicAdd(deg + j, 1);
        my_pass++;
    }
    my_pass = (unsigned)hh_warp_sum((int)my_pass);
    if ((threadIdx.x & 31) == 0 && my_pass) atomicAdd(&s_pass, my_pass);
    __syncthreads();
    if (threadIdx.x == 0 && s_pass) atomicAdd(n_pass, (unsigned long long)s_pass);
}

__global__ void hh_k_iota_i32(int32_t* __restrict__ p, int n) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) p[k] = k;
}

// After the (touch, fragment) pairs are sorted by touch: index[fragment] = its rank among the touched ones, -1 for the
// untouched (touch values are unique; the untouched sort last); out[0] = number touched
__global__ void hh_k_rank_sorted(const unsigned long long* __restrict__ touch_sorted, const int32_t* __restrict__ frag_sorted, int n,
                                 int32_t* __restrict__ index, unsigned long long* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const bool touched = touch_sorted[k] != ~0ull;
    index[frag_sorted[k]] = touched ? k : -1;
    if (touched && (k == n - 1 || touch_sorted[k + 1] == ~0ull)) out[0] = (unsigned long long)(k + 1);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static inline int hh_grid(hh_ctx* ctx, int per_sm) { return ctx->sm_count * per_sm; }

// blocks of 256 threads for a grid-stride kernel over n items: one thread per item, at most 8 blocks per SM
static inline int links_grid(hh_ctx* ctx, int64_t n) {
    return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, hh_grid(ctx, 8)));
}

static int links_alloc_table(hh_links* lk, uint64_t cap, uint64_t** keys, hh_slot** vals) {
    HH_CHECK(hh_dmalloc(keys, cap));
    int rc = hh_dmalloc(vals, cap);
    if (rc != HH_OK) {
        hh_dfree(*keys);
        return rc;
    }
    HH_LAUNCH(lk->ctx, hh_k_links_init, hh_grid(lk->ctx, 8), 256, 0, *keys, *vals, cap);
    return HH_OK;
}

static int links_read_counters(hh_links* lk, unsigned long long out[8]) {
    hh_ctx* ctx = lk->ctx;
    HH_CUDA(cudaMemcpyAsync(ctx->h_scratch, lk->d_counters, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    HH_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 8; ++k) out[k] = ctx->h_scratch[k];
    return HH_OK;
}

// the big hash table of the direct path is allocated on first use (the partitioned path never needs it)
static int links_need_table(hh_links* lk) {
    if (lk->d_keys) return HH_OK;
    uint64_t cap = 1ull << 16;
    const double want = lk->capacity_hint > 0 ? (double)lk->capacity_hint / 0.5 : 0.0;
    while ((double)cap < want) cap <<= 1;
    HH_CHECK(links_alloc_table(lk, cap, &lk->d_keys, &lk->d_vals));
    lk->cap = cap;
    return HH_OK;
}

// make sure `incoming` more distinct keys fit under a 0.7 load factor
static int links_ensure_capacity(hh_links* lk, int64_t incoming) {
    const double max_load = 0.7;
    HH_CHECK(links_need_table(lk));
    if ((double)(lk->known_unique + lk->since_known + incoming) <= max_load * (double)lk->cap) return HH_OK;
    unsigned long long c[8];
    HH_CHECK(links_read_counters(lk, c));
    HH_REQUIRE(c[2] == 0, HH_ERR_CAPACITY, "hh_links: hash table overflow (capacity %llu slots)", (unsigned long long)lk->cap);
    lk->known_unique = (int64_t)c[0];
    lk->since_known = 0;
    if ((double)(lk->known_unique + incoming) <= max_load * (double)lk->cap) return HH_OK;
    uint64_t ncap = lk->cap;
    while ((double)(lk->known_unique + incoming) > max_load * (double)ncap) ncap <<= 1;
    uint64_t* nkeys;
    hh_slot* nvals;
    HH_CHECK(links_alloc_table(lk, ncap, &nkeys, &nvals));
    HH_LAUNCH(lk->ctx, hh_k_links_rehash, hh_grid(lk->ctx, 8), 256, 0, lk->d_keys, lk->d_vals, lk->cap, nkeys, nvals, ncap,
              lk->d_counters);
    HH_CUDA(cudaStreamSynchronize(lk->ctx->stream));
    hh_dfree(lk->d_keys);
    hh_dfree(lk->d_vals);
    lk->d_keys = nkeys;
    lk->d_vals = nvals;
    lk->cap = ncap;
    return HH_OK;
}

static int links_create_common(hh_ctx* ctx, int32_t n_key, const int64_t* key_len, const int32_t* key_rank, const uint8_t* in_nx,
                               int64_t flank_bp, int64_t capacity_hint, int32_t n_src, const int32_t* src_rank,
                               const int32_t* frag_base, int64_t bin_size, hh_links** out) {
    *out = nullptr;
    std::vector<int32_t> len32(n_key);
    for (int32_t c = 0; c < n_key; ++c) {
        HH_REQUIRE(key_len[c] > 0 && key_len[c] <= 0x7fffffffLL, HH_ERR_UNSUPPORTED,
                   "hh_links_create: object %d has length %lld; records carry int32 positions (pos_int_type int32, "
                   "HapHiC_cluster.py:116-147)", c, (long long)key_len[c]);
        HH_REQUIRE(key_rank[c] >= 0 && key_rank[c] < n_key, HH_ERR_ARG, "hh_links_create: name_rank[%d] out of range", c);
        len32[c] = (int32_t)key_len[c];
    }
    hh_links* lk = new (std::nothrow) hh_links();      // value-initialised: every field zero, no partition set
    HH_REQUIRE(lk != nullptr, HH_ERR_NOMEM, "hh_links_create: out of host memory");
    lk->ctx = ctx;
    lk->n_ctg = n_key;
    lk->n_src = frag_base ? n_src : n_key;
    lk->bin_size = bin_size;
    lk->flank_bp = flank_bp;
    lk->kbits = 1;
    while ((1ll << lk->kbits) < (int64_t)n_key) lk->kbits++;
    int rc = HH_OK;
    do {
        if ((rc = hh_dmalloc(&lk->d_len, n_key)) != HH_OK) break;
        if ((rc = hh_dmalloc(&lk->d_rank, n_key)) != HH_OK) break;
        if ((rc = hh_dmalloc(&lk->d_nx, n_key)) != HH_OK) break;
        if ((rc = hh_dmalloc(&lk->d_ctg, n_key)) != HH_OK) break;
        if ((rc = hh_dmalloc(&lk->d_counters, 8)) != HH_OK) break;
        if ((rc = hh_dmalloc(&lk->d_index, n_key)) != HH_OK) break;
        if ((rc = hh_dmalloc(&lk->d_keep, n_key)) != HH_OK) break;
        if ((rc = hh_dmalloc(&lk->d_deg, n_key)) != HH_OK) break;
        if (frag_base) {
            if ((rc = hh_dmalloc(&lk->d_src_rank, n_src)) != HH_OK) break;
            if ((rc = hh_dmalloc(&lk->d_fbase, (size_t)n_src + 1)) != HH_OK) break;
        }
    } while (0);
    if (rc != HH_OK) {
        hh_links_destroy(lk);
        return rc;
    }
    cudaStream_t st = ctx->stream;
    HH_CUDA(cudaMemcpyAsync(lk->d_len, len32.data(), n_key * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    HH_CUDA(cudaMemcpyAsync(lk->d_rank, key_rank, n_key * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    HH_CUDA(cudaMemcpyAsync(lk->d_nx, in_nx, n_key * sizeof(uint8_t), cudaMemcpyHostToDevice, st));
    HH_CUDA(cudaMemsetAsync(lk->d_ctg, 0, n_key * sizeof(unsigned long long), st));
    HH_CUDA(cudaMemsetAsync(lk->d_counters, 0, 8 * sizeof(unsigned long long), st));
    if (frag_base) {
        HH_CUDA(cudaMemcpyAsync(lk->d_src_rank, src_rank, (size_t)n_src * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        HH_CUDA(cudaMemcpyAsync(lk->d_fbase, frag_base, ((size_t)n_src + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    }
    HH_CUDA(cudaStreamSynchronize(st));   // host temporaries go out of scope
    lk->capacity_hint = capacity_hint;
    HH_CUDA(cudaStreamCreateWithFlags(&lk->copy_stream, cudaStreamNonBlocking));
    for (int k = 0; k < 2; ++k) {
        HH_CUDA(cudaEventCreateWithFlags(&lk->ev_copied[k], cudaEventDisableTiming));
        HH_CUDA(cudaEventCreateWithFlags(&lk->ev_consumed[k], cudaEventDisableTiming));
    }
    *out = lk;
    return HH_OK;
}

extern "C" int hh_links_create(hh_ctx* ctx, int32_t n_ctg, const int64_t* ctg_len, const int32_t* name_rank,
                               const uint8_t* in_nx, int64_t flank_bp, int64_t capacity_hint, hh_links** out) {
    HH_REQUIRE(ctx && out && ctg_len && name_rank && in_nx, HH_ERR_ARG, "hh_links_create: NULL argument");
    HH_REQUIRE(n_ctg > 0, HH_ERR_ARG, "hh_links_create: n_ctg must be positive");
    HH_REQUIRE(flank_bp >= 0, HH_ERR_ARG, "hh_links_create: flank_bp must be >= 0");
    hh_scope _scope(ctx);
    return links_create_common(ctx, n_ctg, ctg_len, name_rank, in_nx, flank_bp, capacity_hint, n_ctg, nullptr, nullptr, 0, out);
}

extern "C" int hh_links_create_frags(hh_ctx* ctx, int32_t n_ctg, const int32_t* ctg_rank, const int32_t* frag_base,
                                     int32_t n_frag, const int64_t* frag_len, const int32_t* frag_rank, const uint8_t* frag_in_nx,
                                     int64_t bin_size, int64_t flank_bp, int64_t capacity_hint, hh_links** out) {
    HH_REQUIRE(ctx && out && ctg_rank && frag_base && frag_len && frag_rank && frag_in_nx, HH_ERR_ARG,
               "hh_links_create_frags: NULL argument");
    HH_REQUIRE(n_ctg > 0 && n_frag >= n_ctg, HH_ERR_ARG, "hh_links_create_frags: need n_frag >= n_ctg > 0");
    HH_REQUIRE(flank_bp >= 0 && bin_size > 0, HH_ERR_ARG, "hh_links_create_frags: flank_bp >= 0 and bin_size > 0 required");
    HH_REQUIRE(frag_base[0] == 0 && frag_base[n_ctg] == n_frag, HH_ERR_ARG, "hh_links_create_frags: frag_base must span [0, n_frag]");
    for (int32_t c = 0; c < n_ctg; ++c) {
        HH_REQUIRE(frag_base[c + 1] > frag_base[c], HH_ERR_ARG, "hh_links_create_frags: contig %d has no fragment", c);
        HH_REQUIRE(ctg_rank[c] >= 0 && ctg_rank[c] < n_ctg, HH_ERR_ARG, "hh_links_create_frags: ctg_rank[%d] out of range", c);
    }
    hh_scope _scope(ctx);
    return links_create_common(ctx, n_frag, frag_len, frag_rank, frag_in_nx, flank_bp, capacity_hint, n_ctg, ctg_rank, frag_base,
                               bin_size, out);
}

static int links_env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoi(v) : dflt;
}

// whether records of stream indices below `stream_end` can take the narrow format (see "partition records")
static bool links_narrow(const hh_links* lk, int64_t stream_end) {
    return lk->kbits <= HH_NREC_KBITS && stream_end <= HH_NREC_ZEND;
}

// a new set of partition regions sized for `n_rec` more records, ending at stream index `stream_end`
static int links_new_partset(hh_links* lk, int64_t n_rec, int64_t stream_end) {
    const int npart = 1 << lk->npart_log;
    hh_partset ps;
    memset(&ps, 0, sizeof(ps));
    ps.pcap = (uint64_t)((double)n_rec / npart * 1.5) + 4096;
    ps.sized_for = n_rec;
    ps.narrow = links_narrow(lk, stream_end);
    const size_t bytes = ps.narrow ? sizeof(hh_nrec) : sizeof(int4);
    unsigned char* buf = nullptr;
    HH_CHECK(hh_ws_alloc(lk->ctx, &buf, (size_t)npart * (size_t)ps.pcap * bytes));
    ps.buf = buf;
    int rc = hh_dmalloc(&ps.cursor, (size_t)npart);
    if (rc != HH_OK) {
        hh_ws_free(lk->ctx, ps.buf);
        return rc;
    }
    HH_CUDA(cudaMemsetAsync(ps.cursor, 0, (size_t)npart * sizeof(unsigned long long), lk->ctx->stream));
    lk->psets.push_back(ps);
    lk->set_bytes.push_back((int32_t)bytes);
    return HH_OK;
}

// the spill list holds an eighth of the records the partition sets are sized for, plus 4 Mi.  It is sized with the first
// set and grown when a later call opens another one, so that a stream sent in several calls spills into as much room as the
// same stream sent in one.  The copy of the old list is ordered on the library stream behind every scatter that wrote it
// and ahead of the next one; the spill cursor is unchanged.
static int links_size_spill(hh_links* lk) {
    int64_t sized = 0;
    for (const hh_partset& ps : lk->psets) sized += ps.sized_for;
    const uint64_t need = (uint64_t)(sized / 8) + (4u << 20);
    if (lk->d_spill && need <= lk->spill_cap) return HH_OK;
    int4* grown = nullptr;
    HH_CHECK(hh_ws_alloc(lk->ctx, &grown, (size_t)need));
    if (lk->d_spill) {
        const cudaError_t e = cudaMemcpyAsync(grown, lk->d_spill, (size_t)lk->spill_cap * sizeof(int4), cudaMemcpyDeviceToDevice,
                                              lk->ctx->stream);
        if (e != cudaSuccess) hh_ws_free(lk->ctx, grown);
        HH_CUDA(e);
        hh_ws_free(lk->ctx, lk->d_spill);
    }
    lk->d_spill = grown;
    lk->spill_cap = need;
    return HH_OK;
}

// first records of the stream: direct hash table or partition-then-aggregate.  `total` = records the caller is about to
// stream in this call (the sizing of the partition regions), from stream index `stream_offset`
static int links_choose_mode(hh_links* lk, int64_t total, int64_t stream_offset) {
    if (lk->mode) return HH_OK;
    const int want = links_env_int("HH_LINKS_PARTITION", -1);          // 0 = never, 1 = always (contig mode), -1 = by size
    const bool can = lk->d_fbase == nullptr && lk->d_keys == nullptr;
    const bool big = total >= (16ll << 20) && lk->n_ctg >= 2048;
    if (!can || want == 0 || (want < 0 && !big)) {
        lk->mode = 1;
        return HH_OK;
    }
    lk->mode = 2;
    int lg = 4;
    // ~400k records per partition, at most 512 partitions (the buckets of links_bucket_log split them further at finish)
    while (lg < 9 && ((int64_t)400000 << lg) < total) lg++;
    lk->npart_log = links_env_int("HH_LINKS_NPART_LOG", lg);
    if (lk->npart_log < 1) lk->npart_log = 1;
    if (lk->npart_log > 10) lk->npart_log = 10;
    HH_CHECK(links_new_partset(lk, total, stream_offset + total));
    HH_CHECK(links_size_spill(lk));
    HH_CHECK(hh_dmalloc(&lk->d_spill_cursor, 1));
    HH_CUDA(cudaMemsetAsync(lk->d_spill_cursor, 0, sizeof(unsigned long long), lk->ctx->stream));
    return HH_OK;
}

// records -> the regions of the last partition set, whose records are R
template <typename R>
static int links_launch_scatter(hh_links* lk, R* pbuf, const int4* d_rec, int64_t n_rec, int64_t stream_offset) {
    hh_ctx* ctx = lk->ctx;
    auto kernel = hh_k_part_scatter<R>;
    const int64_t tiles = (n_rec + hh_scatter_tile<R>() - 1) / hh_scatter_tile<R>();
    int grid = 0;
    HH_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HH_STAGE_SMEM));
    HH_CHECK(hh_resident_grid(ctx, kernel, 512, HH_STAGE_SMEM, &grid));
    grid = (int)std::max<int64_t>(1, std::min<int64_t>(tiles, grid));
    const hh_partset& ps = lk->psets.back();
    HH_LAUNCH(ctx, kernel, grid, 512, HH_STAGE_SMEM, d_rec, n_rec, (uint32_t)stream_offset, lk->n_ctg, lk->d_len, lk->d_rank, lk->d_nx,
              lk->flank_bp, lk->npart_log, lk->kbits, pbuf, ps.pcap, ps.cursor, lk->d_spill, lk->spill_cap, lk->d_spill_cursor,
              lk->d_counters);
    return HH_OK;
}

static int links_launch_insert(hh_links* lk, const int4* d_rec, int64_t n_rec, int64_t stream_offset,
                               const uint32_t* d_pos = nullptr) {
    hh_ctx* ctx = lk->ctx;
    if (lk->mode == 2 && d_pos == nullptr) {
        const hh_partset& ps = lk->psets.back();
        return ps.narrow ? links_launch_scatter(lk, reinterpret_cast<hh_nrec*>(ps.buf), d_rec, n_rec, stream_offset)
                         : links_launch_scatter(lk, reinterpret_cast<int4*>(ps.buf), d_rec, n_rec, stream_offset);
    }
    HH_CHECK(links_need_table(lk));
    HH_LAUNCH(ctx, hh_k_links_insert, links_grid(ctx, n_rec), 256, 0, d_rec, n_rec, (uint32_t)stream_offset, lk->n_ctg, lk->d_len,
              lk->d_rank, lk->d_nx, lk->flank_bp, lk->d_keys, lk->d_vals, lk->cap, lk->d_ctg, lk->d_counters, lk->d_src_rank,
              lk->d_fbase, lk->bin_size, lk->n_src, d_pos);
    return HH_OK;
}

// partitioned mode: a call that would outgrow the current set (sized for the first call), or put a stream index beyond
// the narrow format into a narrow set, gets a set of its own
static int links_part_room(hh_links* lk, int64_t n_rec, int64_t stream_offset) {
    hh_partset& ps = lk->psets.back();
    const bool outgrown = ps.sent + n_rec > ps.sized_for + ps.sized_for / 8;
    if (ps.sent > 0 && (outgrown || (ps.narrow && !links_narrow(lk, stream_offset + n_rec)))) {
        HH_CHECK(links_new_partset(lk, n_rec, stream_offset + n_rec));
        lk->psets.back().sent = n_rec;
        return links_size_spill(lk);
    }
    ps.sent += n_rec;
    return HH_OK;
}

// Device records in chunks of 8 Mi (128 MiB), so that the direct table can grow between two kernels.  d_pos = the stream
// index of every record (routed records), or NULL when they are stream_offset, stream_offset + 1, ...
static const int64_t HH_ADD_CHUNK = 1ll << 23;
static int links_add_chunks(hh_links* lk, const int4* d_rec, const uint32_t* d_pos, int64_t n_rec, int64_t stream_offset) {
    for (int64_t off = 0; off < n_rec; off += HH_ADD_CHUNK) {
        const int64_t m = std::min(n_rec - off, HH_ADD_CHUNK);
        if (lk->mode != 2) HH_CHECK(links_ensure_capacity(lk, m));
        HH_CHECK(links_launch_insert(lk, d_rec + off, m, stream_offset + off, d_pos ? d_pos + off : nullptr));
        lk->since_known += m;
    }
    return HH_OK;
}

extern "C" int hh_links_add_async(hh_links* lk, const int32_t* rec_dev, int64_t n_rec, int64_t stream_offset) {
    HH_REQUIRE(lk && (rec_dev || n_rec == 0), HH_ERR_ARG, "hh_links_add_async: NULL argument");
    hh_scope _scope(lk->ctx);
    HH_REQUIRE(!lk->finished, HH_ERR_STATE, "hh_links_add_async: stream already finished");
    HH_REQUIRE(n_rec >= 0 && stream_offset >= 0 && stream_offset + n_rec <= 0xFFFFFFFELL, HH_ERR_UNSUPPORTED,
               "hh_links_add: stream indices must fit 32 bits (offset %lld + %lld records)", (long long)stream_offset,
               (long long)n_rec);
    HH_REQUIRE(((uintptr_t)rec_dev & 15) == 0, HH_ERR_ARG, "hh_links_add: records must be 16-byte aligned");
    if (n_rec == 0) return HH_OK;
    HH_CUDA(cudaSetDevice(lk->ctx->device));
    HH_CHECK(links_choose_mode(lk, n_rec, stream_offset));
    if (lk->mode == 2) HH_CHECK(links_part_room(lk, n_rec, stream_offset));
    HH_CHECK(links_launch_insert(lk, reinterpret_cast<const int4*>(rec_dev), n_rec, stream_offset));
    lk->n_records += n_rec;
    lk->since_known += n_rec;
    if (stream_offset + n_rec > lk->stream_end) lk->stream_end = stream_offset + n_rec;
    return HH_OK;
}

extern "C" int hh_links_add(hh_links* lk, const int32_t* rec, int64_t n_rec, int64_t stream_offset, int mem) {
    HH_REQUIRE(lk && (rec || n_rec == 0), HH_ERR_ARG, "hh_links_add: NULL argument");
    hh_scope _scope(lk->ctx);
    HH_REQUIRE(!lk->finished, HH_ERR_STATE, "hh_links_add: stream already finished");
    HH_REQUIRE(mem == HH_MEM_HOST || mem == HH_MEM_DEVICE, HH_ERR_ARG, "hh_links_add: bad mem flag %d", mem);
    HH_REQUIRE(n_rec >= 0 && stream_offset >= 0 && stream_offset + n_rec <= 0xFFFFFFFELL, HH_ERR_UNSUPPORTED,
               "hh_links_add: stream indices must fit 32 bits (offset %lld + %lld records)", (long long)stream_offset,
               (long long)n_rec);
    if (n_rec == 0) return HH_OK;
    hh_ctx* ctx = lk->ctx;
    HH_CUDA(cudaSetDevice(ctx->device));
    const int64_t CH = HH_ADD_CHUNK;
    HH_CHECK(links_choose_mode(lk, n_rec, stream_offset));
    if (lk->mode == 2) HH_CHECK(links_part_room(lk, n_rec, stream_offset));
    if (mem == HH_MEM_DEVICE) {
        HH_REQUIRE(((uintptr_t)rec & 15) == 0, HH_ERR_ARG, "hh_links_add: records must be 16-byte aligned");
        HH_CHECK(links_add_chunks(lk, reinterpret_cast<const int4*>(rec), nullptr, n_rec, stream_offset));
    } else {
        if (!lk->d_stage[0]) {
            lk->stage_records = CH;
            HH_CUDA(cudaMalloc((void**)&lk->d_stage[0], (size_t)CH * sizeof(int4)));   // plain cudaMalloc: also used by copy_stream
            HH_CUDA(cudaMalloc((void**)&lk->d_stage[1], (size_t)CH * sizeof(int4)));
        }
        int buf = 0;
        for (int64_t off = 0; off < n_rec; off += CH, buf ^= 1) {
            const int64_t m = (n_rec - off < CH) ? (n_rec - off) : CH;
            // the copy engine may not overwrite a staging buffer the insert kernel still reads
            HH_CUDA(cudaStreamWaitEvent(lk->copy_stream, lk->ev_consumed[buf], 0));
            HH_CUDA(cudaMemcpyAsync(lk->d_stage[buf], rec + off * 4, (size_t)m * 16, cudaMemcpyHostToDevice, lk->copy_stream));
            HH_CUDA(cudaEventRecord(lk->ev_copied[buf], lk->copy_stream));
            if (lk->mode != 2) HH_CHECK(links_ensure_capacity(lk, m));
            HH_CUDA(cudaStreamWaitEvent(ctx->stream, lk->ev_copied[buf], 0));
            HH_CHECK(links_launch_insert(lk, lk->d_stage[buf], m, stream_offset + off));
            HH_CUDA(cudaEventRecord(lk->ev_consumed[buf], ctx->stream));
            lk->since_known += m;
        }
        HH_CUDA(cudaStreamSynchronize(ctx->stream));   // the caller may reuse `rec` on return
    }
    lk->n_records += n_rec;
    if (stream_offset + n_rec > lk->stream_end) lk->stream_end = stream_offset + n_rec;
    return HH_OK;
}

// partitioned counting, second phase (see "partition, then aggregate"): the regions are split into dense buckets, every
// bucket is counted in shared memory and the few that a shared-memory table cannot take in a global scratch table;
// entries are appended to an unordered compact list
static void links_free_partsets(hh_links* lk) {
    for (hh_partset& ps : lk->psets) {
        hh_ws_free(lk->ctx, ps.buf);
        hh_dfree(ps.cursor);
    }
    lk->psets.clear();
    hh_ws_free(lk->ctx, lk->d_spill);
    hh_dfree(lk->d_spill_cursor);
}

// log2 of the number of buckets for n_used records: a mean of at most HH_AGG_MEAN records per bucket (200M records:
// 2^17 buckets of about 1.3k records, 256 per partition), at least one bucket per partition region, at most
// 2^HH_SUB_MAX_LOG per region
static int links_bucket_log(int64_t n_used, int npart_log) {
    int b = npart_log;
    while (b < npart_log + HH_SUB_MAX_LOG && (n_used >> b) > HH_AGG_MEAN) b++;
    return b;
}

// records above which a bucket goes to the fallback without trying shared memory: HH_AGG_HOT x the mean bucket, and at
// least HH_AGG_HOT x HH_AGG_MEAN / 2.  Counting a bucket costs about its records, and a CTA of hh_k_bucket_count takes
// about buckets / (3 x SMs) of them (about 330 at 200M records on an H100), so a bucket at the threshold is a tenth of a
// CTA's share.  A hot contig pair above it would make one CTA a straggler; the fallback spreads it over the whole GPU.
static uint64_t links_hot_records(int64_t n_used, int bucket_log) {
    const uint64_t mean = ((uint64_t)n_used + (1ull << bucket_log) - 1) >> bucket_log;
    return (uint64_t)HH_AGG_HOT * (mean > HH_AGG_MEAN / 2 ? mean : HH_AGG_MEAN / 2);
}

// hh_k_bucket_count for keys of 2 kbits bits: 32-bit keys in chunks of 2048 records, 64-bit keys in chunks of 1280 (the
// shared memory of three CTAs per SM)
template <typename K, int ITEMS, typename R>
static int links_bucket_count(hh_links* lk, const void* rec, const int64_t* boff, int nb, uint64_t hot, int kbits, uint32_t* compact,
                              uint64_t compact_cap, unsigned long long* agg, uint32_t* fallback) {
    hh_ctx* ctx = lk->ctx;
    auto kernel = hh_k_bucket_count<K, ITEMS, R>;
    const size_t smem = sizeof(hh_bc_smem<K, ITEMS>);
    HH_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = 0;
    HH_CHECK(hh_resident_grid(ctx, kernel, HH_AGG_THREADS, smem, &grid));
    HH_LAUNCH(ctx, kernel, grid, HH_AGG_THREADS, smem, reinterpret_cast<const R*>(rec), boff, nb, hot, kbits, compact, compact_cap, lk->d_ctg, lk->d_counters, agg,
              fallback);
    return HH_OK;
}

// the records of every partition set (and, with the first, the spill list) per bucket
template <typename R>
static int links_launch_hist(hh_links* lk, const hh_partset& ps, int64_t n_spill, int blog, unsigned int* bcnt) {
    hh_ctx* ctx = lk->ctx;
    auto kernel = hh_k_part_hist<R>;
    int grid = 0;
    HH_CHECK(hh_resident_grid(ctx, kernel, 512, 0, &grid));
    const int64_t tpr = (int64_t)((ps.pcap + HH_PART_TILE - 1) / HH_PART_TILE);
    HH_LAUNCH(ctx, kernel, grid, 512, 0, reinterpret_cast<const R*>(ps.buf), ps.pcap, ps.cursor, lk->npart_log, lk->kbits, tpr,
              lk->d_spill, n_spill, blog, bcnt);
    return HH_OK;
}

// every record of a partition set (and, with the first, of the spill list) to its place in the bucket buffer `out` of D
template <typename R, typename D>
static int links_launch_scatter2(hh_links* lk, const hh_partset& ps, int64_t n_spill, int blog, const int64_t* boff, unsigned int* bfill,
                                 void* out, uint64_t n_out) {
    hh_ctx* ctx = lk->ctx;
    auto kernel = hh_k_part_scatter2<R, D>;
    int grid = 0;
    const size_t smem = (size_t)HH_PART_TILE * sizeof(R);
    HH_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    HH_CHECK(hh_resident_grid(ctx, kernel, 512, smem, &grid));
    const int64_t tpr = (int64_t)((ps.pcap + HH_PART_TILE - 1) / HH_PART_TILE);
    HH_LAUNCH(ctx, kernel, grid, 512, smem, reinterpret_cast<const R*>(ps.buf), ps.pcap, ps.cursor, lk->npart_log, lk->kbits, tpr,
              lk->d_spill, n_spill, blog, boff, bfill, reinterpret_cast<D*>(out), n_out, lk->d_counters);
    return HH_OK;
}

// Device memory of the finish for P records sent, U of them usable, in the narrow format (wide: twice the first and the
// third): the regions (12 B x P + 16 MB at 512 partitions) and the spill list (2 B x P + 64 MB), the bucket buffer
// (8 B x U) and the compact staging list (36 B x U).  The regions and the spill list are released before the staging list
// is allocated, so at most 7.4 GB is in use at once at the benchmark's 200M records (U = 167M).  Released blocks stay in
// the context's workspace cache, which gives them back only when an allocation fails, and the staging list does not fit
// the regions' block: the process holds all four, 10.2 GB (14.0 GB with wide records).  A fallback adds its gathered
// records (16 B each), which take the place of the bucket buffer, and two scratch tables.
static int links_finish_partitioned(hh_links* lk) {
    hh_ctx* ctx = lk->ctx;
    unsigned long long c[8];
    HH_CHECK(links_read_counters(lk, c));
    HH_REQUIRE(c[2] == 0, HH_ERR_CAPACITY,
               "hh_links_finish: the spill list of the partitioned counting overflowed (a few contig pairs own most of the stream): "
               "set HH_LINKS_PARTITION=0 to use the direct hash table");
    lk->n_used = lk->peer_used + (int64_t)c[1];
    const int64_t U = (int64_t)c[1];                       // records in the regions and on the spill list
    HH_REQUIRE(U < (1ll << 31), HH_ERR_UNSUPPORTED,
               "hh_links_finish: %lld usable records; the partitioned counting takes fewer than 2^31: set HH_LINKS_PARTITION=0",
               (long long)U);
    unsigned long long n_spill = 0;
    HH_CUDA(cudaMemcpyAsync(&n_spill, lk->d_spill_cursor, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    HH_CUDA(cudaStreamSynchronize(ctx->stream));
    const int blog = links_bucket_log(U, lk->npart_log);
    const int nb = 1 << blog;
    const uint64_t hot = links_hot_records(U, blog);
    const uint64_t compact_cap = (uint64_t)(U > 0 ? U : 1);       // distinct pairs <= usable records
    unsigned int *d_bcnt = nullptr, *d_bfill = nullptr;
    uint32_t *d_fallback = nullptr, *d_stage_compact = nullptr;  // the exact-size list is cut from the staging list
    int64_t* d_boff = nullptr;
    unsigned long long* d_agg = nullptr;
    unsigned char* d_rec2 = nullptr;                              // the bucket buffer: hh_nrec when narrow, else int4
    int4* d_fb_rec = nullptr;
    int64_t* d_fb_off = nullptr;                                  // fallback: [nf] bucket offsets, [nf + 1] prefix of their records
    uint64_t* skeys[2] = {nullptr, nullptr};
    hh_slot* svals[2] = {nullptr, nullptr};
    hh_dfree(lk->d_compact);
    int rc = [&]() -> int {
        HH_CHECK(hh_dmalloc(&d_bcnt, (size_t)nb));
        HH_CHECK(hh_dmalloc(&d_bfill, (size_t)nb));
        HH_CHECK(hh_dmalloc(&d_boff, (size_t)nb + 1));
        HH_CHECK(hh_dmalloc(&d_fallback, (size_t)nb));
        HH_CHECK(hh_dmalloc(&d_agg, 4));
        const bool narrow = links_narrow(lk, lk->stream_end);
        lk->bucket_bytes = narrow ? (int32_t)sizeof(hh_nrec) : (int32_t)sizeof(int4);
        HH_CHECK(hh_ws_alloc(ctx, &d_rec2, (size_t)compact_cap * (size_t)lk->bucket_bytes));
        HH_CUDA(cudaMemsetAsync(d_bcnt, 0, (size_t)nb * sizeof(unsigned int), ctx->stream));
        HH_CUDA(cudaMemsetAsync(d_bfill, 0, (size_t)nb * sizeof(unsigned int), ctx->stream));
        HH_CUDA(cudaMemsetAsync(d_agg, 0, 4 * sizeof(unsigned long long), ctx->stream));
        // ---- buckets: records per bucket, dense offsets, every record to its bucket
        for (size_t k = 0; k < lk->psets.size(); ++k) {
            const hh_partset& ps = lk->psets[k];
            const int64_t ns = k == 0 ? (int64_t)n_spill : 0;
            HH_CHECK(ps.narrow ? links_launch_hist<hh_nrec>(lk, ps, ns, blog, d_bcnt) : links_launch_hist<int4>(lk, ps, ns, blog, d_bcnt));
        }
        HH_CHECK(hh_exclusive_scan_i32(ctx, reinterpret_cast<const int*>(d_bcnt), d_boff, nb));
        for (size_t k = 0; k < lk->psets.size(); ++k) {
            const hh_partset& ps = lk->psets[k];
            const int64_t ns = k == 0 ? (int64_t)n_spill : 0;
            auto scatter2 = ps.narrow ? (narrow ? links_launch_scatter2<hh_nrec, hh_nrec> : links_launch_scatter2<hh_nrec, int4>)
                                      : (narrow ? links_launch_scatter2<int4, hh_nrec> : links_launch_scatter2<int4, int4>);
            HH_CHECK(scatter2(lk, ps, ns, blog, d_boff, d_bfill, d_rec2, compact_cap));
        }
        links_free_partsets(lk);                               // ordered on the stream behind scatter2
        HH_CHECK(hh_ws_alloc(ctx, &d_stage_compact, (size_t)compact_cap * HH_E_WORDS));
        HH_CUDA(cudaMemsetAsync(lk->d_counters + 0, 0, sizeof(unsigned long long), ctx->stream));     // entry cursor
        HH_CUDA(cudaMemsetAsync(lk->d_counters + 3, 0, sizeof(unsigned long long), ctx->stream));     // nnz_flank
        // ---- every bucket in shared memory
        const int kbits = lk->kbits;                           // key (i << kbits) | j
        auto count = narrow ? links_bucket_count<uint32_t, 8, hh_nrec>
                            : 2 * kbits <= 32 ? links_bucket_count<uint32_t, 8, int4> : links_bucket_count<uint64_t, 5, int4>;
        HH_CHECK(count(lk, d_rec2, d_boff, nb, hot, kbits, d_stage_compact, compact_cap, d_agg, d_fallback));
        unsigned long long agg[4];
        HH_CUDA(cudaMemcpyAsync(agg, d_agg, sizeof(agg), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CHECK(links_read_counters(lk, c));
        lk->agg_buckets = nb;
        lk->agg_smem = (int64_t)agg[2];
        lk->agg_fallback = (int64_t)agg[1];
        lk->scap = HH_AGG_SLOTS;
        // ---- fallback: the listed buckets' records are gathered into one list and counted in batches through two global
        // scratch tables (load <= 0.6 even if every record of the largest batch is a distinct key): launch t emits +
        // clears the table of batch t - 1 and counts batch t into the other
        if (agg[1]) {
            const int nf = (int)agg[1];
            std::vector<uint32_t> fb((size_t)nf);
            std::vector<int64_t> off((size_t)nb + 1), src_off((size_t)nf), pre((size_t)nf + 1, 0);
            HH_CUDA(cudaMemcpyAsync(fb.data(), d_fallback, fb.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
            HH_CUDA(cudaMemcpyAsync(off.data(), d_boff, off.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
            HH_CUDA(cudaStreamSynchronize(ctx->stream));
            std::vector<int64_t> cut(1, 0);                    // batch t = gathered records [cut[t], cut[t + 1])
            for (int k = 0; k < nf; ++k) {
                src_off[k] = off[fb[k]];
                const int64_t n = off[fb[k] + 1] - off[fb[k]];
                if (pre[k] > cut.back() && pre[k] + n - cut.back() > HH_FB_BATCH) cut.push_back(pre[k]);
                pre[k + 1] = pre[k] + n;
            }
            cut.push_back(pre[nf]);
            int64_t worst = 1;
            for (size_t t = 0; t + 1 < cut.size(); ++t) worst = std::max(worst, cut[t + 1] - cut[t]);
            uint64_t scap = 1ull << 12;
            while ((double)scap * 0.6 < (double)worst) scap <<= 1;
            lk->scap = scap;
            HH_CHECK(hh_dmalloc(&d_fb_off, 2 * (size_t)nf + 1));
            HH_CUDA(cudaMemcpyAsync(d_fb_off, src_off.data(), (size_t)nf * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
            HH_CUDA(cudaMemcpyAsync(d_fb_off + nf, pre.data(), ((size_t)nf + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
            HH_CHECK(hh_ws_alloc(ctx, &d_fb_rec, (size_t)pre[nf]));
            if (narrow)
                HH_LAUNCH(ctx, hh_k_gather_buckets<hh_nrec>, hh_grid(ctx, 8), 256, 0, reinterpret_cast<const hh_nrec*>(d_rec2), d_fb_off,
                          d_fb_off + nf, nf, kbits, d_fb_rec);
            else
                HH_LAUNCH(ctx, hh_k_gather_buckets<int4>, hh_grid(ctx, 8), 256, 0, reinterpret_cast<const int4*>(d_rec2), d_fb_off,
                          d_fb_off + nf, nf, kbits, d_fb_rec);
            hh_ws_free(ctx, d_rec2);                           // ordered on the stream behind the gather
            for (int t = 0; t < 2; ++t) HH_CHECK(links_alloc_table(lk, scap, &skeys[t], &svals[t]));
            const int g = hh_grid(ctx, 8);
            const int nbatch = (int)cut.size() - 1;
            for (int t = 0; t <= nbatch; ++t) {
                const int cb = t & 1, eb = cb ^ 1;
                const bool have = t < nbatch;
                HH_LAUNCH(ctx, hh_k_part_step, g, 256, 0, have ? d_fb_rec + cut[t] : (const int4*)nullptr,
                          have ? cut[t + 1] - cut[t] : (int64_t)0, have ? skeys[cb] : (uint64_t*)nullptr,
                          have ? svals[cb] : (hh_slot*)nullptr, t > 0 ? skeys[eb] : (uint64_t*)nullptr,
                          t > 0 ? svals[eb] : (hh_slot*)nullptr, scap, d_stage_compact, compact_cap, lk->d_ctg, lk->d_counters);
            }
            HH_CHECK(links_read_counters(lk, c));
        }
        HH_REQUIRE(c[2] == 0, HH_ERR_CAPACITY,
                   "hh_links_finish: a bucket of the partitioned counting overflowed (code %llu): set HH_LINKS_PARTITION=0", c[2]);
        lk->nnz = (int64_t)c[0];
        lk->nnz_flank = (int64_t)c[3];
        HH_CHECK(hh_dmalloc(&lk->d_compact, (size_t)(lk->nnz > 0 ? lk->nnz : 1) * HH_E_WORDS));
        if (lk->nnz)
            HH_CUDA(cudaMemcpyAsync(lk->d_compact, d_stage_compact, (size_t)lk->nnz * HH_E_WORDS * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                                    ctx->stream));
        return HH_OK;
    }();
    hh_ws_free(ctx, d_stage_compact);
    hh_ws_free(ctx, d_rec2);
    hh_ws_free(ctx, d_fb_rec);
    hh_dfree(d_fb_off);
    hh_dfree(d_bcnt);
    hh_dfree(d_bfill);
    hh_dfree(d_boff);
    hh_dfree(d_fallback);
    hh_dfree(d_agg);
    for (int t = 0; t < 2; ++t) {
        hh_dfree(skeys[t]);
        hh_dfree(svals[t]);
    }
    links_free_partsets(lk);
    HH_CHECK(rc);
    lk->finished = true;
    lk->gen++;                  // the linked index of an earlier table does not apply
    lk->ordered = false;        // dict insertion order is restored by the first hh_links_fetch (links_order_list)
    return HH_OK;
}

extern "C" int hh_links_record_bytes(hh_links* lk, int32_t* set_bytes, int32_t max_sets, int32_t* n_sets, int32_t* bucket_bytes) {
    HH_REQUIRE(lk != nullptr && (max_sets <= 0 || set_bytes), HH_ERR_ARG, "hh_links_record_bytes: NULL argument");
    for (int32_t k = 0; k < max_sets && k < (int32_t)lk->set_bytes.size(); ++k) set_bytes[k] = lk->set_bytes[k];
    if (n_sets) *n_sets = (int32_t)lk->set_bytes.size();
    if (bucket_bytes) *bucket_bytes = lk->bucket_bytes;
    return HH_OK;
}

extern "C" int hh_links_agg_info(hh_links* lk, int64_t* buckets, int64_t* smem_buckets, int64_t* fallback_buckets) {
    HH_REQUIRE(lk != nullptr, HH_ERR_ARG, "hh_links_agg_info: NULL handle");
    if (buckets) *buckets = lk->agg_buckets;
    if (smem_buckets) *smem_buckets = lk->agg_smem;
    if (fallback_buckets) *fallback_buckets = lk->agg_fallback;
    return HH_OK;
}

// Order array -> entries: dst gets, in array order, the entries that d_order[0..S) names (HH_NONE32 = none): slots of the
// hash table (keys, vals) or, with keys = NULL, entries of the list passed as `vals`.  Live items per tile, a scan, the
// gather; the gather from a table also counts the flank entries (counters[3]).
static int links_compact(hh_links* lk, const uint32_t* d_order, int64_t S, const uint64_t* keys, const hh_slot* vals, uint32_t* dst) {
    hh_ctx* ctx = lk->ctx;
    const int64_t nb = (S + HH_CMP_TILE - 1) / HH_CMP_TILE;
    int* d_bcnt = nullptr;
    int64_t* d_boff = nullptr;
    const int rc = [&]() -> int {
        HH_CHECK(hh_dmalloc(&d_bcnt, (size_t)nb));
        HH_CHECK(hh_dmalloc(&d_boff, (size_t)nb + 1));
        HH_LAUNCH(ctx, hh_k_compact_count, (unsigned)nb, 256, 0, d_order, S, d_bcnt);
        HH_CHECK(hh_exclusive_scan_i32(ctx, d_bcnt, d_boff, (int)nb));
        HH_LAUNCH(ctx, hh_k_compact_gather, (unsigned)nb, 256, 0, d_order, S, d_boff, keys, vals, dst, lk->d_counters);
        return HH_OK;
    }();
    hh_dfree(d_bcnt);                 // ordered on the stream behind the kernels
    hh_dfree(d_boff);
    return rc;
}

// The direct table becomes the compact list: in dict insertion order (order[first_full] = slot over the whole stream, then
// compaction), or -- a partition of a routed stream, whose union hh_links_fetch orders lazily -- in slot order.  `who` is
// the entry point that the error texts name.
static int links_finish_direct(hh_links* lk, bool ordered, const char* who) {
    hh_ctx* ctx = lk->ctx;
    HH_CHECK(links_need_table(lk));
    unsigned long long c[8];
    HH_CHECK(links_read_counters(lk, c));
    HH_REQUIRE(c[2] == 0, HH_ERR_CAPACITY, "%s: hash table overflow (capacity %llu slots)%s", who, (unsigned long long)lk->cap,
               ordered ? ": pass a larger capacity_hint or use hh_links_add" : "");
    HH_REQUIRE(c[5] == 0, HH_ERR_ARG,
               "%s: %llu records have a position outside their contig's bins (e.g. record %llu of the stream)%s", who, c[5], c[6] - 1ull,
               ordered ? ": positions must lie in [0, contig length)" : "");
    lk->nnz = (int64_t)c[0];
    lk->n_used = lk->peer_used + (int64_t)c[1];
    HH_CUDA(cudaMemsetAsync(lk->d_counters + 3, 0, sizeof(unsigned long long), ctx->stream));
    if (ordered && lk->nnz > 0 && (int64_t)c[4] + 1 > lk->stream_end) lk->stream_end = (int64_t)c[4] + 1;   // merged peers
    hh_dfree(lk->d_compact);
    HH_CHECK(hh_dmalloc(&lk->d_compact, (size_t)(lk->nnz > 0 ? lk->nnz : 1) * HH_E_WORDS));
    if (lk->nnz > 0) {
        HH_REQUIRE(ordered || lk->cap <= 0xFFFFFFFFull, HH_ERR_UNSUPPORTED, "%s: table too large", who);
        const int64_t S = ordered ? lk->stream_end : (int64_t)lk->cap;
        uint32_t* d_order = nullptr;
        HH_CHECK(hh_dmalloc(&d_order, (size_t)S));
        const int rc = [&]() -> int {
            if (ordered) {
                HH_CUDA(cudaMemsetAsync(d_order, 0xFF, (size_t)S * sizeof(uint32_t), ctx->stream));
                HH_LAUNCH(ctx, hh_k_links_scatter_order, hh_grid(ctx, 8), 256, 0, lk->d_keys, lk->d_vals, lk->cap, d_order, S,
                          lk->d_counters);
            } else {
                HH_LAUNCH(ctx, hh_k_links_mark_slots, hh_grid(ctx, 8), 256, 0, lk->d_keys, lk->cap, d_order);
            }
            HH_CHECK(links_compact(lk, d_order, S, lk->d_keys, lk->d_vals, lk->d_compact));
            return links_read_counters(lk, c);
        }();
        hh_dfree(d_order);
        HH_CHECK(rc);
        HH_REQUIRE(c[2] == 0, HH_ERR_STATE, "%s: first-seen index beyond the stream end (stream_offset misuse)", who);
        lk->nnz_flank = (int64_t)c[3];
    }
    lk->finished = true;
    lk->gen++;                  // the linked index of an earlier table does not apply
    lk->ordered = ordered;
    return HH_OK;
}

static void links_fill_info(hh_links* lk, hh_links_info* info, int64_t table_slots) {
    if (!info) return;
    info->n_records = lk->n_records;
    info->n_used = lk->n_used;
    info->nnz_full = lk->nnz;
    info->nnz_flank = lk->nnz_flank;
    info->table_slots = table_slots;
}

extern "C" int hh_links_finish(hh_links* lk, hh_links_info* info) {
    HH_REQUIRE(lk != nullptr, HH_ERR_ARG, "hh_links_finish: NULL handle");
    hh_scope _scope(lk->ctx);
    HH_CUDA(cudaSetDevice(lk->ctx->device));
    if (!lk->finished) HH_CHECK(lk->mode == 2 ? links_finish_partitioned(lk) : links_finish_direct(lk, true, "hh_links_finish"));
    links_fill_info(lk, info, (int64_t)(lk->mode == 2 ? lk->scap : lk->cap));
    return HH_OK;
}

// AoS compact entries -> the 7 output arrays (SoA), so each goes to the host with one plain copy
// HT slot of the ultra-long-read pair (i, j), -1 when the pair is not on the list (binary search of the sorted keys)
__device__ __forceinline__ int hh_ul_slot(const unsigned long long* __restrict__ keys, const int32_t* __restrict__ slot, int64_t n,
                                          uint32_t i, uint32_t j) {
    const unsigned long long key = ((unsigned long long)i << 32) | j;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return (lo < n && keys[lo] == key) ? slot[lo] : -1;
}

// ul_key / ul_slot / n_ul: the full count and one HT slot of the listed pairs are doubled (HH from the stored counts);
// *overflow is set when a doubled count does not fit 32 bits
__global__ void hh_k_links_split(const uint32_t* __restrict__ compact, int64_t nnz, uint32_t* __restrict__ soa, int64_t ht_off,
                                 const unsigned long long* __restrict__ ul_key, const int32_t* __restrict__ ul_slot, int64_t n_ul,
                                 int* __restrict__ overflow) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        const uint32_t* p = compact + e * HH_E_WORDS;
#pragma unroll
        for (int w = HH_E_I; w <= HH_E_FIRST_FLANK; ++w) soa[w * nnz + e] = p[w];     // the first six words, in entry order
        uint4 h;
        h.y = p[HH_E_HT];
        h.z = p[HH_E_TH];
        h.w = p[HH_E_TT];
        h.x = p[HH_E_FULL] - p[HH_E_HT] - p[HH_E_TH] - p[HH_E_TT];          // HH = full - HT - TH - TT
        const int s = n_ul ? hh_ul_slot(ul_key, ul_slot, n_ul, p[HH_E_I], p[HH_E_J]) : -1;
        if (s >= 0) {
            // selects rather than h[s]: a runtime index would put the four words in local memory
            const uint32_t hs = s == 0 ? h.x : s == 1 ? h.y : s == 2 ? h.z : h.w;
            if (p[HH_E_FULL] > 0x7FFFFFFFu || hs > 0x7FFFFFFFu) atomicExch(overflow, 1);
            soa[HH_E_FULL * nnz + e] = p[HH_E_FULL] * 2u;
            h.x = s == 0 ? h.x * 2u : h.x;
            h.y = s == 1 ? h.y * 2u : h.y;
            h.z = s == 2 ? h.z * 2u : h.z;
            h.w = s == 3 ? h.w * 2u : h.w;
        }
        reinterpret_cast<uint4*>(soa + ht_off)[e] = h;
    }
}

// ---------------------------------------------------------------------------------------------
// routed multi-GPU counting (SURVEY.md 8e): route -> [all-to-all] -> add_routed -> finish_partition ->
// export -> [all-gather] -> adopt
// ---------------------------------------------------------------------------------------------
extern "C" int hh_links_route(hh_links* lk, const int32_t* rec_dev, int64_t n_rec, int64_t stream_offset, int world,
                              int32_t* rec_out_dev, uint32_t* pos_out_dev, int64_t* counts) {
    HH_REQUIRE(lk && counts && (n_rec == 0 || (rec_dev && rec_out_dev && pos_out_dev)), HH_ERR_ARG, "hh_links_route: NULL argument");
    HH_REQUIRE(world >= 1 && world <= HH_MAX_WORLD, HH_ERR_ARG, "hh_links_route: world must be in [1, %d]", HH_MAX_WORLD);
    HH_REQUIRE(n_rec >= 0 && stream_offset >= 0 && stream_offset + n_rec <= 0xFFFFFFFELL, HH_ERR_UNSUPPORTED,
               "hh_links_route: stream indices must fit 32 bits (offset %lld + %lld records)", (long long)stream_offset,
               (long long)n_rec);
    HH_REQUIRE((((uintptr_t)rec_dev | (uintptr_t)rec_out_dev) & 15) == 0, HH_ERR_ARG, "hh_links_route: records must be 16-byte aligned");
    hh_scope _scope(lk->ctx);
    hh_ctx* ctx = lk->ctx;
    HH_CUDA(cudaSetDevice(ctx->device));
    for (int d = 0; d < world; ++d) counts[d] = 0;
    if (n_rec == 0) return HH_OK;
    unsigned long long* d_cnt = nullptr;
    HH_CHECK(hh_dmalloc(&d_cnt, 2 * HH_MAX_WORLD));
    int rc = [&]() -> int {
        HH_CUDA(cudaMemsetAsync(d_cnt, 0, 2 * HH_MAX_WORLD * sizeof(unsigned long long), ctx->stream));
        const int contig_mode = lk->d_fbase == nullptr;
        const int grid = links_grid(ctx, n_rec);
        const int4* rec4 = reinterpret_cast<const int4*>(rec_dev);
        HH_LAUNCH(ctx, hh_k_route_count, grid, 256, 0, rec4, n_rec, lk->n_src, contig_mode, world, d_cnt);
        unsigned long long h[HH_MAX_WORLD];
        HH_CUDA(cudaMemcpyAsync(h, d_cnt, (size_t)world * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        unsigned long long base[HH_MAX_WORLD], acc = 0;
        for (int d = 0; d < world; ++d) {
            counts[d] = (int64_t)h[d];
            base[d] = acc;
            acc += h[d];
        }
        HH_CUDA(cudaMemcpyAsync(d_cnt + HH_MAX_WORLD, base, (size_t)world * sizeof(unsigned long long), cudaMemcpyHostToDevice,
                                ctx->stream));
        HH_LAUNCH(ctx, hh_k_route_scatter, grid, 256, 0, rec4, n_rec, (uint32_t)stream_offset, lk->n_src, contig_mode, world,
                  d_cnt + HH_MAX_WORLD, reinterpret_cast<int4*>(rec_out_dev), pos_out_dev);
        HH_CUDA(cudaStreamSynchronize(ctx->stream));      // `base` is a host temporary; the caller hands the buffers to NCCL next
        return HH_OK;
    }();
    hh_dfree(d_cnt);
    HH_CHECK(rc);
    lk->n_records += n_rec;          // records this rank read from the stream (used or not)
    if (stream_offset + n_rec > lk->stream_end) lk->stream_end = stream_offset + n_rec;
    return HH_OK;
}

extern "C" int hh_links_add_routed(hh_links* lk, const int32_t* rec_dev, const uint32_t* pos_dev, int64_t n_rec) {
    HH_REQUIRE(lk && (n_rec == 0 || (rec_dev && pos_dev)), HH_ERR_ARG, "hh_links_add_routed: NULL argument");
    hh_scope _scope(lk->ctx);
    HH_REQUIRE(!lk->finished, HH_ERR_STATE, "hh_links_add_routed: stream already finished");
    HH_REQUIRE(n_rec >= 0, HH_ERR_ARG, "hh_links_add_routed: negative record count");
    HH_REQUIRE(((uintptr_t)rec_dev & 15) == 0, HH_ERR_ARG, "hh_links_add_routed: records must be 16-byte aligned");
    if (n_rec == 0) return HH_OK;
    HH_CUDA(cudaSetDevice(lk->ctx->device));
    HH_REQUIRE(lk->mode != 2, HH_ERR_STATE, "hh_links_add_routed: this table counts a partitioned stream (hh_links_add of a long stream)");
    lk->mode = 1;
    return links_add_chunks(lk, reinterpret_cast<const int4*>(rec_dev), pos_dev, n_rec, 0);
}

// compact list of a partition table in slot order (no first-seen ordering: the union is ordered lazily by hh_links_fetch)
extern "C" int hh_links_finish_partition(hh_links* lk, hh_links_info* info) {
    HH_REQUIRE(lk != nullptr, HH_ERR_ARG, "hh_links_finish_partition: NULL handle");
    hh_scope _scope(lk->ctx);
    HH_CUDA(cudaSetDevice(lk->ctx->device));
    // a partitioned stream already ends in an unordered entry list
    if (!lk->finished)
        HH_CHECK(lk->mode == 2 ? links_finish_partitioned(lk) : links_finish_direct(lk, false, "hh_links_finish_partition"));
    links_fill_info(lk, info, (int64_t)lk->cap);
    return HH_OK;
}

// the table becomes the union of disjoint partitions: `entries_dev` is the concatenation of every rank's export,
// `ctg_links_dev` / n_records / n_used the sums over ranks, stream_end the length of the whole stream
extern "C" int hh_links_adopt(hh_links* lk, const uint32_t* entries_dev, int64_t n_entries, const int64_t* ctg_links_dev,
                              int64_t n_records, int64_t n_used, int64_t stream_end) {
    HH_REQUIRE(lk && ctg_links_dev && (entries_dev || n_entries == 0), HH_ERR_ARG, "hh_links_adopt: NULL argument");
    HH_REQUIRE(n_entries >= 0 && stream_end >= 0 && stream_end <= 0xFFFFFFFELL, HH_ERR_ARG, "hh_links_adopt: bad sizes");
    hh_scope _scope(lk->ctx);
    hh_ctx* ctx = lk->ctx;
    HH_CUDA(cudaSetDevice(ctx->device));
    // the hash table is not needed any more: every consumer works on the entry list
    hh_dfree(lk->d_keys);
    hh_dfree(lk->d_vals);
    lk->d_keys = nullptr;
    lk->d_vals = nullptr;
    lk->cap = 0;
    hh_dfree(lk->d_compact);
    lk->d_compact = nullptr;
    lk->gen++;                  // the linked index of the old list does not apply, even if this call fails
    HH_CHECK(hh_dmalloc(&lk->d_compact, (size_t)(n_entries > 0 ? n_entries : 1) * HH_E_WORDS));
    HH_CUDA(cudaMemsetAsync(lk->d_counters + 2, 0, 2 * sizeof(unsigned long long), ctx->stream));
    if (n_entries) {
        HH_CUDA(cudaMemcpyAsync(lk->d_compact, entries_dev, (size_t)n_entries * HH_E_WORDS * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                                ctx->stream));
        const int grid = links_grid(ctx, n_entries);
        HH_LAUNCH(ctx, hh_k_list_count_flank, grid, 256, 0, lk->d_compact, n_entries, lk->d_counters);
    }
    HH_CUDA(cudaMemcpyAsync(lk->d_ctg, ctg_links_dev, (size_t)lk->n_ctg * sizeof(int64_t), cudaMemcpyDeviceToDevice, ctx->stream));
    unsigned long long c[8];
    HH_CHECK(links_read_counters(lk, c));
    lk->nnz = n_entries;
    lk->nnz_flank = (int64_t)c[3];
    lk->n_records = n_records;
    lk->n_used = n_used;
    lk->peer_used = 0;
    lk->stream_end = stream_end;
    lk->finished = true;
    lk->ordered = false;
    return HH_OK;
}

// put an adopted / partition list into dict insertion order (first_full ascending; the values are unique stream indices)
static int links_order_list(hh_links* lk) {
    if (lk->ordered || lk->nnz == 0) {
        lk->ordered = true;
        return HH_OK;
    }
    hh_ctx* ctx = lk->ctx;
    const int64_t S = lk->stream_end;
    uint32_t *d_order = nullptr, *d_sorted = nullptr;
    const int rc = [&]() -> int {
        HH_CHECK(hh_dmalloc(&d_order, (size_t)S));
        HH_CHECK(hh_dmalloc(&d_sorted, (size_t)lk->nnz * HH_E_WORDS));
        HH_CUDA(cudaMemsetAsync(d_order, 0xFF, (size_t)S * sizeof(uint32_t), ctx->stream));
        HH_CUDA(cudaMemsetAsync(lk->d_counters + 2, 0, sizeof(unsigned long long), ctx->stream));
        HH_LAUNCH(ctx, hh_k_list_scatter_order, links_grid(ctx, lk->nnz), 256, 0, lk->d_compact, lk->nnz, d_order, S, lk->d_counters);
        HH_CHECK(links_compact(lk, d_order, S, nullptr, reinterpret_cast<const hh_slot*>(lk->d_compact), d_sorted));
        unsigned long long c[8];
        HH_CHECK(links_read_counters(lk, c));
        HH_REQUIRE(c[2] == 0, HH_ERR_STATE, "hh_links: first-seen index beyond the stream end (stream_end misuse in hh_links_adopt)");
        return HH_OK;
    }();
    hh_dfree(d_order);
    if (rc != HH_OK) {
        hh_dfree(d_sorted);
        return rc;
    }
    hh_dfree(lk->d_compact);
    lk->d_compact = d_sorted;
    lk->ordered = true;
    return HH_OK;
}

extern "C" int hh_links_fetch(hh_links* lk, int32_t* key_i, int32_t* key_j, uint32_t* full, uint32_t* flank,
                              uint32_t* first_full, uint32_t* first_flank, uint32_t* ht) {
    HH_REQUIRE(lk != nullptr, HH_ERR_ARG, "hh_links_fetch: NULL handle");
    hh_scope _scope(lk->ctx);
    HH_REQUIRE(lk->finished, HH_ERR_STATE, "hh_links_fetch: call hh_links_finish first");
    if (lk->nnz == 0) return HH_OK;
    hh_ctx* ctx = lk->ctx;
    HH_CUDA(cudaSetDevice(ctx->device));
    HH_CHECK(links_order_list(lk));
    const int64_t nnz = lk->nnz;
    uint32_t* d_soa = nullptr;
    HH_CHECK(hh_dmalloc(&d_soa, (size_t)nnz * 10 + 4));
    int rc = [&]() -> int {
        uint32_t* base = d_soa;
        const int64_t ht_off = (6 * nnz + 3) & ~3ll;      // the 4-wide HT block is written with 16-byte stores
        const int grid = links_grid(ctx, nnz);
        int* d_err = reinterpret_cast<int*>(ctx->d_scratch + 10);
        HH_CUDA(cudaMemsetAsync(d_err, 0, sizeof(int), ctx->stream));
        HH_LAUNCH(ctx, hh_k_links_split, grid, 256, 0, lk->d_compact, nnz, base, ht_off, lk->d_ul_key, lk->d_ul_slot, lk->n_ul, d_err);
        void* dst[6] = {key_i, key_j, full, flank, first_full, first_flank};
        for (int k = 0; k < 6; ++k)
            if (dst[k])
                HH_CUDA(cudaMemcpyAsync(dst[k], base + (size_t)k * nnz, (size_t)nnz * 4, cudaMemcpyDeviceToHost, ctx->stream));
        if (ht) HH_CUDA(cudaMemcpyAsync(ht, base + ht_off, (size_t)nnz * 16, cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaMemcpyAsync(ctx->h_scratch + 10, d_err, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        HH_REQUIRE(*reinterpret_cast<int*>(ctx->h_scratch + 10) == 0, HH_ERR_UNSUPPORTED,
                   "hh_links_fetch: an ultra-long-read doubled link count exceeds 2^32 - 1");
        return HH_OK;
    }();
    hh_dfree(d_soa);
    return rc;
}

// The full count of an entry after reduce_inter_hap_HiC_links (695-707): x - x * w in fp64 with two roundings when its ends
// lie on different haplotypes (then a Python float), else the count (an int).  The same expression as hh_flank_value.
__device__ __forceinline__ double hh_full_value(const uint32_t* __restrict__ p, const int32_t* __restrict__ hap, double w,
                                                bool* is_float) {
    const double x = (double)p[HH_E_FULL];
    *is_float = hap[p[HH_E_I]] != hap[p[HH_E_J]];
    return *is_float ? __dsub_rn(x, __dmul_rn(x, w)) : x;
}

// order[e] = e for the entries that stay (value != 0), HH_NONE32 for the deleted ones; n_kept counts the former
__global__ void __launch_bounds__(256)
hh_k_phased_mark(const uint32_t* __restrict__ compact, int64_t nnz, const int32_t* __restrict__ hap, double w,
                 uint32_t* __restrict__ order, unsigned long long* __restrict__ n_kept) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int kept = 0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
        bool f;
        const bool keep = hh_full_value(compact + e * HH_E_WORDS, hap, w, &f) != 0.0;
        order[e] = keep ? (uint32_t)e : HH_NONE32;
        kept += keep;
    }
    kept = hh_warp_sum(kept);
    if ((threadIdx.x & 31) == 0 && kept) atomicAdd(n_kept, (unsigned long long)kept);
}

// the kept entries -> key_i, key_j, values, is_float (SoA: int32 | int32 | fp64 | uint8 blocks of n)
__global__ void __launch_bounds__(256)
hh_k_phased_split(const uint32_t* __restrict__ kept, int64_t n, const int32_t* __restrict__ hap, double w, int32_t* __restrict__ ki,
                  int32_t* __restrict__ kj, double* __restrict__ val, uint8_t* __restrict__ flt,
                  const unsigned long long* __restrict__ ul_key, const int32_t* __restrict__ ul_slot, int64_t n_ul) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
        const uint32_t* p = kept + e * HH_E_WORDS;
        bool f;
        // an ultra-long-read pair counts twice before the reduction (1936-1985 runs before 2926-2928); 2 x - 2 x w is
        // exactly 2 (x - x w), so the value is the reduced count doubled and zero exactly when that is
        const bool ul = n_ul && hh_ul_slot(ul_key, ul_slot, n_ul, p[HH_E_I], p[HH_E_J]) >= 0;
        val[e] = (ul ? 2.0 : 1.0) * hh_full_value(p, hap, w, &f);
        ki[e] = (int32_t)p[HH_E_I];
        kj[e] = (int32_t)p[HH_E_J];
        flt[e] = f;
    }
}

extern "C" int hh_links_fetch_phased(hh_links* lk, const int32_t* hap, double w, int32_t* key_i, int32_t* key_j, double* values,
                                     uint8_t* is_float, int64_t* n_out) {
    HH_REQUIRE(lk && hap && key_i && key_j && values && is_float && n_out, HH_ERR_ARG, "hh_links_fetch_phased: NULL argument");
    HH_REQUIRE(w >= 0.0 && w <= 1.0, HH_ERR_ARG, "hh_links_fetch_phased: phasing weight %g outside [0, 1]", w);
    hh_scope _scope(lk->ctx);
    HH_REQUIRE(lk->finished, HH_ERR_STATE, "hh_links_fetch_phased: call hh_links_finish first");
    *n_out = 0;
    if (lk->nnz == 0) return HH_OK;
    hh_ctx* ctx = lk->ctx;
    HH_CHECK(links_order_list(lk));
    const int64_t nnz = lk->nnz;
    int32_t* d_hap = nullptr;
    uint32_t *d_order = nullptr, *d_kept = nullptr;
    uint8_t* d_soa = nullptr;
    unsigned long long* d_n = nullptr;
    const int rc = [&]() -> int {
        HH_CHECK(hh_dmalloc(&d_hap, (size_t)lk->n_ctg));
        HH_CHECK(hh_dmalloc(&d_order, (size_t)nnz));
        HH_CHECK(hh_dmalloc(&d_n, 1));
        HH_CUDA(cudaMemcpyAsync(d_hap, hap, (size_t)lk->n_ctg * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
        HH_CUDA(cudaMemsetAsync(d_n, 0, sizeof(unsigned long long), ctx->stream));
        HH_LAUNCH(ctx, hh_k_phased_mark, links_grid(ctx, nnz), 256, 0, lk->d_compact, nnz, d_hap, w, d_order, d_n);
        unsigned long long n_kept = 0;
        HH_CUDA(cudaMemcpyAsync(&n_kept, d_n, sizeof(n_kept), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        const int64_t n = (int64_t)n_kept;
        *n_out = n;
        if (n == 0) return HH_OK;
        // stable: the kept entries stay in dict insertion order
        HH_CHECK(hh_dmalloc(&d_kept, (size_t)n * HH_E_WORDS));
        HH_CHECK(links_compact(lk, d_order, nnz, nullptr, reinterpret_cast<const hh_slot*>(lk->d_compact), d_kept));
        HH_CHECK(hh_dmalloc(&d_soa, (size_t)n * 17));
        int32_t* ki = reinterpret_cast<int32_t*>(d_soa);
        double* val = reinterpret_cast<double*>(d_soa + (size_t)n * 8);
        uint8_t* flt = d_soa + (size_t)n * 16;
        HH_LAUNCH(ctx, hh_k_phased_split, links_grid(ctx, n), 256, 0, d_kept, n, d_hap, w, ki, ki + n, val, flt, lk->d_ul_key,
                  lk->d_ul_slot, lk->n_ul);
        HH_CUDA(cudaMemcpyAsync(key_i, ki, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaMemcpyAsync(key_j, ki + n, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaMemcpyAsync(values, val, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaMemcpyAsync(is_float, flt, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        return HH_OK;
    }();
    hh_dfree(d_hap);
    hh_dfree(d_order);
    hh_dfree(d_kept);
    hh_dfree(d_soa);
    hh_dfree(d_n);
    return rc;
}

extern "C" int hh_links_set_ul_pairs(hh_links* lk, const int32_t* key_i, const int32_t* key_j, const int32_t* ht_slot, int64_t n_pairs) {
    HH_REQUIRE(lk && n_pairs >= 0 && (n_pairs == 0 || (key_i && key_j && ht_slot)), HH_ERR_ARG, "hh_links_set_ul_pairs: bad argument");
    hh_scope _scope(lk->ctx);
    hh_ctx* ctx = lk->ctx;
    HH_CUDA(cudaSetDevice(ctx->device));
    std::vector<std::pair<unsigned long long, int32_t>> pairs((size_t)n_pairs);
    for (int64_t k = 0; k < n_pairs; ++k) {
        HH_REQUIRE(key_i[k] >= 0 && key_i[k] < lk->n_ctg && key_j[k] >= 0 && key_j[k] < lk->n_ctg && key_i[k] != key_j[k] &&
                       ht_slot[k] >= 0 && ht_slot[k] < 4,
                   HH_ERR_ARG, "hh_links_set_ul_pairs: pair %lld is out of range", (long long)k);
        pairs[(size_t)k] = {((unsigned long long)key_i[k] << 32) | (uint32_t)key_j[k], ht_slot[k]};
    }
    std::sort(pairs.begin(), pairs.end());
    for (size_t k = 1; k < pairs.size(); ++k)
        HH_REQUIRE(pairs[k].first != pairs[k - 1].first, HH_ERR_ARG, "hh_links_set_ul_pairs: a contig pair is listed twice");
    hh_dfree(lk->d_ul_key);
    hh_dfree(lk->d_ul_slot);
    lk->d_ul_key = nullptr;
    lk->d_ul_slot = nullptr;
    lk->n_ul = 0;
    if (n_pairs == 0) return HH_OK;
    std::vector<unsigned long long> keys((size_t)n_pairs);
    std::vector<int32_t> slots((size_t)n_pairs);
    for (size_t k = 0; k < pairs.size(); ++k) {
        keys[k] = pairs[k].first;
        slots[k] = pairs[k].second;
    }
    HH_CHECK(hh_dmalloc(&lk->d_ul_key, (size_t)n_pairs));
    HH_CHECK(hh_dmalloc(&lk->d_ul_slot, (size_t)n_pairs));
    HH_CUDA(cudaMemcpyAsync(lk->d_ul_key, keys.data(), keys.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, ctx->stream));
    HH_CUDA(cudaMemcpyAsync(lk->d_ul_slot, slots.data(), slots.size() * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    HH_CUDA(cudaStreamSynchronize(ctx->stream));
    lk->n_ul = n_pairs;
    return HH_OK;
}

extern "C" int hh_links_fetch_ctg(hh_links* lk, int64_t* ctg_links) {
    HH_REQUIRE(lk && ctg_links, HH_ERR_ARG, "hh_links_fetch_ctg: NULL argument");
    HH_CUDA(cudaSetDevice(lk->ctx->device));
    HH_CUDA(cudaMemcpyAsync(ctg_links, lk->d_ctg, (size_t)lk->n_ctg * sizeof(int64_t), cudaMemcpyDeviceToHost, lk->ctx->stream));
    HH_CUDA(cudaStreamSynchronize(lk->ctx->stream));
    return HH_OK;
}

extern "C" int hh_links_export(hh_links* lk, uint32_t* entries_dev, int64_t* ctg_links_dev) {
    HH_REQUIRE(lk != nullptr, HH_ERR_ARG, "hh_links_export: NULL handle");
    HH_REQUIRE(lk->finished, HH_ERR_STATE, "hh_links_export: call hh_links_finish first");
    HH_CUDA(cudaSetDevice(lk->ctx->device));
    if (entries_dev && lk->nnz)
        HH_CUDA(cudaMemcpyAsync(entries_dev, lk->d_compact, (size_t)lk->nnz * HH_E_WORDS * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
                                lk->ctx->stream));
    if (ctg_links_dev)
        HH_CUDA(cudaMemcpyAsync(ctg_links_dev, lk->d_ctg, (size_t)lk->n_ctg * sizeof(int64_t), cudaMemcpyDeviceToDevice,
                                lk->ctx->stream));
    HH_CUDA(cudaStreamSynchronize(lk->ctx->stream));
    return HH_OK;
}

extern "C" int hh_links_merge(hh_links* lk, const uint32_t* entries_dev, int64_t n_entries, const int64_t* ctg_links_dev,
                              int64_t n_records, int64_t n_used) {
    HH_REQUIRE(lk != nullptr, HH_ERR_ARG, "hh_links_merge: NULL handle");
    hh_scope _scope(lk->ctx);
    HH_REQUIRE(lk->mode != 2 && !(lk->finished && lk->d_keys == nullptr), HH_ERR_STATE,
               "hh_links_merge: this table holds an entry list (hh_links_adopt / partitioned counting), not a hash table");
    lk->mode = 1;
    HH_CHECK(links_need_table(lk));
    lk->finished = false;   // a finished table is re-opened: the next hh_links_finish rebuilds the ordered view
    lk->gen++;
    HH_REQUIRE(n_entries >= 0 && (entries_dev || n_entries == 0), HH_ERR_ARG, "hh_links_merge: bad entries");
    hh_ctx* ctx = lk->ctx;
    HH_CUDA(cudaSetDevice(ctx->device));
    if (n_entries) {
        HH_CHECK(links_ensure_capacity(lk, n_entries));
        const int grid = links_grid(ctx, n_entries);
        HH_LAUNCH(ctx, hh_k_links_merge, grid, 256, 0, entries_dev, n_entries, lk->d_keys, lk->d_vals, lk->cap, lk->d_counters);
        lk->since_known += n_entries;
    }
    if (ctg_links_dev)
        HH_LAUNCH(ctx, hh_k_add_u64, (lk->n_ctg + 255) / 256, 256, 0, lk->d_ctg, ctg_links_dev, lk->n_ctg);
    HH_CUDA(cudaStreamSynchronize(ctx->stream));
    lk->n_records += n_records;
    lk->peer_used += n_used;
    return HH_OK;
}

extern "C" int hh_links_linked_index(hh_links* lk, const uint8_t* keep, int32_t* index, int32_t* n_linked) {
    return hh_links_linked_index_phased(lk, keep, 0, nullptr, 0.0, index, n_linked);
}

// The index, the degrees and the passing count depend on the table and on (keep, hap, w, normalize_by_nlinks) only.  They
// are kept with what they were computed from, and a call with the same table generation and the same array contents
// reuses them: bench.py, `haphic cluster` and dist.py call linked_index and then to_matrix with the same arguments.
static bool links_index_current(const hh_links* lk, const uint8_t* keep, int normalize, const int32_t* hap, double w) {
    if (!lk->ix_valid || lk->ix_gen != lk->gen || lk->ix_normalize != normalize) return false;
    if ((hap != nullptr) != !lk->ix_hap.empty()) return false;
    if (hap && (lk->ix_w != w || memcmp(hap, lk->ix_hap.data(), (size_t)lk->n_ctg * sizeof(int32_t)) != 0)) return false;
    return memcmp(keep, lk->ix_keep.data(), (size_t)lk->n_ctg) == 0;
}

extern "C" int hh_links_linked_index_phased(hh_links* lk, const uint8_t* keep, int normalize_by_nlinks, const int32_t* hap,
                                            double w, int32_t* index, int32_t* n_linked) {
    HH_REQUIRE(lk && keep, HH_ERR_ARG, "hh_links_linked_index: NULL argument");
    hh_scope _scope(lk->ctx);
    HH_REQUIRE(lk->finished, HH_ERR_STATE, "hh_links_linked_index: call hh_links_finish first");
    HH_REQUIRE(!hap || (w >= 0.0 && w <= 1.0), HH_ERR_ARG, "hh_links_linked_index_phased: phasing weight %g outside [0, 1]", w);
    hh_ctx* ctx = lk->ctx;
    HH_CUDA(cudaSetDevice(ctx->device));
    const int n_ctg = lk->n_ctg;
    if (!links_index_current(lk, keep, normalize_by_nlinks, hap, w)) {
        lk->ix_valid = false;
        lk->phased = hap != nullptr;
        if (hap) {
            if (!lk->d_hap) HH_CHECK(hh_dmalloc(&lk->d_hap, (size_t)n_ctg));
            HH_CUDA(cudaMemcpyAsync(lk->d_hap, hap, (size_t)n_ctg * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
        }
        unsigned long long *d_touch = nullptr, *d_touch_sorted = nullptr;
        int32_t *d_frag = nullptr, *d_frag_sorted = nullptr;
        uint8_t* d_tmp = nullptr;
        int rc = [&]() -> int {
            HH_CHECK(hh_dmalloc(&d_touch, (size_t)n_ctg * 2));
            HH_CHECK(hh_dmalloc(&d_frag, (size_t)n_ctg * 2));
            d_touch_sorted = d_touch + n_ctg;
            d_frag_sorted = d_frag + n_ctg;
            // touch values are below 2^33 and the untouched ones (all bits set) are 2^34 - 1 in the low 34 bits
            size_t tmp_bytes = 0;
            HH_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_touch, d_touch_sorted, d_frag, d_frag_sorted, n_ctg, 0, 34,
                                                    ctx->stream));
            HH_CHECK(hh_dmalloc(&d_tmp, tmp_bytes));
            HH_CUDA(cudaMemcpyAsync(lk->d_keep, keep, (size_t)n_ctg, cudaMemcpyHostToDevice, ctx->stream));
            HH_CUDA(cudaMemsetAsync(d_touch, 0xFF, (size_t)n_ctg * sizeof(unsigned long long), ctx->stream));
            HH_CUDA(cudaMemsetAsync(lk->d_deg, 0, (size_t)n_ctg * sizeof(int32_t), ctx->stream));
            unsigned long long* d_out = reinterpret_cast<unsigned long long*>(ctx->d_scratch + 8);   // [0] touched  [1] passing
            HH_CUDA(cudaMemsetAsync(d_out, 0, 2 * sizeof(unsigned long long), ctx->stream));
            if (lk->nnz) {
                int grid = 0;
                HH_CHECK(hh_resident_grid(ctx, hh_k_touch, 256, 0, &grid));
                grid = std::min(grid, links_grid(ctx, lk->nnz));
                HH_LAUNCH(ctx, hh_k_touch, grid, 256, 0, lk->d_compact, lk->nnz, lk->d_keep, lk->d_ctg, normalize_by_nlinks,
                          hh_links_hap_dev(lk), w, d_touch, lk->d_deg, d_out + 1);
            }
            HH_LAUNCH(ctx, hh_k_iota_i32, (n_ctg + 255) / 256, 256, 0, d_frag, n_ctg);
            HH_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_touch, d_touch_sorted, d_frag, d_frag_sorted, n_ctg, 0, 34,
                                                    ctx->stream));
            HH_LAUNCH(ctx, hh_k_rank_sorted, (n_ctg + 255) / 256, 256, 0, d_touch_sorted, d_frag_sorted, n_ctg, lk->d_index, d_out);
            HH_CUDA(cudaMemcpyAsync(ctx->h_scratch + 8, d_out, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
            HH_CUDA(cudaStreamSynchronize(ctx->stream));
            lk->n_linked = (int32_t)ctx->h_scratch[8];
            lk->n_pass = (int64_t)ctx->h_scratch[9];
            return HH_OK;
        }();
        hh_dfree(d_touch);
        hh_dfree(d_frag);
        hh_dfree(d_tmp);
        HH_CHECK(rc);
        lk->ix_keep.assign(keep, keep + n_ctg);
        if (hap) lk->ix_hap.assign(hap, hap + n_ctg);
        else lk->ix_hap.clear();
        lk->ix_w = w;
        lk->ix_normalize = normalize_by_nlinks;
        lk->ix_gen = lk->gen;
        lk->ix_valid = true;
    }
    if (index) {
        HH_CUDA(cudaMemcpyAsync(index, lk->d_index, (size_t)n_ctg * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    if (n_linked) *n_linked = lk->n_linked;
    return HH_OK;
}

extern "C" int hh_links_destroy(hh_links* lk) {
    if (!lk) return HH_OK;
    hh_scope _scope(lk->ctx);
    cudaSetDevice(lk->ctx->device);
    cudaStreamSynchronize(lk->ctx->stream);
    if (lk->copy_stream) {
        cudaStreamSynchronize(lk->copy_stream);
        cudaStreamDestroy(lk->copy_stream);
    }
    for (int k = 0; k < 2; ++k) {
        if (lk->ev_copied[k]) cudaEventDestroy(lk->ev_copied[k]);
        if (lk->ev_consumed[k]) cudaEventDestroy(lk->ev_consumed[k]);
        if (lk->d_stage[k]) cudaFree(lk->d_stage[k]);
    }
    hh_dfree(lk->d_src_rank);
    hh_dfree(lk->d_fbase);
    hh_dfree(lk->d_len);
    hh_dfree(lk->d_rank);
    hh_dfree(lk->d_nx);
    hh_dfree(lk->d_ctg);
    hh_dfree(lk->d_keys);
    hh_dfree(lk->d_vals);
    hh_dfree(lk->d_counters);
    hh_dfree(lk->d_compact);
    hh_dfree(lk->d_index);
    hh_dfree(lk->d_keep);
    hh_dfree(lk->d_hap);
    hh_dfree(lk->d_deg);
    hh_dfree(lk->d_ul_key);
    hh_dfree(lk->d_ul_slot);
    links_free_partsets(lk);
    delete lk;
    return HH_OK;
}

// accessors used by hh_matrix.cu
int32_t hh_links_n_ctg(hh_links* lk) { return lk->n_ctg; }
hh_ctx* hh_links_ctx(hh_links* lk) { return lk->ctx; }
const uint32_t* hh_links_compact(hh_links* lk, int64_t* nnz) { *nnz = lk->nnz; return lk->d_compact; }
const unsigned long long* hh_links_ctg_totals(hh_links* lk) { return lk->d_ctg; }
const int32_t* hh_links_index_dev(hh_links* lk, int32_t* n_linked) { *n_linked = lk->n_linked; return lk->d_index; }
const int32_t* hh_links_degree_dev(hh_links* lk, int64_t* n_pass) { *n_pass = lk->n_pass; return lk->d_deg; }
uint8_t* hh_links_keep_dev(hh_links* lk) { return lk->d_keep; }
bool hh_links_finished(hh_links* lk) { return lk->finished; }
const int32_t* hh_links_hap_dev(hh_links* lk) { return lk->phased ? lk->d_hap : nullptr; }
