/*
 * haphic_b200 -- C ABI of the GPU-native (H100, sm_90a) `haphic cluster` hot path.
 *
 * This is the drop-in boundary: a plain C interface (pointers + sizes, no torch / C++ types)
 * that a maintainer of zengxiaofei/HapHiC would bind with ctypes from
 * scripts/HapHiC_cluster.py (see INTEGRATION.md).  The reference has no FFI of its own -- the
 * whole path is in-process Python -- so every entry point below names the reference function
 * (file:line in scripts/HapHiC_cluster.py, v1.0.7) whose work it replaces.
 *
 * Conventions
 *   - every function returns HH_OK (0) or an HH_ERR_* code; hh_last_error() gives the message
 *     (thread-local);
 *   - objects are opaque handles owned by the library until the matching *_destroy;
 *   - `mem` arguments say where a caller buffer lives: HH_MEM_HOST (pageable or pinned host
 *     memory) or HH_MEM_DEVICE (device memory of the context's GPU, e.g. a torch tensor's
 *     data_ptr());  all *_fetch_* outputs are HOST buffers sized by the caller from the
 *     preceding *_info call;
 *   - all calls are synchronous on return unless stated otherwise;
 *   - there is NO CPU fallback: without a CUDA device hh_ctx_create fails.
 *
 * Contig identifiers are dense int32 ids in FASTA order; the host keeps the name <-> id map
 * (fa_dict, HapHiC_cluster.py:87-113).  Where the reference orders by contig NAME
 * (`sorted(((ref, pos+1), (mref, mpos+1)))`, 1629) the caller passes `name_rank`.
 */
#ifndef HAPHIC_B200_H
#define HAPHIC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HH_VERSION 100

enum {
    HH_OK = 0,
    HH_ERR_CUDA = 1,      /* CUDA runtime / launch failure            */
    HH_ERR_ARG = 2,       /* invalid argument                         */
    HH_ERR_CAPACITY = 3,  /* a bounded device structure overflowed    */
    HH_ERR_NOMEM = 4,     /* device allocation failed                 */
    HH_ERR_STATE = 5,     /* call sequence violated                   */
    HH_ERR_UNSUPPORTED = 6
};

enum { HH_MEM_HOST = 0, HH_MEM_DEVICE = 1 };

typedef struct hh_ctx hh_ctx;       /* one GPU + one stream                                   */
typedef struct hh_links hh_links;   /* link counters of one run (full/flank/HT/per-fragment)  */
typedef struct hh_matrix hh_matrix; /* contig x contig link matrix, MCL-ready                 */
typedef struct hh_mcl hh_mcl;       /* Markov-cluster state: M0, pre-expanded M1, iterates     */

int hh_version(void);
const char* hh_last_error(void);

/* ---- context ------------------------------------------------------------------------- */
int hh_ctx_create(int device, hh_ctx** out);
int hh_ctx_destroy(hh_ctx* ctx);
int hh_ctx_sync(hh_ctx* ctx);
/* the cudaStream_t every kernel of this context is launched on (for CUDA-event timing) */
void* hh_ctx_stream(hh_ctx* ctx);
int hh_ctx_device(hh_ctx* ctx);
int hh_ctx_sm_count(hh_ctx* ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
int64_t hh_ctx_launches(hh_ctx* ctx);

/* ---- link counting: parse_alignments_for_ctgs, HapHiC_cluster.py:1596-1655 ----------------
 * One record per read pair: int32 {ctg_a, pos_a, ctg_b, pos_b}, positions 0-based exactly as
 * the generators yield them (1562-1593).  Records with ctg_a == ctg_b are dropped
 * (pairs_generator_inter_ctgs, 1582; BAM filter `refid != mrefid`, 2862), records naming an
 * id outside [0, n_ctg) are skipped (1625).
 *   ctg_len[n_ctg]   contig lengths (frag_len_dict)
 *   name_rank[n_ctg] rank of each contig under Python str ordering of the names (1629)
 *   in_nx[n_ctg]     1 if the contig is in Nx_ctg_set (stat_fragments, 273-288)
 *   flank_bp         args.flank * 1000 (1603); 0 = whole contig (is_flank, 299-307)
 *   capacity_hint    expected number of distinct contig pairs (0 = let the table grow)
 */
int hh_links_create(hh_ctx* ctx, int32_t n_ctg, const int64_t* ctg_len, const int32_t* name_rank,
                    const uint8_t* in_nx, int64_t flank_bp, int64_t capacity_hint, hh_links** out);
/* Fragment mode -- parse_alignments, HapHiC_cluster.py:1658-1752 (some contig longer than bin_size): records
 * still name CONTIGS, the table is keyed by FRAGMENT pairs.  Contig c owns the fragment ids
 * [frag_base[c], frag_base[c+1]); more than one fragment means the contig is split into bins of `bin_size` bp
 * (bin = ceil(coord / bin_size), convert_frags 1662-1670).  Pairs inside one unsplit contig or one bin are
 * dropped (1699, 1715); ends are ordered by contig name then coordinate (1707) and, when a bin is involved,
 * re-ordered by fragment name rank (1719-1720).  Counts the flank links between fragments and the
 * per-fragment totals (1723-1726); its full/HT counters refer to fragment pairs and have no counterpart in the
 * reference -- full_link_dict / HT_link_dict / clm of that run come from a second, contig-level table fed
 * with the same records (hh_links_create with in_nx = 0). */
int hh_links_create_frags(hh_ctx* ctx, int32_t n_ctg, const int32_t* ctg_rank, const int32_t* frag_base,
                          int32_t n_frag, const int64_t* frag_len, const int32_t* frag_rank,
                          const uint8_t* frag_in_nx, int64_t bin_size, int64_t flank_bp, int64_t capacity_hint,
                          hh_links** out);
/* stream `n_rec` more records; `stream_offset` is the index of rec[0] in the whole read stream
 * (first-seen order of dict keys is reproduced from it; use the running total on one GPU, the
 * shard offset when the stream is split over ranks).  May be called repeatedly. */
int hh_links_add(hh_links* lk, const int32_t* rec, int64_t n_rec, int64_t stream_offset, int mem);
/* asynchronous variant for device-resident records: returns after enqueueing (no growth check:
 * the caller guarantees capacity_hint was sufficient; overflow is reported by hh_links_finish) */
int hh_links_add_async(hh_links* lk, const int32_t* rec_dev, int64_t n_rec, int64_t stream_offset);

typedef struct {
    int64_t n_records;   /* records seen                                        */
    int64_t n_used;      /* records counted (passed the id / inter-contig tests) */
    int64_t nnz_full;    /* len(full_link_dict)                                  */
    int64_t nnz_flank;   /* len(flank_link_dict)                                 */
    int64_t table_slots; /* hash-table capacity at the end                       */
} hh_links_info;

/* close the stream: orders the distinct pairs by first appearance (dict insertion order) */
int hh_links_finish(hh_links* lk, hh_links_info* info);
/* how the finish of a partitioned count (long streams; hh_links_finish or hh_links_finish_partition) aggregated: the
 * number of hash buckets, those counted in a shared-memory table, and those counted by the global-table fallback
 * (too many records or distinct pairs for shared memory).  All 0 for a table counted directly.  Any pointer may be NULL. */
int hh_links_agg_info(hh_links* lk, int64_t* buckets, int64_t* smem_buckets, int64_t* fallback_buckets);
/* bytes per record of the partitioned count: of every partition set opened so far, in order (the first max_sets of them
 * to set_bytes, their number to *n_sets), and of the bucket buffer of its finish (*bucket_bytes, 0 before the finish).
 * 8 = the narrow format (at most 65,536 objects and stream indices below 2^29), 16 = the wide one.  No sets and 0 for a
 * table counted directly.  set_bytes may be NULL when max_sets <= 0, the other pointers always. */
int hh_links_record_bytes(hh_links* lk, int32_t* set_bytes, int32_t max_sets, int32_t* n_sets, int32_t* bucket_bytes);

/* full_link_dict / flank_link_dict / HT_link_dict as parallel arrays of nnz_full entries in
 * full_link_dict insertion order (1649).  key_i/key_j: contig ids with name(key_i) < name(key_j).
 * first_full / first_flank: stream index of the record that created the key in the respective
 * dict (first_flank = 0xFFFFFFFF when flank == 0).  ht[4*e + 2*ti + tj]: HT_link_dict counts,
 * ti/tj = 1 for the `_T` half (`coord*2 > len`, 404-416).  Any pointer may be NULL. */
int hh_links_fetch(hh_links* lk, int32_t* key_i, int32_t* key_j, uint32_t* full, uint32_t* flank,
                   uint32_t* first_full, uint32_t* first_flank, uint32_t* ht);
/* full_link_dict after reduce_inter_hap_HiC_links (695-707, --gfa with >= 2 haplotype files): hap[n_ctg] (host) is the
 * haplotype index of every contig, w in [0, 1] the phasing weight.  An entry whose ends differ in hap becomes x - x * w
 * (fp64, two roundings, x = the full count) and is a Python float (is_float = 1); the others keep their count (is_float = 0).
 * Entries that become exactly 0 are deleted; the rest keep dict insertion order.  The outputs are host buffers of nnz_full
 * entries, of which the first *n_out are written. */
int hh_links_fetch_phased(hh_links* lk, const int32_t* hap, double w, int32_t* key_i, int32_t* key_j, double* values,
                          uint8_t* is_float, int64_t* n_out);
/* The contig pairs that ultra-long reads join (add_HT_links_based_on_ul 1912-1933 and the full links of
 * add_flank_and_full_links_based_on_ul 1936-1985): key_i / key_j [n_pairs] (host) as in hh_links_fetch (name(key_i) <
 * name(key_j)), ht_slot the HT_link_dict slot 2 * ti + tj of the joined semi-contigs.  From then on hh_links_fetch returns
 * those entries with the full count and that HT slot doubled (HH still derived from the stored counts) and
 * hh_links_fetch_phased doubles the full count before the reduction; the stored counts are not changed.  A doubled count
 * above 2^32 - 1 fails the fetch.  Pairs absent from the table are ignored; n_pairs = 0 detaches the list. */
int hh_links_set_ul_pairs(hh_links* lk, const int32_t* key_i, const int32_t* key_j, const int32_t* ht_slot, int64_t n_pairs);
/* ctg_link_dict (1638-1639): per-contig flank-link totals, [n_ctg] */
int hh_links_fetch_ctg(hh_links* lk, int64_t* ctg_links);
/* multi-GPU: export the finished table as device arrays / merge a peer's export into this
 * table (a finished table is re-opened; call hh_links_finish again afterwards).  An export is 9 uint32 per entry: {i, j, full, flank, first_full,
 * first_flank, HT, TH, TT}.  ctg totals travel separately (int64 [n_ctg]). */
int hh_links_export(hh_links* lk, uint32_t* entries_dev, int64_t* ctg_links_dev);
int hh_links_merge(hh_links* lk, const uint32_t* entries_dev, int64_t n_entries, const int64_t* ctg_links_dev,
                   int64_t n_records, int64_t n_used);
/* Routed multi-GPU counting (SURVEY.md 8e "route each pair to its owner"): every contig pair is owned by one rank
 * (hash of the unordered contig pair), so the partition tables are disjoint and nothing is reduced afterwards.
 *   hh_links_route:  split this rank's shard of the stream (device records, global index of rec[0] = stream_offset)
 *     into `world` destination groups: rec_out_dev [n_rec][4] / pos_out_dev [n_rec] receive records and their stream
 *     indices grouped by owner, counts[world] (host) the group sizes.  Records that can never be used (same contig,
 *     ids outside the FASTA) are dropped here.  The caller exchanges the groups (all-to-all).
 *   hh_links_add_routed: count records with explicit stream indices (any order).
 *   hh_links_finish_partition: compact list of this rank's partition (unordered); hh_links_export hands it out.
 *   hh_links_adopt: the table becomes the union of all partitions (entries = concatenated exports [n][9],
 *     ctg_links / n_records / n_used summed over ranks, stream_end = length of the whole stream).  The index,
 *     the matrix and hh_links_fetch (which restores dict insertion order on first use) work as after hh_links_finish. */
int hh_links_route(hh_links* lk, const int32_t* rec_dev, int64_t n_rec, int64_t stream_offset, int world,
                   int32_t* rec_out_dev, uint32_t* pos_out_dev, int64_t* counts);
int hh_links_add_routed(hh_links* lk, const int32_t* rec_dev, const uint32_t* pos_dev, int64_t n_rec);
int hh_links_finish_partition(hh_links* lk, hh_links_info* info);
int hh_links_adopt(hh_links* lk, const uint32_t* entries_dev, int64_t n_entries, const int64_t* ctg_links_dev,
                   int64_t n_records, int64_t n_used, int64_t stream_end);
int hh_links_destroy(hh_links* lk);

/* ---- dict_to_matrix, HapHiC_cluster.py:310-373 ------------------------------------------------
 * Two steps because the reference appends kept-but-unlinked fragments in Python set order
 * (355-359), which only the host can reproduce:
 *   hh_links_linked_index: first-seen index of every fragment that occurs in flank_link_dict
 *     restricted to `keep` (327-349); index[c] = -1 otherwise; *n_linked = len(frags_in_dict).
 *   hh_matrix_from_links: builds the symmetric fp32 matrix, with self loops = 1 when add_self_loops (351-364);
 *     `tail[n_tail]` lists the kept-but-unlinked contig ids in the order they get the following
 *     indices.  normalize_by_nlinks != 0 applies links / sqrt(tot_i * tot_j) first (718-724).  A matrix of more than
 *     2^22 fragments (n_linked + n_tail) is refused with HH_ERR_ARG.
 */
int hh_links_linked_index(hh_links* lk, const uint8_t* keep, int32_t* index, int32_t* n_linked);
int hh_matrix_from_links(hh_links* lk, const uint8_t* keep, const int32_t* tail, int32_t n_tail,
                         int normalize_by_nlinks, int add_self_loops, hh_matrix** out);
/* The same two steps on the phasing-reduced flank_link_dict (reduce_inter_hap_HiC_links, 695-707, with --gfa of >= 2
 * haplotype files): hap[n_ctg] (host) is the haplotype index of every fragment of the table's id space, w in [0, 1] the
 * phasing weight.  An entry whose ends differ in hap becomes x - x * w (fp64, two roundings; x = the flank count, or the
 * normalised value when normalize_by_nlinks) and is absent when that is exactly 0: it then sets no first-seen index and no
 * matrix entry.  hap = NULL is the unphased call above (which is this one with hap = NULL); hh_matrix_from_links_phased
 * recomputes the indices with its own arguments, so give both calls the same keep / normalize_by_nlinks / hap / w. */
int hh_links_linked_index_phased(hh_links* lk, const uint8_t* keep, int normalize_by_nlinks, const int32_t* hap, double w,
                                 int32_t* index, int32_t* n_linked);
int hh_matrix_from_links_phased(hh_links* lk, const uint8_t* keep, const int32_t* tail, int32_t n_tail,
                                int normalize_by_nlinks, int add_self_loops, const int32_t* hap, double w, hh_matrix** out);
/* hh_matrix_from_links_phased with the ultra-long-read boost of add_flank_and_full_links_based_on_ul (1936-1985): ul_path and
 * ul_parent [n_ctg] (host) give every fragment of the table the path id of its contig (-1 = on no path) and the id of its
 * contig (a bin's parent).  An entry whose ends lie on two different contigs of one path counts twice, after normalisation
 * and before the phasing reduction.  Doubling deletes no entry, so the first-seen indices are those of
 * hh_links_linked_index_phased with the same keep / normalize_by_nlinks / hap / w.  ul_path = NULL is
 * hh_matrix_from_links_phased. */
int hh_matrix_from_links_ex(hh_links* lk, const uint8_t* keep, const int32_t* tail, int32_t n_tail, int normalize_by_nlinks,
                            int add_self_loops, const int32_t* hap, double w, const int32_t* ul_path, const int32_t* ul_parent,
                            hh_matrix** out);
/* rank-sum statistic of filter_fragments, HapHiC_cluster.py:864-892, on a matrix WITHOUT self loops: for every
 * fragment, sort its row by links descending (ties by matrix index, a stable list.sort(reverse=True)), take
 * the first topN fragments and sum min(rank_a(b), rank_b(a)) over their pairs.  rank_sum[n] (host) is
 * indexed by matrix index.  topN <= 32. */
int hh_matrix_rank_sums(hh_matrix* m, int topN, int64_t* rank_sum);
/* the same matrix from a host CSC (symmetric, self loops included) -- the entry point when host
 * code edited the link dict (allele-aware removal, UL boosts, phasing weights: 2911-2928) */
int hh_matrix_from_csc(hh_ctx* ctx, int32_t n, const int64_t* indptr, const int32_t* indices,
                       const float* data, hh_matrix** out);
int hh_matrix_info(hh_matrix* m, int32_t* n, int64_t* nnz);
/* canonical CSC (row-sorted) of the raw link matrix, host buffers: indptr[n+1], indices/data[nnz] */
int hh_matrix_fetch_csc(hh_matrix* m, int64_t* indptr, int32_t* indices, float* data);
int hh_matrix_destroy(hh_matrix* m);

/* ---- reassignment statistics over the full links: output_statistics, HapHiC_cluster.py:2279-2478 ---------------------
 * For every form of full_link_dict: integer counts (is_float all 0), or ints and Python floats after a fractional phasing
 * weight or a link scaling; every result is the reference's fp64 arithmetic in the reference's order, bit for bit.
 *   hh_stats_create: the full links (n_entries in dict insertion order, values exact integers or floats, is_float per
 *     entry), kept on the device for every later call.  n_entries < 2^30.
 *   hh_stats_rank: parse_link_dict (2245-2258) and the ranking of 2373 for group[n_ctg] (host; -1 = ungrouped, else
 *     < n_groups): the links of every contig into every group, summed by sequential fp64 adds in the order parse_link_dict
 *     visits them (first end of entry 0, second end of entry 0, first end of entry 1, ...), a sum being a float iff one of
 *     its links is; each contig's groups ranked by sum descending, ties by the first visit.  *n_ranked = number of
 *     (contig, group) sums.
 *   hh_stats_fetch_ranked: those sums in (contig, rank) order, host buffers of n_ranked entries (any may be NULL).
 *   hh_stats_best: the three per-contig quantities of 2373-2400 over the last ranking, host buffers of n_ctg entries:
 *     has = the contig has a ranked list; top_links / top_is_float = links to the first group; top_density =
 *     cal_link_density to it; others = the sum of the densities of the other ranked groups in rank order (CPython >= 3.12
 *     sum() with its Neumaier compensation when `compensated`, else plain adds) / (n_groups - 1), 0 when n_groups == 1;
 *     ratio = top_density / others (inf or nan when others == 0).  group_re[n_groups] = RE sites of every group,
 *     ctg_re[n_ctg] = RE sites of every contig. */
typedef struct hh_stats hh_stats;
int hh_stats_create(hh_ctx* ctx, int32_t n_ctg, const int32_t* key_i, const int32_t* key_j, const double* values,
                    const uint8_t* is_float, int64_t n_entries, hh_stats** out);
int hh_stats_rank(hh_stats* st, const int32_t* group, int32_t n_groups, int64_t* n_ranked);
int hh_stats_fetch_ranked(hh_stats* st, int32_t* ctg, int32_t* group, double* links, uint8_t* is_float);
int hh_stats_best(hh_stats* st, const int64_t* group_re, int32_t n_groups, const int64_t* ctg_re, int compensated, uint8_t* has,
                  double* top_links, uint8_t* top_is_float, double* top_density, double* others, double* ratio);
int hh_stats_destroy(hh_stats* st);

/* ---- Markov clustering: run_mcl_clustering / mcl / prune, HapHiC_cluster.py:1987-2062, 2132-2162
 * hh_mcl_create does 2144 (column-L1 normalise, M0) and 2146-2149 (pre-expansion M1 = M0^e, kept
 * resident and shared by the whole inflation sweep).  [col_lo, col_hi) is the block of columns
 * this context owns (0, n for one GPU): M1 and every iterate are computed for owned columns only.
 */
int hh_mcl_create(hh_matrix* m, int expansion, int32_t col_lo, int32_t col_hi, hh_mcl** out);
/* The same with the engine of the pre-expansion (2146-2149) chosen by the caller:
 *   HH_PREEXP_SPARSE  Gustavson SpGEMM on a shared-memory column accumulator (the reference's sparse mode,
 *                     mkl_matrix_power 2017-2023);
 *   HH_PREEXP_DENSE   the product as a symmetric dense GEMM on the tensor cores (wgmma / TMA; 16-bit operand
 *                     planes that reproduce the fp32 product to 2^-23, fp32 accumulation) -- the reference's dense mode
 *                     (`--dense_matrix`, numpy.linalg.matrix_power 2035 / 2149);
 *   HH_PREEXP_AUTO    whichever is estimated cheaper for this matrix (hh_mcl_create; env HH_MCL_PREEXP overrides).
 * Both engines give M1 within fp32 rounding of the exact product; every later step is shared. */
enum { HH_PREEXP_AUTO = 0, HH_PREEXP_SPARSE = 1, HH_PREEXP_DENSE = 2 };
int hh_mcl_create_ex(hh_matrix* m, int expansion, int32_t col_lo, int32_t col_hi, int preexp_mode, hh_mcl** out);
/* The engine hh_mcl_create_ex would pick for `requested` (SPARSE or DENSE; AUTO reads the free device memory now).  A sweep
 * over column blocks resolves it once and passes the result to every block, so that all columns of M1 come from one engine. */
int hh_mcl_choose_preexp(hh_matrix* m, int expansion, int requested, int* mode);
/* Device bytes an engine created with hh_mcl_create_ex(m, expansion, lo, lo + ncols, mode) holds at its peak, for iterates
 * pruned at `pruning`: m1_bytes = its dense block of M1 (grows with ncols), fixed_bytes = what does not depend on ncols
 * (M0 slots, the global column accumulators above 57,600 vertices, the GEMM operand planes of one K chunk, the unpruned
 * power slots of expansion > 2, the two iterate slots and the small per-vertex arrays).  mode must be SPARSE or DENSE. */
int hh_mcl_footprint(hh_matrix* m, int expansion, int32_t ncols, int mode, double pruning, size_t* m1_bytes, size_t* fixed_bytes);
/* free device memory plus the idle blocks of this context's workspace cache (released on demand by any allocation) */
int hh_ctx_mem_available(hh_ctx* ctx, size_t* bytes);
typedef struct {
    int32_t mode;          /* HH_PREEXP_SPARSE or HH_PREEXP_DENSE: what ran                              */
    int32_t a_planes;      /* dense: 16-bit planes of the count operand (1: integer counts, 3: weights)    */
    int32_t passes;        /* dense: tensor-core passes per k-block                                        */
    int32_t cta_group;     /* dense: 1 = one CTA per 128 x 128 tile                                          */
    int32_t stages;        /* dense: shared-memory pipeline stages                                         */
    int32_t chunk_kb;      /* dense: 64-wide k-blocks accumulated by wgmma between two round-to-nearest adds */
    float total_ms;        /* device time of the pre-expansion                                             */
    float densify_ms;      /* dense: operand planes from the CSC                                           */
    float gemm_ms;         /* dense: the GEMM kernel                                                       */
    float clip_ms;         /* dense: sparse correction for link counts above `clip` (0 when there are none) */
    double flops;          /* dense: tensor-core flops issued                                              */
    int64_t products;      /* sparse: Gustavson products (dense: products of the clip correction)          */
    float clip;            /* dense: counts enter the GEMM as min(count, clip): 2048 (f16 plane) / 256 (bf16) */
    int32_t b_planes;      /* dense: planes of the M0 operand (2: f16 hi + lo, 22 bits; 3: exact bf16)      */
    int32_t fmt_a, fmt_b;  /* dense: operand formats, 0 = bf16, 1 = f16                                    */
    int32_t k_chunks;      /* dense: launches the K range was cut into (operand planes of one chunk at a time) */
} hh_preexp_info;
int hh_mcl_preexp_info(hh_mcl* mc, hh_preexp_info* info);
/* normalize_ms / preexp_ms: device time of the two kernels hh_mcl_create ran */
int hh_mcl_info(hh_mcl* mc, int32_t* n, int64_t* nnz_m0, int64_t* preexp_products, float* normalize_ms,
                float* preexp_ms);
/* M0 as canonical CSC / owned block of M1 as dense column-major fp32 [n * (col_hi-col_lo)] */
int hh_mcl_fetch_m0(hh_mcl* mc, int64_t* indptr, int32_t* indices, float* data);
int hh_mcl_fetch_m1(hh_mcl* mc, float* dense);
/* columns [col_lo, col_hi) of M1 (absolute indices inside the owned block), dense column-major fp32 [n * (col_hi-col_lo)] */
int hh_mcl_fetch_m1_cols(hh_mcl* mc, int32_t col_lo, int32_t col_hi, float* dense);

typedef struct {
    int32_t rounds;          /* iterations executed ("after N rounds", 2047-2060)          */
    int32_t converged;       /* 1 if the convergence test (2044-2055) fired                 */
    int64_t nnz;             /* stored entries of the returned matrix                       */
    int64_t products;        /* sum over iterations of Gustavson products (flops / 2)       */
    int64_t bytes;           /* sum over iterations of algorithmic bytes (SURVEY.md 8d)     */
} hh_mcl_result;

/* one mcl() call (2026-2062) on one GPU owning all columns.  iter_nnz / iter_products /
 * iter_delta / iter_ms: optional host arrays of max_iter entries receiving per-iteration statistics
 * (iter_ms = device time of the iteration's column kernel, CUDA events on the context stream). */
int hh_mcl_run(hh_mcl* mc, double inflation, int max_iter, double pruning, hh_mcl_result* res,
               int64_t* iter_nnz, int64_t* iter_products, float* iter_delta, float* iter_ms);
/* the matrix hh_mcl_run (or the last hh_mcl_step + hh_mcl_commit) left, canonical CSC, host */
int hh_mcl_fetch_result(hh_mcl* mc, int64_t* indptr, int32_t* indices, float* data);

/* step-wise interface for column-sharded multi-GPU runs (one rank per GPU):
 *   begin -> { step -> pack -> [host: all-gather] -> unpack(peer blocks) -> commit } ...
 * hh_mcl_step computes iteration `it` (0-based; it == 0 streams the dense M1, 2030) for the owned
 * columns and returns their stats; *delta is max(|M - L| - 1e-5|L|) over owned columns (2045);
 * *kernel_ms the device time of the column kernel.
 * hh_mcl_pack writes the owned block as {len[col_hi-col_lo] int32} and packed {idx int32, val
 * fp32}[nnz_owned] into caller-provided DEVICE buffers; hh_mcl_unpack installs a peer's block. */
int hh_mcl_begin(hh_mcl* mc, double inflation, double pruning);
int hh_mcl_step(hh_mcl* mc, int it, int64_t* nnz_owned, int64_t* products, float* delta, float* kernel_ms);
int hh_mcl_pack(hh_mcl* mc, int32_t* len_dev, int32_t* idx_dev, float* val_dev);
int hh_mcl_unpack(hh_mcl* mc, int32_t col_lo, int32_t col_hi, const int32_t* len_dev,
                  const int32_t* idx_dev, const float* val_dev, int64_t nnz_block);
int hh_mcl_commit(hh_mcl* mc);
/* which engines the last hh_mcl_step ran (tests assert with it that the path they target was taken).  Counts are of the
 * columns this context computed in that step. */
typedef struct {
    int32_t it;              /* iteration number of the step (-1: no step since hh_mcl_begin)                      */
    int32_t iter0;           /* 1: hh_k_iter0 streamed the dense M1                                              */
    int32_t iter0_w;         /* its W (row blocks per column)                                                    */
    int32_t blk;             /* 1: the window components were multiplied by the block GEMM on the tensor cores   */
    int32_t blk_f16;         /* block GEMM operands: 1 = two f16 planes of M * 2^14 (four passes), 0 = three bf16 */
    int32_t blk_chunk;       /* block GEMM: k-blocks accumulated by wgmma between two round-to-nearest adds      */
    int64_t blk_ldk;         /* block GEMM: row pitch of the operand planes (largest window component, padded)   */
    int32_t n_win;           /* columns of window components (hh_k_col_win, or the block GEMM's epilogue)       */
    int32_t n_big;           /* columns of components wider than the window                                      */
    int32_t wmax;            /* window accumulator size                                                          */
    int32_t small;           /* 1: the nearly-converged branch ran hh_k_col_small                                */
    int32_t small_cols;      /* columns hh_k_col_small finished                                                  */
    int32_t small_overflow;  /* columns it sent to its overflow list (finished by hh_k_col)                      */
    int32_t col;             /* 1: hh_k_col<product, prune> was launched                                         */
    int32_t col_cols;        /* columns it was given (the overflow list, the wide components, or all owned)      */
    int32_t col_w;           /* its W                                                                            */
    int32_t col_smem;        /* 1: shared-memory accumulator, 0: global                                          */
    int32_t col_track;       /* TRACK (dirty-chunk bitmap)                                                       */
    int32_t col_flat;        /* FLAT (flat 32-entry walk)                                                        */
} hh_mcl_step_info_t;
int hh_mcl_step_info(hh_mcl* mc, hh_mcl_step_info_t* info);
/* change the block of columns the following steps compute (between hh_mcl_commit and hh_mcl_step, after iteration 0;
 * reset by hh_mcl_begin).  Column shards switch to (0, n) once the iterate is tiny: no exchange is needed any more
 * because every rank then computes the identical full iterate. */
int hh_mcl_set_block(hh_mcl* mc, int32_t col_lo, int32_t col_hi);
int hh_mcl_destroy(hh_mcl* mc);

/* ---- assembly correction (--correct_nrounds): correct_assembly and its helpers, HapHiC_cluster.py:943-1536 -----------
 * Contigs are the ids 0 .. n_ctg-1 of the input FASTA; `resolution` = --correct_resolution.  Fragments under examination
 * start as all contigs; after a round that is not the last they are the pieces of the fragments broken in it, with ids
 * n_frag, n_frag + 1, ... (n_frag as reported by that round) in breakpoint-list order, left to right.
 *   hh_correct_create: coverage arrays of len//res + 1 int32 bins per contig (1307-1311 / 1370-1374).
 *   hh_correct_add: the coverage pass over a batch of records {ctg_a, pos_a, ctg_b, pos_b} (parse_pairs_for_correction
 *     1321-1342, parse_bam_for_correction 1380-1396): same-contig records of contigs in the FASTA add 1 to the bins
 *     [lo//res, hi//res] (numpy slice semantics) and are kept as links; every other record is ignored.
 *   hh_correct_round: detect_break_points (943-1014) on the fragments under examination; unless last_round, the coverage
 *     and link updates of break_and_update_ctgs (1063-1113, 1151-1153, 1176-1178, 1192-1197).
 *   hh_correct_fetch_breaks: the round's breakpoints (fragment id, bin, coverage), n_breaks entries in the order of the
 *     fragments under examination, ascending bins (a breakpoint sits at bin * res on its fragment).
 *   hh_correct_info / hh_correct_fetch_cov: fragments under examination and their coverage slices, concatenated in order
 *     (frag[n_active], nbins[n_active], cov[active_bins]).
 *   hh_correct_set_layout: the corrected contigs, decided on the host (final_break_pos_dict / final_break_frag_dict,
 *     1116-1170, and the re-ordered fa_dict): source contig c owns the entries [src_base[c], src_base[c+1]) of
 *     piece_start (ascending, 0 first) / piece_id (id in the corrected fa_dict); an unbroken contig has one entry.
 *   hh_correct_remap: convert_ctg of the *_for_correction generators (1401-1536): an end on contig c goes to the piece
 *     with the largest start <= pos, at pos - start; ids outside [0, n_ctg) are kept.  rec_in / rec_out in `mem`. */
typedef struct hh_correct hh_correct;
typedef struct {
    int32_t n_examined;  /* fragments examined in this round                            */
    int32_t n_broken;    /* len(ctg_break_point_dict) (1214)                            */
    int32_t n_breaks;    /* breakpoints in all                                           */
    int32_t n_frag;      /* fragment ids before the round: the pieces' ids start here    */
    int64_t n_links;     /* same-contig records kept by the coverage pass                */
} hh_correct_round_info;
int hh_correct_create(hh_ctx* ctx, int32_t n_ctg, const int64_t* ctg_len, int64_t resolution, hh_correct** out);
int hh_correct_add(hh_correct* cr, const int32_t* rec, int64_t n_rec, int mem);
int hh_correct_round(hh_correct* cr, double median_cov_ratio, double region_len_ratio, int64_t min_region_cutoff,
                     int last_round, hh_correct_round_info* info);
int hh_correct_fetch_breaks(hh_correct* cr, int32_t* frag, int32_t* bin, int32_t* cov);
int hh_correct_info(hh_correct* cr, int32_t* n_active, int64_t* active_bins, int64_t* n_links);
int hh_correct_fetch_cov(hh_correct* cr, int32_t* frag, int32_t* nbins, int32_t* cov);
int hh_correct_set_layout(hh_correct* cr, const int32_t* src_base, const int64_t* piece_start, const int32_t* piece_id,
                          int32_t n_pieces);
int hh_correct_remap(hh_correct* cr, const int32_t* rec_in, int32_t* rec_out, int64_t n_rec, int mem);
int hh_correct_destroy(hh_correct* cr);

/* ---- contact maps (`haphic plot`, scripts/HapHiC_plot.py v1.0.7) ------------------------- *
 * The AGP layout is resolved on the host (parse_agp 41-103, generate_contact_matrix 106-150); the device gets, per contig
 * id, in_set (the contig is in ctg_set) and a dense run of (contig, aln bin) slots: slot_base[c] .. slot_base[c+1]-1 are
 * aln bins 0, 1, ... of contig c.  cand_off[slot] .. cand_off[slot+1]-1 are that slot's entries of ctg_aln_dict, in list
 * order: the closed raw range [cand_lo, cand_hi] and the total bin of its ctg_dict mapping (overwrites already resolved),
 * or -1 when that scaffold is not kept.  An empty slot is an aln bin the contig has no list for (the KeyError).
 *   hh_contact_create: the nb x nb count matrix (int32 while the records added cannot make a symmetrised entry reach 2^31,
 *     widened to int64 on the device by the add that would).
 *   hh_contact_load: a finished handle holding an nb x nb symmetrised int64 count matrix (a `contact_matrix.pkl`,
 *     load_pickle 266-288), for the KR / normalisation calls.
 *   hh_contact_add / hh_contact_add_async: parse_pairs / parse_bam with convert_group_bin_id (153-245) over records
 *     {id_a, pos_a, id_b, pos_b} (0-based positions, ids < 0 or >= n_ctg are not in ctg_set), in stream order across
 *     calls.  Host batches are staged through pinned double buffers; _async takes device records and returns at once.
 *   hh_contact_error: the first offending record in stream order (index -1: none), which end (0 / 1), its contig id and
 *     1-based position: the reference raises "Cannot find alignment position" for it.
 *   hh_contact_finish: contact_matrix + contact_matrix.T with the diagonal halved (854-856), in place.
 *   hh_contact_info / hh_contact_fetch: nb, bytes per stored count, records added; the symmetrised counts as int64.
 *   hh_contact_kr: bnewt (291-404) on n_prob diagonal blocks (off, n) of counts + 1e-5, all advanced together;
 *     x_out holds the problems' x one after the other, status 1 = "Unable to converge" (1000 outer / 10000 inner steps).
 *   hh_contact_normalize: normalize_matrix (407-504).  mode 0 = KR: x_whole[i] A_ij x_whole[j], replaced inside the blocks
 *     by x_blocks (indexed by bin), 0 where the count is 0; 1 = log10(count + 1); 2 = counts.  out (nb x nb fp64 host
 *     array, may be NULL) gets the matrix; the off-diagonal block entries (unmasked) are sorted on the device and their
 *     median's two middle values (equal for an odd count) returned with the count. */
typedef struct hh_contact hh_contact;
int hh_contact_create(hh_ctx* ctx, int32_t n_ctg, const uint8_t* in_set, const int64_t* slot_base, const int64_t* cand_off,
                      const int64_t* cand_lo, const int64_t* cand_hi, const int32_t* cand_bin, int32_t nb, int64_t bin_size,
                      hh_contact** out);
int hh_contact_load(hh_ctx* ctx, int32_t nb, const int64_t* counts, hh_contact** out);
int hh_contact_add(hh_contact* h, const int32_t* rec, int64_t n_rec, int mem);
int hh_contact_add_async(hh_contact* h, const int32_t* rec_dev, int64_t n_rec);
int hh_contact_error(hh_contact* h, int64_t* index, int32_t* end, int32_t* ctg, int64_t* pos);
int hh_contact_finish(hh_contact* h);
int hh_contact_info(hh_contact* h, int32_t* nb, int32_t* count_bytes, int64_t* n_records);
int hh_contact_fetch(hh_contact* h, int64_t* out);
int hh_contact_kr(hh_contact* h, int32_t n_prob, const int32_t* off, const int32_t* n, double tol, double delta, double Delta,
                  int32_t max_outer, int32_t max_inner, double* x_out, int32_t* n_outer, int64_t* n_inner, int32_t* status);
int hh_contact_normalize(hh_contact* h, int mode, int32_t n_blk, const int32_t* blk_off, const int32_t* blk_n,
                         const double* x_blocks, const double* x_whole, double* out, double* median_lo, double* median_hi,
                         int64_t* n_values);
int hh_contact_destroy(hh_contact* h);

/* ---- host-side I/O around the path (native, no CUDA) ------------------------------------------------
 * .pairs / .pairs.gz reader: pairs_generator / pairs_generator_inter_ctgs, HapHiC_cluster.py:1539-1583.  Skips blank
 * and '#' lines, takes `cols[1], int(cols[2])-1, cols[3], int(cols[4])-1`, writes the two BED lines per pair
 * to `bed_path` (may be NULL) and returns int32 records {id_a, pos_a, id_b, pos_b} (id -1 = name not in the table);
 * with inter_only pairs whose two names are equal are dropped (1582).  names_blob = n_names NUL-terminated names.
 * The text is cut at line boundaries and parsed on `threads` host threads (0 = all cores, at most 16); bgzipped
 * input is inflated block-parallel, other gzip streams by zlib. */
typedef struct hh_pairs_reader hh_pairs_reader;
int hh_pairs_open(const char* path, const char* names_blob, int32_t n_names, const char* bed_path, int inter_only,
                  int threads, hh_pairs_reader** out);
int hh_pairs_next(hh_pairs_reader* r, int32_t* rec, int64_t max_records, int64_t* n_out);   /* *n_out == 0: end of file */
int hh_pairs_close(hh_pairs_reader* r);
/* the inverse, for fixtures and benchmarks: n_rec records {id_a, pos_a, id_b, pos_b} (0-based positions) as 4DN .pairs text
 * `r{first_index + i}\tname_a\tpos_a+1\tname_b\tpos_b+1\t+\t-`; append != 0 continues an existing file without the header */
int hh_pairs_write(const char* path, const char* names_blob, int32_t n_names, const int32_t* rec, int64_t n_rec, int64_t first_index,
                   int append, int threads);
/* BAM input (bam_generator, HapHiC_cluster.py:1586-1593, with the htslib filters `flag.read1 [&& refid != mrefid]` of
 * 2855 / 2862): BGZF blocks are inflated on `threads` host threads; one record per read1 alignment,
 * (id(reference_name), reference_start, id(next_reference_name), next_reference_start), ids through the BAM header's
 * reference names (-1 = not in the FASTA / unmapped).  hh_bam_header_text gives the SAM header (sorting order check,
 * check_sorting_order 1347-1359); the pointer stays valid until hh_bam_close. */
typedef struct hh_bam_reader hh_bam_reader;
int hh_bam_open(const char* path, const char* names_blob, int32_t n_names, int inter_only, int threads, hh_bam_reader** out);
int hh_bam_header_text(hh_bam_reader* r, const char** text, int64_t* len);
int hh_bam_next(hh_bam_reader* r, int32_t* rec, int64_t max_records, int64_t* n_out);
int hh_bam_close(hh_bam_reader* r);
/* Ultra-long read alignments (`--ul`, parse_ul_alignments 1763-1869): hh_ul_open reads the whole BAM once (BGZF inflated
 * on `threads` threads) with the htslib filter !flag.unmap, drops alignments with MAPQ < min_mapq, reference length <
 * min_alignment_length or more than max_distance_to_end from both ends of the reference (lengths from the BAM header), and
 * runs the primary (flag 0 / 16) / supplementary (0x800, same read, other reference, query-interval overlap and gap tests)
 * state machine; each primary with accepted supplementaries yields one event from the one with the highest AS (first on a
 * tie).  hh_ul_info / hh_ul_fetch hand out the header's references (names NUL-separated, names_bytes in all, lengths) and
 * the events [n_events][4] in file order: left semi-contig, right semi-contig (2 * reference index + 0 for `_H`, 1 for
 * `_T`), primary reference, supplementary reference.  Any output pointer may be NULL. */
typedef struct hh_ul_reader hh_ul_reader;
int hh_ul_open(const char* path, int threads, int32_t min_mapq, int64_t min_alignment_length, int64_t max_distance_to_end,
               double max_overlap_ratio, int64_t max_gap_len, hh_ul_reader** out);
int hh_ul_info(hh_ul_reader* r, int32_t* n_ref, int64_t* names_bytes, int64_t* n_events, int64_t* n_records);
int hh_ul_fetch(hh_ul_reader* r, char* names, int64_t* ref_len, int32_t* events);
int hh_ul_close(hh_ul_reader* r);

/* paired_links.clm straight from the record stream (update_clm_dict 395-401 + output_clm 376-392): for every contig
 * pair with >= 2 links, in dict insertion order, four lines (orientations ++ +- -+ --)
 * `{ci}{s} {cj}{s}\t{2*links}\t{every ascending distance printed twice}`.  rec = n_rec int32 records
 * {id_a, pos_a, id_b, pos_b} in stream order (same-contig records and ids outside [0, n_names) are skipped),
 * ctg_len / name_rank per contig id.  Grouping, the per-pair sorts and the text formatting run on `threads` host
 * threads (0 = all cores, at most 16). */
int hh_clm_from_records(const char* path, const char* names_blob, int32_t n_names, const int32_t* rec, int64_t n_rec,
                        const int64_t* ctg_len, const int32_t* name_rank, int threads);
/* full_links.pkl / HT_links.pkl (output_pickle, 710-715) written from the fetched arrays, without materialising the
 * Python dicts: the file loads (pickle.load) as `defaultdict(int, {(name_i, name_j): value})` in entry order.
 * Give values_i64 or values_f64 for one entry per pair, or ht[n_entries][4] = {HH, HT, TH, TT} for HT_link_dict, whose
 * keys are (name_i + '_H'|'_T', name_j + '_H'|'_T') for the non-zero counters (update_HT_link_dict, 404-416). */
int hh_pickle_links(const char* path, const char* names_blob, int32_t n_names, const int32_t* key_i, const int32_t* key_j,
                    int64_t n_entries, const int64_t* values_i64, const double* values_f64, const uint32_t* ht);
/* full_links.pkl after a fractional phasing weight: reduced entries are Python floats, the others stay ints.  Entry e is
 * written as the float values[e] when is_float[e], else as the int (int64_t)values[e]. */
int hh_pickle_links_mixed(const char* path, const char* names_blob, int32_t n_names, const int32_t* key_i, const int32_t* key_j,
                          int64_t n_entries, const double* values, const uint8_t* is_float);

#ifdef __cplusplus
}
#endif
#endif /* HAPHIC_B200_H */
