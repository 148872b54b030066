// Internal (non-ABI) declarations shared between the translation units of libhaphic_b200.
#pragma once
#include "hh_common.cuh"

struct hh_matrix {
    hh_ctx* ctx;
    int32_t n;
    int64_t nnz;
    int64_t* d_colptr;   // [n+1]
    int32_t* d_row;      // [nnz]  rows are NOT sorted inside a column
    float* d_val;        // [nnz]
    int32_t* d_index;    // [n_index] contig id -> matrix index (-1 = absent); NULL for hh_matrix_from_csc
    int32_t n_index;
};

// The words of one entry of the compact link table (HH_E_WORDS x uint32).  The order is the hh_links_export /
// hh_links_adopt wire format.
enum { HH_E_I, HH_E_J, HH_E_FULL, HH_E_FLANK, HH_E_FIRST_FULL, HH_E_FIRST_FLANK, HH_E_HT, HH_E_TH, HH_E_TT, HH_E_WORDS };

// How the matrix sees one entry of the compact link table: the flank count, or
// links / (tot_i * tot_j) ** 0.5 in fp64 with normalize (normalize_by_nlinks, 718-724), then x 2 when ul_path != NULL and
// the two ends lie on two different contigs (ul_parent) of one ultra-long-read path (add_flank_and_full_links_based_on_ul,
// 1936-1985), then -- when hap != NULL and the two ends lie on different haplotypes -- x - x * w with two roundings
// (reduce_inter_hap_HiC_links, 695-707).  Returns false when the entry is not in the (reduced) flank_link_dict: no flank
// link, or reduced to exactly 0.  hh_k_touch and hh_k_mat_group both decide through this one function, so pattern,
// values and first-seen indices cannot disagree; doubling never makes a value 0, so the index pass may leave ul_path NULL.
__device__ __forceinline__ bool hh_flank_value(const uint32_t* __restrict__ p, const unsigned long long* __restrict__ ctg_tot,
                                               int normalize, const int32_t* __restrict__ hap, double w,
                                               const int32_t* __restrict__ ul_path, const int32_t* __restrict__ ul_parent,
                                               double* x_out) {
    if (p[HH_E_FLANK] == 0) return false;
    double x;
    if (normalize) {
        const unsigned long long prod = ctg_tot[p[HH_E_I]] * ctg_tot[p[HH_E_J]];
        x = (double)p[HH_E_FLANK] / pow((double)prod, 0.5);
    } else {
        x = (double)p[HH_E_FLANK];
    }
    if (ul_path != nullptr) {
        const int32_t pi = ul_path[p[HH_E_I]];
        if (pi >= 0 && pi == ul_path[p[HH_E_J]] && ul_parent[p[HH_E_I]] != ul_parent[p[HH_E_J]]) x *= 2.0;
    }
    if (hap != nullptr && hap[p[HH_E_I]] != hap[p[HH_E_J]]) x = __dsub_rn(x, __dmul_rn(x, w));
    if (x == 0.0) return false;
    *x_out = x;
    return true;
}

// hh_links accessors (hh_links.cu)
int32_t hh_links_n_ctg(hh_links* lk);
hh_ctx* hh_links_ctx(hh_links* lk);
const uint32_t* hh_links_compact(hh_links* lk, int64_t* nnz);
const unsigned long long* hh_links_ctg_totals(hh_links* lk);
const int32_t* hh_links_index_dev(hh_links* lk, int32_t* n_linked);   // the table's copy: hh_matrix_from_links never writes it
const int32_t* hh_links_degree_dev(hh_links* lk, int64_t* n_pass);   // per-fragment degree and passing entries of that index
uint8_t* hh_links_keep_dev(hh_links* lk);
bool hh_links_finished(hh_links* lk);
const int32_t* hh_links_hap_dev(hh_links* lk);   // haplotypes of the last phased hh_links_linked_index_phased; NULL = none
