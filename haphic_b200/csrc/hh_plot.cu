// `haphic plot` on the device (scripts/HapHiC_plot.py, v1.0.7): the genome-wide contact matrix binned from the record
// stream, its symmetrisation, Knight-Ruiz balancing of every scaffold block and of the whole matrix, the normalised
// matrix and the median that sets vmax.
//
//   parse_pairs / parse_bam, convert_group_bin_id (153-245)        hh_contact_add / hh_contact_add_async
//   contact_matrix + contact_matrix.T, diagonal / 2 (854-856)     hh_contact_finish
//   bnewt (291-404) on every block and on the whole matrix        hh_contact_kr
//   normalize_matrix (407-504): d @ A @ d, log10, vmax median     hh_contact_normalize
//
// Counting.  A CTA resolves a tile of 2048 records to bin-pair keys (bin_a * nb + bin_b), sorts the tile in shared memory
// (cub::BlockRadixSort over only the bits nb * nb needs) and issues one global atomicAdd per run of equal keys.  Hi-C pairs
// pile up on and next to the diagonal, so a per-record atomic would serialise on a few hundred entries; after the sort a
// diagonal-heavy tile issues a handful.
//
// Storage.  The counts are int32 while the records added so far cannot make any symmetrised entry (c_ij + c_ji <= records)
// reach 2^31; the add that would cross it first widens the matrix to int64 on the device.
//
// KR.  The outer Newton / inner CG control of bnewt runs here on the host, one state machine per problem (a scaffold block
// or the whole matrix).  Every round advances all problems that are still iterating by one matrix-vector product, with
// three launches for all of them: a vector kernel (one CTA per problem: the CG direction / x update), the product (a warp per
// four rows, reading the count matrix directly and adding 1e-5 in fp64), and a vector kernel that fuses p.w, the CG updates,
// the dot products and the min / max / gamma reductions.  One CTA per problem makes every reduction deterministic.
#include <cub/cub.cuh>
#include <math.h>
#include <algorithm>
#include <climits>
#include <vector>

#include "hh_common.cuh"

namespace {

constexpr int CNT_THREADS = 256;
constexpr int CNT_ITEMS = 8;
constexpr int CNT_TILE = CNT_THREADS * CNT_ITEMS;
constexpr int64_t ADD_CHUNK = (int64_t)1 << 22;      // records per staged host copy
constexpr int64_t FETCH_ROWS_BYTES = (int64_t)256 << 20;

struct Layout {
    const uint8_t* in_set;      // [n_ctg] contig has a W line in a kept scaffold (ctg_set)
    const int64_t* slot_base;   // [n_ctg + 1] first (contig, aln bin) slot of a contig; aln bins 0 .. count - 1
    const int64_t* cand_off;    // [n_slot + 1] candidate ranges of a slot, in ctg_aln_dict list order
    const int64_t* lo;          // [n_cand] closed raw range
    const int64_t* hi;
    const int32_t* bin;         // [n_cand] total bin, -1 = the range's scaffold is not kept, -2 = no such scaffold bin
    int32_t n_ctg;
    int64_t bin_size;
};

enum { RES_OK = 0, RES_SKIP = 1, RES_ERR = 2 };

// convert_group_bin_id (155-167) for a 1-based position
__device__ __forceinline__ int resolve_end(const Layout& L, int32_t c, int64_t p, int32_t* out) {
    const int64_t q = p - 1;
    const int64_t ab = q >= 0 ? q / L.bin_size : -((-q + L.bin_size - 1) / L.bin_size);
    const int64_t s0 = L.slot_base[c], s1 = L.slot_base[c + 1];
    if (ab < 0 || ab >= s1 - s0) return RES_ERR;
    const int64_t k0 = L.cand_off[s0 + ab], k1 = L.cand_off[s0 + ab + 1];
    if (k0 == k1) return RES_ERR;
    for (int64_t k = k0; k < k1; ++k) {
        if (L.lo[k] <= p && p <= L.hi[k]) {
            const int32_t b = L.bin[k];
            if (b < 0) return b == -1 ? RES_SKIP : RES_ERR;
            *out = b;
            return RES_OK;
        }
    }
    return RES_SKIP;
}

template <typename CountT>
__device__ __forceinline__ void count_add(CountT* p, int64_t v);
template <>
__device__ __forceinline__ void count_add<int32_t>(int32_t* p, int64_t v) { atomicAdd(p, (int)v); }
template <>
__device__ __forceinline__ void count_add<int64_t>(int64_t* p, int64_t v) {
    atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
}

// err[0] = min over offending records of (stream index << 1 | end), err[1] / err[2] = that end's contig / position
template <typename KeyT, typename CountT>
__global__ void __launch_bounds__(CNT_THREADS) k_contact_count(const int4* __restrict__ rec, int64_t n, int64_t stream_base,
                                                                Layout L, CountT* __restrict__ M, int32_t nb, int end_bit,
                                                                unsigned long long* __restrict__ err) {
    using Sort = cub::BlockRadixSort<KeyT, CNT_THREADS, CNT_ITEMS>;
    using Disc = cub::BlockDiscontinuity<KeyT, CNT_THREADS>;
    using Scan = cub::BlockScan<int, CNT_THREADS>;
    __shared__ union {
        typename Sort::TempStorage sort;
        typename Disc::TempStorage disc;
        typename Scan::TempStorage scan;
    } tmp;
    const KeyT NONE = ~(KeyT)0;
    const int64_t base = (int64_t)blockIdx.x * CNT_TILE;
    KeyT key[CNT_ITEMS];
#pragma unroll
    for (int it = 0; it < CNT_ITEMS; ++it) {
        const int64_t r = base + it * CNT_THREADS + threadIdx.x;
        key[it] = NONE;
        if (r >= n) continue;
        const int4 v = hh_ld_stream(rec + r);
        if (v.x < 0 || v.x >= L.n_ctg || v.z < 0 || v.z >= L.n_ctg || !L.in_set[v.x] || !L.in_set[v.z]) continue;
        int32_t ba = 0, bb = 0;
        int res = resolve_end(L, v.x, (int64_t)v.y + 1, &ba);
        int end = 0;
        if (res == RES_OK) {
            res = resolve_end(L, v.z, (int64_t)v.w + 1, &bb);
            end = 1;
        }
        if (res == RES_ERR) {
            atomicMin(err, (unsigned long long)(stream_base + r) << 1 | (unsigned long long)end);
            continue;
        }
        if (res == RES_OK) key[it] = (KeyT)ba * (KeyT)nb + (KeyT)bb;
    }
    Sort(tmp.sort).Sort(key, 0, end_bit + 1);      // bit end_bit sorts NONE (all ones) behind every key
    __syncthreads();
    bool head[CNT_ITEMS], tail[CNT_ITEMS];
    Disc(tmp.disc).FlagHeadsAndTails(head, tail, key, cub::Inequality());
    __syncthreads();
    int hpos[CNT_ITEMS];
#pragma unroll
    for (int it = 0; it < CNT_ITEMS; ++it) hpos[it] = head[it] ? (int)threadIdx.x * CNT_ITEMS + it : 0;
    Scan(tmp.scan).InclusiveScan(hpos, hpos, cub::Max());
#pragma unroll
    for (int it = 0; it < CNT_ITEMS; ++it) {
        if (!tail[it] || key[it] == NONE) continue;
        const int run = (int)threadIdx.x * CNT_ITEMS + it - hpos[it] + 1;
        count_add<CountT>(M + (int64_t)key[it], run);
    }
}

// the contig and 1-based position of the first offending end, recorded by the batch that holds it
__global__ void k_contact_err_info(const int4* __restrict__ rec, int64_t n, int64_t stream_base,
                                   unsigned long long* __restrict__ err) {
    const unsigned long long e = err[0];
    if (e == ~0ull) return;
    const int64_t idx = (int64_t)(e >> 1);
    if (idx < stream_base || idx >= stream_base + n) return;
    const int4 v = rec[idx - stream_base];
    err[1] = (unsigned long long)(int64_t)((e & 1) ? v.z : v.x);
    err[2] = (unsigned long long)((int64_t)((e & 1) ? v.w : v.y) + 1);
}

__global__ void k_widen(const int32_t* __restrict__ in, int64_t* __restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = in[i];
}

// M <- M + M^T with the diagonal kept, one 32 x 32 tile pair per CTA through shared memory
template <typename CountT>
__global__ void __launch_bounds__(256) k_symmetrise(CountT* __restrict__ M, int32_t nb) {
    const int I = blockIdx.y, J = blockIdx.x;
    if (I > J) return;
    __shared__ CountT a[32][33], b[32][33];
    const int tx = threadIdx.x, ty = threadIdx.y;
    for (int r = ty; r < 32; r += 8) {
        const int64_t ri = (int64_t)I * 32 + r, rj = (int64_t)J * 32 + r;
        const int64_t ci = (int64_t)I * 32 + tx, cj = (int64_t)J * 32 + tx;
        a[r][tx] = (ri < nb && cj < nb) ? M[ri * nb + cj] : 0;
        b[r][tx] = (rj < nb && ci < nb) ? M[rj * nb + ci] : 0;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int64_t ri = (int64_t)I * 32 + r, rj = (int64_t)J * 32 + r;
        const int64_t ci = (int64_t)I * 32 + tx, cj = (int64_t)J * 32 + tx;
        if (I == J) {
            if (ri < nb && ci < nb) M[ri * nb + ci] = (r == tx) ? a[r][r] : (CountT)(a[r][tx] + a[tx][r]);
        } else {
            if (ri < nb && cj < nb) M[ri * nb + cj] = a[r][tx] + b[tx][r];
            if (rj < nb && ci < nb) M[rj * nb + ci] = b[r][tx] + a[tx][r];
        }
    }
}

__global__ void k_narrow(const int64_t* __restrict__ in, int32_t* __restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = (int32_t)in[i];
}

template <typename CountT>
__global__ void k_rows_to_i64(const CountT* __restrict__ M, int64_t n, int64_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = (int64_t)M[i];
}

// ------------------------------------------------------------------------------------------------------------------------
// KR (bnewt)
// ------------------------------------------------------------------------------------------------------------------------
enum { PRE_INIT, PRE_XUPD, PRE_FIRST, PRE_NEXT };
enum { XU_KEEP, XU_STEP, XU_Y };
enum { MV_X, MV_XP };
enum { POST_OUTER, POST_CG };
enum { S_RHO, S_PW, S_ALPHA, S_MINY, S_MAXY, S_GLO, S_GHI, S_RHONEW, S_N };
enum { V_X, V_V, V_RK, V_Y, V_P, V_Z, V_W, V_U, V_N };

struct KrCmd {
    int32_t off, n;         // block of the count matrix: rows and columns off .. off + n - 1
    int64_t vbase;          // first element of the problem's vectors
    int64_t unit_base;      // first four-row unit of the problem in the product's grid
    int32_t pre, xu, mv, post;
    double c1, c2, c3;      // PRE_XUPD: gamma, alpha;  PRE_NEXT: beta, alpha, rho_km1
};

constexpr int KR_VEC_THREADS = 1024;
constexpr int KR_ROWS = 4;
constexpr int KR_MV_WARPS = 8;

__device__ __forceinline__ double block_sum(double v, double* sh) {
    v = hh_warp_sum(v);
    __syncthreads();
    if (hh_lane() == 0) sh[hh_warp()] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < 32) {
        t = threadIdx.x < blockDim.x / 32 ? sh[threadIdx.x] : 0.0;
        t = hh_warp_sum(t);
        if (threadIdx.x == 0) sh[32] = t;
    }
    __syncthreads();
    return sh[32];
}
__device__ __forceinline__ double block_min(double v, double* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(HH_FULL_MASK, v, o));
    __syncthreads();
    if (hh_lane() == 0) sh[hh_warp()] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        double t = threadIdx.x < blockDim.x / 32 ? sh[threadIdx.x] : INFINITY;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t = fmin(t, __shfl_xor_sync(HH_FULL_MASK, t, o));
        if (threadIdx.x == 0) sh[32] = t;
    }
    __syncthreads();
    return sh[32];
}

// phase 0: the command's pre op (before the product); phase 1: its post op.  One CTA per problem.
__global__ void __launch_bounds__(KR_VEC_THREADS) k_kr_vec(const KrCmd* __restrict__ cmds, double* __restrict__ V, int64_t L,
                                                           double* __restrict__ sc, int phase, double delta, double Delta) {
    __shared__ double sh[33];
    const KrCmd c = cmds[blockIdx.x];
    double* x = V + V_X * L + c.vbase;
    double* v = V + V_V * L + c.vbase;
    double* rk = V + V_RK * L + c.vbase;
    double* y = V + V_Y * L + c.vbase;
    double* p = V + V_P * L + c.vbase;
    double* Z = V + V_Z * L + c.vbase;
    double* w = V + V_W * L + c.vbase;
    double* u = V + V_U * L + c.vbase;
    double* s = sc + (int64_t)blockIdx.x * S_N;
    const int n = c.n;
    if (phase == 0) {
        if (c.pre == PRE_INIT) {
            for (int i = threadIdx.x; i < n; i += blockDim.x) x[i] = u[i] = 1.0;
        } else if (c.pre == PRE_XUPD) {
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                double xi = x[i];
                if (c.xu == XU_STEP) xi = __dmul_rn(xi, __dadd_rn(y[i], __dmul_rn(c.c1, __dmul_rn(c.c2, p[i]))));
                else if (c.xu == XU_Y) xi = __dmul_rn(xi, y[i]);
                x[i] = u[i] = xi;
            }
        } else if (c.pre == PRE_FIRST) {
            double acc = 0.0;
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const double z = __ddiv_rn(rk[i], v[i]);
                y[i] = 1.0;
                Z[i] = p[i] = z;
                u[i] = __dmul_rn(x[i], z);
                acc = __fma_rn(rk[i], z, acc);
            }
            acc = block_sum(acc, sh);
            if (threadIdx.x == 0) s[S_RHO] = acc;
        } else {   // PRE_NEXT
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const double po = p[i];
                y[i] = __dadd_rn(y[i], __dmul_rn(c.c2, po));
                const double pn = __dadd_rn(Z[i], __dmul_rn(c.c1, po));
                p[i] = pn;
                u[i] = __dmul_rn(x[i], pn);
            }
            if (threadIdx.x == 0) s[S_RHO] = c.c3;
        }
        return;
    }
    if (c.post == POST_OUTER) {
        double acc = 0.0;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const double r = __dsub_rn(1.0, v[i]);
            rk[i] = r;
            acc = __fma_rn(r, r, acc);
        }
        acc = block_sum(acc, sh);
        if (threadIdx.x == 0) s[S_RHO] = acc;
        return;
    }
    // POST_CG
    double pw = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) pw = __fma_rn(p[i], w[i], pw);
    pw = block_sum(pw, sh);
    const double alpha = __ddiv_rn(s[S_RHO], pw);
    double mn = INFINITY, mx = -INFINITY, glo = INFINITY, ghi = INFINITY, rho = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double ap = __dmul_rn(alpha, p[i]);
        const double yi = y[i];
        const double yn = __dadd_rn(yi, ap);
        mn = fmin(mn, yn);
        mx = fmax(mx, yn);
        if (ap < 0.0) glo = fmin(glo, __ddiv_rn(__dsub_rn(delta, yi), ap));
        if (yn > Delta) ghi = fmin(ghi, __ddiv_rn(__dsub_rn(Delta, yi), ap));
        const double r = __dsub_rn(rk[i], __dmul_rn(alpha, w[i]));
        rk[i] = r;
        const double z = __ddiv_rn(r, v[i]);
        Z[i] = z;
        rho = __fma_rn(r, z, rho);
    }
    mn = block_min(mn, sh);
    mx = -block_min(-mx, sh);
    glo = block_min(glo, sh);
    ghi = block_min(ghi, sh);
    rho = block_sum(rho, sh);
    if (threadIdx.x == 0) {
        s[S_PW] = pw;
        s[S_ALPHA] = alpha;
        s[S_MINY] = mn;
        s[S_MAXY] = mx;
        s[S_GLO] = glo;
        s[S_GHI] = ghi;
        s[S_RHONEW] = rho;
    }
}

// t = A u over each command's block (A = counts + 1e-5 in fp64), then v = x * t (MV_X) or w = x * t + v * p (MV_XP).  A
// warp takes four consecutive rows so that each u[j] it loads serves four matrix entries.
template <typename CountT>
__global__ void __launch_bounds__(KR_MV_WARPS * 32) k_kr_mv(const CountT* __restrict__ M, int32_t ld, const KrCmd* __restrict__ cmds,
                                                              int n_cmd, int64_t n_units, double* __restrict__ V, int64_t L) {
    const int64_t unit = (int64_t)blockIdx.x * KR_MV_WARPS + hh_warp();
    if (unit >= n_units) return;
    int lo = 0, hi = n_cmd - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (cmds[mid].unit_base <= unit) lo = mid;
        else hi = mid - 1;
    }
    const KrCmd c = cmds[lo];
    const int i0 = (int)(unit - c.unit_base) * KR_ROWS;
    const int n = c.n;
    const double* u = V + V_U * L + c.vbase;
    const CountT* row[KR_ROWS];
    bool live[KR_ROWS];
#pragma unroll
    for (int r = 0; r < KR_ROWS; ++r) {
        live[r] = i0 + r < n;
        row[r] = M + (int64_t)(c.off + (live[r] ? i0 + r : i0)) * ld + c.off;
    }
    double acc[KR_ROWS] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 4
    for (int j = hh_lane(); j < n; j += 32) {
        const double uj = u[j];
#pragma unroll
        for (int r = 0; r < KR_ROWS; ++r)
            if (live[r]) acc[r] = __fma_rn(__dadd_rn((double)__ldg(row[r] + j), 1e-5), uj, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < KR_ROWS; ++r) acc[r] = hh_warp_sum(acc[r]);
    if (hh_lane() < KR_ROWS && live[hh_lane()]) {
        const int rr = hh_lane();
        double t = acc[0];
#pragma unroll
        for (int r = 1; r < KR_ROWS; ++r)
            if (rr == r) t = acc[r];
        const int64_t gi = c.vbase + i0 + rr;
        const double xt = __dmul_rn(V[V_X * L + gi], t);
        if (c.mv == MV_X) V[V_V * L + gi] = xt;
        else V[V_W * L + gi] = __dadd_rn(xt, __dmul_rn(V[V_V * L + gi], V[V_P * L + gi]));
    }
}

// ------------------------------------------------------------------------------------------------------------------------
// normalised output and the vmax median
// ------------------------------------------------------------------------------------------------------------------------
enum { NORM_KR = 0, NORM_LOG10 = 1, NORM_NONE = 2 };

template <typename CountT>
__device__ __forceinline__ double norm_value(CountT raw, int mode, bool intra, int64_t i, int64_t j, const double* xb,
                                             const double* xw) {
    if (mode == NORM_LOG10) return log10((double)((int64_t)raw + 1));
    if (mode == NORM_NONE) return (double)raw;
    const double a = __dadd_rn((double)raw, 1e-5);
    const double* x = intra ? xb : xw;
    return __dmul_rn(__dmul_rn(x[i], a), x[j]);
}

// rows row0 .. row0 + rows - 1 of the normalised matrix; KR entries whose count is 0 are 0
template <typename CountT>
__global__ void k_norm_rows(const CountT* __restrict__ M, int32_t nb, int64_t row0, int mode, const int32_t* __restrict__ blk,
                            const double* __restrict__ xb, const double* __restrict__ xw, double* __restrict__ out) {
    const int64_t i = row0 + blockIdx.y;
    const int32_t bi = blk[i];
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nb; j += (int64_t)gridDim.x * blockDim.x) {
        const CountT raw = M[i * nb + j];
        double val = 0.0;
        if (mode != NORM_KR || raw != 0) val = norm_value<CountT>(raw, mode, bi >= 0 && blk[j] == bi, i, j, xb, xw);
        out[(int64_t)blockIdx.y * nb + j] = val;
    }
}

// the off-diagonal entries of every scaffold block, unmasked (the values normalize_matrix collects into non_diagonal_list)
template <typename CountT>
__global__ void k_gather_intra(const CountT* __restrict__ M, int32_t nb, int n_blk, const int32_t* __restrict__ boff,
                               const int32_t* __restrict__ bn, const int64_t* __restrict__ row_base,
                               const int64_t* __restrict__ val_base, int mode, const double* __restrict__ xb,
                               double* __restrict__ out) {
    const int64_t gr = blockIdx.x;
    int lo = 0, hi = n_blk - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (row_base[mid] <= gr) lo = mid;
        else hi = mid - 1;
    }
    const int n = bn[lo];
    const int64_t r = gr - row_base[lo];
    const int64_t i = boff[lo] + r;
    double* o = out + val_base[lo] + r * (n - 1);
    for (int64_t q = threadIdx.x; q < n; q += blockDim.x) {
        if (q == r) continue;
        const int64_t j = boff[lo] + q;
        o[q < r ? q : q - 1] = norm_value<CountT>(M[i * nb + j], mode, true, i, j, xb, xb);
    }
}

}  // namespace

struct hh_contact {
    hh_ctx* ctx;
    int32_t n_ctg, nb;
    int64_t n_slot, n_cand, bin_size;
    uint8_t* d_in_set;
    int64_t *d_slot_base, *d_cand_off, *d_lo, *d_hi;
    int32_t* d_bin;
    int32_t* d_m32;
    int64_t* d_m64;
    int64_t n_records;
    bool finished;
    unsigned long long* d_err;     // [3]
    int4* d_stage[2];
    cudaStream_t copy_stream;
    cudaEvent_t ev_copied[2], ev_consumed[2];
};

static Layout contact_layout(const hh_contact* h) {
    Layout L;
    L.in_set = h->d_in_set;
    L.slot_base = h->d_slot_base;
    L.cand_off = h->d_cand_off;
    L.lo = h->d_lo;
    L.hi = h->d_hi;
    L.bin = h->d_bin;
    L.n_ctg = h->n_ctg;
    L.bin_size = h->bin_size;
    return L;
}

static int contact_free(hh_contact* h) {
    hh_dfree(h->d_in_set);
    hh_dfree(h->d_slot_base);
    hh_dfree(h->d_cand_off);
    hh_dfree(h->d_lo);
    hh_dfree(h->d_hi);
    hh_dfree(h->d_bin);
    hh_dfree(h->d_m32);
    hh_dfree(h->d_m64);
    hh_dfree(h->d_err);
    for (int b = 0; b < 2; ++b) {
        if (h->d_stage[b]) cudaFree(h->d_stage[b]);
        h->d_stage[b] = nullptr;
        if (h->ev_copied[b]) cudaEventDestroy(h->ev_copied[b]);
        if (h->ev_consumed[b]) cudaEventDestroy(h->ev_consumed[b]);
        h->ev_copied[b] = h->ev_consumed[b] = nullptr;
    }
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    h->copy_stream = nullptr;
    return HH_OK;
}

template <typename T>
static int upload(hh_ctx* ctx, T** d, const T* h, int64_t n) {
    HH_CHECK(hh_dmalloc(d, (size_t)n));
    if (n > 0) HH_CUDA(cudaMemcpyAsync(*d, h, (size_t)n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return HH_OK;
}

static int contact_widen(hh_contact* h) {
    const int64_t nn = (int64_t)h->nb * h->nb;
    HH_CHECK(hh_dmalloc(&h->d_m64, (size_t)nn));
    HH_LAUNCH(h->ctx, k_widen, h->ctx->sm_count * 8, 256, 0, h->d_m32, h->d_m64, nn);
    hh_dfree(h->d_m32);
    return HH_OK;
}

static int contact_launch(hh_contact* h, const int4* d_rec, int64_t n) {
    hh_ctx* ctx = h->ctx;
    if (!h->d_m64 && h->n_records + n > INT_MAX) HH_CHECK(contact_widen(h));
    const uint64_t nn = (uint64_t)h->nb * (uint64_t)h->nb;
    int end_bit = 1;
    while (end_bit < 64 && (nn - 1) >> end_bit) ++end_bit;     // bits of the largest key
    const int64_t grid = (n + CNT_TILE - 1) / CNT_TILE;
    const Layout L = contact_layout(h);
    const bool k32 = nn <= 0xFFFFFFFFull;
    if (k32 && !h->d_m64)
        HH_LAUNCH(ctx, (k_contact_count<uint32_t, int32_t>), grid, CNT_THREADS, 0, d_rec, n, h->n_records, L, h->d_m32, h->nb, end_bit, h->d_err);
    else if (k32)
        HH_LAUNCH(ctx, (k_contact_count<uint32_t, int64_t>), grid, CNT_THREADS, 0, d_rec, n, h->n_records, L, h->d_m64, h->nb, end_bit, h->d_err);
    else if (!h->d_m64)
        HH_LAUNCH(ctx, (k_contact_count<uint64_t, int32_t>), grid, CNT_THREADS, 0, d_rec, n, h->n_records, L, h->d_m32, h->nb, end_bit, h->d_err);
    else
        HH_LAUNCH(ctx, (k_contact_count<uint64_t, int64_t>), grid, CNT_THREADS, 0, d_rec, n, h->n_records, L, h->d_m64, h->nb, end_bit, h->d_err);
    HH_LAUNCH(ctx, k_contact_err_info, 1, 1, 0, d_rec, n, h->n_records, h->d_err);
    h->n_records += n;
    return HH_OK;
}

extern "C" {

int hh_contact_create(hh_ctx* ctx, int32_t n_ctg, const uint8_t* in_set, const int64_t* slot_base, const int64_t* cand_off,
                      const int64_t* cand_lo, const int64_t* cand_hi, const int32_t* cand_bin, int32_t nb, int64_t bin_size,
                      hh_contact** out) {
    HH_REQUIRE(ctx && out && in_set && slot_base && cand_off && n_ctg > 0 && nb > 0 && bin_size > 0, HH_ERR_ARG,
               "hh_contact_create: bad arguments");
    *out = nullptr;
    hh_scope _scope(ctx);
    const int64_t n_slot = slot_base[n_ctg];
    HH_REQUIRE(n_slot >= 0 && cand_off[0] == 0, HH_ERR_ARG, "hh_contact_create: bad slot table");
    const int64_t n_cand = cand_off[n_slot];
    HH_REQUIRE(n_cand == 0 || (cand_lo && cand_hi && cand_bin), HH_ERR_ARG, "hh_contact_create: NULL candidate arrays");
    for (int64_t k = 0; k < n_cand; ++k)
        HH_REQUIRE(cand_bin[k] >= -2 && cand_bin[k] < nb, HH_ERR_ARG, "hh_contact_create: bin %d out of [-2, %d)", cand_bin[k], nb);
    hh_contact* h = new (std::nothrow) hh_contact();
    HH_REQUIRE(h, HH_ERR_NOMEM, "hh_contact_create: out of host memory");
    h->ctx = ctx;
    h->n_ctg = n_ctg;
    h->nb = nb;
    h->n_slot = n_slot;
    h->n_cand = n_cand;
    h->bin_size = bin_size;
    int rc = HH_OK;
    do {
        if ((rc = upload(ctx, &h->d_in_set, in_set, n_ctg)) != HH_OK) break;
        if ((rc = upload(ctx, &h->d_slot_base, slot_base, (int64_t)n_ctg + 1)) != HH_OK) break;
        if ((rc = upload(ctx, &h->d_cand_off, cand_off, n_slot + 1)) != HH_OK) break;
        if ((rc = upload(ctx, &h->d_lo, cand_lo, n_cand)) != HH_OK) break;
        if ((rc = upload(ctx, &h->d_hi, cand_hi, n_cand)) != HH_OK) break;
        if ((rc = upload(ctx, &h->d_bin, cand_bin, n_cand)) != HH_OK) break;
        if ((rc = hh_dmalloc(&h->d_m32, (size_t)nb * (size_t)nb)) != HH_OK) break;
        if ((rc = hh_dmalloc(&h->d_err, 3)) != HH_OK) break;
        cudaError_t e = cudaMemsetAsync(h->d_m32, 0, (size_t)nb * (size_t)nb * sizeof(int32_t), ctx->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(h->d_err, 0xFF, 3 * sizeof(unsigned long long), ctx->stream);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking);
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) {
            e = cudaEventCreateWithFlags(&h->ev_copied[b], cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_consumed[b], cudaEventDisableTiming);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) {
            hh_set_error("hh_contact_create: %s", cudaGetErrorString(e));
            rc = HH_ERR_CUDA;
        }
    } while (0);
    if (rc != HH_OK) {
        contact_free(h);
        delete h;
        return rc;
    }
    *out = h;
    return HH_OK;
}

int hh_contact_load(hh_ctx* ctx, int32_t nb, const int64_t* counts, hh_contact** out) {
    HH_REQUIRE(ctx && counts && out && nb > 0, HH_ERR_ARG, "hh_contact_load: bad arguments");
    *out = nullptr;
    hh_scope _scope(ctx);
    const int64_t nn = (int64_t)nb * nb;
    int64_t mx = 0;
    for (int64_t i = 0; i < nn; ++i) {
        HH_REQUIRE(counts[i] >= 0, HH_ERR_ARG, "hh_contact_load: negative count at %lld", (long long)i);
        mx = std::max(mx, counts[i]);
    }
    hh_contact* h = new (std::nothrow) hh_contact();
    HH_REQUIRE(h, HH_ERR_NOMEM, "hh_contact_load: out of host memory");
    h->ctx = ctx;
    h->nb = nb;
    h->finished = true;
    int rc = HH_OK;
    int64_t* stage = nullptr;
    if (mx > INT_MAX) {
        rc = hh_dmalloc(&h->d_m64, (size_t)nn);
        if (rc == HH_OK && cudaMemcpyAsync(h->d_m64, counts, (size_t)nn * 8, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) {
            hh_set_error("hh_contact_load: upload failed");
            rc = HH_ERR_CUDA;
        }
    } else {
        // counts that fit int32 are narrowed on the device in row chunks: the products then read 4 bytes per entry
        const int64_t rows = std::max<int64_t>(1, std::min<int64_t>(nb, FETCH_ROWS_BYTES / ((int64_t)nb * 8)));
        rc = hh_dmalloc(&h->d_m32, (size_t)nn);
        if (rc == HH_OK) rc = hh_dmalloc(&stage, (size_t)(rows * nb));
        for (int64_t r0 = 0; r0 < nb && rc == HH_OK; r0 += rows) {
            const int64_t m = std::min<int64_t>(rows, nb - r0) * nb;
            cudaError_t e = cudaMemcpyAsync(stage, counts + r0 * nb, (size_t)m * 8, cudaMemcpyHostToDevice, ctx->stream);
            if (e == cudaSuccess) {
                k_narrow<<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(stage, h->d_m32 + r0 * nb, m);
                ctx->launches++;
                e = cudaGetLastError();
            }
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
            if (e != cudaSuccess) {
                hh_set_error("hh_contact_load: %s", cudaGetErrorString(e));
                rc = HH_ERR_CUDA;
            }
        }
    }
    if (rc == HH_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) {
        hh_set_error("hh_contact_load: upload failed");
        rc = HH_ERR_CUDA;
    }
    hh_dfree(stage);
    if (rc != HH_OK) {
        contact_free(h);
        delete h;
        return rc;
    }
    *out = h;
    return HH_OK;
}

int hh_contact_add(hh_contact* h, const int32_t* rec, int64_t n_rec, int mem) {
    HH_REQUIRE(h && (rec || n_rec == 0) && n_rec >= 0, HH_ERR_ARG, "hh_contact_add: bad arguments");
    HH_REQUIRE(mem == HH_MEM_HOST || mem == HH_MEM_DEVICE, HH_ERR_ARG, "hh_contact_add: bad mem flag %d", mem);
    hh_scope _scope(h->ctx);
    HH_REQUIRE(!h->finished, HH_ERR_STATE, "hh_contact_add: the matrix is already finished");
    if (n_rec == 0) return HH_OK;
    hh_ctx* ctx = h->ctx;
    if (mem == HH_MEM_DEVICE) {
        HH_REQUIRE(((uintptr_t)rec & 15) == 0, HH_ERR_ARG, "hh_contact_add: records must be 16-byte aligned");
        HH_CHECK(contact_launch(h, reinterpret_cast<const int4*>(rec), n_rec));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        return HH_OK;
    }
    if (!h->d_stage[0]) {
        HH_CUDA(cudaMalloc((void**)&h->d_stage[0], (size_t)ADD_CHUNK * sizeof(int4)));
        HH_CUDA(cudaMalloc((void**)&h->d_stage[1], (size_t)ADD_CHUNK * sizeof(int4)));
    }
    int buf = 0;
    for (int64_t off = 0; off < n_rec; off += ADD_CHUNK, buf ^= 1) {
        const int64_t m = std::min(ADD_CHUNK, n_rec - off);
        // the copy engine may not overwrite a staging buffer the count kernel still reads
        HH_CUDA(cudaStreamWaitEvent(h->copy_stream, h->ev_consumed[buf], 0));
        HH_CUDA(cudaMemcpyAsync(h->d_stage[buf], rec + off * 4, (size_t)m * 16, cudaMemcpyHostToDevice, h->copy_stream));
        HH_CUDA(cudaEventRecord(h->ev_copied[buf], h->copy_stream));
        HH_CUDA(cudaStreamWaitEvent(ctx->stream, h->ev_copied[buf], 0));
        HH_CHECK(contact_launch(h, h->d_stage[buf], m));
        HH_CUDA(cudaEventRecord(h->ev_consumed[buf], ctx->stream));
    }
    HH_CUDA(cudaStreamSynchronize(ctx->stream));      // the caller may reuse `rec` on return
    return HH_OK;
}

int hh_contact_add_async(hh_contact* h, const int32_t* rec_dev, int64_t n_rec) {
    HH_REQUIRE(h && (rec_dev || n_rec == 0) && n_rec >= 0, HH_ERR_ARG, "hh_contact_add_async: bad arguments");
    hh_scope _scope(h->ctx);
    HH_REQUIRE(!h->finished, HH_ERR_STATE, "hh_contact_add_async: the matrix is already finished");
    HH_REQUIRE(((uintptr_t)rec_dev & 15) == 0, HH_ERR_ARG, "hh_contact_add_async: records must be 16-byte aligned");
    if (n_rec == 0) return HH_OK;
    return contact_launch(h, reinterpret_cast<const int4*>(rec_dev), n_rec);
}

int hh_contact_error(hh_contact* h, int64_t* index, int32_t* end, int32_t* ctg, int64_t* pos) {
    HH_REQUIRE(h && index && end && ctg && pos, HH_ERR_ARG, "hh_contact_error: NULL argument");
    hh_scope _scope(h->ctx);
    unsigned long long e[3];
    HH_CUDA(cudaMemcpyAsync(e, h->d_err, sizeof(e), cudaMemcpyDeviceToHost, h->ctx->stream));
    HH_CUDA(cudaStreamSynchronize(h->ctx->stream));
    *index = e[0] == ~0ull ? -1 : (int64_t)(e[0] >> 1);
    *end = e[0] == ~0ull ? -1 : (int32_t)(e[0] & 1);
    *ctg = (int32_t)(int64_t)e[1];
    *pos = (int64_t)e[2];
    return HH_OK;
}

int hh_contact_finish(hh_contact* h) {
    HH_REQUIRE(h, HH_ERR_ARG, "hh_contact_finish: NULL handle");
    hh_scope _scope(h->ctx);
    HH_REQUIRE(!h->finished, HH_ERR_STATE, "hh_contact_finish: called twice");
    const int T = (h->nb + 31) / 32;
    const dim3 grid(T, T), block(32, 8);
    if (h->d_m64) HH_LAUNCH(h->ctx, k_symmetrise<int64_t>, grid, block, 0, h->d_m64, h->nb);
    else HH_LAUNCH(h->ctx, k_symmetrise<int32_t>, grid, block, 0, h->d_m32, h->nb);
    HH_CUDA(cudaStreamSynchronize(h->ctx->stream));
    h->finished = true;
    return HH_OK;
}

int hh_contact_info(hh_contact* h, int32_t* nb, int32_t* count_bytes, int64_t* n_records) {
    HH_REQUIRE(h, HH_ERR_ARG, "hh_contact_info: NULL handle");
    if (nb) *nb = h->nb;
    if (count_bytes) *count_bytes = h->d_m64 ? 8 : 4;
    if (n_records) *n_records = h->n_records;
    return HH_OK;
}

int hh_contact_fetch(hh_contact* h, int64_t* out) {
    HH_REQUIRE(h && out, HH_ERR_ARG, "hh_contact_fetch: NULL argument");
    hh_scope _scope(h->ctx);
    HH_REQUIRE(h->finished, HH_ERR_STATE, "hh_contact_fetch: hh_contact_finish first");
    hh_ctx* ctx = h->ctx;
    const int64_t nb = h->nb, nn = nb * nb;
    if (h->d_m64) {
        HH_CUDA(cudaMemcpyAsync(out, h->d_m64, (size_t)nn * 8, cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        return HH_OK;
    }
    // int32 counts are widened on the device in row chunks, each chunk copied straight into the caller's int64 array
    const int64_t rows = std::max<int64_t>(1, std::min<int64_t>(nb, FETCH_ROWS_BYTES / (nb * 8)));
    int64_t* stage = nullptr;
    HH_CHECK(hh_dmalloc(&stage, (size_t)(rows * nb)));
    int rc = HH_OK;
    for (int64_t r0 = 0; r0 < nb && rc == HH_OK; r0 += rows) {
        const int64_t m = std::min(rows, nb - r0) * nb;
        k_rows_to_i64<int32_t><<<ctx->sm_count * 4, 256, 0, ctx->stream>>>(h->d_m32 + r0 * nb, m, stage);
        ctx->launches++;
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(out + r0 * nb, stage, (size_t)m * 8, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) {
            hh_set_error("hh_contact_fetch: %s", cudaGetErrorString(e));
            rc = HH_ERR_CUDA;
        }
    }
    hh_dfree(stage);
    return rc;
}

int hh_contact_kr(hh_contact* h, int32_t n_prob, const int32_t* off, const int32_t* n, double tol, double delta, double Delta,
                  int32_t max_outer, int32_t max_inner, double* x_out, int32_t* n_outer, int64_t* n_inner, int32_t* status) {
    HH_REQUIRE(h && n_prob > 0 && off && n && x_out && n_outer && n_inner && status, HH_ERR_ARG, "hh_contact_kr: bad arguments");
    hh_scope _scope(h->ctx);
    HH_REQUIRE(h->finished, HH_ERR_STATE, "hh_contact_kr: hh_contact_finish first");
    hh_ctx* ctx = h->ctx;
    struct Prob {
        int32_t off, n;
        int64_t vbase;
        KrCmd next;
        double rho_km1, rho_km2, rout, rold, eta, innertol;
        int32_t nn, mm, k, i;
        int64_t inner;
        bool first, active;
    };
    std::vector<Prob> P((size_t)n_prob);
    int64_t L = 0;
    for (int q = 0; q < n_prob; ++q) {
        HH_REQUIRE(n[q] > 0 && off[q] >= 0 && (int64_t)off[q] + n[q] <= h->nb, HH_ERR_ARG,
                   "hh_contact_kr: block %d (%d + %d) outside the %d-bin matrix", q, off[q], n[q], h->nb);
        Prob& p = P[(size_t)q];
        memset(&p, 0, sizeof(p));
        p.off = off[q];
        p.n = n[q];
        p.vbase = L;
        p.first = p.active = true;
        p.eta = 0.1;
        p.next.pre = PRE_INIT;
        p.next.mv = MV_X;
        p.next.post = POST_OUTER;
        L += n[q];
        status[q] = 0;
    }
    const double g = 0.9, etamax = 0.1, stop_tol = tol * 0.5, rt = tol * tol;
    double* V = nullptr;
    KrCmd* d_cmd = nullptr;
    double* d_sc = nullptr;
    HH_CHECK(hh_dmalloc(&V, (size_t)(V_N * L)));
    int rc = HH_OK;
    KrCmd* h_cmd = nullptr;
    double* h_sc = nullptr;
    std::vector<int> act;
    auto fail = [&](const char* what, cudaError_t e) {
        hh_set_error("hh_contact_kr: %s: %s", what, cudaGetErrorString(e));
        rc = HH_ERR_CUDA;
    };
    cudaError_t e = cudaMallocHost((void**)&h_cmd, sizeof(KrCmd) * (size_t)n_prob);
    if (e == cudaSuccess) e = cudaMallocHost((void**)&h_sc, sizeof(double) * S_N * (size_t)n_prob);
    if (e != cudaSuccess) fail("pinned buffers", e);
    if (rc == HH_OK) rc = hh_dmalloc(&d_cmd, (size_t)n_prob);
    if (rc == HH_OK) rc = hh_dmalloc(&d_sc, (size_t)(S_N * n_prob));
    bool stop = false;
    while (rc == HH_OK && !stop) {
        act.clear();
        int64_t units = 0;
        for (int q = 0; q < n_prob; ++q) {
            Prob& p = P[(size_t)q];
            if (!p.active) continue;
            KrCmd c = p.next;
            c.off = p.off;
            c.n = p.n;
            c.vbase = p.vbase;
            c.unit_base = units;
            units += (p.n + KR_ROWS - 1) / KR_ROWS;
            h_cmd[act.size()] = c;
            act.push_back(q);
        }
        if (act.empty()) break;
        const int na = (int)act.size();
        e = cudaMemcpyAsync(d_cmd, h_cmd, sizeof(KrCmd) * (size_t)na, cudaMemcpyHostToDevice, ctx->stream);
        if (e != cudaSuccess) { fail("command upload", e); break; }
        k_kr_vec<<<na, KR_VEC_THREADS, 0, ctx->stream>>>(d_cmd, V, L, d_sc, 0, delta, Delta);
        const int64_t mv_grid = (units + KR_MV_WARPS - 1) / KR_MV_WARPS;
        if (h->d_m64) k_kr_mv<int64_t><<<(unsigned)mv_grid, KR_MV_WARPS * 32, 0, ctx->stream>>>(h->d_m64, h->nb, d_cmd, na, units, V, L);
        else k_kr_mv<int32_t><<<(unsigned)mv_grid, KR_MV_WARPS * 32, 0, ctx->stream>>>(h->d_m32, h->nb, d_cmd, na, units, V, L);
        k_kr_vec<<<na, KR_VEC_THREADS, 0, ctx->stream>>>(d_cmd, V, L, d_sc, 1, delta, Delta);
        ctx->launches += 3;
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpyAsync(h_sc, d_sc, sizeof(double) * S_N * (size_t)na, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { fail("round", e); break; }
        for (int a = 0; a < na; ++a) {
            Prob& p = P[(size_t)act[(size_t)a]];
            const double* s = h_sc + (size_t)a * S_N;
            KrCmd& nx = p.next;
            bool outer_next = false;
            if (p.next.post == POST_OUTER) {
                // end of an outer step: rk = 1 - v and rho = rk . rk are fresh
                const double r = s[S_RHO];
                if (p.first) {
                    p.rho_km1 = p.rout = p.rold = r;
                    p.first = false;
                } else {
                    p.rho_km1 = p.rout = r;
                    p.inner += p.k;
                    const double rat = p.rout / p.rold;
                    p.rold = p.rout;
                    const double res_norm = sqrt(p.rout);
                    const double eta_o = p.eta;
                    p.eta = g * rat;
                    if (g * (eta_o * eta_o) > 0.1) p.eta = std::max(p.eta, g * (eta_o * eta_o));
                    p.eta = std::max(std::min(p.eta, etamax), stop_tol / res_norm);
                }
                if (!(p.rout > rt)) {
                    p.active = false;
                    continue;
                }
                if (++p.nn > max_outer) {
                    status[act[(size_t)a]] = 1;
                    stop = true;
                    continue;
                }
                p.mm = 0;
                p.i++;
                p.k = 0;
                p.innertol = std::max((p.eta * p.eta) * p.rout, rt);
                if (p.rho_km1 > p.innertol) {
                    if (++p.mm > max_inner) {
                        status[act[(size_t)a]] = 1;
                        stop = true;
                        continue;
                    }
                    p.k = 1;
                    nx.pre = PRE_FIRST;
                    nx.mv = MV_XP;
                    nx.post = POST_CG;
                } else {
                    nx.pre = PRE_XUPD;
                    nx.xu = XU_KEEP;
                    outer_next = true;
                }
            } else {
                // end of an inner CG step
                p.rho_km1 = s[S_RHO];
                const double alpha = s[S_ALPHA];
                nx.pre = PRE_XUPD;
                nx.c2 = alpha;
                if (s[S_MINY] <= delta) {
                    if (delta == 0) nx.xu = XU_Y;
                    else {
                        nx.xu = XU_STEP;
                        nx.c1 = s[S_GLO];
                    }
                    outer_next = true;
                } else if (s[S_MAXY] >= Delta) {
                    nx.xu = XU_STEP;
                    nx.c1 = s[S_GHI];
                    outer_next = true;
                } else {
                    p.rho_km2 = p.rho_km1;
                    p.rho_km1 = s[S_RHONEW];
                    if (p.rho_km1 > p.innertol) {
                        if (++p.mm > max_inner) {
                            status[act[(size_t)a]] = 1;
                            stop = true;
                            continue;
                        }
                        p.k++;
                        nx.pre = PRE_NEXT;
                        nx.c1 = p.rho_km1 / p.rho_km2;
                        nx.c3 = p.rho_km1;
                        nx.mv = MV_XP;
                        nx.post = POST_CG;
                    } else {
                        nx.xu = XU_STEP;
                        nx.c1 = 1.0;
                        outer_next = true;
                    }
                }
            }
            if (outer_next) {
                nx.mv = MV_X;
                nx.post = POST_OUTER;
            }
        }
    }
    for (int q = 0; q < n_prob && rc == HH_OK; ++q) {
        const Prob& p = P[(size_t)q];
        n_outer[q] = p.i;
        n_inner[q] = p.inner;
        e = cudaMemcpyAsync(x_out + p.vbase, V + V_X * L + p.vbase, sizeof(double) * (size_t)p.n, cudaMemcpyDeviceToHost, ctx->stream);
        if (e != cudaSuccess) fail("x download", e);
    }
    if (rc == HH_OK) {
        e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) fail("x download", e);
    }
    if (h_cmd) cudaFreeHost(h_cmd);
    if (h_sc) cudaFreeHost(h_sc);
    hh_dfree(d_cmd);
    hh_dfree(d_sc);
    hh_dfree(V);
    return rc;
}

int hh_contact_normalize(hh_contact* h, int mode, int32_t n_blk, const int32_t* blk_off, const int32_t* blk_n,
                         const double* x_blocks, const double* x_whole, double* out, double* median_lo, double* median_hi,
                         int64_t* n_values) {
    HH_REQUIRE(h && (n_blk == 0 || (blk_off && blk_n)) && n_blk >= 0 && median_lo && median_hi && n_values, HH_ERR_ARG,
               "hh_contact_normalize: bad arguments");
    HH_REQUIRE(mode == NORM_KR || mode == NORM_LOG10 || mode == NORM_NONE, HH_ERR_ARG, "hh_contact_normalize: bad mode %d", mode);
    HH_REQUIRE(mode != NORM_KR || (x_blocks && x_whole), HH_ERR_ARG, "hh_contact_normalize: KR needs both scalings");
    hh_scope _scope(h->ctx);
    HH_REQUIRE(h->finished, HH_ERR_STATE, "hh_contact_normalize: hh_contact_finish first");
    hh_ctx* ctx = h->ctx;
    const int64_t nb = h->nb;
    std::vector<int32_t> blk((size_t)nb, -1);
    std::vector<int64_t> row_base((size_t)n_blk + 1, 0), val_base((size_t)n_blk + 1, 0);
    for (int b = 0; b < n_blk; ++b) {
        HH_REQUIRE(blk_n[b] > 0 && blk_off[b] >= 0 && (int64_t)blk_off[b] + blk_n[b] <= nb, HH_ERR_ARG,
                   "hh_contact_normalize: block %d outside the matrix", b);
        for (int32_t i = 0; i < blk_n[b]; ++i) blk[(size_t)(blk_off[b] + i)] = b;
        row_base[(size_t)b + 1] = row_base[(size_t)b] + blk_n[b];
        val_base[(size_t)b + 1] = val_base[(size_t)b] + (int64_t)blk_n[b] * (blk_n[b] - 1);
    }
    const int64_t n_val = val_base[(size_t)n_blk];
    int32_t *d_blk = nullptr, *d_boff = nullptr, *d_bn = nullptr;
    int64_t *d_rb = nullptr, *d_vb = nullptr;
    double *d_xb = nullptr, *d_xw = nullptr, *d_val = nullptr, *d_sorted = nullptr, *stage = nullptr;
    void* d_tmp = nullptr;
    int rc = HH_OK;
    auto fail = [&](const char* what, cudaError_t e) {
        hh_set_error("hh_contact_normalize: %s: %s", what, cudaGetErrorString(e));
        rc = HH_ERR_CUDA;
    };
    do {
        if ((rc = upload(ctx, &d_blk, blk.data(), nb)) != HH_OK) break;
        if ((rc = upload(ctx, &d_boff, blk_off, n_blk)) != HH_OK) break;
        if ((rc = upload(ctx, &d_bn, blk_n, n_blk)) != HH_OK) break;
        if ((rc = upload(ctx, &d_rb, row_base.data(), (int64_t)n_blk + 1)) != HH_OK) break;
        if ((rc = upload(ctx, &d_vb, val_base.data(), (int64_t)n_blk + 1)) != HH_OK) break;
        if (mode == NORM_KR) {
            if ((rc = upload(ctx, &d_xb, x_blocks, nb)) != HH_OK) break;
            if ((rc = upload(ctx, &d_xw, x_whole, nb)) != HH_OK) break;
        }
        // vmax: median of the intra-scaffold off-diagonal values, sorted on the device
        *n_values = n_val;
        *median_lo = *median_hi = NAN;
        if (n_val > 0) {
            if ((rc = hh_dmalloc(&d_val, (size_t)n_val)) != HH_OK) break;
            if ((rc = hh_dmalloc(&d_sorted, (size_t)n_val)) != HH_OK) break;
            const int64_t rows = row_base[(size_t)n_blk];
            if (h->d_m64) k_gather_intra<int64_t><<<(unsigned)rows, 256, 0, ctx->stream>>>(h->d_m64, h->nb, n_blk, d_boff, d_bn, d_rb, d_vb, mode, d_xb, d_val);
            else k_gather_intra<int32_t><<<(unsigned)rows, 256, 0, ctx->stream>>>(h->d_m32, h->nb, n_blk, d_boff, d_bn, d_rb, d_vb, mode, d_xb, d_val);
            ctx->launches++;
            cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) { fail("gather", e); break; }
            size_t tmp_bytes = 0;
            e = cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, d_val, d_sorted, n_val, 0, 64, ctx->stream);
            if (e != cudaSuccess) { fail("sort size", e); break; }
            char* t = nullptr;
            if ((rc = hh_dmalloc(&t, tmp_bytes)) != HH_OK) break;
            d_tmp = t;
            e = cub::DeviceRadixSort::SortKeys(d_tmp, tmp_bytes, d_val, d_sorted, n_val, 0, 64, ctx->stream);
            ctx->launches++;
            if (e != cudaSuccess) { fail("sort", e); break; }
            const int64_t mid = n_val / 2;
            const int64_t lo_i = (n_val % 2) ? mid : mid - 1;
            e = cudaMemcpyAsync(median_lo, d_sorted + lo_i, 8, cudaMemcpyDeviceToHost, ctx->stream);
            if (e == cudaSuccess) e = cudaMemcpyAsync(median_hi, d_sorted + mid, 8, cudaMemcpyDeviceToHost, ctx->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
            if (e != cudaSuccess) { fail("median", e); break; }
        }
        if (out) {
            const int64_t rows = std::max<int64_t>(1, std::min<int64_t>(nb, FETCH_ROWS_BYTES / (nb * 8)));
            if ((rc = hh_dmalloc(&stage, (size_t)(rows * nb))) != HH_OK) break;
            const unsigned gx = (unsigned)std::min<int64_t>((nb + 255) / 256, 64);
            for (int64_t r0 = 0; r0 < nb; r0 += rows) {
                const int64_t m = std::min(rows, nb - r0);
                const dim3 grid(gx, (unsigned)m);
                if (h->d_m64) k_norm_rows<int64_t><<<grid, 256, 0, ctx->stream>>>(h->d_m64, h->nb, r0, mode, d_blk, d_xb, d_xw, stage);
                else k_norm_rows<int32_t><<<grid, 256, 0, ctx->stream>>>(h->d_m32, h->nb, r0, mode, d_blk, d_xb, d_xw, stage);
                ctx->launches++;
                cudaError_t e = cudaGetLastError();
                if (e == cudaSuccess) e = cudaMemcpyAsync(out + r0 * nb, stage, (size_t)(m * nb) * 8, cudaMemcpyDeviceToHost, ctx->stream);
                if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
                if (e != cudaSuccess) { fail("rows", e); break; }
            }
        }
    } while (0);
    cudaStreamSynchronize(ctx->stream);
    hh_dfree(d_blk);
    hh_dfree(d_boff);
    hh_dfree(d_bn);
    hh_dfree(d_rb);
    hh_dfree(d_vb);
    hh_dfree(d_xb);
    hh_dfree(d_xw);
    hh_dfree(d_val);
    hh_dfree(d_sorted);
    if (d_tmp) {
        char* t = (char*)d_tmp;
        hh_dfree(t);
    }
    hh_dfree(stage);
    return rc;
}

int hh_contact_destroy(hh_contact* h) {
    if (!h) return HH_OK;
    hh_scope _scope(h->ctx);
    cudaStreamSynchronize(h->ctx->stream);
    if (h->copy_stream) cudaStreamSynchronize(h->copy_stream);
    contact_free(h);
    delete h;
    return HH_OK;
}

}  // extern "C"
