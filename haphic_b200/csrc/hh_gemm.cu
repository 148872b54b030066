// Dense-block pre-expansion on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
// What it computes (scripts/HapHiC_cluster.py:2144-2149, dense mode 2035 / 2149): the one-off pre-expansion
//     M1 = M0 . M0,   M0 = normalize(link_matrix, 'l1', axis=0)
// for the part of the product that is a true GEMM.  With C the symmetric link matrix and s its column sums,
//     M1[r, c] = ( sum_k C[r, k] * M0[c, k] ) / s[c]          (C[k, c] = C[c, k],  M0[c, k] = C[c, k] / s[k])
// so S[r, c] = sum_k C[r, k] * M0[c, k] is a "TN" GEMM of two row-major (K-major) n x n operands and S is symmetric:
// only tiles on or above the diagonal are computed; the epilogue writes M1[r, c] = S / s[c] and the mirror image
// M1[c, r] = S / s[r].
//
// Precision.  The reference multiplies fp32 by fp32.  Tensor cores take bf16, so each operand is split into bf16
// "planes" whose sum is the fp32 value EXACTLY:
//   A = C      link counts are integers: <= 256 -> one plane, < 65536 -> two, anything else (weights) three;
//   B = M0     three planes (8 + 8 + 8 significant bits).
// A bf16 x bf16 product is exact in fp32, so the passes (plane_a, plane_b) below reproduce the fp32 product up to
// dropped terms of relative size 2^-24.  The accumulation inside the tensor core is not IEEE round-to-nearest, so a
// tile's K range is cut into chunks: each chunk accumulates in the wgmma accumulator registers and is then added to a
// second set of fp32 registers with round-to-nearest (HH_GEMM_CHUNK k-blocks per chunk).
//
#include "hh_common.cuh"
#include "hh_internal.cuh"
#include "hh_gemm.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <algorithm>

// ---------------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t hg_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void hg_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void hg_fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void hg_mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
    } while (!ok);
}
__device__ __forceinline__ void hg_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void hg_mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

__device__ __forceinline__ void hg_tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint32_t mbar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
                 "l"(tm), "r"(mbar), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void hg_prefetch_tmap(const CUtensorMap* tm) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}

// shared-memory matrix descriptor (sm_90 wgmma) of a K-major tile stored as [rows][64 16-bit] with the 128-byte swizzle TMA
// applies: 8-row groups 1024 bytes apart (SBO), layout type 1 = SWIZZLE_128B.  The start address moves by 32 bytes per K = 16
// step inside the swizzle atom.
__device__ __forceinline__ uint64_t hg_make_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
    d |= (uint64_t)1 << 16;               // leading byte offset: unused for swizzled K-major layouts
    d |= (uint64_t)(1024 >> 4) << 32;     // stride byte offset
    d |= (uint64_t)1 << 62;               // SWIZZLE_128B
    return d;
}

__device__ __forceinline__ void hg_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void hg_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void hg_wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D (+)= A[smem] . B[smem]^T for one warpgroup: M = 64 rows of A, N = 128 rows of B, K = 16, 16-bit operands (bf16 or f16),
// fp32 accumulator in 64 registers per thread.  accumulate == 0 overwrites D.
#define HG_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define HG_WGMMA_BODY(TYPES)                                                                                                      \
    asm volatile(                                                                                                                 \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                                         \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TYPES " "                                                                  \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                                 \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                                        \
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                                         \
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "                                       \
        "%64, %65, p, 1, 1, 0, 0;\n\t}"                                                                                           \
        : HG_ACC8(0), HG_ACC8(8), HG_ACC8(16), HG_ACC8(24), HG_ACC8(32), HG_ACC8(40), HG_ACC8(48), HG_ACC8(56)                   \
        : "l"(adesc), "l"(bdesc), "r"(accumulate))
template <bool F16>
__device__ __forceinline__ void hg_wgmma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if (F16) HG_WGMMA_BODY("f16.f16");
    else HG_WGMMA_BODY("bf16.bf16");
}

// ---------------------------------------------------------------------------------------------------------------------
// the GEMM kernel
// ---------------------------------------------------------------------------------------------------------------------
// Kernel shape (one persistent CTA per SM, tile 128 x 128, BLOCK_K = 64 16-bit = one 128-byte swizzle atom):
//   warpgroup 0      TMA producer (one thread): per k-block one 128x64 box per operand plane (cp.async.bulk.tensor,
//                    SWIZZLE_128B) into a ring of shared-memory stages, completion on the stage's "full" mbarrier;
//   warpgroups 1, 2  rows 0-63 / 64-127 of the tile: wgmma (m64n128k16) for every pass and k step into register
//                    accumulators, then release the stage on its "empty" mbarrier (one arrival per warp).  Every
//                    HH_GEMM_CHUNK k-blocks the chunk accumulator is added to a second set of fp32 registers with
//                    round-to-nearest; after the last chunk the tile and its mirror image are scaled and stored.
#define HG_THREADS 384
#define HG_TILE 128
#define HG_PLANE_BYTES 16384        // 128 rows x 64 16-bit elements
#define HG_MAX_STAGES 4

struct hh_gemm_args {
    const hh_gemm_item* items;
    int n_items;
    int n;                 // matrix dimension
    int na, nb;            // planes of A / of B per k-block (1..3)
    int npass;
    int pa[8], pb[8];      // pass list: plane of A, plane of B
    int chunk_kb;          // k-blocks accumulated by the tensor core before they are added into the round-to-nearest registers
    int stages;
    float* m1;             // dense column-major [ld x (col_hi - col_lo)]
    long long ld;
    int col_lo, col_hi;
    const float* inv_s;    // 1 / column sum
    float out_scale;       // applied instead when inv_s == NULL
    int accumulate;        // 1: the epilogue adds to what the output holds (K range processed in several launches)
};

template <bool F16>
__global__ void __launch_bounds__(HG_THREADS, 1)
hh_k_syrk(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const hh_gemm_args a) {
    extern __shared__ uint8_t hg_smem_raw[];
    __shared__ __align__(8) uint64_t s_full[HG_MAX_STAGES];
    __shared__ __align__(8) uint64_t s_empty[HG_MAX_STAGES];

    const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
    const uint32_t smem_base = (hg_smem_u32(hg_smem_raw) + 1023u) & ~1023u;
    const uint32_t stage_bytes = (uint32_t)(a.na + a.nb) * HG_PLANE_BYTES;
    const int S = a.stages;

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            hg_mbar_init(hg_smem_u32(&s_full[s]), 1);
            hg_mbar_init(hg_smem_u32(&s_empty[s]), 8);        // every consumer warp
        }
        hg_fence_barrier_init();
        hg_prefetch_tmap(&tmA);
        hg_prefetch_tmap(&tmB);
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------------------------------------- TMA producer
        if (threadIdx.x == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int it = blockIdx.x; it < a.n_items; it += gridDim.x) {
                const hh_gemm_item w = a.items[it];
                for (int seg = 0; seg < 2; ++seg) {
                    for (int kb = w.kb_lo[seg]; kb < w.kb_hi[seg]; ++kb) {
                        hg_mbar_wait(hg_smem_u32(&s_empty[s]), ph ^ 1u);
                        const uint32_t bar = hg_smem_u32(&s_full[s]);
                        hg_mbar_expect_tx(bar, stage_bytes);
                        const uint32_t dst = smem_base + (uint32_t)s * stage_bytes;
                        for (int p = 0; p < a.na; ++p) hg_tma_load_3d(dst + (uint32_t)p * HG_PLANE_BYTES, &tmA, bar, kb * 64, w.m0, p);
                        for (int p = 0; p < a.nb; ++p)
                            hg_tma_load_3d(dst + (uint32_t)(a.na + p) * HG_PLANE_BYTES, &tmB, bar, kb * 64, w.n0, p);
                        if (++s == S) {
                            s = 0;
                            ph ^= 1u;
                        }
                    }
                }
            }
        }
        return;
    }

    // ----------------------------------------------------------------------------------------------- consumers
    const int e = wg - 1;                          // rows 64 e .. 64 e + 63 of the tile
    const int wq = (threadIdx.x >> 5) & 3;         // warp within the warpgroup
    int s = 0;
    uint32_t ph = 0;
    float acc[64], racc[64];
    for (int it = blockIdx.x; it < a.n_items; it += gridDim.x) {
        const hh_gemm_item w = a.items[it];
        const int total = (w.kb_hi[0] - w.kb_lo[0]) + (w.kb_hi[1] - w.kb_lo[1]);
#pragma unroll
        for (int j = 0; j < 64; ++j) {
            acc[j] = 0.f;
            racc[j] = 0.f;
        }
        int in_chunk = 0;
        for (int t = 0; t < total; ++t) {
            hg_mbar_wait(hg_smem_u32(&s_full[s]), ph);
            const uint32_t st = smem_base + (uint32_t)s * stage_bytes;
            hg_wgmma_fence();
            for (int p = 0; p < a.npass; ++p) {
                const uint64_t ad = hg_make_desc(st + (uint32_t)a.pa[p] * HG_PLANE_BYTES + (uint32_t)e * (64u * 128u));
                const uint64_t bd = hg_make_desc(st + (uint32_t)(a.na + a.pb[p]) * HG_PLANE_BYTES);
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    hg_wgmma<F16>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (in_chunk | p | k) ? 1u : 0u);
            }
            hg_wgmma_commit();
            hg_wgmma_wait0();
            __syncwarp();
            if (lane == 0) hg_mbar_arrive(hg_smem_u32(&s_empty[s]));      // this warp's reads of the stage are complete
            if (++s == S) {
                s = 0;
                ph ^= 1u;
            }
            if (++in_chunk == a.chunk_kb || t + 1 == total) {
#pragma unroll
                for (int j = 0; j < 64; ++j) racc[j] = __fadd_rn(racc[j], acc[j]);
                in_chunk = 0;
            }
        }
        // ---- scale and store: out[r, c] = D * scale[c]; mirror image out[c, r] = D * scale[r].
        // Accumulator layout of m64nN: register 4 q + 2 h + b holds row 16 wq + lane / 4 + 8 h, column 8 q + 2 (lane % 4) + b.
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = w.m0 + 64 * e + 16 * wq + (lane >> 2) + 8 * h;
            if (r >= w.m_end) continue;
            if (w.flags & HH_GEMM_DIRECT) {
                float* __restrict__ dst = a.m1 + (ptrdiff_t)(r - w.out_row0);
#pragma unroll
                for (int q = 0; q < 16; ++q) {
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        const int c = w.n0 + 8 * q + 2 * (lane & 3) + b;
                        if (c < w.n_end && c >= a.col_lo && c < a.col_hi) {
                            float* __restrict__ o = dst + (size_t)(c - a.col_lo) * (size_t)a.ld;
                            const float x = racc[4 * q + 2 * h + b];
                            const float v = a.inv_s ? x * __ldg(a.inv_s + c) : x * a.out_scale;
                            *o = a.accumulate ? __fadd_rn(*o, v) : v;
                        }
                    }
                }
            }
            if ((w.flags & HH_GEMM_MIRROR) && r >= a.col_lo && r < a.col_hi) {
                const float sr = a.inv_s ? __ldg(a.inv_s + r) : a.out_scale;
                float* __restrict__ dst = a.m1 + (size_t)(r - a.col_lo) * (size_t)a.ld - (ptrdiff_t)w.out_row0;
#pragma unroll
                for (int q = 0; q < 16; ++q) {
                    const int c = w.n0 + 8 * q + 2 * (lane & 3);
                    const float v0 = racc[4 * q + 2 * h] * sr, v1 = racc[4 * q + 2 * h + 1] * sr;
                    if (c + 1 < w.n_end && w.out_row0 == 0) {
                        float2 v = make_float2(v0, v1);
                        if (a.accumulate) {
                            const float2 old = *reinterpret_cast<const float2*>(dst + c);
                            v = make_float2(__fadd_rn(old.x, v.x), __fadd_rn(old.y, v.y));
                        }
                        *reinterpret_cast<float2*>(dst + c) = v;
                    } else {
                        if (c < w.n_end) dst[c] = a.accumulate ? __fadd_rn(dst[c], v0) : v0;
                        if (c + 1 < w.n_end) dst[c + 1] = a.accumulate ? __fadd_rn(dst[c + 1], v1) : v1;
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// operand preparation: CSC of the symmetric link matrix -> dense row-major bf16 planes
// ---------------------------------------------------------------------------------------------------------------------
// column sums in fp64 (sklearn normalize accumulates in double, 2144) and their fp32 reciprocals
__global__ void hh_k_gemm_colsum(const int64_t* __restrict__ colptr, const float* __restrict__ val, int n, double* __restrict__ s,
                                 float* __restrict__ inv_s, int* __restrict__ flags) {
    const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (c >= n) return;
    const int lane = threadIdx.x & 31;
    double t = 0.0;
    for (int64_t p = colptr[c] + lane; p < colptr[c + 1]; p += 32) t += fabs((double)val[p]);
    t = hh_warp_sum(t);
    if (lane == 0) {
        s[c] = t;
        inv_s[c] = (t != 0.0) ? (float)(1.0 / t) : 1.f;
        if (t >= 8388608.0) atomicOr(flags, 4);          // 2^-e_k of the scaled f16 encoding would leave the subnormal range
    }
}

// flags[0] |= 1 if some value is not an integer in [0, 65536); |= 2 if some value exceeds 256; |= 8 if some value exceeds 2048
__global__ void hh_k_gemm_valstats(const float* __restrict__ val, int64_t nnz, int* __restrict__ flags) {
    int f = 0;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += (int64_t)gridDim.x * blockDim.x) {
        const float v = val[p];
        if (!(v >= 0.f && v < 65536.f && v == floorf(v))) f |= 1;
        if (v > 256.f) f |= 2;
        if (v > 2048.f) f |= 8;
    }
    f = __reduce_or_sync(HH_FULL_MASK, f);
    if ((threadIdx.x & 31) == 0 && f) atomicOr(flags, f);
}

__device__ __forceinline__ void hg_split3(float x, unsigned short& h1, unsigned short& h2, unsigned short& h3) {
    const uint32_t b1 = __float_as_uint(x) & 0xFFFF0000u;          // bf16 by truncation: the remainder stays exact
    const float r1 = x - __uint_as_float(b1);
    const uint32_t b2 = __float_as_uint(r1) & 0xFFFF0000u;
    const float r2 = r1 - __uint_as_float(b2);
    h1 = (unsigned short)(b1 >> 16);
    h2 = (unsigned short)(b2 >> 16);
    h3 = (unsigned short)(__float_as_uint(r2) >> 16);              // at most 8 significant bits are left
}

// One CTA per column c of the CSC = row c of both operands.  Two encodings of  S[r, c] = sum_k C[r, k] * M0[c, k]:
//   exact bf16   A[c, k] = min(C[c, k], clip) in na planes,  B[c, k] = fp32(A[c, k] / s[k]) in three bf16 planes (8 + 8 + 8 bits);
//   scaled f16   A[c, k] = min(C[c, k], clip) * 2^-e_k  (ONE plane: an integer times a power of two is exact in bf16 up to 256 and
//                in f16 up to 2048, subnormals included while e_k <= 24),
//                B[c, k] = fp32(A / s[k]) * 2^e_k in (count, 2 count]  as TWO f16 planes hi + lo = 22 significant bits, round to
//                nearest: every product is within 2^-23 relative of the fp32 product, in two passes instead of three.
//                2^e_k is the power of two above the column sum s[k]: it cancels inside every product.
// The row is assembled in shared memory (segments of HG_SEG columns, up to three planes at a time) and written with
// coalesced 16-byte stores: every element of the padded row is written exactly once, so the planes need no memset and no
// read-modify-write of partially written sectors.
#define HG_SEG 32768
__global__ void __launch_bounds__(1024)
hh_k_gemm_densify(const int64_t* __restrict__ colptr, const int32_t* __restrict__ row, const float* __restrict__ val, int n,
                  const double* __restrict__ s, unsigned short* __restrict__ A, int na, unsigned short* __restrict__ B, int nb, long long ldk,
                  long long plane, float clip, int scaled, int a_f16, long long k0) {
    // the planes hold the K range [k0, k0 + ldk) of the operands (the whole range unless the product is cut along K)
    extern __shared__ __align__(16) unsigned short hg_row[];        // [3][HG_SEG]
    const int c = blockIdx.x;
    const int64_t p0 = colptr[c], p1 = colptr[c + 1];
    for (int group = 0; group < 2; ++group) {                       // 0: planes of A, 1: planes of B
        const int np = group ? nb : na;
        unsigned short* __restrict__ out = (group ? B : A) + (size_t)c * (size_t)ldk;
        for (long long seg0 = k0; seg0 < k0 + ldk; seg0 += HG_SEG) {
            const int seg_n = (int)((k0 + ldk - seg0 < HG_SEG) ? (k0 + ldk - seg0) : HG_SEG);      // multiple of 64
            uint4* z = reinterpret_cast<uint4*>(hg_row);
            for (int q = threadIdx.x; q < 3 * HG_SEG / 8; q += blockDim.x) z[q] = make_uint4(0u, 0u, 0u, 0u);
            __syncthreads();
            for (int64_t p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
                const long long k = row[p];
                if (k < seg0 || k >= seg0 + seg_n) continue;
                const float v = fminf(val[p], clip);      // counts above `clip` are finished by the caller's sparse correction
                const double sk = s[k];
                unsigned short h1 = 0, h2 = 0, h3 = 0;
                if (!scaled) {
                    float x = v;
                    if (group) x = (sk != 0.0) ? (float)((double)v / sk) : v;
                    hg_split3(x, h1, h2, h3);
                } else {
                    // s[k] in [2^(e-1), 2^e), 0 <= e <= 24: the exponent field of the double; 2^e and 2^-e as floats
                    const int e = (sk != 0.0) ? (int)((__double2hiint(sk) >> 20) & 0x7ff) - 1022 : 0;
                    if (!group) {
                        const float xa = v * __int_as_float((127 - e) << 23);
                        h1 = a_f16 ? __half_as_ushort(__float2half_rn(xa)) : (unsigned short)(__float_as_uint(xa) >> 16);
                    } else {
                        const float x = (sk != 0.0) ? (float)((double)v / sk) : v;
                        const float xs = x * __int_as_float((127 + e) << 23);
                        const __half hi = __float2half_rn(xs);
                        const __half lo = __float2half_rn(xs - __half2float(hi));
                        h1 = __half_as_ushort(hi);
                        h2 = __half_as_ushort(lo);
                    }
                }
                const int kk = (int)(k - seg0);
                hg_row[kk] = h1;
                if (np > 1) hg_row[HG_SEG + kk] = h2;
                if (np > 2) hg_row[2 * HG_SEG + kk] = h3;
            }
            __syncthreads();
            for (int pl = 0; pl < np; ++pl) {
                const uint4* src = reinterpret_cast<const uint4*>(hg_row + (size_t)pl * HG_SEG);
                uint4* dst = reinterpret_cast<uint4*>(out + (size_t)pl * (size_t)plane + (size_t)(seg0 - k0));
                for (int q = threadIdx.x; q < seg_n / 8; q += blockDim.x) dst[q] = src[q];
            }
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
typedef CUresult (*hg_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int hg_encode(CUtensorMap* tm, void* base, int rows, int kdim, long long ldk, long long plane_elems, int planes, int fmt) {
    static hg_encode_fn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        HH_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        HH_REQUIRE(p != nullptr && q == cudaDriverEntryPointSuccess, HH_ERR_CUDA, "hh_gemm: the driver does not export cuTensorMapEncodeTiled");
        fn = reinterpret_cast<hg_encode_fn>(p);
    }
    const cuuint64_t dims[3] = {(cuuint64_t)kdim, (cuuint64_t)rows, (cuuint64_t)planes};
    const cuuint64_t strides[2] = {(cuuint64_t)ldk * 2ull, (cuuint64_t)plane_elems * 2ull};
    const cuuint32_t box[3] = {64u, 128u, 1u};
    const cuuint32_t estr[3] = {1u, 1u, 1u};
    const CUresult r = fn(tm, fmt == HH_GEMM_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    HH_REQUIRE(r == CUDA_SUCCESS, HH_ERR_CUDA, "hh_gemm: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HH_OK;
}

static int hg_env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoi(v) : dflt;
}

template <bool F16>
static int hg_launch(hh_ctx* ctx, const CUtensorMap& tmA, const CUtensorMap& tmB, const hh_gemm_args& a, size_t smem) {
    auto kern = hh_k_syrk<F16>;
    HH_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int grid = ctx->sm_count;
    if (grid > a.n_items) grid = a.n_items;
    if (grid < 1) grid = 1;
    HH_LAUNCH(ctx, kern, grid, HG_THREADS, smem, tmA, tmB, a);
    return HH_OK;
}

int hh_gemm_run(hh_ctx* ctx, const hh_gemm_operand& A, const hh_gemm_operand& B, const hh_gemm_item* d_items, int n_items, int npass,
                const int* pa, const int* pb, int chunk_kb, float* out, long long ld, int col_lo, int col_hi, const float* scale,
                int* stages_out, float out_scale, int accumulate) {
    HH_REQUIRE(n_items >= 1 && npass >= 1 && npass <= 8, HH_ERR_ARG, "hh_gemm_run: bad work list");
    HH_REQUIRE(A.fmt == B.fmt, HH_ERR_ARG, "hh_gemm_run: wgmma takes one 16-bit format for both operands");
    CUtensorMap tmA, tmB;
    HH_CHECK(hg_encode(&tmA, (void*)A.base, A.rows, A.kdim, A.ldk, A.plane, A.planes, A.fmt));
    HH_CHECK(hg_encode(&tmB, (void*)B.base, B.rows, B.kdim, B.ldk, B.plane, B.planes, B.fmt));
    hh_gemm_args a;
    memset(&a, 0, sizeof(a));
    a.items = d_items;
    a.n_items = n_items;
    a.na = A.planes;
    a.nb = B.planes;
    a.npass = npass;
    for (int p = 0; p < npass; ++p) {
        a.pa[p] = pa[p];
        a.pb[p] = pb[p];
    }
    a.chunk_kb = chunk_kb < 1 ? (1 << 30) : chunk_kb;           // 0 = accumulate the whole K range in the tensor core
    const size_t stage_bytes = (size_t)(A.planes + B.planes) * HG_PLANE_BYTES;
    int stages = (int)((ctx->smem_optin - 2048) / stage_bytes);
    if (stages > HG_MAX_STAGES) stages = HG_MAX_STAGES;
    HH_REQUIRE(stages >= 2, HH_ERR_UNSUPPORTED, "hh_gemm: shared memory too small for two pipeline stages");
    a.stages = stages;
    if (stages_out) *stages_out = stages;
    a.m1 = out;
    a.ld = ld;
    a.col_lo = col_lo;
    a.col_hi = col_hi;
    a.inv_s = scale;
    a.out_scale = out_scale;
    a.accumulate = accumulate;
    const size_t smem = (size_t)stages * stage_bytes + 1024;
    return A.fmt == HH_GEMM_F16 ? hg_launch<true>(ctx, tmA, tmB, a, smem) : hg_launch<false>(ctx, tmA, tmB, a, smem);
}

static const int HG_P1[3][2] = {{0, 0}, {0, 1}, {0, 2}};
static const int HG_P3[6][2] = {{0, 0}, {0, 1}, {1, 0}, {0, 2}, {1, 1}, {2, 0}};

// pass list for `na` (1 or 3) planes of A against three planes of B: every product of relative size >= 2^-16 (na = 1: exact)
int hh_gemm_passes(int na, int* pa, int* pb) {
    const int(*pl)[2] = na == 1 ? HG_P1 : HG_P3;
    const int np = na == 1 ? 3 : 6;
    for (int p = 0; p < np; ++p) {
        pa[p] = pl[p][0];
        pb[p] = pl[p][1];
    }
    return np;
}

// The K range is cut into equal chunks when the operand planes of the whole range would exceed ~16 GB (a fifth of an 80 GB
// device; 150k contigs: 135 GB): planes of one chunk at a time, the epilogue of every chunk after the first adds to M1.  The
// cut depends on n and the encoding only, so every column block of M1 is cut alike and stays bit-identical.
void hh_gemm_kchunks(int n, int planes, long long* kw_out, int* kchunks_out) {
    const long long ldk = ((long long)n + 63) & ~63ll;
    const double plane_bytes_all = (double)planes * (double)(ldk * (long long)n) * 2.0;
    int kchunks = (int)(plane_bytes_all / 16.0e9) + 1;
    kchunks = hg_env_int("HH_GEMM_KCHUNKS", kchunks);
    if (kchunks < 1) kchunks = 1;
    const long long kw = ((((long long)n + kchunks - 1) / kchunks) + 63) & ~63ll;      // chunk width, multiple of 64
    *kw_out = kw;
    *kchunks_out = (int)(((long long)n + kw - 1) / kw);
}

size_t hh_gemm_preexpand_plane_bytes(int n) {
    size_t most = 0;
    for (int planes : {3, 4, 6}) {            // scaled f16 (1 + 2), exact bf16 (1 + 3), weights (3 + 3)
        long long kw = 0;
        int kc = 0;
        hh_gemm_kchunks(n, planes, &kw, &kc);
        const size_t b = (size_t)planes * (size_t)kw * (size_t)n * 2;
        if (b > most) most = b;
    }
    return most;
}

int hh_gemm_preexpand(hh_ctx* ctx, const hh_matrix* m, int col_lo, int col_hi, float* d_m1, long long ld, const hh_gemm_item* h_items,
                      int n_items, hh_gemm_stats* st) {
    const int n = m->n;
    HH_REQUIRE(n >= 1 && n_items >= 1, HH_ERR_ARG, "hh_gemm_preexpand: empty problem");
    double* d_s = nullptr;
    float* d_inv = nullptr;
    int* d_flags = nullptr;
    unsigned short *d_A = nullptr, *d_B = nullptr;
    hh_gemm_item* d_items = nullptr;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
    int rc = [&]() -> int {
        for (int k = 0; k < 3; ++k) HH_CUDA(cudaEventCreate(&ev[k]));
        HH_CHECK(hh_dmalloc(&d_s, (size_t)n));
        HH_CHECK(hh_dmalloc(&d_inv, (size_t)n));
        HH_CHECK(hh_dmalloc(&d_flags, 1));
        HH_CUDA(cudaEventRecord(ev[0], ctx->stream));
        HH_CUDA(cudaMemsetAsync(d_flags, 0, sizeof(int), ctx->stream));
        HH_LAUNCH(ctx, hh_k_gemm_colsum, (n + 7) / 8, 256, 0, m->d_colptr, m->d_val, n, d_s, d_inv, d_flags);
        HH_LAUNCH(ctx, hh_k_gemm_valstats, ctx->sm_count * 8, 256, 0, m->d_val, m->nnz, d_flags);
        int flags = 0;
        HH_CUDA(cudaMemcpyAsync(&flags, d_flags, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        // Integer link counts (the usual case): the scaled encoding, one plane of min(count, clip) against two f16 planes of M0,
        // two passes, clip 2048; the excess over `clip` is the caller's sparse correction.  It needs column sums below 2^23 (the
        // scaled counts may be f16 subnormals, exact down to 2^-24).  Otherwise, or with HH_GEMM_FMT=bf16, the exact encoding:
        // one bf16 plane of min(count, 256) against three bf16 planes of M0, three passes.  (kind::f16 takes ONE format for both
        // operands.)
        // Anything else (weights of --normalize_by_nlinks, allele-aware scaling): three exact bf16 planes each, six passes.
        const char* fmt_env = getenv("HH_GEMM_FMT");
        int enc = 2;                                             // 0 = exact bf16, 2 = scaled f16
        if (fmt_env && !strcmp(fmt_env, "bf16")) enc = 0;
        if (flags & (1 | 4)) enc = 0;
        const int na = (flags & 1) ? 3 : 1;
        const int nb = enc ? 2 : 3;
        const float clip = (flags & 1) ? 3.0e38f : (enc == 2 ? 2048.f : 256.f);
        const int fmt_a = enc == 2 ? HH_GEMM_F16 : HH_GEMM_BF16, fmt_b = enc ? HH_GEMM_F16 : HH_GEMM_BF16;
        // The K range is cut into equal chunks when the operand planes of the whole range would exceed ~16 GB (a fifth of an
        // 80 GB device; 150k contigs: 135 GB): planes of one chunk at a time, the epilogue of every chunk after the first adds to M1.  The cut depends on
        // n and the encoding only, so every rank of a sharded run cuts alike and M1 stays bit-identical for any world size.
        long long kw = 0;
        int kchunks = 0;
        hh_gemm_kchunks(n, na + nb, &kw, &kchunks);
        const long long plane_c = kw * (long long)n;
        HH_CHECK(hh_ws_alloc(ctx, &d_A, (size_t)plane_c * (size_t)na));
        HH_CHECK(hh_ws_alloc(ctx, &d_B, (size_t)plane_c * (size_t)nb));
        // rows [n, ld) of every M1 column stay zero
        HH_CUDA(cudaMemsetAsync(d_m1, 0, (size_t)ld * (size_t)(col_hi - col_lo) * sizeof(float), ctx->stream));
        HH_CHECK(hh_dmalloc(&d_items, (size_t)n_items));
        int pa[8], pb[8];
        int npass = hh_gemm_passes(na, pa, pb);
        if (enc) {                                               // (A, B hi), (A, B lo)
            npass = 2;
            pa[0] = pa[1] = 0;
            pb[0] = 0;
            pb[1] = 1;
        }
        // k-blocks accumulated by the tensor core between two drains into the round-to-nearest registers: the tensor core's
        // accumulate truncates, so the bias grows with the number of accumulations (4 MMAs per k-block and pass); on dense
        // inputs (every product of similar size) 64 truncating accumulations reach 2.5e-6 of relative error.  Three k-blocks
        // = 24 accumulations, the same as three bf16 passes drained every second k-block, keeps every test input below 2e-6.
        const int chunk = hg_env_int("HH_GEMM_CHUNK", npass > 3 ? 1 : (npass == 3 ? 2 : 3));
        int stages = 0;
        float densify_ms = 0.f, gemm_ms = 0.f;
        const float stats_ms = 0.f;                              // column sums + value statistics: a fraction of a millisecond
        std::vector<hh_gemm_item> items_c(h_items, h_items + n_items);
        for (int kc = 0; kc < kchunks; ++kc) {
            const long long k0 = (long long)kc * kw;
            const long long k1 = std::min((long long)n, k0 + kw);
            HH_CUDA(cudaEventRecord(ev[0], ctx->stream));
            {
                auto kd = hh_k_gemm_densify;
                const size_t dsm = (size_t)3 * HG_SEG * sizeof(unsigned short);
                HH_CUDA(cudaFuncSetAttribute(kd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm));
                HH_LAUNCH(ctx, kd, n, 1024, dsm, m->d_colptr, m->d_row, m->d_val, n, d_s, d_A, na, d_B, nb, kw, plane_c, clip, enc ? 1 : 0,
                          enc == 2 ? 1 : 0, k0);
            }
            const int nkb_c = (int)((k1 - k0 + 63) / 64);
            for (auto& w : items_c) {
                w.kb_lo[0] = 0;
                w.kb_hi[0] = nkb_c;
            }
            HH_CUDA(cudaMemcpyAsync(d_items, items_c.data(), (size_t)n_items * sizeof(hh_gemm_item), cudaMemcpyHostToDevice, ctx->stream));
            hh_gemm_operand A = {d_A, na, n, (int)(k1 - k0), kw, plane_c, fmt_a};
            hh_gemm_operand B = {d_B, nb, n, (int)(k1 - k0), kw, plane_c, fmt_b};
            HH_CUDA(cudaEventRecord(ev[1], ctx->stream));
            HH_CHECK(hh_gemm_run(ctx, A, B, d_items, n_items, npass, pa, pb, chunk, d_m1, ld, col_lo, col_hi, d_inv, &stages, 1.0f,
                                 kc > 0 ? 1 : 0));
            HH_CUDA(cudaEventRecord(ev[2], ctx->stream));
            HH_CUDA(cudaStreamSynchronize(ctx->stream));         // items_c is rewritten for the next chunk
            float t0 = 0.f, t1 = 0.f;
            HH_CUDA(cudaEventElapsedTime(&t0, ev[0], ev[1]));
            HH_CUDA(cudaEventElapsedTime(&t1, ev[1], ev[2]));
            densify_ms += t0;
            gemm_ms += t1;
        }
        HH_CUDA(cudaEventRecord(ev[2], ctx->stream));
        HH_CUDA(cudaStreamSynchronize(ctx->stream));
        if (st) {
            memset(st, 0, sizeof(*st));
            st->a_planes = na;
            st->clipped = (clip < 1.0e38f && (flags & (clip > 256.f ? 8 : 2))) ? 1 : 0;
            st->clip = clip;
            st->fmt_a = fmt_a;
            st->fmt_b = fmt_b;
            st->b_planes = nb;
            st->passes = npass;
            st->cta_group = 1;                                   // one CTA per tile
            st->stages = stages;
            st->chunk_kb = chunk < 1 ? (1 << 30) : chunk;
            st->densify_ms = densify_ms + stats_ms;
            st->gemm_ms = gemm_ms;
            st->k_chunks = kchunks;
            double kb = 0.0;
            for (int i = 0; i < n_items; ++i) kb += (double)((h_items[i].kb_hi[0] - h_items[i].kb_lo[0]) + (h_items[i].kb_hi[1] - h_items[i].kb_lo[1]));
            const double tile = (double)HG_TILE;
            st->flops = 2.0 * tile * tile * 64.0 * kb * (double)npass;
        }
        return HH_OK;
    }();
    hh_dfree(d_s);
    hh_dfree(d_inv);
    hh_dfree(d_flags);
    hh_ws_free(ctx, d_A);
    hh_ws_free(ctx, d_B);
    hh_dfree(d_items);
    for (int k = 0; k < 3; ++k)
        if (ev[k]) cudaEventDestroy(ev[k]);
    return rc;
}


// ---------------------------------------------------------------------------------------------------------------------
// block-diagonal products of the Markov-cluster iterations (hh_mcl.cu): operand planes of the component blocks
// ---------------------------------------------------------------------------------------------------------------------
// Bt[c, kk] = M[lo + kk, c] for the columns c of `list` (lo = first row of c's component): one CTA per column assembles the
// row of its planes in shared memory and writes all ldk elements (zeros beyond the component).  Two encodings:
//   three bf16 planes, the exact fp32 value (8 + 8 + 8 bits by truncation);
//   two f16 planes of M * 2^14, hi + lo = 22 significant bits (entries of a pruned column-stochastic iterate lie in
//   [pruning, 1]: scaled they are f16 normals for every pruning >= 2^-14; the product carries 2^28, removed in the epilogue).
#define HG_BLK_SHIFT 14
__global__ void __launch_bounds__(128)
hh_k_blk_densify(const int* __restrict__ len, const uint2* __restrict__ ent, int cap, const int* __restrict__ list, int nlist,
                 const int* __restrict__ comp_lo, const int* __restrict__ comp_hi, unsigned short* __restrict__ Bt, long long ldk,
                 long long plane, int f16) {
    extern __shared__ __align__(16) unsigned short hb_row[];        // [3][ldk]
    const int j = list[blockIdx.x];
    const int lo = comp_lo[j], width = comp_hi[j] - lo;
    uint4* z = reinterpret_cast<uint4*>(hb_row);
    for (int q = threadIdx.x; q < (int)(3 * ldk / 8); q += 128) z[q] = make_uint4(0u, 0u, 0u, 0u);
    __syncthreads();
    const int L = len[j];
    const uint2* __restrict__ e = ent + (size_t)j * (size_t)cap;
    for (int p = threadIdx.x; p < L; p += 128) {
        const uint2 t = e[p];
        const unsigned kk = t.x - (unsigned)lo;
        if (kk < (unsigned)width) {
            unsigned short h1, h2, h3 = 0;
            if (f16) {
                const float xs = ldexpf(__uint_as_float(t.y), HG_BLK_SHIFT);
                const __half hi = __float2half_rn(xs);
                h1 = __half_as_ushort(hi);
                h2 = __half_as_ushort(__float2half_rn(xs - __half2float(hi)));
            } else {
                hg_split3(__uint_as_float(t.y), h1, h2, h3);
            }
            hb_row[kk] = h1;
            hb_row[ldk + kk] = h2;
            hb_row[2 * ldk + kk] = h3;
        }
    }
    __syncthreads();
    for (int pl = 0; pl < (f16 ? 2 : 3); ++pl) {
        const uint4* src = reinterpret_cast<const uint4*>(hb_row + (size_t)pl * (size_t)ldk);
        uint4* dst = reinterpret_cast<uint4*>(Bt + (size_t)pl * (size_t)plane + (size_t)j * (size_t)ldk);
        for (int q = threadIdx.x; q < (int)(ldk / 8); q += 128) dst[q] = src[q];
    }
}

// A[r, kk] = M[r, lo + kk] = Bt[lo + kk, r - lo]: the transpose inside every component block; zeros beyond the component and
// for rows of components wider than ldk (those are not multiplied).  grid (ceil(n / 32), ldk / 32, 3), block (32, 8).
__global__ void __launch_bounds__(256)
hh_k_blk_transpose(const unsigned short* __restrict__ Bt, unsigned short* __restrict__ A, int n, const int* __restrict__ comp_lo,
                   const int* __restrict__ comp_hi, long long ldk, long long plane) {
    __shared__ unsigned short tile[32][34];
    const int r0 = blockIdx.x * 32, kk0 = blockIdx.y * 32;
    const unsigned short* __restrict__ src = Bt + (size_t)blockIdx.z * (size_t)plane;
    unsigned short* __restrict__ dst = A + (size_t)blockIdx.z * (size_t)plane;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int rl = min(r0 + 31, n - 1);
    const bool same = (r0 + 31 < n) && comp_lo[r0] == comp_lo[rl];
    if (same) {
        const int lo = comp_lo[r0], width = comp_hi[r0] - lo;
        const bool fits = width <= (int)ldk;
        for (int y = ty; y < 32; y += 8) {
            const int kk = kk0 + y;
            tile[y][tx] = (fits && kk < width) ? src[(size_t)(lo + kk) * (size_t)ldk + (size_t)(r0 - lo + tx)] : (unsigned short)0;
        }
        __syncthreads();
        for (int y = ty; y < 32; y += 8) dst[(size_t)(r0 + y) * (size_t)ldk + (size_t)(kk0 + tx)] = tile[tx][y];
    } else {
        for (int y = ty; y < 32; y += 8) {
            const int r = r0 + y;
            if (r >= n) continue;
            const int lo = comp_lo[r], width = comp_hi[r] - lo;
            const int kk = kk0 + tx;
            dst[(size_t)r * (size_t)ldk + (size_t)kk] =
                (width <= (int)ldk && kk < width) ? src[(size_t)(lo + kk) * (size_t)ldk + (size_t)(r - lo)] : (unsigned short)0;
        }
    }
}

float hh_gemm_blk_out_scale(int f16) { return f16 ? ldexpf(1.0f, -2 * HG_BLK_SHIFT) : 1.0f; }

int hh_gemm_blk_operands(hh_ctx* ctx, const int* d_len, const void* d_ent, int cap, const int* d_list, int nlist, const int* d_comp_lo,
                         const int* d_comp_hi, int n, unsigned short* d_A, unsigned short* d_Bt, long long ldk, int f16) {
    const long long plane = ldk * (long long)n;
    auto kd = hh_k_blk_densify;
    const size_t dsm = (size_t)3 * (size_t)ldk * sizeof(unsigned short);
    HH_CUDA(cudaFuncSetAttribute(kd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm));
    if (nlist > 0)
        HH_LAUNCH(ctx, kd, nlist, 128, dsm, d_len, reinterpret_cast<const uint2*>(d_ent), cap, d_list, nlist, d_comp_lo, d_comp_hi, d_Bt, ldk,
                  plane, f16);
    dim3 grid((unsigned)((n + 31) / 32), (unsigned)(ldk / 32), f16 ? 2u : 3u), block(32, 8);
    hh_k_blk_transpose<<<grid, block, 0, ctx->stream>>>(d_Bt, d_A, n, d_comp_lo, d_comp_hi, ldk, plane);
    ctx->launches++;
    HH_CUDA(cudaGetLastError());
    return HH_OK;
}

int hh_gemm_tile_size() { return HG_TILE; }

// work list of the whole-matrix product: every tile pair (a <= b) on or above the diagonal whose result (columns of
// tile b) or mirror image (columns of tile a) falls into the owned column block [col_lo, col_hi).  A column shard
// computes every element exactly as the single-GPU run does (same tile, same orientation), so M1 is bit-identical
// for any number of shards.
int hh_gemm_items_full(int n, int col_lo, int col_hi, std::vector<hh_gemm_item>& out) {
    const int T = hh_gemm_tile_size();
    const int nt = (n + T - 1) / T;
    const int nkb = (n + 63) / 64;
    out.clear();
    auto owned = [&](int t) {
        const int c0 = t * T, c1 = std::min(n, c0 + T);
        return c1 > col_lo && c0 < col_hi;
    };
    // Rasterisation.  Item i runs on CTA (i mod CTAs), so one item per SM (132 on an H100) form a wave that streams its
    // operand panels together: the wave should be a compact block of tiles.  A panels (one plane) are two to three times
    // cheaper than B panels (two or three planes), so super-blocks are SB_M = 16 tiles tall and SB_N = 8 wide (128 tiles ~
    // one wave): per k-block a wave then reads 16 + 2 * 8 = 32 panel blocks instead of 1 + 2 * 132.
    const int SB_M = 16, SB_N = 8;
    for (int bb = 0; bb < nt; bb += SB_N) {
        for (int ba = 0; ba <= std::min(nt - 1, bb + SB_N - 1); ba += SB_M) {
            for (int ta = ba; ta < std::min(nt, ba + SB_M); ++ta) {
                for (int tb = std::max(bb, ta); tb < std::min(nt, bb + SB_N); ++tb) {
                    int flags = 0;
                    if (owned(tb)) flags |= HH_GEMM_DIRECT;
                    if (tb > ta && owned(ta)) flags |= HH_GEMM_MIRROR;
                    if (!flags) continue;
                    hh_gemm_item w;
                    memset(&w, 0, sizeof(w));
                    w.m0 = ta * T;
                    w.n0 = tb * T;
                    w.m_end = n;
                    w.n_end = n;
                    w.kb_lo[0] = 0;
                    w.kb_hi[0] = nkb;
                    w.flags = flags;
                    out.push_back(w);
                }
            }
        }
    }
    return HH_OK;
}
