"""Host reference of the tensor-core pre-expansion M1 = M0 . M0 (csrc/hh_gemm.cu: hh_k_gemm_densify + hh_k_syrk +
hh_k_clip_fix in hh_mcl_create_ex).  Used by tests/test_gpu_gemm_scale.py and checked itself in tests/test_gemm_oracle.py.

  exact_m1_cols     the fp64 product M0 @ M0[:, cols] of the fp32 matrix M0, from SciPy sparse products (seconds at
                    n = 50k, where a dense n^3 would take hours).
  encode / emulate_m1_cols
                    the operand planes hh_k_gemm_densify writes, element for element (scaled f16: one plane of
                    min(C, 2048) * 2^-e_k against f16 hi + lo of fp32(C / s) * 2^e_k; exact bf16: hg_split3, the three-way
                    truncating split), and the fp64 product of those planes over the library's pass list.  Switches
                    reproduce plausible defects (flushed subnormals, a dropped lo plane, e_k off by one on one side, a K
                    range left out, a missing clip correction), so the tests can show that the 2e-6 bar catches each.
  expected_preexp   the choice hh_gemm_preexpand makes from the data and the HH_GEMM_FMT / HH_GEMM_KCHUNKS settings:
                    encoding, planes, passes, clip, K chunks and densify segments.
  the input generators the GPU tests use (random counts, a hub column, one planted large count).

Nothing under haphic_b200/ imports this module."""

import numpy as np
import scipy.sparse as sp

BAR = 2e-6                      # DESIGN.md section 2: every stored entry of M1 within 2e-6 relative of the exact product
# DESIGN.md section 2: what the truncating tensor-core accumulation and the fp32 clip correction reach on the inputs that
# exceed BAR (the six-pass weights encoding at C3, a hub column under the f16 drain period, 4,095 clipped counts in a column)
ACCUMULATION_BAND = 5e-6
HG_SEG = 32768                  # columns of one operand row that hh_k_gemm_densify assembles at a time
F16_CLIP, BF16_CLIP = 2048.0, 256.0
COLSUM_F16_LIMIT = 2.0 ** 23    # a column sum at or above it forces the exact bf16 encoding
PLANE_BUDGET = 16.0e9           # bytes of operand planes per K chunk
BF16, F16 = 0, 1                # hh_preexp_info.fmt_a / fmt_b
PASSES_1 = [(0, 0), (0, 1), (0, 2)]
PASSES_3 = [(0, 0), (0, 1), (1, 0), (0, 2), (1, 1), (2, 0)]      # every plane pair of relative size >= 2^-16
PASSES_F16 = [(0, 0), (0, 1)]


# ---------------------------------------------------------------------------------------------------------------------------
# the exact product
# ---------------------------------------------------------------------------------------------------------------------------
def colsums(link):
    """fp64 column sums of |C| (hh_k_gemm_colsum; sklearn normalize)."""
    link = sp.csc_matrix(link)
    return np.asarray(abs(link).sum(axis=0, dtype=np.float64)).ravel()


def normalize(link):
    """M0 = fp32(fp64(C) / s), column by column (what hh_mcl_create stores and Mcl.m0() returns)."""
    link = sp.csc_matrix(link, dtype=np.float32)
    s = colsums(link)
    col = np.repeat(np.arange(link.shape[1]), np.diff(link.indptr))
    with np.errstate(divide="ignore", invalid="ignore"):
        v = np.where(s[col] != 0, link.data.astype(np.float64) / s[col], link.data)
    return sp.csc_matrix((v.astype(np.float32), link.indices, link.indptr), shape=link.shape)


def exact_m1_cols(m0, cols):
    """fp64 M0 @ M0[:, cols] as a dense [n, len(cols)] array; m0 is the fp32 M0 (scipy sparse)."""
    m = sp.csc_matrix(m0, dtype=np.float64)
    return np.asarray((m @ m[:, cols]).todense())


def rel_error(got, ref):
    """(pattern_equal, max relative error over the stored entries of ref)."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    nz = ref != 0
    same = bool(np.array_equal(got != 0, nz))
    if not nz.any():
        return same, 0.0
    return same, float((np.abs(got[nz] - ref[nz]) / ref[nz]).max())


# ---------------------------------------------------------------------------------------------------------------------------
# the path hh_gemm_preexpand chooses
# ---------------------------------------------------------------------------------------------------------------------------
def expected_preexp(link, fmt=None, kchunks=None):
    """What hh_gemm_preexpand does with the link matrix `link`, HH_GEMM_FMT = fmt and HH_GEMM_KCHUNKS = kchunks (None =
    unset).  Keys as in Mcl.preexp, plus `weights`, `clipped`, `kw` (K chunk width) and `segments` (densify segments per
    chunk)."""
    link = sp.csc_matrix(link, dtype=np.float32)
    n = link.shape[0]
    v = link.data
    s = colsums(link)
    # hh_k_gemm_valstats flag 1: some value is not an integer in [0, 65536); hh_k_gemm_colsum flag 4: a column sum >= 2^23
    weights = bool(np.any(~((v >= 0) & (v < np.float32(65536)) & (v == np.floor(v)))))
    exact = fmt == "bf16" or weights or (n > 0 and s.max() >= COLSUM_F16_LIMIT)
    a_planes = 3 if weights else 1
    b_planes = 3 if exact else 2
    passes = 6 if weights else (3 if exact else 2)
    clip = float(np.float32(3.0e38)) if weights else (BF16_CLIP if exact else F16_CLIP)
    clipped = (not weights) and len(v) > 0 and float(v.max()) > clip
    ldk = (n + 63) // 64 * 64
    plane_bytes = float(a_planes + b_planes) * float(ldk) * float(n) * 2.0
    k = int(plane_bytes / PLANE_BUDGET) + 1 if kchunks is None else int(kchunks)
    k = max(k, 1)
    kw = ((n + k - 1) // k + 63) // 64 * 64
    k_chunks = (n + kw - 1) // kw
    fmt_ab = BF16 if exact else F16
    return {"mode": "dense", "weights": weights, "fmt_a": fmt_ab, "fmt_b": fmt_ab, "a_planes": a_planes, "b_planes": b_planes,
            "passes": passes, "clip": clip, "clipped": clipped, "k_chunks": k_chunks, "kw": kw,
            "segments": (kw + HG_SEG - 1) // HG_SEG, "chunk_kb": 1 if passes > 3 else (2 if passes == 3 else 3)}


# ---------------------------------------------------------------------------------------------------------------------------
# operand encodings of hh_k_gemm_densify
# ---------------------------------------------------------------------------------------------------------------------------
def split3(x):
    """hg_split3: x = h1 + h2 + h3 exactly, each a bf16 value obtained by truncation (returned as fp64 arrays)."""
    x = np.asarray(x, np.float32)
    mask = np.uint32(0xFFFF0000)
    b1 = (x.view(np.uint32) & mask).view(np.float32)
    r1 = (x - b1).astype(np.float32)
    b2 = (r1.view(np.uint32) & mask).view(np.float32)
    r2 = (r1 - b2).astype(np.float32)
    b3 = (r2.view(np.uint32) & mask).view(np.float32)
    return [b.astype(np.float64) for b in (b1, b2, b3)]


def exponent(s):
    """e with s in [2^(e-1), 2^e) (the exponent field of the double minus 1022); 0 for s == 0."""
    _m, e = np.frexp(np.asarray(s, np.float64))
    return np.where(np.asarray(s) != 0, e, 0).astype(np.int64)


def _f16(x, flush):
    h = np.asarray(x, np.float32).astype(np.float16)                   # round to nearest even, subnormals kept
    if flush:
        h = np.where(np.abs(h) < np.float16(2.0 ** -14), np.float16(0), h)
    return h


def encode(link, enc, flush_subnormals=False, drop_lo=False, e_off_a=0):
    """Operand planes of hh_k_gemm_densify on the pattern of `link`: value (r, k) of plane p of A is A_p[r, k], of B is
    B_p[r, k] (row r of either operand; C is symmetric).  enc = "f16" (scaled), "bf16" (exact, one count plane) or
    "weights" (three planes each side).  Returns (A planes, B planes, pass list, the unscaled planes' exponents e_k) with
    every plane a scipy CSC of fp64 values.
    Defects: flush_subnormals (f16 values below 2^-14 become 0), drop_lo (the f16 lo plane of B is zero), e_off_a (A is
    scaled with 2^-(e_k + e_off_a) while B keeps 2^e_k)."""
    link = sp.csc_matrix(link, dtype=np.float32)
    link.sort_indices()
    s = colsums(link)
    col = np.repeat(np.arange(link.shape[1]), np.diff(link.indptr))
    sk = s[col]
    clip = {"f16": F16_CLIP, "bf16": BF16_CLIP, "weights": np.float32(3.0e38)}[enc]
    v = np.minimum(link.data, np.float32(clip))                          # fminf(val, clip)
    with np.errstate(divide="ignore", invalid="ignore"):
        x = np.where(sk != 0, v.astype(np.float64) / sk, v).astype(np.float32)      # fp32(A / s[k])
    e = exponent(s)[col]

    def plane(vals):
        return sp.csc_matrix((np.asarray(vals, np.float64), link.indices, link.indptr), shape=link.shape)

    if enc == "f16":
        ea = e + e_off_a
        xa = (v * np.ldexp(np.float32(1), -ea).astype(np.float32)).astype(np.float32)
        a = [_f16(xa, flush_subnormals)]
        xs = (x * np.ldexp(np.float32(1), e).astype(np.float32)).astype(np.float32)
        hi = _f16(xs, flush_subnormals)
        lo = _f16((xs - hi.astype(np.float32)).astype(np.float32), flush_subnormals)
        if drop_lo:
            lo = np.zeros_like(lo)
        b = [hi, lo]
        return [plane(p.astype(np.float64)) for p in a], [plane(p.astype(np.float64)) for p in b], PASSES_F16, e
    if enc == "bf16":
        return [plane(split3(v)[0])], [plane(p) for p in split3(x)], PASSES_1, e
    return [plane(p) for p in split3(v)], [plane(p) for p in split3(x)], PASSES_3, e


def emulate_m1_cols(link, cols, enc, clip_fix=True, drop_k=None, **defects):
    """M1[:, cols] as the library computes it, with the tensor-core sums taken exactly: S = sum over the pass list of
    A_pa . B_pb^T in fp64 from the encoded planes, times fp32(1 / s[c]); plus, when counts were clipped and clip_fix is set,
    the clip correction M0 . M0l + M0l . M0s (hh_k_clip_fix) in fp64.  drop_k = (k0, k1) leaves that K range out of the
    GEMM (a lost densify segment or K chunk).  Returns a dense [n, len(cols)] fp64 array."""
    link = sp.csc_matrix(link, dtype=np.float32)
    n = link.shape[0]
    cols = np.arange(n)[cols]
    A, B, passes, _e = encode(link, enc, **defects)
    if drop_k is not None:
        keep = np.ones(n)
        keep[drop_k[0]:drop_k[1]] = 0.0
        A = [a @ sp.diags(keep) for a in A]
    Bc = [sp.csr_matrix(b)[cols, :].T.tocsc() for b in B]               # [k, c] = B[c, k]
    S = None
    for pa, pb in passes:
        t = A[pa] @ Bc[pb]
        S = t if S is None else S + t
    s = colsums(link)
    with np.errstate(divide="ignore"):
        inv = np.where(s != 0, (1.0 / s).astype(np.float32), np.float32(1)).astype(np.float64)
    m1 = np.asarray(S.todense()) * inv[cols][None, :]
    clip = {"f16": F16_CLIP, "bf16": BF16_CLIP, "weights": None}[enc]
    if clip_fix and clip is not None and link.nnz and link.data.max() > clip:
        c64 = sp.csc_matrix(link, dtype=np.float64)
        s_col = sp.diags(np.where(s != 0, 1.0 / np.where(s != 0, s, 1.0), 1.0))
        m0 = c64 @ s_col
        big = c64.copy()
        big.data = np.maximum(big.data - clip, 0.0)
        big.eliminate_zeros()
        small = c64.copy()
        small.data = np.minimum(small.data, clip)
        m0l, m0s = big @ s_col, small @ s_col
        m1 += np.asarray((m0 @ m0l[:, cols] + m0l @ m0s[:, cols]).todense())
    return m1


# ---------------------------------------------------------------------------------------------------------------------------
# inputs of the GPU tests
# ---------------------------------------------------------------------------------------------------------------------------
def _symmetric(n, i, j, v):
    """Symmetric CSC from upper-or-lower pairs (duplicates summed, diagonal dropped) plus self loops 1."""
    keep = i != j
    i, j, v = i[keep], j[keep], np.asarray(v, np.float64)[keep]
    lo, hi = np.minimum(i, j), np.maximum(i, j)
    u = sp.coo_matrix((v, (lo, hi)), shape=(n, n)).tocsr()
    u.sum_duplicates()
    m = u + u.T + sp.identity(n, dtype=np.float64, format="csr")
    m = sp.csc_matrix(m, dtype=np.float32)
    m.sort_indices()
    return m


def random_counts(n, per_col, maxc, seed):
    """Symmetric integer link counts, about `per_col` entries per column, geometric counts capped at maxc, self loops 1."""
    rng = np.random.default_rng(seed)
    m = max(1, int(n * per_col / 2))
    i = rng.integers(0, n, m)
    j = rng.integers(0, n, m)
    v = np.minimum(rng.geometric(0.4, m), maxc)
    a = _symmetric(n, i, j, v)
    a.data = np.minimum(a.data, np.float32(maxc))
    return a


# K cuts at size: n > 32768 * 1.8, so one K chunk has two densify segments (the second partial), and the default cut of the
# scaled f16 encoding (3 planes of n x n) is two chunks
KCUT_N, KCUT_PER_COL, KCUT_MAXC, KCUT_SEED = 60000, 300, 50, 60
KCUT_SHARDS = [(0, 100), (32700, 32900), (59900, 60000)]


def kcut_matrix():
    return random_counts(KCUT_N, KCUT_PER_COL, KCUT_MAXC, KCUT_SEED)


def hub_matrix(hub_sum, n=6200, hub=3001, seed=5):
    """A sparse random background (counts <= 8) plus one hub column (and row) of sum `hub_sum` (self loop included):
    4095 neighbours with count 2048 and the rest of the sum in neighbours with count 1.  With hub_sum = 2^23 - 1 the hub's
    e_k is 23 and its count-1 entries enter the scaled f16 plane as the subnormal 2^-23."""
    rng = np.random.default_rng(seed)
    ones = int(hub_sum) - 1 - 4095 * 2048
    assert 0 <= ones and 4095 + ones <= n - 1
    others = np.delete(np.arange(n), hub)
    nb = rng.permutation(others)[: 4095 + ones]
    m = n * 10
    i = rng.integers(0, n, m)
    j = rng.integers(0, n, m)
    bg = (i != hub) & (j != hub)
    v = np.minimum(rng.geometric(0.5, m), 8)
    ii = np.concatenate([i[bg], np.full(len(nb), hub)])
    jj = np.concatenate([j[bg], nb])
    vv = np.concatenate([v[bg], np.full(4095, 2048), np.ones(ones)])
    return _symmetric(n, ii, jj, vv)


def planted_count(value, n=300, per_col=12, seed=17):
    """Random counts <= 20 plus one pair (7, 250) with link count `value`, the matrix maximum."""
    a = sp.lil_matrix(random_counts(n, per_col, 20, seed))
    a[7, 250] = value
    a[250, 7] = value
    a = sp.csc_matrix(a, dtype=np.float32)
    a.sort_indices()
    return a
