"""Host reference of ONE Markov-clustering iteration (expansion, inflation, prune, normalise, convergence term), applied to
the device's own previous iterate.  Used by tests/test_gpu_mcl_steps.py to check every iteration engine of hh_mcl_step step
by step, and checked itself in tests/test_mcl_step_oracle.py.

Two expansions:
  expand_ordered  what the sequential engines (hh_k_col, hh_k_col_win, hh_k_col_small) promise: every cell (r, j) of the
                  product receives fp32 fused multiply-adds of P[r, i] * P[i, j] in ascending i, starting from 0.  The
                  relabelling of hh_mcl_commit ranks vertices by (component, index), so ascending new index inside a
                  component is ascending original index: the oracle works in original indices, as Mcl.result() returns them.
  expand_exact    the product in fp64 (the tensor-core block GEMM is held to a rounding band around it).
The epilogue restates hh_inflate and the E1-E3 phases of the column kernels; `delta` the fp32 convergence term."""

import math

import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

U = 2.0 ** -23          # one fp32 ulp, relative, upper bound


def canon(m, dtype=np.float32):
    m = sp.csc_matrix(m, dtype=dtype, copy=True)
    m.eliminate_zeros()
    m.sort_indices()
    return m


# ---------------------------------------------------------------------------------------------------------------------------
# exact fp32 fused multiply-add
# ---------------------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32(a * b + c) rounded once, element-wise.  The fp64 product of two fp32 values is exact (48 bits); the sum is
    formed with TwoSum and rounded to odd in fp64 (53 >= 24 + 2 bits), which makes the final cast to fp32 a correct
    rounding of the exact a * b + c."""
    a = np.asarray(a, np.float32).astype(np.float64)
    b = np.asarray(b, np.float32).astype(np.float64)
    c = np.asarray(c, np.float32).astype(np.float64)
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    even = (s.view(np.int64) & 1) == 0
    fix = (err != 0) & even
    if np.any(fix):
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------------
# expansion
# ---------------------------------------------------------------------------------------------------------------------------
def _product_terms(A, B, col_mask=None):
    """Every product term A[r, i] * B[i, j] of A.B as flat arrays (j, r, a = A[r, i], b = B[i, j]), ordered by j, then
    ascending i, then r.  col_mask restricts the columns j."""
    n = B.shape[1]
    lens_b = np.diff(B.indptr)
    col_of = np.repeat(np.arange(n, dtype=np.int64), lens_b)
    ent = np.arange(len(B.indices), dtype=np.int64)
    if col_mask is not None:
        ent = ent[np.asarray(col_mask, bool)[col_of]]
    ib = B.indices[ent].astype(np.int64)
    cnt = np.diff(A.indptr)[ib]
    tot = int(cnt.sum())
    first = np.cumsum(cnt) - cnt
    off = np.arange(tot, dtype=np.int64) - np.repeat(first, cnt)
    src = np.repeat(A.indptr[ib].astype(np.int64), cnt) + off
    return np.repeat(col_of[ent], cnt), A.indices[src].astype(np.int64), A.data[src], np.repeat(B.data[ent], cnt)


def power(A, B, col_mask=None):
    """A.B (columns col_mask) with one fp32 fma per product, each cell summed in ascending i from 0: fp32 CSC.  Also one
    factor A . A^(k-1) of mkl_matrix_power (--expansion k > 2)."""
    A, B = canon(A), canon(B)
    n = A.shape[0]
    j, r, a, b = _product_terms(A, B, col_mask)
    key = j * n + r
    order = np.argsort(key, kind="stable")            # cells grouped, ascending i kept inside a cell
    ks = key[order]
    start = np.ones(len(ks), bool)
    start[1:] = ks[1:] != ks[:-1]
    cell = np.cumsum(start) - 1                       # cell id per sorted term
    first = np.nonzero(start)[0]
    rank = np.arange(len(ks)) - first[cell]
    acc = np.zeros(len(first), np.float32)
    a, b = a[order], b[order]
    by_rank = np.argsort(rank, kind="stable")
    bounds = np.searchsorted(rank[by_rank], np.arange(int(rank.max(initial=-1)) + 2))
    for t in range(len(bounds) - 1):
        sel = by_rank[bounds[t]:bounds[t + 1]]
        c = cell[sel]                                 # distinct cells: one term of rank t each
        acc[c] = fma32(a[sel], b[sel], acc[c])
    keys = ks[first]
    return canon(sp.csc_matrix((acc, (keys % n, keys // n)), shape=A.shape))


def expand_ordered(P, col_mask=None):
    """P.P as the sequential engines compute it (columns col_mask)."""
    return power(P, P, col_mask)


def expand_exact(P, col_mask=None, dense_from=64):
    """P.P (columns col_mask) in fp64.  Components of at least `dense_from` vertices are multiplied as dense blocks."""
    P = canon(P, np.float64)
    n = P.shape[0]
    _nc, lab = connected_components(P, directed=True, connection="weak")
    size = np.bincount(lab)
    want = np.ones(n, bool) if col_mask is None else np.asarray(col_mask, bool)
    big = size[lab] >= dense_from
    rows, cols, vals = [], [], []
    small_cols = want & ~big
    if small_cols.any():
        Ps = P @ sp.diags(small_cols.astype(np.float64))
        X = sp.coo_matrix(P @ Ps)
        rows.append(X.row), cols.append(X.col), vals.append(X.data)
    for comp in np.unique(lab[want & big]):
        S = np.nonzero(lab == comp)[0]
        D = P[S][:, S].toarray()
        X = D @ D
        rr, cc = np.nonzero(X)
        keep = want[S[cc]]
        rows.append(S[rr[keep]]), cols.append(S[cc[keep]]), vals.append(X[rr[keep], cc[keep]])
    if not rows:
        return sp.csc_matrix(P.shape, dtype=np.float64)
    return canon(sp.csc_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=P.shape),
                 np.float64)


# ---------------------------------------------------------------------------------------------------------------------------
# epilogue
# ---------------------------------------------------------------------------------------------------------------------------
def special_mode(r):
    """hh_inflate's multiplicative modes: the exponents (as fp32) evaluated with correctly rounded * and sqrt."""
    return {2.0: "sq", 1.5: "x15", 3.0: "cube", 2.5: "x25"}.get(float(np.float32(r)))


def inflate32(x, r):
    """hh_inflate in fp32: x*x, x*sqrt(x), (x*x)*x, (x*x)*sqrt(x) for r = 2, 1.5, 3, 2.5; np.power otherwise (the device
    uses powf there, which is only held to an ulp bound)."""
    x = np.asarray(x, np.float32)
    m = special_mode(r)
    if m == "sq":
        return x * x
    if m == "x15":
        return x * np.sqrt(x)
    if m == "cube":
        return (x * x) * x
    if m == "x25":
        return (x * x) * np.sqrt(x)
    return np.power(x, np.float32(r))


def _colsum_exact(v, indptr):
    """fp64-rounded exact column sums (math.fsum)."""
    lst = v.tolist()
    return np.array([math.fsum(lst[a:b]) for a, b in zip(indptr[:-1].tolist(), indptr[1:].tolist())], np.float64)


def _first_max(x, rows, indptr):
    """Per non-empty column: position of its first maximum (lowest row among ties), -1 for empty columns."""
    ncols = len(indptr) - 1
    col = np.repeat(np.arange(ncols), np.diff(indptr))
    order = np.lexsort((rows, -x.astype(np.float64), col))
    pos = np.full(ncols, -1, np.int64)
    nonempty = np.diff(indptr) > 0
    pos[nonempty] = order[indptr[:-1][nonempty]]
    return pos


def epilogue(X, r, pruning, s1=None, s2=None):
    """hh_k_col's E1-E3 on the product X (fp32 CSC): y = inflate32(x); S1 = exact fp64 column sum; x1 = fp32(y / S1);
    keep x1 >= fp32(pruning), else the first maximum (lowest row); S2 = exact sum of the kept x1; x2 = fp32(x1 / S2)
    (1.0 for a kept maximum).  s1 / s2 replace the column sums (the one-ulp recomputation of a single column).
    Returns (fp32 CSC result, dict of the intermediates)."""
    X = canon(X)
    n, ncols = X.shape
    y = inflate32(X.data, r)
    lens = np.diff(X.indptr)
    col = np.repeat(np.arange(ncols), lens)
    nz = y != 0
    y, rows, col = y[nz], X.indices[nz], col[nz]
    indptr = np.concatenate([[0], np.cumsum(np.bincount(col, minlength=ncols))])
    S1 = _colsum_exact(y.astype(np.float64), indptr) if s1 is None else np.asarray(s1, np.float64)
    S1c = S1[col]
    x1 = np.where(S1c != 0, (y.astype(np.float64) / np.where(S1c != 0, S1c, 1.0)), y).astype(np.float32)
    surv = (x1 >= np.float32(pruning)) & (x1 > 0)
    cnt = np.bincount(col[surv], minlength=ncols)
    fm = _first_max(x1, rows, indptr)
    need = (cnt == 0) & (fm >= 0)
    need[need] = x1[fm[need]] > 0
    keep = surv.copy()
    keep[fm[need]] = True
    kp = np.concatenate([[0], np.cumsum(np.bincount(col[keep], minlength=ncols))])
    S2 = _colsum_exact(x1[keep].astype(np.float64), kp) if s2 is None else np.asarray(s2, np.float64)
    S2[need] = x1[fm[need]].astype(np.float64)
    x2 = (x1[keep].astype(np.float64) / S2[col[keep]]).astype(np.float32)
    res = sp.csc_matrix((x2, rows[keep], kp), shape=(n, ncols))
    return res, {"S1": S1, "S2": S2, "need_max": need, "x1": x1, "rows": rows, "col": col, "indptr": indptr}


def delta(M, L):
    """max(|M - L| - 1e-5 |L|) over the union pattern in non-contracted fp32, floored at 0 (hh_k_col's E4/E5 and
    oracle.convergence_delta)."""
    M, L = canon(M), canon(L)
    n = M.shape[0]

    def keys(A):
        return np.repeat(np.arange(A.shape[1], dtype=np.int64), np.diff(A.indptr)) * n + A.indices

    km, kl = keys(M), keys(L)
    ku = np.union1d(km, kl)
    m = np.zeros(len(ku), np.float32)
    l = np.zeros(len(ku), np.float32)
    m[np.searchsorted(ku, km)] = M.data
    l[np.searchsorted(ku, kl)] = L.data
    d = np.abs(m - l) - np.float32(1e-5) * np.abs(l)
    return np.float32(max(np.float32(0), d.max(initial=np.float32(0))))


# ---------------------------------------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------------------------------------
def columns_equal(A, B):
    """Per column: True where the two fp32 CSC matrices hold bit-identical columns."""
    A, B = canon(A), canon(B)
    ncols = A.shape[1]
    la, lb = np.diff(A.indptr), np.diff(B.indptr)
    eq = la == lb
    ca = np.repeat(np.arange(ncols), la)
    cb = np.repeat(np.arange(ncols), lb)
    bad = np.zeros(ncols, bool)
    both = eq[ca]
    # columns of equal length: compare entry by entry (same positions in both arrays after the length check)
    ia = np.nonzero(both)[0]
    ib = np.nonzero(eq[cb])[0]
    diff = (A.indices[ia] != B.indices[ib]) | (A.data[ia].view(np.uint32) != B.data[ib].view(np.uint32))
    bad[ca[ia][diff]] = True
    return eq & ~bad


def exact_bit_check(dev, X, r, pruning, col_mask=None):
    """The device iterate `dev` against epilogue(X) (columns col_mask).  Columns that differ are recomputed with S1
    and/or S2 moved by one fp64 ulp; returns (columns that still differ, columns explained by a one-ulp sum)."""
    want, im = epilogue(X, r, pruning)
    ok = columns_equal(dev, want)
    if col_mask is not None:
        ok |= ~np.asarray(col_mask, bool)
    bad = np.nonzero(~ok)[0]
    one_ulp, still = [], []
    if len(bad):
        D = canon(dev)
        for j in bad.tolist():
            xj = X[:, [j]]
            hit = False
            s1 = im["S1"][j]
            for a in (s1, np.nextafter(s1, 0), np.nextafter(s1, np.inf)):
                _r, im2 = epilogue(xj, r, pruning, s1=[a])
                s2 = im2["S2"][0]
                for b in (s2, np.nextafter(s2, 0), np.nextafter(s2, np.inf)):
                    got, _ = epilogue(xj, r, pruning, s1=[a], s2=[b])
                    if columns_equal(D[:, [j]], got)[0]:
                        hit = True
                        break
                if hit:
                    break
            (one_ulp if hit else still).append(j)
    return still, one_ulp


def band_check(dev, X64, r, pruning, e_y, col_mask=None):
    """The device iterate `dev` against the exact epilogue of the fp64 product X64, given a relative error bound e_y on
    the inflated values y = x^r.  Returns a dict:
      pattern_bad   kept / dropped entries of the device outside the borderline band |x1/pruning - 1| <= 2 e_y
      max_bad       need-max columns whose kept row is not within the band of the column maximum
      x2_err        largest |x2_dev - x2| / x2 on the device's pattern, x2 = x1 / (sum of the exact x1 the device kept)
      x2_bar        2 e_y + 2^-22."""
    X = canon(X64, np.float64)
    D = canon(dev)
    n, ncols = X.shape
    cols = np.arange(ncols) if col_mask is None else np.nonzero(col_mask)[0]
    band = 2.0 * e_y
    pattern_bad = max_bad = 0
    worst = 0.0
    for j in cols.tolist():
        a0, a1 = X.indptr[j], X.indptr[j + 1]
        rows = X.indices[a0:a1]
        y = X.data[a0:a1] ** float(np.float32(r))
        S1 = y.sum()
        x1 = y / S1 if S1 != 0 else y
        d0, d1 = D.indptr[j], D.indptr[j + 1]
        drows, dvals = D.indices[d0:d1], D.data[d0:d1].astype(np.float64)
        pos = np.searchsorted(rows, drows)
        if np.any(pos >= len(rows)) or np.any(rows[np.minimum(pos, len(rows) - 1)] != drows):
            pattern_bad += 1                          # a kept row the exact product does not have
            continue
        kept = np.zeros(len(rows), bool)
        kept[pos] = True
        exact_keep = x1 >= pruning
        border = np.abs(x1 / pruning - 1.0) <= band
        diff = kept != exact_keep
        if np.any(diff & ~border):
            # the one legitimate non-borderline difference: a column without (non-borderline) survivors keeps its maximum
            need_max = len(drows) == 1 and not np.any(exact_keep & ~border)
            if not need_max:
                pattern_bad += 1
                continue
            if x1[pos[0]] < x1.max() * (1.0 - band):
                max_bad += 1
        S2 = x1[kept].sum()
        x2 = x1[pos] / S2
        worst = max(worst, float(np.max(np.abs(dvals - x2) / x2)))
    return {"pattern_bad": pattern_bad, "max_bad": max_bad, "x2_err": worst, "x2_bar": band + 2.0 ** -22}
