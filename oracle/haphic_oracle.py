"""CPU oracle for the `haphic cluster` hot path -- TEST INFRASTRUCTURE, NOT PRODUCT.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` legs may import this module.  The product path
(``haphic_b200``) never does and fails loudly when the CUDA library is missing.

This is a restatement (numpy / scipy.sparse primitives / plain Python loops) of
the algorithm in the reference ``scripts/HapHiC_cluster.py`` (zengxiaofei/HapHiC
v1.0.7).  Every function cites the reference lines it follows.  The reference
is Python and cannot travel to the GPU box, so parity is PINNED by the golden
fixtures in ``tests/golden/*.npz`` that ``tests/golden/make_golden.py`` produced
by running the unmodified reference in the build container
(``tests/test_oracle_golden.py`` checks this module against every one of them).

Third-party arithmetic restated here because it is not under /root/reference:
* scikit-learn 1.5.1 ``preprocessing.normalize(norm='l1', axis=0)`` on CSC input
  = per column an fp64 sum accumulated sequentially in stored order, then
  ``x = float32(float64(x) / sum)``; all-zero columns untouched
  (sklearn/utils/sparsefuncs_fast.pyx ``inplace_csr_row_normalize_l1``).
* sparse_dot_mkl 0.9.4 / Intel MKL 2024.2 ``dot_product_mkl`` = fp32 CSC x CSC
  SpGEMM, accumulation order unspecified; restated as Gustavson column products
  accumulated in fp32 (``scipy.sparse`` ``@``, which is what the golden fixtures
  used as the MKL stand-in).

Contig names are replaced by integer ids throughout; where the reference orders
by name (Python ``str`` comparison, HapHiC_cluster.py:1629) the caller passes
``name_rank`` (rank of each contig id under that ordering).
"""

from __future__ import annotations

from collections import OrderedDict
from decimal import Decimal

import numpy as np
import scipy.sparse as sp


# --------------------------------------------------------------------------------------
# link counting  (HapHiC_cluster.py:1596-1655, 299-307, 395-416)
# --------------------------------------------------------------------------------------

def is_flank(coord: int, length: int, flank: int) -> bool:
    """HapHiC_cluster.py:299-307 -- 1-based ``coord``; ``flank`` in bp (0 = whole contig)."""
    if flank and (coord <= flank or coord > length - flank):
        return True
    return not flank


def count_links_loop(pairs, lengths, name_rank, in_nx, flank_bp):
    """One Python iteration per read pair, as the reference does (1622-1653).

    pairs: int array [P,4] (ctg_a, pos_a, ctg_b, pos_b), 0-based positions; ids outside
    [0, n) stand for names missing from the FASTA (skipped, 1625); a == b is dropped by
    the generator before the loop (1582).
    Returns insertion-ordered dicts keyed by id tuples:
      full {(i,j): n}, flank {(i,j): n}, HT {(i,ti,j,tj): n}, clm {(i,j): [4 distances per link]},
      ctg_links {i: n}.
    """
    n = len(lengths)
    full, flank_d, HT, clm, ctg_links = OrderedDict(), OrderedDict(), OrderedDict(), OrderedDict(), OrderedDict()
    for a, pa, b, pb in np.asarray(pairs).tolist():
        if a == b:                                   # pairs_generator_inter_ctgs, 1582
            continue
        if not (0 <= a < n and 0 <= b < n):          # 1625
            continue
        # sorted(((ref, pos+1), (mref, mpos+1))) by name (1629)
        if name_rank[a] < name_rank[b]:
            i, ci, j, cj = a, pa + 1, b, pb + 1
        else:
            i, ci, j, cj = b, pb + 1, a, pa + 1
        li, lj = int(lengths[i]), int(lengths[j])
        key = (i, j)
        if in_nx[i] and in_nx[j] and is_flank(ci, li, flank_bp) and is_flank(cj, lj, flank_bp):   # 1636-1639
            flank_d[key] = flank_d.get(key, 0) + 1
            ctg_links[i] = ctg_links.get(i, 0) + 1
            ctg_links[j] = ctg_links.get(j, 0) + 1
        a0, b0 = ci - 1, cj - 1                       # update_clm_dict, 395-401
        clm.setdefault(key, []).extend((li - a0 + b0, li - a0 + lj - b0, a0 + b0, a0 + lj - b0))
        ti, tj = int(ci * 2 > li), int(cj * 2 > lj)   # update_HT_link_dict, 404-416
        hk = (i, ti, j, tj)
        HT[hk] = HT.get(hk, 0) + 1
        full[key] = full.get(key, 0) + 1              # 1649
    return full, flank_d, HT, clm, ctg_links


def build_c(force=False):
    """gcc-compile oracle/haphic_oracle.c into oracle/_build/ (git-ignored) and return the ctypes library."""
    import ctypes
    import os
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    src = os.path.join(here, "haphic_oracle.c")
    out_dir = os.path.join(here, "_build")
    lib = os.path.join(out_dir, "libhaphic_oracle.so")
    if force or not os.path.exists(lib) or os.path.getmtime(lib) < os.path.getmtime(src):
        os.makedirs(out_dir, exist_ok=True)
        subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-o", lib, src], check=True)
    cdll = ctypes.CDLL(lib)
    cdll.hho_count_links.restype = ctypes.c_int64
    return cdll


def count_links_c(pairs, lengths, name_rank, in_nx, flank_bp, cap=None):
    """The same loop in plain C (oracle/haphic_oracle.c): single core, hash table, entries in first-seen order.
    Returns the arrays of count_links_numpy that do not involve the clm distances."""
    import ctypes as C
    lib = build_c()
    rec = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 4)
    n = len(lengths)
    lengths = np.ascontiguousarray(lengths, dtype=np.int64)
    name_rank = np.ascontiguousarray(name_rank, dtype=np.int32)
    in_nx = np.ascontiguousarray(in_nx, dtype=np.uint8)
    cap = int(cap if cap is not None else max(16, min(len(rec), n * (n - 1) // 2)))
    ki, kj = np.empty(cap, np.int32), np.empty(cap, np.int32)
    full, flank = np.empty(cap, np.int64), np.empty(cap, np.int64)
    ff, fl = np.empty(cap, np.int64), np.empty(cap, np.int64)
    ht = np.empty((cap, 4), np.int64)
    tot = np.empty(n, np.int64)
    used = C.c_int64()
    p = lambda x: x.ctypes.data_as(C.c_void_p)       # noqa: E731
    nnz = lib.hho_count_links(p(rec), C.c_int64(len(rec)), C.c_int32(n), p(lengths), p(name_rank), p(in_nx), C.c_int64(flank_bp),
                              C.c_int64(cap), p(ki), p(kj), p(full), p(flank), p(ff), p(fl), p(ht), p(tot), C.byref(used))
    if nnz < 0:
        raise MemoryError("count_links_c: more than {} contig pairs".format(cap))
    ki, kj, full, flank, ff, fl, ht = ki[:nnz], kj[:nnz], full[:nnz], flank[:nnz], ff[:nnz], fl[:nnz], ht[:nnz]
    sel = np.nonzero(flank > 0)[0]
    sel = sel[np.argsort(fl[sel], kind="stable")]
    return {"n_used": int(used.value), "full_keys": np.stack([ki, kj], 1), "full_vals": full, "full_first": ff,
            "flank_keys": np.stack([ki[sel], kj[sel]], 1), "flank_vals": flank[sel], "flank_first": fl[sel],
            "ht": ht, "ctg_link_total": tot}


# --------------------------------------------------------------------------------------
# fragment mode: contigs longer than bin_size split into bins  (HapHiC_cluster.py:1658-1752, 188-296)
# --------------------------------------------------------------------------------------

def frag_records(pairs, frag_base, bin_size):
    """parse_alignments' record handling (1696-1723) as a mapping of contig records into fragment space, after which
    fragment-mode counting is contig-mode counting (count_links_* over fragment lengths / name ranks / Nx).

    pairs: int [P, 4] (ctg_a, pos_a, ctg_b, pos_b), 0-based positions, ids of SOURCE contigs; frag_base [n_src + 1]:
    contig c owns fragment ids [frag_base[c], frag_base[c+1]), more than one = split into bins of bin_size bp.
    An end on a split contig at pos goes to bin k = ceil((pos + 1) / bin_size) (convert_frags, 1662-1670): fragment
    frag_base[c] + k - 1 at position pos - (k - 1) * bin_size.  Rows are kept, so stream indices stay:
      * ids outside [0, n_src) -> (-1, ., -1, .): skipped (1703);
      * an intra-contig record whose ends share a bin number -> a == b: skipped (1699 / 1715), whether the bin exists or not;
      * otherwise a bin outside 1..nbins -> (-1, ., -1, .) and REFUSED: the reference raises a KeyError (1723).
    Returns (mapped int32 [P, 4], n_refused, stream indices of the refused records)."""
    pairs = np.asarray(pairs).reshape(-1, 4)
    step = 1 << 24                                     # int64 temporaries of 16 Mi records at a time
    if len(pairs) > step:
        out = np.empty((len(pairs), 4), np.int32)
        bad = []
        for lo in range(0, len(pairs), step):
            out[lo:lo + step], _, b = frag_records(pairs[lo:lo + step], frag_base, bin_size)
            bad.append(b + lo)
        bad = np.concatenate(bad)
        return out, len(bad), bad
    p = pairs.astype(np.int64)
    fb = np.asarray(frag_base, dtype=np.int64)
    n_src = len(fb) - 1
    a, pa, b, pb = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
    ok = (a >= 0) & (a < n_src) & (b >= 0) & (b < n_src)
    a0, b0 = np.where(ok, a, 0), np.where(ok, b, 0)

    def to_frag(c, pos):
        nb = fb[c + 1] - fb[c]
        k = -(-(pos + 1) // bin_size)                  # Python ceil: floor division, so any int32 position agrees
        split = nb > 1
        missing = split & ((k < 1) | (k > nb))
        return np.where(split, fb[c] + k - 1, fb[c]), np.where(split, pos - (k - 1) * bin_size, pos), missing, k

    fa, qa, miss_a, ka = to_frag(a0, pa)
    fbb, qb, miss_b, kb = to_frag(b0, pb)
    same_bin = ok & (a0 == b0) & (ka == kb)
    refused = ok & (miss_a | miss_b) & ~same_bin
    fa = np.where(same_bin, fb[a0], fa)
    fbb = np.where(same_bin, fb[a0], fbb)
    use = ok & ~refused
    out = np.stack([np.where(use, fa, -1), np.where(use, qa, 0), np.where(use, fbb, -1), np.where(use, qb, 0)], 1)
    bad = np.nonzero(refused)[0]
    return out.astype(np.int32), len(bad), bad


def count_frag_links_c(pairs, frag_base, bin_size, frag_len, frag_rank, frag_in_nx, flank_bp, cap=None):
    """Every field of a fragment-mode table: count_links_c over frag_records.  Returns count_links_c's dict plus
    "mapped", "n_refused" and "refused" (stream indices)."""
    mapped, n_bad, bad = frag_records(pairs, frag_base, bin_size)
    ref = count_links_c(mapped, frag_len, frag_rank, frag_in_nx, flank_bp, cap=cap)
    ref.update(mapped=mapped, n_refused=n_bad, refused=bad)
    return ref


def count_frag_links_loop(pairs, names, lengths, bin_size, nx_frags, flank_bp):
    """One Python iteration per record of parse_alignments (1696-1733) on name strings, with the reference's tuple sorts
    and its fragment layout (stat_fragments, 228-264: contigs longer than bin_size split into '{ctg}_bin{k}').  For small
    inputs; independent of frag_records.

    pairs: int [P, 4] of contig ids into ``names`` (ids outside stand for names missing from the FASTA); nx_frags: the
    set of Nx fragment names.  A record that would raise a KeyError in the reference (1723) is noted and skipped.
    Returns a dict of insertion-ordered dicts keyed by names: "flank" {(frag_i, frag_j): n}, "frag_links" {frag: n},
    "full" {(ctg_i, ctg_j): n} and "HT" {(ctg_i_H/T, ctg_j_H/T): n} (inter-contig records only, 1736-1746),
    "ctg_pair_to_frag" {(ctg_i, ctg_j): {(frag_i, frag_j)}}, plus "frag_len" {frag: length} and "raises" (stream
    indices of the records that would raise; the first is where the reference stops)."""
    fa_dict = {n: int(ln) for n, ln in zip(names, np.asarray(lengths).tolist())}
    split = {n for n, ln in fa_dict.items() if ln > bin_size}
    frag_len = OrderedDict()
    for n, ln in fa_dict.items():
        if n in split:
            nbins = -(-ln // bin_size)
            for m in range(nbins):
                frag_len["{}_bin{}".format(n, m + 1)] = bin_size if m + 1 < nbins else ln - m * bin_size
        else:
            frag_len[n] = ln

    def convert(ctg, coord):                                   # 1662-1670
        if ctg in split:
            k = -(-coord // bin_size)
            return "{}_bin{}".format(ctg, k), coord - (k - 1) * bin_size, True
        return ctg, coord, False

    full, flank_d, HT, frag_links, c2f = OrderedDict(), OrderedDict(), OrderedDict(), OrderedDict(), OrderedDict()
    raises = []
    n = len(names)
    for r, (a, pa, b, pb) in enumerate(np.asarray(pairs).reshape(-1, 4).tolist()):
        ref = names[a] if 0 <= a < n else None
        mref = names[b] if 0 <= b < n else None
        if ref == mref and ref not in split:                  # 1699
            continue
        if ref is None or mref is None:                        # 1703
            continue
        (ctg_i, coord_i), (ctg_j, coord_j) = sorted(((ref, pa + 1), (mref, pb + 1)))     # 1707
        frag_i, fc_i, i_bin = convert(ctg_i, coord_i)
        frag_j, fc_j, j_bin = convert(ctg_j, coord_j)
        if frag_i == frag_j:                                   # 1715
            continue
        if i_bin or j_bin:                                     # 1719-1720
            (frag_i, fc_i), (frag_j, fc_j) = sorted(((frag_i, fc_i), (frag_j, fc_j)))
        if frag_i not in frag_len or frag_j not in frag_len:  # 1723: KeyError
            raises.append(r)
            continue
        key = (frag_i, frag_j)
        if frag_i in nx_frags and frag_j in nx_frags and is_flank(fc_i, frag_len[frag_i], flank_bp) and \
                is_flank(fc_j, frag_len[frag_j], flank_bp):   # 1726-1729
            flank_d[key] = flank_d.get(key, 0) + 1
            frag_links[frag_i] = frag_links.get(frag_i, 0) + 1
            frag_links[frag_j] = frag_links.get(frag_j, 0) + 1
        c2f.setdefault((ctg_i, ctg_j), set()).add(key)         # 1732-1733
        if ref != mref:                                        # 1736-1746
            full[(ctg_i, ctg_j)] = full.get((ctg_i, ctg_j), 0) + 1
            li, lj = fa_dict[ctg_i], fa_dict[ctg_j]
            hk = (ctg_i + ("_T" if coord_i * 2 > li else "_H"), ctg_j + ("_T" if coord_j * 2 > lj else "_H"))
            HT[hk] = HT.get(hk, 0) + 1
    return {"flank": flank_d, "frag_links": frag_links, "full": full, "HT": HT, "ctg_pair_to_frag": c2f,
            "frag_len": frag_len, "raises": raises}


def count_links_numpy(pairs, lengths, name_rank, in_nx, flank_bp, with_clm=True):
    """Vectorised restatement of the same loop; identical outputs as arrays.

    Returns a dict of arrays; every *_keys array is in dict-insertion (first-seen) order.
    """
    p = np.asarray(pairs, dtype=np.int64)
    n = len(lengths)
    lengths = np.asarray(lengths, dtype=np.int64)
    name_rank = np.asarray(name_rank, dtype=np.int64)
    in_nx = np.asarray(in_nx).astype(bool)
    a, pa, b, pb = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
    ok = (a != b) & (a >= 0) & (a < n) & (b >= 0) & (b < n)
    idx = np.nonzero(ok)[0]
    a, pa, b, pb = a[idx], pa[idx], b[idx], pb[idx]
    swap = name_rank[a] > name_rank[b]
    i = np.where(swap, b, a)
    j = np.where(swap, a, b)
    ci = np.where(swap, pb, pa) + 1
    cj = np.where(swap, pa, pb) + 1
    li, lj = lengths[i], lengths[j]

    def flank_ok(c, ln):
        if not flank_bp:
            return np.ones(len(c), dtype=bool)
        return (c <= flank_bp) | (c > ln - flank_bp)

    fl = in_nx[i] & in_nx[j] & flank_ok(ci, li) & flank_ok(cj, lj)
    key = i * n + j

    def first_seen_unique(k, stream):
        u, first, cnt = np.unique(k, return_index=True, return_counts=True)
        order = np.argsort(stream[first], kind="stable")
        return u[order], stream[first][order], cnt[order]

    fk, f_first, f_cnt = first_seen_unique(key, idx)
    lk, l_first, l_cnt = first_seen_unique(key[fl], idx[fl])
    ti = (ci * 2 > li).astype(np.int64)
    tj = (cj * 2 > lj).astype(np.int64)
    hk, _h_first, h_cnt = first_seen_unique(key * 4 + ti * 2 + tj, idx)
    # per-fragment totals (ctg_link_dict); insertion order = first touch, i before j
    tot = np.bincount(i[fl], minlength=n) + np.bincount(j[fl], minlength=n)
    touch = np.full(n, np.iinfo(np.int64).max)
    np.minimum.at(touch, i[fl], idx[fl] * 2)
    np.minimum.at(touch, j[fl], idx[fl] * 2 + 1)
    touched = np.nonzero(tot > 0)[0]
    touched = touched[np.argsort(touch[touched], kind="stable")]
    if not with_clm:      # the per-pair Python loop below is for fixture sizes; at BASELINE sizes only the counters are compared
        return {
            "n_used": len(idx),
            "full_keys": np.stack([fk // n, fk % n], axis=1).astype(np.int32), "full_vals": f_cnt.astype(np.int64),
            "full_first": f_first,
            "flank_keys": np.stack([lk // n, lk % n], axis=1).astype(np.int32), "flank_vals": l_cnt.astype(np.int64),
            "flank_first": l_first,
            "HT_keys": np.stack([(hk // 4) // n, (hk % 4) // 2, (hk // 4) % n, hk % 2], axis=1).astype(np.int32),
            "HT_vals": h_cnt.astype(np.int64),
            "ctg_link_ids": touched.astype(np.int32), "ctg_link_vals": tot[touched].astype(np.int64),
            "ctg_link_total": tot.astype(np.int64),
        }
    # clm: per key, distances in stream order (4 per link)
    a0, b0 = ci - 1, cj - 1
    dist = np.stack([li - a0 + b0, li - a0 + lj - b0, a0 + b0, a0 + lj - b0], axis=1)
    srt = np.argsort(key, kind="stable")
    ukey, start = np.unique(key[srt], return_index=True)
    # re-order segments into first-seen order
    seg_first = idx[srt][start]
    seg_order = np.argsort(seg_first, kind="stable")
    seg_len = np.diff(np.append(start, len(srt)))
    clm_vals, clm_off = [], [0]
    for s in seg_order.tolist():
        rows = srt[start[s]:start[s] + seg_len[s]]
        clm_vals.append(dist[rows].reshape(-1))
        clm_off.append(clm_off[-1] + 4 * len(rows))
    return {
        "n_used": len(idx),
        "full_keys": np.stack([fk // n, fk % n], axis=1).astype(np.int32), "full_vals": f_cnt.astype(np.int64),
        "full_first": f_first,
        "flank_keys": np.stack([lk // n, lk % n], axis=1).astype(np.int32), "flank_vals": l_cnt.astype(np.int64),
        "flank_first": l_first,
        "HT_keys": np.stack([(hk // 4) // n, (hk % 4) // 2, (hk // 4) % n, hk % 2], axis=1).astype(np.int32),
        "HT_vals": h_cnt.astype(np.int64),
        "ctg_link_ids": touched.astype(np.int32), "ctg_link_vals": tot[touched].astype(np.int64),
        "ctg_link_total": tot.astype(np.int64),
        "clm_keys": np.stack([ukey[seg_order] // n, ukey[seg_order] % n], axis=1).astype(np.int32),
        "clm_offsets": np.asarray(clm_off, dtype=np.int64),
        "clm_vals": (np.concatenate(clm_vals) if clm_vals else np.zeros(0, np.int64)).astype(np.int64),
    }


def clm_text(clm_keys, clm_offsets, clm_vals, names):
    """output_clm, HapHiC_cluster.py:376-392: pairs with >= 2 links, 4 orientation lines each,
    sorted distances each printed twice, count doubled."""
    ori = (("+", "+"), ("+", "-"), ("-", "+"), ("-", "-"))
    out = []
    for (i, j), s, e in zip(np.asarray(clm_keys).tolist(), clm_offsets[:-1].tolist(), clm_offsets[1:].tolist()):
        lst = clm_vals[s:e]
        if len(lst) < 8:
            continue
        for k in range(4):
            d = np.sort(lst[k::4]).tolist()
            out.append("{}{} {}{}\t{}\t{}\n".format(names[i], ori[k][0], names[j], ori[k][1], len(d) * 2,
                                                     " ".join("{0} {0}".format(v) for v in d)))
    return "".join(out)


def normalize_by_nlinks(flank_keys, flank_vals, ctg_link_total):
    """HapHiC_cluster.py:718-724: links / sqrt(tot_i * tot_j) in Python float (fp64)."""
    k = np.asarray(flank_keys, dtype=np.int64)
    t = np.asarray(ctg_link_total, dtype=np.int64)
    prod = (t[k[:, 0]] * t[k[:, 1]]).astype(object)         # exact Python ints, as the reference
    return np.array([float(v) / (int(q) ** 0.5) for v, q in zip(np.asarray(flank_vals).tolist(), prod.tolist())],
                    dtype=np.float64)


# --------------------------------------------------------------------------------------
# dict -> matrix  (HapHiC_cluster.py:310-373)
# --------------------------------------------------------------------------------------

def assign_matrix_index(flank_keys, keep, tail_order=None):
    """First-seen index assignment (327-349) over the flank dict restricted to ``keep``;
    kept-but-unlinked fragments follow (355-359) in ``tail_order`` (the reference uses set
    iteration order there; ascending id when not given).  Returns int32 [n], -1 = not in matrix."""
    keep = np.asarray(keep).astype(bool)
    n = len(keep)
    index = np.full(n, -1, dtype=np.int32)
    nxt = 0
    for i, j in np.asarray(flank_keys).tolist():
        if not (keep[i] and keep[j]):
            continue
        if index[i] < 0:
            index[i] = nxt
            nxt += 1
        if index[j] < 0:
            index[j] = nxt
            nxt += 1
    rest = [f for f in (tail_order if tail_order is not None else range(n)) if keep[f] and index[f] < 0]
    for f in rest:
        index[f] = nxt
        nxt += 1
    assert nxt == int(keep.sum())
    return index


def dict_to_matrix(flank_keys, flank_vals, keep, tail_order=None, add_self_loops=True):
    """Symmetric fp32 CSC with self loops = 1 on raw values (351-371)."""
    index = assign_matrix_index(flank_keys, keep, tail_order)
    k = np.asarray(flank_keys, dtype=np.int64).reshape(-1, 2)
    sel = (index[k[:, 0]] >= 0) & (index[k[:, 1]] >= 0)
    r, c = index[k[sel, 0]], index[k[sel, 1]]
    v = np.asarray(flank_vals)[sel]
    shape = int((index >= 0).sum())
    rows = np.concatenate([r, c] + ([np.arange(shape)] if add_self_loops else []))
    cols = np.concatenate([c, r] + ([np.arange(shape)] if add_self_loops else []))
    data = np.concatenate([v, v] + ([np.ones(shape)] if add_self_loops else []))
    m = sp.coo_matrix((data, (rows, cols)), shape=(shape, shape), dtype=np.float32).tocsc()
    m.sort_indices()
    return m, index


# --------------------------------------------------------------------------------------
# Markov clustering  (HapHiC_cluster.py:1987-2095, 2132-2242)
# --------------------------------------------------------------------------------------

def col_normalize_l1(m: sp.csc_matrix) -> sp.csc_matrix:
    """sklearn normalize(norm='l1', axis=0) on CSC: sequential fp64 column sums in stored
    order (np.bincount accumulates sequentially in fp64), x = fp32(fp64(x)/sum); zero columns kept."""
    m = sp.csc_matrix(m, dtype=np.float32, copy=True)
    n = m.shape[1]
    col = np.repeat(np.arange(n), np.diff(m.indptr))
    s = np.bincount(col, weights=np.abs(m.data).astype(np.float64), minlength=n)
    d = s[col]
    nz = d != 0
    out = m.data.astype(np.float64)
    out[nz] = out[nz] / d[nz]
    m.data = out.astype(np.float32)
    return m


def expand(m: sp.csc_matrix, expansion: int) -> sp.csc_matrix:
    """mkl_matrix_power (2017-2023): A . A^(e-1), fp32 SpGEMM."""
    r = m
    for _ in range(expansion - 1):
        r = sp.csc_matrix(m @ r, dtype=np.float32)
    return r


def inflate(m: sp.csc_matrix, inflation: float) -> sp.csc_matrix:
    """matrix.power(r) in fp32 then column L1 normalise (2038)."""
    m = sp.csc_matrix(m, dtype=np.float32, copy=True)
    # fp32 array ** Python float: numpy computes in fp32 with the exponent cast to fp32
    m.data = np.power(m.data, np.float32(inflation))
    return col_normalize_l1(m)


def prune(m: sp.csc_matrix, pruning: float) -> sp.csc_matrix:
    """prune (1987-2014): keep x >= pruning, re-insert each column's FIRST maximum (lowest
    row among ties, scipy argmax on sorted indices), then column L1 normalise."""
    m = sp.csc_matrix(m, dtype=np.float32, copy=True)
    m.sort_indices()
    n = m.shape[1]
    keep = m.data >= pruning
    lens = np.diff(m.indptr)
    for jcol in np.nonzero(lens)[0].tolist():
        s, e = m.indptr[jcol], m.indptr[jcol + 1]
        d = m.data[s:e]
        am = int(np.argmax(d))                # first maximum in row order
        if d[am] > 0:
            keep[s + am] = True
    col = np.repeat(np.arange(n), lens)
    out = sp.csc_matrix((m.data[keep], (m.indices[keep], col[keep])), shape=m.shape, dtype=np.float32)
    out.sort_indices()
    return col_normalize_l1(out)


def convergence_delta(m: sp.csc_matrix, last: sp.csc_matrix) -> float:
    """max(|M - L| - 1e-5*|L|) with implicit zeros taking part (2044-2046), fp32 arithmetic."""
    d = abs(m - last) - np.float32(1e-5) * abs(last)
    d = sp.csc_matrix(d)
    mx = float(d.data.max()) if d.nnz else 0.0
    if d.nnz < d.shape[0] * d.shape[1]:
        mx = max(mx, 0.0)
    return mx


def mcl(m1: sp.csc_matrix, expansion: int, inflation: float, iters: int, pruning: float, trace=None):
    """mcl (2026-2062).  Returns (matrix, n_rounds, converged).  ``trace`` (list) receives each
    iteration's pruned matrix."""
    matrix = m1
    last = None
    n_done = 0
    for n in range(iters):
        if n != 0:
            matrix = expand(matrix, expansion)
        matrix = inflate(matrix, inflation)
        matrix = prune(matrix, pruning)
        n_done = n + 1
        if trace is not None:
            trace.append(matrix.copy())
        if n > 1 and convergence_delta(matrix, last) <= 1e-8:
            return matrix, n_done, True
        last = matrix.copy()
    return matrix, n_done, False


def interpret_result(result: sp.csc_matrix):
    """interpret_result (2065-2095): attractor rows with non-zero diagonal; their non-zero
    columns form a cluster; None if any node is in two clusters or in none."""
    r = sp.csr_matrix(result)
    r.eliminate_zeros()
    r.sort_indices()
    shape = r.shape[0]
    attractors = np.nonzero(r.diagonal())[0]
    clusters = set()
    for a in attractors.tolist():
        clusters.add(tuple(r.indices[r.indptr[a]:r.indptr[a + 1]].tolist()))
    nodes = set()
    for c in clusters:
        for v in c:
            if v in nodes:
                return None
            nodes.add(v)
    if len(nodes) != shape:
        return None
    return list(clusters)


def inflation_sweep(min_inflation, max_inflation, step):
    """arange over Decimals (2139-2141, 2155): returns the list of Decimal inflations."""
    start = Decimal(str(min_inflation))
    st = Decimal(str(step))
    end = Decimal(str(max_inflation)) + st
    return list(np.arange(start, end, st))


def run_mcl_sweep(link_matrix, expansion, inflations, max_iter, pruning):
    """run_mcl_clustering's numeric part (2144-2162): normalise, pre-expand, sweep.
    Returns list of (inflation, final matrix, rounds, converged, clusters-or-None)."""
    m0 = col_normalize_l1(sp.csc_matrix(link_matrix, dtype=np.float32))
    m1 = expand(m0, expansion)
    out = []
    for r in inflations:
        fin, rounds, conv = mcl(m1, expansion, float(r), max_iter, pruning)
        out.append((r, fin, rounds, conv, interpret_result(fin)))
    return out


def labels_from_clusters(clusters, n):
    lab = np.full(n, -1, dtype=np.int32)
    for c in clusters:
        lab[list(c)] = min(c)
    return lab
