"""numpy restatement of the per-record / per-bin parts of assembly correction (scripts/HapHiC_cluster.py v1.0.7), used by
the tests at sizes the reference cannot reach and checked itself against the reference's own results
(tests/golden/correct_*.npz)."""

import numpy as np


def pyslice(i, n):
    """A numpy slice bound on an array of n elements: negative counts from the end; clamped to [0, n]."""
    i = np.asarray(i, np.int64)
    return np.where(i < 0, np.maximum(i + n, 0), np.minimum(i, n))


def coverage(records, lengths, res):
    """parse_pairs_for_correction (1321-1342): {contig id: int32 coverage of len//res + 1 bins} and the same-contig links
    {contig id: int [m, 2] (lo, hi)}.  `cov[lo//res : hi//res + 1] += 1`, bins past the end dropped (numpy slicing)."""
    rec = np.asarray(records, np.int64)
    n = len(lengths)
    same = (rec[:, 0] == rec[:, 2]) & (rec[:, 0] >= 0) & (rec[:, 0] < n)
    r = rec[same]
    lo, hi = np.minimum(r[:, 1], r[:, 3]), np.maximum(r[:, 1], r[:, 3])
    cov, links = {}, {}
    order = np.argsort(r[:, 0], kind="stable")
    cuts = np.searchsorted(r[order, 0], np.arange(n + 1))
    for c in range(n):
        nb = int(lengths[c]) // res + 1
        sel = order[cuts[c]:cuts[c + 1]]
        s = pyslice(lo[sel] // res, nb)
        e = pyslice(hi[sel] // res + 1, nb)
        d = np.zeros(nb + 1, np.int64)
        ok = s < e
        np.add.at(d, s[ok], 1)
        np.add.at(d, e[ok], -1)
        cov[c] = np.cumsum(d[:-1]).astype(np.int32)
        links[c] = np.stack([lo[sel], hi[sel]], axis=1)
    return cov, links


def detect(cov, frag_len, res, median_cov_ratio=0.2, region_len_ratio=0.1, min_region_cutoff=5000):
    """detect_break_points (943-1014) for one fragment: [(position, coverage)] relative to the fragment."""
    cov = np.asarray(cov)
    m = np.median(cov)
    if not m:
        return []
    high = (cov >= m * median_cov_ratio).astype(np.int8)
    d = np.diff(np.concatenate([[0], high, [0]]))
    starts, ends = np.nonzero(d == 1)[0], np.nonzero(d == -1)[0]      # runs of high bins [start, end)
    if len(starts) < 2:
        return []
    large = (ends - starts) * res >= max(min_region_cutoff, frag_len * region_len_ratio)
    ls, le = starts[large], ends[large]
    if len(ls) < 2:
        return []
    cands = []
    for k in range(len(ls) - 1):
        v = cov[le[k]:ls[k + 1]]
        z = np.nonzero(v == 0)[0]
        if len(z):
            cands.append((int(le[k] + z[0]), 0))
        else:
            j = int(np.argmin(v))
            cands.append((int(le[k] + j), int(v[j])))
    if any(c == 0 for _, c in cands):
        return [(b * res, 0) for b, c in cands if c == 0]
    b, c = min(cands, key=lambda x: x[1])         # first of the smallest: the stable sort of 1008
    return [(b * res, c)]


def correct_rounds(records, lengths, res, nrounds, median_cov_ratio=0.2, region_len_ratio=0.1, min_region_cutoff=5000):
    """Items 1-3 of correct_assembly (1200-1243) without the names: every round's examined coverage arrays (dict order)
    and breakpoints [(position in that list, [(position, coverage)])].  After a round that is not the last, break_and_update_ctgs
    (1063-1113, 1151-1153, 1176-1178): links spanning a non-zero breakpoint are subtracted from the parent's coverage and
    dropped; the others move to the piece holding both ends (pos_shift), except that a fragment not starting at 1 files the
    links of all its pieces but the last under a name no fragment has (1050); pieces slice the parent's coverage."""
    cov, links = coverage(records, lengths, res)
    frags = [dict(cov=cov[c], links=links[c], start=1, length=int(lengths[c])) for c in range(len(lengths))]
    rounds = []
    for r in range(nrounds):
        brk = [(i, detect(f["cov"], f["length"], res, median_cov_ratio, region_len_ratio, min_region_cutoff))
               for i, f in enumerate(frags)]
        brk = [(i, b) for i, b in brk if b]
        rounds.append(([f["cov"].copy() for f in frags], brk))
        if not brk or r + 1 == nrounds:
            break
        nxt = []
        for i, b in brk:
            f = frags[i]
            c = f["cov"].astype(np.int64)
            lo, hi = f["links"][:, 0], f["links"][:, 1]
            ok = np.ones(len(lo), bool)
            if b[0][1] != 0:                       # one breakpoint: subtract the links spanning closed(bp, bp + res)
                bp = b[0][0]
                span = (lo <= bp + res) & (hi >= bp)
                d = np.zeros(len(c) + 1, np.int64)
                np.add.at(d, pyslice(lo[span] // res, len(c)), -1)
                np.add.at(d, pyslice(hi[span] // res + 1, len(c)), 1)
                ok = ~span
                c = c + np.cumsum(d[:-1])
            points = [p for p, _ in b]
            jl = np.searchsorted(points, lo, side="right")
            jh = np.searchsorted(points, hi, side="right")
            ok &= (jl == jh) & (lo >= 0)
            if f["start"] != 1:
                ok &= jl == len(points)
            bounds = [0] + points + [None]
            for j in range(len(points) + 1):
                p0, p1 = bounds[j], bounds[j + 1]
                sel = ok & (jl == j)
                nxt.append(dict(cov=c[p0 // res: None if p1 is None else p1 // res].astype(np.int32),
                                links=np.stack([lo[sel] - p0, hi[sel] - p0], axis=1), start=f["start"] + p0,
                                length=(f["length"] if p1 is None else p1) - p0))
        frags = nxt
    return rounds


def convert(records, n_src, layout):
    """convert_ctg (1405-1411) with the piece table of hh_correct_set_layout: (src_base, piece_start, piece_id)."""
    base, start, pid = (np.asarray(a, np.int64) for a in layout)
    src = np.repeat(np.arange(n_src, dtype=np.int64), np.diff(base))
    key = (src << 33) + start                     # ascending: sources in order, starts ascending inside a source
    rec = np.asarray(records, np.int64).copy()
    for s in (0, 2):
        c = rec[:, s]
        ok = (c >= 0) & (c < n_src)
        cc, pos = c[ok], rec[ok, s + 1]
        idx = np.maximum(np.searchsorted(key, (cc << 33) + pos, side="right") - 1, base[cc])   # last start <= pos
        rec[ok, s] = pid[idx]
        rec[ok, s + 1] = pos - start[idx]
    return rec.astype(np.int32)
